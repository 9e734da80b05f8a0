"""lio::MapBuilder with the cube map, the surround map and the registered full cloud in HBM (csrc/cubemap.cu, lio_mb_*) against
the oracle's restatement (oracle/o_mapbuilder.cc MapBuilderOracle).  Tolerances follow test_point_mapping_gpu.py: the first
frame is bit-exact; later frames differ by the float Gauss-Newton's reduction order."""
import numpy as np
import pytest

from oracle import map_builder_py as mbo
from tests.test_oracle_map_builder import mapping_frames

pytestmark = pytest.mark.gpu

POS_TOL, QUAT_TOL = 2e-4, 2e-5


def _close(a, b, rel=0.005):
    return abs(a - b) <= 2 + rel * b


def _check_frame(f, mg, mo, tg, ig, to, io, full):
    assert mg.centre() == mo.centre()
    assert ig["optimised"] == io["optimised"] and ig["surround_published"] == io["surround_published"]
    sg_map, so_map = mg.surround_map(), mo.surround_map()
    rg, ro = mg.registered_full_cloud(), mo.registered_full_cloud()
    assert rg.shape == ro.shape == full.shape
    if f == 0:
        # empty map: no optimisation on either side; insert, per-cube VoxelGrid, surround VoxelGrid and the full cloud are bit-exact
        assert ig == io and ig["iterations"] == 0
        assert np.array_equal(tg, to) and np.array_equal(mg.transform_aft_mapped, mo.transform_aft_mapped)
        for which in ("corner", "surf"):
            so, sg = mo.cube_sizes(which), mg.cube_sizes(which)
            assert np.array_equal(so, sg)
            for idx in np.nonzero(so)[0]:
                assert np.array_equal(mg.cube(idx, which), mo.cube(idx, which)), (which, idx)
        assert np.array_equal(sg_map, so_map)
        assert np.array_equal(rg, ro)
        return
    if io["optimised"]:
        assert abs(ig["iterations"] - io["iterations"]) <= 1, (f, ig, io)
    else:
        assert ig["iterations"] == 0 and io["iterations"] == 0
    for key in ("corner_from_map", "surf_from_map"):
        assert _close(ig[key], io[key]), (f, key, ig[key], io[key])
    assert np.abs(tg[4:] - to[4:]).max() <= POS_TOL and np.abs(tg[:4] - to[:4]).max() <= QUAT_TOL, (f, tg, to)
    ag, ao = mg.transform_aft_mapped, mo.transform_aft_mapped
    assert np.abs(ag[4:] - ao[4:]).max() <= POS_TOL and np.abs(ag[:4] - ao[:4]).max() <= QUAT_TOL
    for which in ("corner", "surf"):
        so, sg = mo.cube_sizes(which), mg.cube_sizes(which)
        assert np.array_equal(so > 0, sg > 0)
        assert np.abs(so - sg).sum() <= 2 + 0.005 * so.sum()
    assert _close(ig["surround_size"], io["surround_size"]) and _close(sg_map.shape[0], so_map.shape[0])
    # registered full cloud: the pose difference moves a point by at most POS_TOL + ~2 QUAT_TOL * range
    rng = np.linalg.norm(full[:, :3], axis=1)
    assert np.all(np.abs(rg[:, :3] - ro[:, :3]).max(1) <= POS_TOL + 4 * QUAT_TOL * rng + 1e-5), f
    assert np.array_equal(rg[:, 3], ro[:, 3])


def _drive(oracle, frames, **cfg):
    from lio_mapping_b200.map_builder import MapBuilder
    mo = mbo.MapBuilderOracle(**cfg)
    mg = MapBuilder(max_points=1 << 17, max_full_points=max(fr[2].shape[0] for fr in frames), **cfg)
    return mg, mo


@pytest.mark.parametrize("kind", ["vlp16", "hdl64"])
def test_map_builder_process_map_parity(oracle, kind):
    """11 frames of a drifting odometry: three surround maps (frames 0, 5, 10) and both branches of the skip_count gate."""
    frames = mapping_frames(oracle, kind, 11)
    mg, mo = _drive(oracle, frames)
    published, gates = [], set()
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        to, io = mo.process_map(corner, surf, full, tf_odom)
        tg, ig = mg.ProcessMap(corner, surf, full, tf_odom)
        _check_frame(f, mg, mo, tg, ig, to, io, full)
        gates.add(ig["optimised"])
        if ig["surround_published"]:
            published.append(f)
    assert published == [0, 5, 10] and gates == {True, False}


def test_map_builder_without_4d_parity(oracle):
    """enable_4d = 0: TransformAssociateToMap and OptimizeTransformTobeMapped (variant 0) under the same gate."""
    frames = mapping_frames(oracle, "vlp16", 6)
    mg, mo = _drive(oracle, frames, enable_4d=0)
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        to, io = mo.process_map(corner, surf, full, tf_odom)
        tg, ig = mg.ProcessMap(corner, surf, full, tf_odom)
        _check_frame(f, mg, mo, tg, ig, to, io, full)


def test_map_builder_recentres_when_the_sensor_leaves_the_centre_cubes(oracle):
    """The drive of test_point_mapping_recentres_when_the_sensor_leaves_the_centre_cubes: same directory centre and cube placement."""
    frames = mapping_frames(oracle, "vlp16", 2)
    mg, mo = _drive(oracle, frames)
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        tf = tf_odom.copy()
        tf[4:] += np.array([430.0, -260.0, 120.0], np.float32) * (f + 1)
        mo.process_map(corner, surf, full, tf)
        mg.ProcessMap(corner, surf, full, tf)
        assert mg.centre() == mo.centre() and mg.centre() != (10, 10, 5)
        for which in ("corner", "surf"):
            assert np.array_equal(mo.cube_sizes(which) > 0, mg.cube_sizes(which) > 0)


def test_map_builder_surround_overflow_passes_the_cloud_through(oracle):
    """A map_filter_size small enough for PCL's voxel-index overflow check: the surround map is its input, bit for bit."""
    frames = mapping_frames(oracle, "vlp16", 1)
    mg, mo = _drive(oracle, frames, map_filter_size=1e-4)
    corner, surf, full, tf_odom, _ = frames[0]
    to, io = mo.process_map(corner, surf, full, tf_odom)
    tg, ig = mg.ProcessMap(corner, surf, full, tf_odom)
    assert ig == io and np.array_equal(tg, to)
    so = mo.surround_map()
    assert so.shape[0] == sum(mo.cube_sizes(w).sum() for w in ("corner", "surf"))   # nothing merged
    assert np.array_equal(mg.surround_map(), so)


def test_map_builder_chain_from_the_estimator(oracle):
    """lio_est -> /local_laser_odom + the clouds of the scan received O - 1 scans earlier -> MapBuilder, on the GPU and in the
    oracle from the same inputs; the mapped pose stays near the ground-truth lidar pose."""
    from lio_mapping_b200 import estimator, ops, scenario
    from lio_mapping_b200.map_builder import MapBuilder
    from lio_mapping_b200.point_processor import PointProcessor
    W = O = 5
    scn = scenario.Scenario("vlp16", n_total=O + 6)
    sensor = scn.sensor
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max(s.shape[0] for s in scn.raw))
    stage_a = []
    for k in range(len(scn.raw)):
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        # /laser_cloud_corner_last and /laser_cloud_surf_last as the estimator pushes them with cutoff_deskew (Estimator.cc:678-693);
        # cloud_in_rings is the full cloud that PointOdometry's pass-through carries
        stage_a.append(dict(less_flat=pp.cloud("surface_points_less_flat"), corner=ops.voxel_grid(pp.cloud("corner_points_less_sharp"), 0.2),
                            full=pp.cloud("cloud_in_rings")))
        stage_a[-1]["surf"] = ops.voxel_grid(stage_a[-1]["less_flat"], 0.4)
    eg = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 16, **scenario.EST_CFG["vlp16"])
    scenario.warm_start(eg, scn, W, lambda k: stage_a[k]["surf"],
                        lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    mg = MapBuilder(max_points=1 << 16, max_full_points=max(s["full"].shape[0] for s in stage_a))
    mo = mbo.MapBuilderOracle()
    for f, k in enumerate(range(W, O + 6)):
        scenario.feed_imu(eg, scn, k)
        eg.process_scan(stage_a[k]["less_flat"])
        tf = eg.local_laser_odom()
        j = k - (O - 1)
        gt_pos = scn.gt_p[j] - scn.gt_R[j] @ scn.t_lb
        assert np.linalg.norm(tf[4:] - gt_pos) < 0.05, (k, tf, gt_pos)
        a = stage_a[j]
        to, io = mo.process_map(a["corner"], a["surf"], a["full"], tf)
        tg, ig = mg.ProcessMap(a["corner"], a["surf"], a["full"], tf)
        _check_frame(f, mg, mo, tg, ig, to, io, a["full"])
        assert np.linalg.norm(tg[4:] - gt_pos) < 0.08
