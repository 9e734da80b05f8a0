"""The lidar-only pipeline PointProcessor -> PointOdometry -> PointMapping with its clouds kept in HBM (lio_po_process_dev,
lio_po_clouds_dev, lio_pm_process_dev) and PointMapping::PublishResults on the GPU (lio_pm_enable_publish): the device entries
against the host entries bit for bit, the published clouds against the oracle's restatement (oracle/o_pm_publish.cc), the whole
chain against the host-copy chain and the oracle chain, and the error paths."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from lio_mapping_b200 import synth

pytestmark = pytest.mark.gpu

STAGE_A = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")
PO_CLOUDS = ("last_corner", "last_surf", "full")
_CUDART = None


def _cudart():
    global _CUDART
    if _CUDART is None:
        import torch
        libs = glob.glob(os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*"))
        _CUDART = C.CDLL(libs[0] if libs else "libcudart.so")
        _CUDART.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return _CUDART


def read_dev(ptr, n, dtype=np.float32, width=4):
    """n rows of `width` values at a device pointer, copied to the host (cudaMemcpy, device to host)."""
    out = np.zeros((max(n, 1), width), dtype)
    if n:
        assert _cudart().cudaMemcpy(out.ctypes.data, C.c_void_p(ptr), out[:n].nbytes, 2) == 0
    return out[:n]


def raw_sweeps(kind, n, seed0=70, t0=1.0):
    """Motion-distorted sweeps of the drive tests.test_oracle_point_odometry.sweeps uses, and the sensor poses at their ends."""
    sensor, scene, traj = synth.default_config(kind)
    out = []
    for f in range(n):
        t_end = t0 + 0.1 * f
        sw = synth.make_sweep(sensor, scene, traj, t_end, seed=seed0 + f, distort=True)
        p, R, _, _, _ = traj.state(np.array(t_end))
        out.append((np.ascontiguousarray(sw, np.float32), (R, p)))
    return sensor, out


class StageA:
    """Device stage A of one sweep at a time: the five clouds PointOdometry takes, as device pointers and as host copies."""

    def __init__(self, sensor, max_points):
        from lio_mapping_b200.point_processor import PointProcessor
        self.pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_points)
        self.n_dev = [self.pp.cloud_count_dev(name) for name in STAGE_A]

    def run(self, raw):
        import torch
        self.raw = torch.from_numpy(raw).cuda()
        self.pp.process_device(self.raw.data_ptr(), self.raw.shape[0])
        return [self.pp.cloud_dev(name) for name in STAGE_A]

    def host(self):
        return [self.pp.cloud(name) for name in STAGE_A]


@pytest.mark.parametrize("kind", ["vlp16", "hdl64"])
def test_po_process_dev_equals_host(kind):
    """lio_po_process_dev on stage A's device outputs against lio_po_process_host on the same clouds downloaded, io_ratio 2, over
    8 distorted sweeps, the last two after EnableOdom(False): poses, info, the published clouds (through clouds_dev and cloud) and
    /compact_data bit-equal.  A call with a device count above its bound fails with LIO_ERR_CAPACITY and leaves no trace."""
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.point_odometry import PointOdometry
    sensor, sw = raw_sweeps(kind, 8)
    max_raw = max(s.shape[0] for s, _ in sw)
    sa = StageA(sensor, max_raw)
    ph = PointOdometry(0.1, 2, 25, max_full_points=max_raw + 3)
    pd = PointOdometry(0.1, 2, 25, max_full_points=max_raw + 3)
    published = []
    for f, (raw, _) in enumerate(sw):
        if f == 6:
            ph.EnableOdom(False); pd.EnableOdom(False)
        ptrs = sa.run(raw)
        clouds = sa.host()
        n = [c.shape[0] for c in clouds]
        if f == 3:      # one bound below its device count: refused before anything changes
            with pytest.raises(_lib.LioError, match="CAPACITY"):
                pd.ProcessDev(ptrs, sa.n_dev, [n[0], n[1], n[2], n[3], n[4] - 1])
        th, eh, ih = ph.Process(*clouds)
        td, ed, idv = pd.ProcessDev(ptrs, sa.n_dev, [c + 3 for c in n])
        assert np.array_equal(th, td) and np.array_equal(eh, ed) and ih == idv, (f, ih, idv)
        dptr, dn, hn = pd.clouds_dev()
        assert np.array_equal(read_dev(dn, 3, np.int32, 1)[:, 0], hn)
        for k, which in enumerate(PO_CLOUDS):
            ch = ph.cloud(which)
            assert hn[k] == ch.shape[0]
            assert np.array_equal(pd.cloud(which), ch) and np.array_equal(read_dev(dptr[k], hn[k]), ch), (f, which)
        if ih["published"]:
            published.append(f)
            assert np.array_equal(ph.compact_data(), pd.compact_data())
        if 1 <= f < 6:
            assert ih["iterations"] >= 1
    assert published == [1, 3, 5, 7]


def _pm_dev_inputs(corner, surf, full=None):
    import torch
    arrs = [np.ascontiguousarray(a, np.float32).reshape(-1, 4) for a in (corner, surf, full if full is not None else np.zeros((0, 4)))]
    dev = [torch.from_numpy(a).cuda() if a.shape[0] else None for a in arrs]
    n = torch.tensor([a.shape[0] for a in arrs], dtype=torch.int32, device="cuda")
    return dev, [d.data_ptr() if d is not None else 0 for d in dev], n, [a.shape[0] for a in arrs]


def _same_map(pa, pb):
    assert pa.centre() == pb.centre()
    for which in ("corner", "surf"):
        sa, sb = pa.cube_sizes(which), pb.cube_sizes(which)
        assert np.array_equal(sa, sb)
        for idx in np.nonzero(sa)[0]:
            assert np.array_equal(pa.cube(idx, which), pb.cube(idx, which)), (which, idx)


@pytest.mark.parametrize("kind", ["vlp16", "hdl64"])
def test_pm_process_dev_equals_host_without_publishing(oracle, kind):
    """lio_pm_process_dev on a handle that does not publish against lio_pm_process_host over the PointMapping parity drive: pose,
    info, centre and every cube bit-equal.  The full cloud is not read: NULL with a bound 0, and any count in its slot."""
    from lio_mapping_b200.point_mapping import PointMapping
    from tests.test_point_mapping_gpu import _frames
    ph, pd = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
    for f, (corner, surf, tf_odom, _) in enumerate(_frames(oracle, kind, 6)):
        th, ih = ph.Process(corner, surf, tf_odom)
        keep, ptrs, n, nn = _pm_dev_inputs(corner, surf)
        n[2] = 1 << 30
        td, ad, idv = pd.ProcessDev(ptrs, n.data_ptr(), [nn[0] + 7, nn[1], 0], tf_odom)
        assert np.array_equal(th, td) and ih == {k: idv[k] for k in ih}, f
        assert not idv["surround_published"] and idv["surround_size"] == 0
        _same_map(ph, pd)


def test_pm_process_dev_equals_host_across_recentring(oracle):
    from lio_mapping_b200.point_mapping import PointMapping
    from tests.test_point_mapping_gpu import _frames
    ph, pd = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
    for f, (corner, surf, tf_odom, _) in enumerate(_frames(oracle, "vlp16", 2)):
        tf = tf_odom.copy()
        tf[4:] += np.array([430.0, -260.0, 120.0], np.float32) * (f + 1)
        th, ih = ph.Process(corner, surf, tf)
        keep, ptrs, n, nn = _pm_dev_inputs(corner, surf)
        td, _, idv = pd.ProcessDev(ptrs, n.data_ptr(), nn, tf)
        assert np.array_equal(th, td) and ih == {k: idv[k] for k in ih}
        assert pd.centre() != (10, 10, 5)
        _same_map(ph, pd)


def test_publish_results(oracle):
    """PointMapping::PublishResults on a publishing handle over 11 HDL-64 frames: the surround map exactly on calls 1, 6 and 11,
    bit-equal to the oracle's VoxelGrid(0.6) of the device's own surround cubes; the registered cloud bit-equal to the oracle's
    PointAssociateToMap of the input with the returned tobe; aft following TransformUpdate; the first frame bit-exact against the
    oracle restatement, later frames within the PointMapping tolerances; poses and cubes bit-identical to a plain handle."""
    from lio_mapping_b200.point_mapping import PointMapping
    from oracle import pm_publish_py as pmp
    from tests.test_oracle_map_builder import mapping_frames
    frames = mapping_frames(oracle, "hdl64", 11)
    max_full = max(fr[2].shape[0] for fr in frames)
    pub, plain = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
    pub.EnablePublish(0.6, max_full)
    po = pmp.PointMappingPublishOracle()
    published = []
    aft_prev = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    for f, (corner, surf, full, tf_odom, tf_true) in enumerate(frames):
        keep, ptrs, n, nn = _pm_dev_inputs(corner, surf, full)
        tg, ag, ig = pub.ProcessDev(ptrs, n.data_ptr(), nn, tf_odom)
        tp, ap, ip = plain.ProcessDev(ptrs, n.data_ptr(), [nn[0], nn[1], 0], tf_odom)
        to, ao, io = po.process(corner, surf, full, tf_odom)
        # publishing changes nothing of Process
        assert np.array_equal(tg, tp) and np.array_equal(ag, ap) and {k: ig[k] for k in ("iterations", "corner_from_map", "surf_from_map")} == \
            {k: ip[k] for k in ("iterations", "corner_from_map", "surf_from_map")}
        _same_map(pub, plain)
        # /aft_mapped_to_init
        optimised = ig["corner_from_map"] > 10 and ig["surf_from_map"] > 100
        assert np.array_equal(ag, tg if optimised else aft_prev), f
        aft_prev = ag
        # /cloud_registered
        reg = pub.registered_full_cloud()
        assert np.array_equal(reg, pmp.associate_to_map(full, tg))
        rp, rn = pub.registered_full_cloud_dev()
        assert rn == full.shape[0] and np.array_equal(read_dev(rp, rn), reg)
        # /laser_cloud_surround
        assert ig["surround_published"] == io["surround_published"]
        if ig["surround_published"]:
            published.append(f)
            idx = po.surround_idx()
            acc = np.concatenate([c for i in idx for c in (pub.cube(i, "corner"), pub.cube(i, "surf"))])
            sur = pub.surround_map()
            assert sur.shape[0] == ig["surround_size"] and np.array_equal(sur, oracle.voxel_grid(acc, 0.6)), f
            sp, sn = pub.surround_map_dev()
            assert sn == sur.shape[0] and np.array_equal(read_dev(sp, sn), sur)
        if f == 0:
            assert ig == io and np.array_equal(tg, to) and np.array_equal(ag, ao)
            assert np.array_equal(pub.surround_map(), po.surround_map()) and np.array_equal(reg, po.registered_full_cloud())
            for which in ("corner", "surf"):
                so = po.cube_sizes(which)
                assert np.array_equal(so, pub.cube_sizes(which))
                for i in np.nonzero(so)[0]:
                    assert np.array_equal(pub.cube(i, which), po.cube(i, which))
        else:
            assert abs(ig["iterations"] - io["iterations"]) <= 1
            for key in ("corner_from_map", "surf_from_map"):
                assert abs(ig[key] - io[key]) <= 2 + 0.005 * io[key], (f, key, ig[key], io[key])
            assert np.abs(tg[4:] - to[4:]).max() <= 2e-4 and np.abs(tg[:4] - to[:4]).max() <= 2e-5, (f, tg, to)
            if ig["surround_published"]:
                so = po.surround_map()
                assert abs(sur.shape[0] - so.shape[0]) <= 2 + 0.005 * so.shape[0]
            assert np.linalg.norm(tg[4:] - tf_true[4:]) < 0.08
    assert published == [0, 5, 10]


def _quat_diff(a, b):
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def test_lidar_chain_against_host_copies_and_the_oracle(oracle):
    """Stage A (process_device) -> PointOdometry.ProcessDev -> (io_ratio gate) -> PointMapping.ProcessDev with publishing, all on
    one stream, over 12 distorted VLP-16 sweeps: poses bit-identical to the host-copy chain on the same stage-A outputs
    (downloads, Process, compact_data, compact_decode, PointMapping.Process); against the oracle chain (stage_a ->
    PointOdometryOracle -> PointMappingPublishOracle) the same gate decisions and poses within the odometry and mapping
    tolerances; the mapped position within 0.08 m of the ground truth."""
    from lio_mapping_b200 import wire
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from oracle import pm_publish_py as pmp
    from tests import helpers
    sensor, sw = raw_sweeps("vlp16", 12)
    max_raw = max(s.shape[0] for s, _ in sw)
    sa = StageA(sensor, max_raw)
    od, oh = PointOdometry(0.1, 2, 25, max_full_points=max_raw), PointOdometry(0.1, 2, 25, max_full_points=max_raw)
    md, mh = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
    md.EnablePublish(0.6, max_raw)
    oo, mo = oracle.PointOdometryOracle(0.1, 2, 25), pmp.PointMappingPublishOracle()
    calls = 0
    for f, (raw, pose) in enumerate(sw):
        ptrs = sa.run(raw)
        td, _, idv = od.ProcessDev(ptrs, sa.n_dev, [1 << 17] * 4 + [max_raw])
        if idv["published"]:
            cptr, cn_dev, cn = od.clouds_dev()
            tm_d, am_d, im_d = md.ProcessDev(cptr, cn_dev, cn, td)
        # host copies of the same device stage-A outputs
        th, _, ih = oh.Process(*sa.host())
        assert np.array_equal(th, td) and ih == idv
        if ih["published"]:
            tf7, c, s, full = wire.compact_decode(oh.compact_data())
            tm_h, im_h = mh.Process(c, s, tf7)
            assert np.array_equal(tm_h, tm_d) and im_h == {k: im_d[k] for k in im_h}, f
            assert np.array_equal(md.registered_full_cloud(), pmp.associate_to_map(full, tm_d))
        # the oracle chain
        r = oracle.stage_a(raw, sensor.lower_deg, sensor.upper_deg, sensor.rings)
        to, _, io = oo.process(r["sharp"], r["less_sharp"], r["flat"], r["less_flat"], r["cloud_in_rings"])
        assert io["published"] == idv["published"] and io["frame_count"] == idv["frame_count"]
        scale = max(1.0, float(np.abs(to[4:]).max()))
        assert np.abs(td[4:] - to[4:]).max() <= 3e-4 * scale and _quat_diff(td[:4], to[:4]) <= 5e-5, (f, td, to)
        if io["published"]:
            calls += 1
            tm_o, _, im_o = mo.process(oo.cloud("last_corner"), oo.cloud("last_surf"), oo.cloud("full"), to)
            assert im_o["surround_published"] == im_d["surround_published"] == (calls in (1, 6))
            assert np.abs(tm_d[4:] - tm_o[4:]).max() <= 2e-4 and _quat_diff(tm_d[:4], tm_o[:4]) <= 2e-5, (f, tm_d, tm_o)
            _, _, tf_true = helpers.rel_transform(sw[0][1], pose)
            assert np.linalg.norm(tm_d[4:] - tf_true[4:]) < 0.08, (f, tm_d, tf_true)
    assert calls == 6


def test_errors():
    """Capacity and argument errors of the device entries and of lio_pm_enable_publish."""
    import torch
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.map_builder import MapBuilder
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    pts = torch.zeros((256, 4), dtype=torch.float32, device="cuda")
    cnt = torch.full((5,), 8, dtype=torch.int32, device="cuda")
    p, c = pts.data_ptr(), [cnt.data_ptr() + 4 * k for k in range(5)]
    # lio_po_process_dev
    po = PointOdometry(0.1, 1, 25, max_feature_points=64, max_full_points=64)
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        po.ProcessDev([p] * 5, c, [8, 65, 8, 8, 8])           # a bound above the capacity
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        po.ProcessDev([p] * 5, c, [8, 8, 8, 8, 65])
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        po.ProcessDev([p] * 5, c, [8, 8, 7, 8, 8])            # a device count above its bound
    with pytest.raises(_lib.LioError, match="INVALID"):
        po.ProcessDev([p, 0, p, p, p], c, [8] * 5)            # NULL cloud with a bound
    with pytest.raises(_lib.LioError, match="INVALID"):
        po.ProcessDev([p] * 5, [c[0], 0, c[2], c[3], c[4]], [8] * 5)   # NULL count
    ts, _, info = po.ProcessDev([p] * 5, c, [8] * 5)
    assert info["frame_count"] == 0 and np.array_equal(ts, [0, 0, 0, 1, 0, 0, 0])   # the refused calls left no trace
    ptr3, n_dev, n_host = po.clouds_dev()
    assert n_host == [8, 8, 8] and all(ptr3)
    # lio_pm_process_dev
    pm = PointMapping(max_points=64)
    n3 = torch.tensor([8, 80, 0], dtype=torch.int32, device="cuda")
    tf = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        pm.ProcessDev([p, p, 0], n3.data_ptr(), [8, 100, 0], tf)   # bound capped at the capacity, count above it
    with pytest.raises(_lib.LioError, match="INVALID"):
        pm.ProcessDev([p, 0, 0], n3.data_ptr(), [8, 8, 0], tf)
    with pytest.raises(_lib.LioError, match="INVALID"):
        pm.ProcessDev([p, p, 0], 0, [8, 8, 0], tf)
    # lio_pm_enable_publish: late, twice, on a map builder; a publishing handle refuses the host entry and a NULL full cloud
    with pytest.raises(_lib.LioError, match="INVALID"):
        pm.EnablePublish(0.6, 64)
    fresh = PointMapping(max_points=64)
    for fn in ("surround_map_dev", "registered_full_cloud_dev"):
        with pytest.raises(_lib.LioError, match="INVALID"):
            getattr(fresh, fn)()
    fresh.EnablePublish(0.6, 64)
    with pytest.raises(_lib.LioError, match="INVALID"):
        fresh.EnablePublish(0.6, 64)
    with pytest.raises(_lib.LioError, match="INVALID"):
        fresh.Process(np.zeros((8, 4), np.float32), np.zeros((8, 4), np.float32), tf)
    with pytest.raises(_lib.LioError, match="INVALID"):
        fresh.ProcessDev([p, p, 0], n3.data_ptr(), [8, 8, 8], tf)
    assert fresh.surround_map_dev()[1] == 0 and fresh.registered_full_cloud_dev()[1] == 0
    mb = MapBuilder(max_points=64, max_full_points=64)
    with pytest.raises(_lib.LioError, match="INVALID"):
        mb.EnablePublish(0.6, 64)
    with pytest.raises(_lib.LioError, match="INVALID"):
        mb.ProcessDev([p, p, p], n3.data_ptr(), [8, 8, 8], tf)
