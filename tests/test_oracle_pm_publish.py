"""PointMapping::Process + PublishResults restated (oracle/o_pm_publish.cc PointMappingPublishOracle): the Process part is
PointMappingOracle's bit for bit, the surround map follows the publishing schedule and equals a numpy concatenation + VoxelGrid
of the oracle's own cubes, the registered cloud is the full cloud in the map frame and /aft_mapped_to_init follows TransformUpdate."""
import numpy as np
from scipy.spatial.transform import Rotation

from oracle import pm_publish_py as pmp
from tests.test_oracle_map_builder import mapping_frames, numpy_voxel_grid


def test_process_is_point_mapping_and_publish_results_follow_the_reference(oracle):
    frames = mapping_frames(oracle, "vlp16", 7)
    po = oracle.PointMappingOracle()
    pp = pmp.PointMappingPublishOracle()
    published = []
    aft_prev = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        to, io = po.process(corner, surf, tf_odom)
        tp, ap, ip = pp.process(corner, surf, full, tf_odom)
        # the Process part is PointMappingOracle's
        assert np.array_equal(tp, to) and {k: ip[k] for k in io} == io, f
        assert pp.centre() == po.centre()
        for which in ("corner", "surf"):
            assert np.array_equal(pp.cube_sizes(which), po.cube_sizes(which))
        # /aft_mapped_to_init: TransformUpdate behind the optimiser's early return
        optimised = io["corner_from_map"] > 10 and io["surf_from_map"] > 100
        assert np.array_equal(ap, tp if optimised else aft_prev), f
        aft_prev = ap
        # /cloud_registered: the full cloud through PointAssociateToMap with the final tobe
        reg = pp.registered_full_cloud()
        assert np.array_equal(reg, pmp.associate_to_map(full, tp))
        ref = Rotation.from_quat(tp[:4].astype(np.float64)).apply(full[:, :3].astype(np.float64)) + tp[4:].astype(np.float64)
        assert np.abs(reg[:, :3] - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()) and np.array_equal(reg[:, 3], full[:, 3])
        # /laser_cloud_surround: calls 1, 6, ... ; every surround cube's corner then surf cloud, VoxelGrid(0.6)
        idx = pp.surround_idx()
        assert len(idx) == 125
        if ip["surround_published"]:
            published.append(f)
            acc = np.concatenate([c for i in idx for c in (pp.cube(i, "corner"), pp.cube(i, "surf"))])
            sur = pp.surround_map()
            assert sur.shape[0] == ip["surround_size"]
            assert np.array_equal(sur, oracle.voxel_grid(acc, 0.6))
            ref = numpy_voxel_grid(acc, 0.6)
            assert ref.shape == sur.shape and np.abs(sur - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    assert published == [0, 5]
    assert 0 < pp.surround_map().shape[0]


def test_associate_to_map_against_float64():
    rng = np.random.default_rng(3)
    cloud = rng.uniform(-40, 40, (500, 4)).astype(np.float32)
    rot = Rotation.from_euler("zyx", [0.7, -0.2, 0.1])
    tf7 = np.array([*rot.as_quat(), 3.0, -1.5, 0.25], np.float32)
    out = pmp.associate_to_map(cloud, tf7)
    ref = Rotation.from_quat(tf7[:4].astype(np.float64)).apply(cloud[:, :3].astype(np.float64)) + tf7[4:].astype(np.float64)
    assert np.abs(out[:, :3] - ref).max() <= 2e-5 and np.array_equal(out[:, 3], cloud[:, 3])
