"""lio::MapBuilder, oracle restatement (oracle/o_mapbuilder.cc MapBuilderOracle): the 4-D pose association against an
independent float64 statement, the optimisation and publishing schedules, and the surround map against numpy."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from lio_mapping_b200 import synth
from oracle import map_builder_py as mbo
from tests import helpers


def mapping_frames(oracle, kind, n, seed0=40):
    """Stage-A corner / surf clouds, the full cloud and a drifting odometry pose per frame (the drive of the PointMapping
    parity test, plus cloud_in_rings as the full-resolution cloud)."""
    sensor, scene, traj = synth.default_config(kind)
    out = []
    p0 = R0 = None
    for f in range(n):
        t_end = 1.0 + 0.1 * f
        sw = synth.make_sweep(sensor, scene, traj, t_end, seed=seed0 + f, distort=False)
        r = oracle.stage_a(sw, sensor.lower_deg, sensor.upper_deg, sensor.rings)
        p, R, _, _, _ = traj.state(np.array(t_end))
        if f == 0:
            p0, R0 = p, R
        _, _, tf7 = helpers.rel_transform((R0, p0), (R, p))
        tf_odom = tf7.copy(); tf_odom[4:] += np.array([0.03, -0.02, 0.01], np.float32) * f      # accumulated odometry error
        out.append((r["less_sharp"], r["less_flat"], r["cloud_in_rings"], tf_odom, tf7))
    return out


def surround_indices(centre, pos):
    """laser_cloud_surround_idx_ (MapBuilder.cc:431-486): every in-range cube of the 5 x 5 x 5 block, i-j-k loop order."""
    def cube_of(v, cen):
        c = int((float(v) + 25.0) / 50.0) + cen
        return c - 1 if float(v) + 25.0 < 0 else c
    ci, cj, ck = (cube_of(pos[a], centre[a]) for a in range(3))
    return [i + 21 * j + 441 * k for i in range(ci - 2, ci + 3) for j in range(cj - 2, cj + 3) for k in range(ck - 2, ck + 3)
            if 0 <= i < 21 and 0 <= j < 21 and 0 <= k < 11]


def numpy_voxel_grid(pts, leaf):
    """pcl::VoxelGrid as test_voxel_grid_oracle_vs_numpy states it (centroids in ascending voxel index order)."""
    inv = np.float32(1.0) / np.float32(leaf)
    ijk = np.floor(pts[:, :3] * inv).astype(np.int64)
    ijk -= np.floor(pts[:, :3].min(0) * inv).astype(np.int64)
    div = ijk.max(0) + 1
    key = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    uk, inv_idx = np.unique(key, return_inverse=True)
    ref = np.zeros((uk.shape[0], 4), np.float64)
    np.add.at(ref, inv_idx, pts.astype(np.float64))
    return ref / np.bincount(inv_idx)[:, None]


def _tf(rot: Rotation, pos):
    q = rot.as_quat()     # x y z w
    return np.array([*q, *pos], np.float32)


def _ypr(tf7):
    """yaw, pitch, roll (rad) of a tf7 in float64, the R2ypr convention R = Rz(yaw) Ry(pitch) Rx(roll)."""
    return Rotation.from_quat(np.asarray(tf7[:4], np.float64)).as_euler("ZYX")


def _compose(a, b):   # float64 a * b of two tf7
    ra, rb = Rotation.from_quat(np.asarray(a[:4], np.float64)), Rotation.from_quat(np.asarray(b[:4], np.float64))
    return ra * rb, ra.apply(np.asarray(b[4:], np.float64)) + np.asarray(a[4:], np.float64)


def _inverse(a):
    r = Rotation.from_quat(np.asarray(a[:4], np.float64)).inv()
    return _tf(r, -r.apply(np.asarray(a[4:], np.float64)))


def _wrap(d):
    return (d + np.pi) % (2 * np.pi) - np.pi


CASES = [
    # (tobe, bef, sum) as (yaw, pitch, roll) in degrees + position
    (((10, 2, -3), (1, 2, 3)), ((5, 1, 1), (0.5, 0.2, 0.1)), ((8, 3, -2), (1.5, 0.1, 0.3))),
    # yaw of tobe * incre just past -180 while sum's is just below +180: the yaw difference crosses +-180 deg
    (((-176, 1, 2), (40, -20, 3)), ((170, 0.5, 1), (30, -10, 1)), ((178, 4, -5), (31, -9, 1.2))),
    # |yaw| near 180 and a large roll: trace of the rotation <= 0, the matrix-to-quaternion conversion's diagonal branch
    (((150, 0, 0), (0, 0, 0)), ((0, 0, 0), (0, 0, 0)), ((20, 5, 170), (2, -1, 0.5))),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_transform_4d_associate_vs_float64(oracle, case):
    tobe, bef, s = [_tf(Rotation.from_euler("ZYX", e, degrees=True), p) for e, p in CASES[case]]
    out = mbo.associate_to_map(tobe, bef, s, enable_4d=True)
    plain = mbo.associate_to_map(tobe, bef, s, enable_4d=False)
    # position: full_transform.pos, the same composition as TransformAssociateToMap, bit for bit
    assert np.array_equal(out[4:], plain[4:])
    r_full, p_full = _compose(tobe, _tf(*_compose(_inverse(bef), s)))
    assert np.abs(out[4:] - p_full).max() <= 1e-5 * max(1.0, np.abs(p_full).max())
    # rotation: roll and pitch of sum, yaw of tobe * incre (float round-off)
    y_out, y_sum, y_full = _ypr(out), _ypr(s), r_full.as_euler("ZYX")
    assert np.abs(_wrap(y_out[1:] - y_sum[1:])).max() < 2e-5, (y_out, y_sum)
    assert abs(_wrap(y_out[0] - y_full[0])) < 2e-5, (y_out, y_full)
    if case == 1:
        assert abs(y_full[0] - y_sum[0]) > np.pi   # the raw difference really wraps
    if case == 2:
        R = Rotation.from_quat(out[:4].astype(np.float64)).as_matrix()
        assert np.trace(R) <= 0
    # the quaternion is Eigen's conversion of the float product, not renormalised: unit to float precision
    assert abs(np.linalg.norm(out[:4].astype(np.float64)) - 1.0) < 1e-6


def test_matrix_to_quaternion_branches(oracle):
    """Eigen's Matrix3 -> Quaternion assignment: trace branch (w largest) and the largest-diagonal branch for each axis,
    against scipy's quaternion up to sign; the branch fixes the sign (w > 0, resp. the component of the largest diagonal > 0)."""
    rots = [Rotation.from_euler("ZYX", (20, 10, 5), degrees=True), Rotation.from_rotvec([np.pi * 0.9, 0.1, 0.0]),
            Rotation.from_rotvec([0.0, np.pi * 0.95, 0.2]), Rotation.from_rotvec([0.1, 0.0, -np.pi * 0.97])]
    for branch, r in enumerate(rots):
        R = r.as_matrix()
        q = mbo.matrix_to_quat(R.astype(np.float32)).astype(np.float64)
        ref = r.as_quat()
        assert min(np.abs(q - ref).max(), np.abs(q + ref).max()) < 1e-6, (branch, q, ref)
        big = 3 if branch == 0 else int(np.argmax(np.diag(R)))
        assert q[big] > 0 and np.argmax(np.abs(q)) == big


def test_map_builder_schedules(oracle):
    """skip_count = 2: the gate chooses OptimizeMap on frames 0, 2, 4, ... (frame 0 finds an empty map and returns early);
    the surround map is published on frames 0, 5, 10; aft follows tobe on every frame that updates it."""
    frames = mapping_frames(oracle, "vlp16", 11)
    mb = mbo.MapBuilderOracle()
    for f, (corner, surf, full, tf_odom, tf_true) in enumerate(frames):
        tobe, info = mb.process_map(corner, surf, full, tf_odom)
        assert info["optimised"] == (f % 2 == 0)
        if f % 2 == 1 or f == 0:
            assert info["iterations"] == 0
        else:
            assert info["iterations"] >= 1
        assert info["surround_published"] == (f in (0, 5, 10))
        if f >= 1:
            assert np.array_equal(mb.transform_aft_mapped, tobe)
        assert mb.registered_full_cloud().shape == full.shape


@pytest.mark.parametrize("leaf,overflow", [(0.2, False), (1e-4, True)])
def test_surround_map_vs_numpy(oracle, leaf, overflow):
    """Surround map = concatenation of the surround cubes (corner then surf per cube, loop order) through VoxelGrid; with a
    leaf small enough for PCL's dx * dy * dz > INT32_MAX check it is the plain concatenation."""
    frames = mapping_frames(oracle, "vlp16", 6)
    mb = mbo.MapBuilderOracle(map_filter_size=leaf)
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        tobe, info = mb.process_map(corner, surf, full, tf_odom)
        if not info["surround_published"]:
            continue
        idx = surround_indices(mb.centre(), tobe[4:])
        acc = np.concatenate([c for i in idx for c in (mb.cube(i, "corner"), mb.cube(i, "surf"))], 0)
        got = mb.surround_map()
        assert info["surround_size"] == got.shape[0]
        if overflow:
            assert np.array_equal(got, acc)
        else:
            ref = numpy_voxel_grid(acc, leaf)
            assert got.shape == ref.shape and got.shape[0] < acc.shape[0]
            assert np.abs(got - ref).max() <= 1e-4, f
    # the registered full cloud is PointAssociateToMap with the final tobe, intensity kept
    R = Rotation.from_quat(tobe[:4].astype(np.float64)).as_matrix()
    ref = full[:, :3].astype(np.float64) @ R.T + tobe[4:]
    got = mb.registered_full_cloud()
    assert np.abs(got[:, :3] - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())
    assert np.array_equal(got[:, 3], full[:, 3])
