"""The oracle's restatement of the estimator's /local/* publication (oracle/o_local_clouds.cc) on the CPU: TransformToEnd with
keep_intensity against an independent float64 statement, and the corner / surf / full bookkeeping on clouds tagged by frame."""
import numpy as np

from tests import helpers


def _quat_mul_vec(q, v):   # q = (x, y, z, w), rows of v
    u = np.asarray(q[:3], np.float64)
    t = 2.0 * np.cross(u, v)
    return v + q[3] * t + np.cross(u, t)


def _slerp_id(s, q):   # identity.slerp(s, q) (Eigen QuaternionBase::slerp), float64
    d = q[3]
    if abs(d) >= 1 - np.finfo(np.float32).eps:
        s0, s1 = 1 - s, s
    else:
        th = np.arccos(abs(d))
        s0, s1 = np.sin((1 - s) * th) / np.sin(th), np.sin(s * th) / np.sin(th)
    if d < 0:
        s1 = -s1
    return np.array([s1 * q[0], s1 * q[1], s1 * q[2], s0 + s1 * q[3]])


def transform_to_end_f64(cloud, tf7, time_factor=10.0, keep_intensity=False):
    """Estimator.cc:62-103 in float64: p -= s t; p = q_e (q_s^-1 p) + t with q_s = slerp(identity, q_e, s), s = 10 frac(I)."""
    c = np.asarray(cloud, np.float64).copy()
    q = np.asarray(tf7[:4], np.float64); t = np.asarray(tf7[4:], np.float64)
    for i in range(c.shape[0]):
        s = time_factor * (c[i, 3] - np.trunc(c[i, 3]))
        p = c[i, :3] - s * t
        qs = _slerp_id(s, q)
        qs = np.array([-qs[0], -qs[1], -qs[2], qs[3]]) / np.linalg.norm(qs)
        c[i, :3] = _quat_mul_vec(q, _quat_mul_vec(qs, p[None])[0][None])[0] + t
        if not keep_intensity:
            c[i, 3] -= np.trunc(c[i, 3])
    return c


def _tagged_cloud(rng, n, tag, spacing=None):
    if spacing:   # on a grid wider than the 0.2 m corner leaf: the VoxelGrid keeps every point as it is
        g = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(n // 16 + 1), indexing="ij"), -1).reshape(-1, 3)[:n]
        xyz = g * spacing + 0.37
    else:
        xyz = rng.uniform(-30, 30, (n, 3))
    frac = (np.arange(n) % 97) * 0.001          # relative time in [0, 0.1): s = 10 frac in [0, 1)
    return np.concatenate([xyz, (tag + frac)[:, None]], 1).astype(np.float32)


def test_transform_to_end_keep_intensity_matches_float64(oracle):
    from oracle import local_clouds_py as lc
    rng = np.random.default_rng(3)
    cloud = _tagged_cloud(rng, 400, 7.0)
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    ang = 0.03
    tf7 = np.array([*(np.sin(ang / 2) * ax), np.cos(ang / 2), 0.4, -0.2, 0.05], np.float32)
    for keep in (True, False):
        got = lc.transform_to_end(cloud, tf7, 10.0, keep_intensity=keep)
        ref = transform_to_end_f64(cloud, tf7.astype(np.float64), 10.0, keep_intensity=keep)
        rng_m = np.linalg.norm(cloud[:, :3], axis=1)
        assert np.all(np.abs(got[:, :3] - ref[:, :3]).max(1) <= 2e-6 * (1 + rng_m))
        if keep:
            assert np.array_equal(got[:, 3], cloud[:, 3])
        else:
            assert np.array_equal(got[:, 3], cloud[:, 3] - np.trunc(cloud[:, 3]))
    # the existing call (no keep_intensity) is unchanged
    assert np.array_equal(lc.transform_to_end(cloud, tf7, 10.0), oracle.transform_to_end(cloud, tf7, 10.0))


class _Staging:
    """Stages frame k's corner / full cloud before each init_frame of helpers.warm_start."""

    def __init__(self, est, clouds):
        self.est, self.clouds = est, clouds

    def __getattr__(self, name):
        return getattr(self.est, name)

    def init_frame(self, k, *args):
        self.est.set_scan_clouds(*self.clouds(k))
        self.est.init_frame(k, *args)


def test_local_clouds_bookkeeping_on_tagged_frames(oracle):
    """W = 4, O = 3 (pivot 1, so SlideWindow accumulates): after scan k the published clouds are frame k - (O - 1)'s; surf is the
    frame's own down-sampled cloud, corner its VoxelGrid, full its raw cloud (warm-start frames) or de-skewed with the
    transform_es_ of the scan that pushed it, intensity kept."""
    from oracle import local_clouds_py as lc
    W, O = 4, 3
    n_total = W + 4
    seq = helpers.Sequence(oracle, "vlp16", n_total=n_total)
    rng = np.random.default_rng(5)
    corner = [_tagged_cloud(rng, 40, float(k), spacing=1.0) for k in range(n_total)]
    full = [_tagged_cloud(rng, 300, float(k)) for k in range(n_total)]
    eo = lc.LocalCloudsEstimator(corner_filter_size=0.2, window_size=W, opt_window_size=O, opt_extrinsic=0)
    helpers.warm_start(_Staging(eo, lambda k: (corner[k], full[k])), seq, oracle, W, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: oracle.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    es = {}
    for k in range(W, n_total):
        eo.set_scan_clouds(corner[k], full[k])
        helpers.feed_scan(eo, seq, k)
        es[k] = eo.transform_es()
        j = k - (O - 1)
        pub = eo.local_clouds()
        if j < W:   # warm-start frames: stored verbatim
            assert np.array_equal(pub["corner"], corner[j])
        else:
            assert np.array_equal(pub["corner"], oracle.voxel_grid(corner[j], 0.2))
            # grid spacing > leaf: every point and its tag survive the VoxelGrid (in voxel order)
            assert np.array_equal(np.unique(pub["corner"], axis=0), np.unique(corner[j], axis=0))
        assert np.array_equal(pub["surf"], oracle.voxel_grid(seq.less_flat[j], 0.4))
        assert eo.frame(W - O + 1).shape[0] > pub["surf"].shape[0]   # the slot itself holds the prepended pivot cloud
        if j < W:
            assert np.array_equal(pub["full"], full[j])
        else:
            assert not np.allclose(es[j][4:], 0)
            assert np.array_equal(pub["full"], lc.transform_to_end(full[j], es[j], 10.0, keep_intensity=True))
            ref = transform_to_end_f64(full[j], es[j].astype(np.float64), 10.0, keep_intensity=True)
            assert np.abs(pub["full"][:, :3] - ref[:, :3]).max() < 1e-4
        assert np.array_equal(pub["full"][:, 3], full[j][:, 3])
        # /local_laser_odom of the same frame: the oracle formula on the window state W - O
        assert np.array_equal(eo.local_laser_odom(), lc.local_laser_odom_of(eo.states()[W - O], eo.extrinsic()))
