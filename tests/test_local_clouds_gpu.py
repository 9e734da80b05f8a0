"""The estimator's /local/* publication (lio_est_enable_local_clouds & co.), /local_laser_odom, the map builder's device-input
entry (lio_mb_process_map_dev) and the device-resident chain stage A -> estimator -> map builder, against the oracle
(oracle/o_local_clouds.cc, oracle/o_mapbuilder.cc)."""
import ctypes as C

import numpy as np
import pytest

from tests import helpers

pytestmark = pytest.mark.gpu

SUMMARY_SOLVER_KEYS = ["iterations", "successful", "termination", "initial_cost", "final_cost", "cost_pim", "cost_ppp", "cost_marg",
                       "turn_off", "convergence_flag", "map_size", "num_features", "odom_iters", "has_prior", "linearizations",
                       "cost_evals"]


def _stage_a(oracle, seq):
    """corner_points_less_sharp and cloud_in_rings of every sweep of seq (the oracle's stage A, like seq.less_flat)."""
    corner, full = [], []
    for sw in seq.raw:
        r = oracle.stage_a(sw, seq.sensor.lower_deg, seq.sensor.upper_deg, seq.sensor.rings)
        corner.append(r["less_sharp"]); full.append(r["cloud_in_rings"])
    return corner, full


class _Staging:
    def __init__(self, est, clouds):
        self.est, self.clouds = est, clouds

    def __getattr__(self, name):
        return getattr(self.est, name)

    def init_frame(self, k, *args):
        self.est.set_scan_clouds(*self.clouds(k))
        self.est.init_frame(k, *args)


def _pair(oracle, seq, W, O, corner, full, local=True, **cfg):
    """(oracle LocalCloudsEstimator, GPU estimator) warm-started from frames 0..W-1; warm-start corner clouds are down-sampled."""
    from lio_mapping_b200 import estimator
    from oracle import local_clouds_py as lc
    max_full = max(f.shape[0] for f in full)
    eo = lc.LocalCloudsEstimator(corner_filter_size=0.2, window_size=W, opt_window_size=O, **cfg)
    eg = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    if local:
        eg.enable_local_clouds(0.2, 1 << 14, max_full)
    clouds = lambda k: (oracle.voxel_grid(corner[k], 0.2), full[k])
    for e, mk in ((eo, lambda a, g: oracle.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)),
                  (eg, lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))):
        helpers.warm_start(_Staging(e, clouds) if (local or e is eo) else e, seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
    return eo, eg


def _check_full(go, gg, tol):
    """Equal counts and intensities; coordinates within 3e-4 m + tol * range.  transform_es_ is rounded differently on the two
    sides (the device evaluates the Twist algebra in double, the oracle in Eigen's float order) and comes from slightly different
    IMU-propagated states, so a de-skewed point moves by up to ~1e-4 m between them."""
    assert go.shape == gg.shape
    assert np.array_equal(go[:, 3], gg[:, 3])
    rng = np.linalg.norm(go[:, :3], axis=1)
    assert np.all(np.abs(go[:, :3] - gg[:, :3]).max(1) <= 3e-4 + tol * rng)


def test_local_clouds_match_the_oracle_cutoff_deskew(oracle):
    """HDL-64 config (enable_deskew = cutoff_deskew = 1), W = 5 / O = 4, 8 scans after the warm start: corner and surf are
    bit-equal; the full cloud has the oracle's count and intensities, coordinates within 3e-4 m + 2e-5 x range (_check_full).
    The extrinsic is held constant like in test_window_solve_parity_with_deskew: transform_es_ conjugates the IMU motion with it."""
    W, O = 5, 4
    seq = helpers.Sequence(oracle, "hdl64", n_total=W + 8)
    corner, full = _stage_a(oracle, seq)
    eo, eg = _pair(oracle, seq, W, O, corner, full, opt_extrinsic=0)
    for k in range(W, W + 8):
        for e in (eo, eg):
            e.set_scan_clouds(corner[k], full[k])
            helpers.feed_scan(e, seq, k)
        po, pg = eo.local_clouds(), eg.local_clouds()
        assert np.array_equal(po["corner"], pg["corner"]), k
        assert np.array_equal(po["surf"], pg["surf"]), k
        assert pg["surf"].shape[0] < eg.frame(W - O + 1).shape[0]   # the own cloud, not the accumulated slot
        _check_full(po["full"], pg["full"], 2e-5)


def test_local_clouds_match_the_oracle_with_deskew(oracle):
    """enable_deskew && !cutoff_deskew on a distorted VLP-16 drive: the corner cloud is de-skewed with the surf cloud's
    transform_es_ before its VoxelGrid; tolerances of test_window_solve_parity_with_deskew."""
    W = 5
    seq = helpers.Sequence(oracle, "vlp16", n_total=9, distort=True)
    corner, full = _stage_a(oracle, seq)
    eo, eg = _pair(oracle, seq, W, W, corner, full, opt_extrinsic=0, enable_deskew=1, cutoff_deskew=0)
    for k in range(W, 9):
        for e in (eo, eg):
            e.set_scan_clouds(corner[k], full[k])
            helpers.feed_scan(e, seq, k)
        po, pg = eo.local_clouds(), eg.local_clouds()
        for name in ("corner", "surf"):
            fo, fg = po[name], pg[name]
            assert abs(fg.shape[0] - fo.shape[0]) <= 3, (k, name)
            if fg.shape[0] == fo.shape[0] and fo.shape[0]:
                assert np.abs(fg[:, :3] - fo[:, :3]).max() < 0.4
                assert np.median(np.abs(fg[:, :3] - fo[:, :3]).max(axis=1)) < 1e-5
        _check_full(po["full"], pg["full"], 1e-4)


def test_local_clouds_opt_in_changes_nothing(oracle, vlp_seq_lc):
    """Window states, features and the solver summary are identical with local clouds on and off."""
    seq, corner, full = vlp_seq_lc
    W = 5
    _, on = _pair(oracle, seq, W, W, corner, full, local=True, opt_extrinsic=0)
    _, off = _pair(oracle, seq, W, W, corner, full, local=False, opt_extrinsic=0)
    for k in range(W, W + 4):
        on.set_scan_clouds(corner[k], full[k])
        helpers.feed_scan(on, seq, k)
        helpers.feed_scan(off, seq, k)
        assert np.array_equal(on.states(), off.states())
        s1, s0 = on.summary(), off.summary()
        assert [s1[key] for key in SUMMARY_SOLVER_KEYS] == [s0[key] for key in SUMMARY_SOLVER_KEYS]
        for f in range(W + 1):
            for a, b in zip(on.features(f), off.features(f)):
                assert np.array_equal(a, b)


@pytest.fixture(scope="module")
def vlp_seq_lc(oracle):
    seq = helpers.Sequence(oracle, "vlp16", n_total=10)
    corner, full = _stage_a(oracle, seq)
    return seq, corner, full


def test_local_clouds_errors_and_buffer_lifetime(oracle, vlp_seq_lc):
    import torch
    from lio_mapping_b200 import _lib, estimator
    seq, corner, full = vlp_seq_lc
    W = 5
    L = _lib.lib()
    _, ref = _pair(oracle, seq, W, W, corner, full, opt_extrinsic=0)
    _, eg = _pair(oracle, seq, W, W, corner, full, opt_extrinsic=0)
    # late enable
    assert L.lio_est_enable_local_clouds(eg.h, 0.2, 1 << 14, 1 << 18) == -2
    # a push with nothing staged: LIO_ERR_INVALID before the window advances, the context stays usable
    s = np.ascontiguousarray(seq.less_flat[W], np.float32)
    tt, acc, gyr = seq.imu[W]
    for e in (ref, eg):
        last = seq.t[W - 1]
        for j in range(len(tt)):
            e.process_imu(tt[j] - last, acc[j], gyr[j], tt[j])
            last = tt[j]
    assert L.lio_est_process_scan_host(eg.h, s, s.shape[0]) == -2
    # over capacity: LIO_ERR_CAPACITY, nothing staged
    big = np.zeros(((1 << 14) + 1, 4), np.float32)
    assert L.lio_est_set_scan_clouds_host(eg.h, big, big.shape[0], full[W], full[W].shape[0]) == -3
    assert L.lio_est_process_scan_host(eg.h, s, s.shape[0]) == -2
    # staged from device buffers that the caller overwrites right after the call (stream-ordered on the shared stream)
    c_dev = torch.from_numpy(np.ascontiguousarray(corner[W], np.float32)).cuda()
    f_dev = torch.from_numpy(np.ascontiguousarray(full[W], np.float32)).cuda()
    n_dev = torch.tensor([corner[W].shape[0], full[W].shape[0]], dtype=torch.int32, device="cuda")
    eg.set_scan_clouds_dev(c_dev.data_ptr(), n_dev.data_ptr(), c_dev.shape[0], f_dev.data_ptr(), n_dev.data_ptr() + 4, f_dev.shape[0])
    c_dev.fill_(123.0); f_dev.fill_(-5.0); n_dev.fill_(0)
    eg.process_scan(s)
    # host staging: the caller's arrays are free on return
    hc, hf = corner[W].copy(), full[W].copy()
    ref.set_scan_clouds(hc, hf)
    hc[:] = 7.0; hf[:] = 7.0
    ref.process_scan(s)
    assert np.array_equal(eg.states(), ref.states())
    pe, pr = eg.local_clouds(), ref.local_clouds()
    for name in ("corner", "surf", "full"):
        assert np.array_equal(pe[name], pr[name]), name
    # each staged pair is consumed by one push
    s1 =np.ascontiguousarray(seq.less_flat[W + 1], np.float32)
    assert L.lio_est_process_scan_host(eg.h, s1, s1.shape[0]) == -2
    # local clouds off: the entries refuse
    off = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17)
    assert L.lio_est_set_scan_clouds_host(off.h, hc, hc.shape[0], hf, hf.shape[0]) == -2
    n = C.c_int()
    assert L.lio_est_local_clouds_download(off.h, 0, hc, hc.shape[0], C.byref(n)) == -2


def test_local_laser_odom_matches_the_oracle_formula(oracle, vlp_seq_lc):
    """lio_est_local_laser_odom equals the oracle's double-precision statement on the same state and a float64 numpy one."""
    from lio_mapping_b200 import synth
    from oracle import local_clouds_py as lc
    seq, corner, full = vlp_seq_lc
    W, O = 5, 3
    _, eg = _pair(oracle, seq, W, O, corner, full, local=False, opt_extrinsic=1)
    for k in range(W, W + 3):
        helpers.feed_scan(eg, seq, k)
        tf = eg.local_laser_odom()
        s = eg.states()[W - O]
        ex = eg.extrinsic()
        assert np.array_equal(tf, lc.local_laser_odom_of(s, ex))
        q = s[3:7] / np.linalg.norm(s[3:7])
        rot = synth.quat_to_rot(q) @ synth.quat_to_rot(ex[:4].astype(np.float64) / np.linalg.norm(ex[:4].astype(np.float64))).T
        pos = s[:3] - rot @ ex[4:].astype(np.float64)
        qr = synth.rot_to_quat(rot)
        qr = qr if np.dot(qr, tf[:4]) >= 0 else -qr
        assert np.abs(tf[:4] - qr).max() <= 1e-6 and np.abs(tf[4:] - pos).max() <= 1e-6 * max(1.0, np.abs(pos).max())


def test_process_map_dev_equals_host(oracle):
    """lio_mb_process_map_dev and lio_mb_process_map_host on the same 11 HDL-64 frames: everything bit-equal."""
    import torch
    from lio_mapping_b200.map_builder import MapBuilder
    from tests.test_oracle_map_builder import mapping_frames
    frames = mapping_frames(oracle, "hdl64", 11)
    max_full = max(fr[2].shape[0] for fr in frames)
    mh = MapBuilder(max_points=1 << 17, max_full_points=max_full)
    md = MapBuilder(max_points=1 << 17, max_full_points=max_full)
    gates, published = set(), []
    for f, (corner, surf, full, tf_odom, _) in enumerate(frames):
        th, ih = mh.ProcessMap(corner, surf, full, tf_odom)
        dev = [torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1, 4)).cuda() for a in (corner, surf, full)]
        n = torch.tensor([a.shape[0] for a in dev], dtype=torch.int32, device="cuda")
        td, idv = md.ProcessMapDev([a.data_ptr() for a in dev], n.data_ptr(), [a.shape[0] + 5 for a in dev], tf_odom)
        assert np.array_equal(th, td) and ih == idv, f
        assert np.array_equal(mh.transform_aft_mapped, md.transform_aft_mapped)
        assert mh.centre() == md.centre()
        for which in ("corner", "surf"):
            sh, sd = mh.cube_sizes(which), md.cube_sizes(which)
            assert np.array_equal(sh, sd)
            for idx in np.nonzero(sh)[0]:
                assert np.array_equal(mh.cube(idx, which), md.cube(idx, which))
        assert np.array_equal(mh.surround_map(), md.surround_map())
        assert np.array_equal(mh.registered_full_cloud(), md.registered_full_cloud())
        gates.add(ih["optimised"])
        if ih["surround_published"]:
            published.append(f)
    assert gates == {True, False} and published == [0, 5, 10]
    # a device count above its bound: LIO_ERR_CAPACITY at the down-sampling read-back
    corner, surf, full, tf_odom, _ = frames[0]
    dev = [torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1, 4)).cuda() for a in (corner, surf, full)]
    n = torch.tensor([a.shape[0] for a in dev], dtype=torch.int32, device="cuda")
    from lio_mapping_b200 import _lib
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        md.ProcessMapDev([a.data_ptr() for a in dev], n.data_ptr(), [a.shape[0] - 1 for a in dev], tf_odom)


def test_device_resident_chain_against_the_oracle(oracle):
    """PointProcessor.process_device -> set_scan_clouds_dev + process_scan_dev -> ProcessMapDev on one stream (no cloud leaves
    HBM), frame by frame against the oracle estimator feeding MapBuilderOracle from its own /local/*: same gate and publishing
    decisions, map sizes within the map-builder tolerances, mapped poses within 5 mm, and the mapped pose within 0.08 m of the
    ground truth."""
    import torch
    from lio_mapping_b200 import _lib, estimator, scenario
    from lio_mapping_b200.map_builder import MapBuilder
    from lio_mapping_b200.point_processor import PointProcessor
    from oracle import local_clouds_py as lc
    from oracle import map_builder_py as mbo
    W = O = 5
    scn = scenario.Scenario("vlp16", n_total=O + 7)
    sensor = scn.sensor
    max_raw = max(s.shape[0] for s in scn.raw)
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_raw)
    st_a = [oracle.stage_a(scn.raw[k], sensor.lower_deg, sensor.upper_deg, sensor.rings) for k in range(len(scn.raw))]
    cfg = dict(scenario.EST_CFG["vlp16"], opt_extrinsic=0)
    eg = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    eg.enable_local_clouds(0.2, 1 << 15, max_raw)
    eo = lc.LocalCloudsEstimator(corner_filter_size=0.2, window_size=W, opt_window_size=O, **cfg)
    clouds = lambda k: (oracle.voxel_grid(st_a[k]["less_sharp"], 0.2), st_a[k]["cloud_in_rings"])
    mk_g = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    mk_o = lambda a, g: oracle.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    scenario.warm_start(_Staging(eg, clouds), scn, W, lambda k: oracle.voxel_grid(st_a[k]["less_flat"], 0.4), mk_g)
    scenario.warm_start(_Staging(eo, clouds), scn, W, lambda k: oracle.voxel_grid(st_a[k]["less_flat"], 0.4), mk_o)
    L = _lib.lib()
    ptr = {w: pp.cloud_dev(name) for w, name in ((1, "cloud_in_rings"), (3, "corner_points_less_sharp"), (5, "surface_points_less_flat"))}
    cnt = {}
    for w in ptr:
        p = C.c_void_p()
        _lib.check(L.lio_pp_cloud_count_dev(pp._h, w, C.byref(p)), "lio_pp_cloud_count_dev")
        cnt[w] = p.value
    mg = MapBuilder(max_points=1 << 16, max_full_points=max_raw)
    mo = mbo.MapBuilderOracle()
    pub_ptrs, pub_n, pub_max = eg.local_clouds_dev()
    for f, k in enumerate(range(W, O + 7)):
        raw = torch.from_numpy(np.ascontiguousarray(scn.raw[k], np.float32)).cuda()
        pp.process_device(raw.data_ptr(), raw.shape[0])
        scenario.feed_imu(eg, scn, k)
        eg.set_scan_clouds_dev(ptr[3], cnt[3], 1 << 15, ptr[1], cnt[1], max_raw)
        eg.process_scan_dev(ptr[5], cnt[5], 1 << 17)
        tg, ig = mg.ProcessMapDev(pub_ptrs, pub_n, pub_max, eg.local_laser_odom())
        scenario.feed_imu(eo, scn, k)
        eo.set_scan_clouds(st_a[k]["less_sharp"], st_a[k]["cloud_in_rings"])
        eo.process_scan(st_a[k]["less_flat"])
        po = eo.local_clouds()
        to, io = mo.process_map(po["corner"], po["surf"], po["full"], eo.local_laser_odom())
        assert ig["optimised"] == io["optimised"] and ig["surround_published"] == io["surround_published"], f
        assert abs(ig["corner_from_map"] - io["corner_from_map"]) <= 2 + 0.005 * io["corner_from_map"]
        assert abs(ig["surf_from_map"] - io["surf_from_map"]) <= 2 + 0.005 * io["surf_from_map"]
        # the two estimators' poses and de-skewed clouds differ by their own rounding, which the scan matching can amplify
        assert np.abs(tg[4:] - to[4:]).max() <= 5e-3 and np.abs(tg[:4] - to[:4]).max() <= 1e-3, (f, tg, to)
        rg, ro = mg.registered_full_cloud(), mo.registered_full_cloud()
        # intensity = ring + relative time from each side's own stage A (device kernels vs the oracle): equal to float rounding
        assert rg.shape == ro.shape and np.abs(rg[:, 3] - ro[:, 3]).max() <= 1e-4
        j = k - (O - 1)
        gt_pos = scn.gt_p[j] - scn.gt_R[j] @ scn.t_lb
        assert np.linalg.norm(tg[4:] - gt_pos) < 0.08, (k, tg, gt_pos)
