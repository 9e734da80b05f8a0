"""The device estimator's global cube map after initialisation (lio_est_attach_map / lio_est_map_poses): the pre-initialisation map
of a publishing PointMapping handed to the estimator, the per-scan prediction of transform_tobe_mapped_, UpdateMapDatabase of the
oldest optimised frame and PublishResults (Estimator.cc:703-723, :776-812)."""
import numpy as np
import pytest

from tests import helpers
from tests.test_local_clouds_gpu import SUMMARY_SOLVER_KEYS, _Staging, _stage_a

pytestmark = pytest.mark.gpu


def _quat_R(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _T(tf7):
    T = np.eye(4)
    T[:3, :3] = _quat_R(tf7[:4]); T[:3, 3] = np.asarray(tf7[4:], np.float64)
    return T


def _T_state(s16):
    return _T(np.r_[s16[3:7], s16[0:3]])


class _Setup:
    """GPU estimator with local clouds (eg), the same without a map (eb), a publishing PointMapping fed the warm-start sweeps
    (pm, attached to eg) and a second one fed identically (pr, the replay map)."""

    def __init__(self, oracle, W, O, n_scans, **cfg):
        from lio_mapping_b200 import estimator
        from lio_mapping_b200.point_mapping import PointMapping
        self.W, self.O = W, O
        self.seq = seq = helpers.Sequence(oracle, "hdl64", n_total=W + n_scans)
        self.corner, self.full = _stage_a(oracle, seq)
        self.corner_ds = [oracle.voxel_grid(c, 0.2) for c in self.corner]
        max_full = max(f.shape[0] for f in self.full)
        self.ests = []
        for _ in range(2):
            e = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
            e.enable_local_clouds(0.2, 1 << 14, max_full)
            helpers.warm_start(_Staging(e, lambda k: (self.corner_ds[k], self.full[k])), seq, oracle, W, pose_noise=0.01, seed=1,
                               make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
            self.ests.append(e)
        self.eg, self.eb = self.ests
        self.pm, self.pr = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
        tlb = seq.tf_lb7()
        for p in (self.pm, self.pr):
            p.EnablePublish(0.6, max_full)
        for k in range(W):   # the pre-initialisation mapper, fed the ground-truth lidar pose as /laser_odom_to_init
            T = _T_state(seq.state16(k, None)) @ np.linalg.inv(_T(tlb))
            sum7 = np.r_[helpers.synth.rot_to_quat(T[:3, :3]), T[:3, 3]].astype(np.float32)
            keep, ptrs, n, nn = _dev_inputs(self.corner[k], self.less_flat(k), self.full[k])
            _, self.aft0, _ = self.pm.ProcessDev(ptrs, n.data_ptr(), nn, sum7)
            self.pr.ProcessDev(ptrs, n.data_ptr(), nn, sum7)

    def less_flat(self, k):
        return self.seq.less_flat[k]

    def imu(self, e, k):
        tt, acc, gyr = self.seq.imu[k]
        last = self.seq.t[k - 1]
        for j in range(len(tt)):
            e.process_imu(tt[j] - last, acc[j], gyr[j], tt[j])
            last = tt[j]


def _dev_inputs(corner, surf, full):
    import torch
    arrs = [np.ascontiguousarray(a, np.float32).reshape(-1, 4) for a in (corner, surf, full)]
    dev = [torch.from_numpy(a).cuda() for a in arrs]
    n = torch.tensor([a.shape[0] for a in arrs], dtype=torch.int32, device="cuda")
    return dev, [d.data_ptr() for d in dev], n, [a.shape[0] for a in arrs]


def _same_map(pa, pb):
    assert pa.centre() == pb.centre()
    for which in ("corner", "surf"):
        sa, sb = pa.cube_sizes(which), pb.cube_sizes(which)
        assert np.array_equal(sa, sb), which
        for idx in np.nonzero(sa)[0]:
            assert np.array_equal(pa.cube(idx, which), pb.cube(idx, which)), (which, idx)


CONFIGS = [
    pytest.param(5, 4, {}, id="W5O4-cutoff_deskew"),                                   # HDL-64 config: enable_deskew = cutoff_deskew = 1
    pytest.param(4, 4, {}, id="W4O4-cutoff_deskew"),                                   # W == O: the inserted clouds have left the window
    pytest.param(5, 4, dict(cutoff_deskew=0), id="W5O4-enable_deskew"),
    pytest.param(5, 4, dict(enable_deskew=0, cutoff_deskew=0), id="W5O4-no_deskew"),
    pytest.param(4, 4, dict(enable_deskew=0, cutoff_deskew=0), id="W4O4-no_deskew"),   # W == O: logical frame 0, no copy
]


@pytest.mark.parametrize("W,O,extra", CONFIGS)
def test_attached_map_follows_the_reference(oracle, W, O, extra):
    """Over O + 5 scans: (1) the map changes nothing of the estimator (states, solver summary, local clouds bit-equal to an estimator
    without a map); (2) tobe follows tobe * lb * (prev^-1 * curr) * lb^-1 of the device's own states to float rounding; (3) no insert
    on the first O scans, then one insert per scan, bit-exact: the replay map (identical before the attach) takes the clouds the
    aliasing rules select from the device's own slots and published corner clouds, with the reported pose, the frozen valid list and
    centre, through lio_pm_update_map_database_host, and every cube stays bit-equal; (4) the surround map every 5th call counting on
    from the warm-start calls, bit-equal to VoxelGrid(0.6) of the device's surround cubes; the registered cloud bit-equal to
    PointAssociateToMap of the raw staged full cloud with tobe; aft frozen at its pre-attach value."""
    from oracle import global_map_py as gmo
    from oracle import pm_publish_py as pmp
    s = _Setup(oracle, W, O, O + 5, opt_extrinsic=0, **extra)
    eg, eb, pm, pr = s.eg, s.eb, s.pm, s.pr
    _same_map(pm, pr)
    valid, surround = pm.cube_lists()
    centre = pm.centre()
    aft0 = s.aft0
    eg.attach_map(pm)
    tobe, aft, _, info = eg.map_poses()
    assert np.array_equal(aft, aft0) and not info["inserted"]
    deskew = bool(eg.cfg["enable_deskew"] or eg.cfg["cutoff_deskew"])
    pivot = W - O
    pub_corner = {}                 # frame id -> its published (down-sampled) corner cloud
    own_prev = None                 # logical frame 0 after the previous scan (W == O: the frame the next scan inserts)
    calls = W                       # the warm-start process calls published on calls 1, 6, ...
    tlb = s.seq.tf_lb7().astype(np.float64)
    for i in range(O + 5):
        k = W + i
        for e in (eg, eb):
            e.set_scan_clouds(s.corner[k], s.full[k])
            s.imu(e, k)
        st = eg.states()
        tobe_prev = tobe.astype(np.float64)
        for e in (eg, eb):
            e.process_scan(s.less_flat(k))
        # (1) nothing of the estimator changes
        assert np.array_equal(eg.states(), eb.states()), i
        sg, sb = eg.summary(), eb.summary()
        assert {q: sg[q] for q in SUMMARY_SOLVER_KEYS} == {q: sb[q] for q in SUMMARY_SOLVER_KEYS}, i
        lg, lb_ = eg.local_clouds(), eb.local_clouds()
        assert all(np.array_equal(lg[q], lb_[q]) for q in lg), i
        for fr in range(W - O + 1, W + 1):
            assert all(np.array_equal(a, b) for a, b in zip(eg.features(fr), eb.features(fr))), (i, fr)
        # (2) the prediction
        tobe, aft, ins, info = eg.map_poses()
        d = np.linalg.inv(_T_state(st[W - 1])) @ _T_state(st[W])
        ref = _T(tobe_prev) @ _T(tlb) @ d @ np.linalg.inv(_T(tlb))
        got = _T(tobe.astype(np.float64))
        assert np.abs(got[:3, :3] - ref[:3, :3]).max() < 2e-5 and np.abs(got[:3, 3] - ref[:3, 3]).max() < 2e-5 * (1 + np.abs(ref[:3, 3]).max()), i
        assert np.array_equal(tobe, gmo.predict(tobe_prev.astype(np.float32), st[W - 1], st[W], s.seq.tf_lb7())), i   # the oracle formula
        assert np.array_equal(aft, aft0)
        # (3) the insert
        assert info["inserted"] == (i >= O), i
        if info["inserted"]:
            f = i + pivot - 1 if deskew else i + pivot          # frame id (warm-start frames 0..W-1, scan i is frame W + i)
            if deskew and pivot == 0:
                surf = own_prev
            else:
                surf = eg.frame(pivot - 1 if deskew else pivot)
            corner = pub_corner[f] if f in pub_corner else s.corner_ds[f]
            assert info["points"] == corner.shape[0] + surf.shape[0]
            pr.UpdateMapDatabase(corner, surf, valid, ins, centre)
            _same_map(pm, pr)
        pub_corner[i + pivot + 1] = lg["corner"]
        own_prev = eg.frame(0)
        # (4) publication
        calls += 1
        assert info["surround_published"] == (calls % 5 == 1), i
        if info["surround_published"]:
            acc = np.concatenate([pm.cube(idx, w) for idx in surround for w in ("corner", "surf")] + [np.zeros((0, 4), np.float32)])
            assert np.array_equal(pm.surround_map(), oracle.voxel_grid(acc, 0.6)), i
            assert info["surround_size"] == pm.surround_map().shape[0]
        assert np.array_equal(pm.registered_full_cloud(), pmp.associate_to_map(s.full[k], tobe)), i
    assert pm.centre() == centre and all(np.array_equal(a, b) for a, b in zip(pm.cube_lists(), (valid, surround)))


def test_attach_errors(oracle):
    """Every refusal of lio_est_attach_map / lio_est_map_poses and of the attached PointMapping's own entries; a refused attach
    changes nothing, and after the estimator is destroyed the map is released."""
    from lio_mapping_b200 import _lib, estimator
    from lio_mapping_b200.point_mapping import PointMapping
    W, O = 4, 4
    s = _Setup(oracle, W, O, 1)
    eg, pm = s.eg, s.pm
    with pytest.raises(_lib.LioError):
        eg.map_poses()                                            # nothing attached
    fresh = PointMapping(max_points=1 << 15)
    fresh.EnablePublish(0.6, 1 << 18)
    with pytest.raises(_lib.LioError):
        eg.attach_map(fresh)                                      # no process call yet
    plain = PointMapping(max_points=1 << 15)
    keep, ptrs, n, nn = _dev_inputs(s.corner[0], s.less_flat(0), s.full[0])
    plain.ProcessDev(ptrs, n.data_ptr(), [nn[0], nn[1], 0], np.array([0, 0, 0, 1, 0, 0, 0], np.float32))
    with pytest.raises(_lib.LioError):
        eg.attach_map(plain)                                      # does not publish
    leaf = PointMapping(max_points=1 << 15, surf_filter_size=0.5)
    leaf.EnablePublish(0.6, 1 << 18)
    leaf.ProcessDev(ptrs, n.data_ptr(), nn, np.array([0, 0, 0, 1, 0, 0, 0], np.float32))
    with pytest.raises(_lib.LioError):
        eg.attach_map(leaf)                                       # leaf sizes differ from the estimator's
    small = PointMapping(max_points=1 << 15)
    small.EnablePublish(0.6, 16)
    keep1, ptrs1, n1, _ = _dev_inputs(s.corner[0], s.less_flat(0), np.zeros((1, 4), np.float32))
    small.ProcessDev(ptrs1, n1.data_ptr(), [s.corner[0].shape[0], s.less_flat(0).shape[0], 1], np.array([0, 0, 0, 1, 0, 0, 0], np.float32))
    assert _lib.lib().lio_est_attach_map(eg.h, small.h) == -3    # LIO_ERR_CAPACITY: max_full_points below the estimator's
    no_lc = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17)
    helpers.warm_start(no_lc, s.seq, oracle, W, make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3)))
    with pytest.raises(_lib.LioError):
        no_lc.attach_map(pm)                                      # local clouds off
    no_init = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17)
    no_init.enable_local_clouds(0.2, 1 << 14, 1 << 18)
    with pytest.raises(_lib.LioError):
        no_init.attach_map(pm)                                    # before finish_init
    no_imu = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, imu_factor=0)
    no_imu.enable_local_clouds(0.2, 1 << 14, 1 << 18)
    helpers.warm_start(_Staging(no_imu, lambda k: (s.corner_ds[k], s.full[k])), s.seq, oracle, W,
                       make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3)))
    with pytest.raises(_lib.LioError, match="imu_factor"):
        no_imu.attach_map(pm)                                     # warm-started, imu_factor = 0
    eg.attach_map(pm)
    with pytest.raises(_lib.LioError):
        eg.attach_map(pm)                                         # twice
    with pytest.raises(_lib.LioError):
        s.eb.attach_map(pm)                                       # attached to another estimator
    with pytest.raises(_lib.LioError):
        pm.ProcessDev(ptrs, n.data_ptr(), nn, np.array([0, 0, 0, 1, 0, 0, 0], np.float32))
    with pytest.raises(_lib.LioError):
        pm.UpdateMapDatabase(s.corner_ds[0], s.less_flat(0), [0], np.array([0, 0, 0, 1, 0, 0, 0], np.float32), (10, 10, 5))
    assert _lib.lib().lio_pm_destroy(pm.h) == -2                  # LIO_ERR_INVALID
    pm.centre(); pm.update_stats(); pm.cube_sizes("surf"); pm.surround_map(); pm.registered_full_cloud()   # accessors keep working
    k = W
    eg.set_scan_clouds(s.corner[k], s.full[k])
    s.imu(eg, k)
    eg.process_scan(s.less_flat(k))
    s.eb.set_scan_clouds(s.corner[k], s.full[k])
    s.imu(s.eb, k)
    s.eb.process_scan(s.less_flat(k))
    with pytest.raises(_lib.LioError):
        s.eb.attach_map(s.pr)                                     # after the first scan
    eg.close()
    assert _lib.lib().lio_pm_destroy(pm.h) == 0                   # released
    pm.h = None


def test_staging_inside_an_open_scan_is_refused(oracle):
    """Stepwise API with a map attached: /cloud_registered registers the staged full cloud when the scan closes, so staging the next
    scan's clouds between open_scan and close_scan is refused (the estimator stays usable), and the registered cloud is the open
    scan's own; staging after close_scan works."""
    from lio_mapping_b200 import _lib
    from oracle import pm_publish_py as pmp
    W, O = 4, 4
    s = _Setup(oracle, W, O, 2)
    eg = s.eg
    eg.attach_map(s.pm)
    k = W
    eg.set_scan_clouds(s.corner[k], s.full[k])
    s.imu(eg, k)
    eg.open_scan(s.less_flat(k))
    with pytest.raises(_lib.LioError, match="stage"):
        eg.set_scan_clouds(s.corner[k + 1], s.full[k + 1])
    eg.close_scan()
    tobe, _, _, _ = eg.map_poses()
    assert np.array_equal(s.pm.registered_full_cloud(), pmp.associate_to_map(s.full[k], tobe))
    eg.set_scan_clouds(s.corner[k + 1], s.full[k + 1])
    s.imu(eg, k + 1)
    eg.process_scan(s.less_flat(k + 1))
    tobe, _, _, _ = eg.map_poses()
    assert np.array_equal(s.pm.registered_full_cloud(), pmp.associate_to_map(s.full[k + 1], tobe))


def test_attached_map_against_the_oracle_chain(oracle):
    """HDL-64 W 5 / O 4, O + 5 scans: the device estimator with the attached map beside the oracle chain (GlobalMapEstimator:
    orc::Estimator + PointMappingPublishOracle fed the same pre-initialisation calls).  Same insert and publish decisions on every
    scan.  The pre-initialisation maps differ by the mapper's parity (float GN on the device against the oracle's order), so:
    insert poses within 2e-4 m / 2e-5 (the mapping tolerance of tests/test_lidar_chain_gpu.py, the window states themselves agree
    to ~1e-7); /cloud_registered with the oracle's count and points within 2e-4 m + 2e-5 x range of it (the same pose bound at
    the cloud's range); every cube's point count within 3 % + 3 points of the oracle's, summed over each cloud within 1 %."""
    from oracle import global_map_py as gmo
    W, O = 5, 4
    s = _Setup(oracle, W, O, O + 5, opt_extrinsic=0)
    go = gmo.GlobalMapEstimator(corner_filter_size=0.2, window_size=W, opt_window_size=O, opt_extrinsic=0)
    tlb = s.seq.tf_lb7()
    for k in range(W):
        T = _T_state(s.seq.state16(k, None)) @ np.linalg.inv(_T(tlb))
        go.pre_init_process(s.corner[k], s.less_flat(k), s.full[k], np.r_[helpers.synth.rot_to_quat(T[:3, :3]), T[:3, 3]].astype(np.float32))
    helpers.warm_start(_Staging(go, lambda k: (s.corner_ds[k], s.full[k])), s.seq, oracle, W, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: oracle.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    eg = s.eg
    eg.attach_map(s.pm)
    for i in range(O + 5):
        k = W + i
        for e in (eg, go):
            e.set_scan_clouds(s.corner[k], s.full[k])
            s.imu(e, k)
            e.process_scan(s.less_flat(k))
        tg, ag, ig, infg = eg.map_poses()
        to, ao, io, info = go.map_poses()
        assert (infg["inserted"], infg["surround_published"]) == (info["inserted"], info["surround_published"]), i
        if infg["inserted"]:
            assert np.abs(ig[4:] - io[4:]).max() <= 2e-4 and min(np.abs(ig[:4] - io[:4]).max(), np.abs(ig[:4] + io[:4]).max()) <= 2e-5, i
        rg, ro = s.pm.registered_full_cloud(), go.cloud("registered")
        assert rg.shape == ro.shape and np.array_equal(rg[:, 3], ro[:, 3])
        assert np.all(np.abs(rg[:, :3] - ro[:, :3]).max(1) <= 2e-4 + 2e-5 * np.linalg.norm(ro[:, :3], axis=1)), i
    for which in ("corner", "surf"):
        sg, so = s.pm.cube_sizes(which), go.cube_sizes(which)
        assert np.all(np.abs(sg - so) <= 0.03 * so + 3), which
        assert abs(int(sg.sum()) - int(so.sum())) <= 0.01 * so.sum(), which


def test_device_resident_chain_equals_host_entries(oracle):
    """Stage A (process_device) -> lio_po_process_dev -> lio_pm_process_dev over the warm-start sweeps -> attach ->
    lio_est_set_scan_clouds_dev / lio_est_process_scan_dev on stage A's outputs in HBM, against the same chain through host copies
    (stage-A downloads, PointOdometry.Process, compact_data, the mapper fed uploaded copies, set_scan_clouds / process_scan from
    host arrays): states, map poses and info, the registered cloud and every cube bit-identical."""
    from lio_mapping_b200 import estimator, wire
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from tests.test_lidar_chain_gpu import StageA
    W, O = 5, 4
    s = _Setup(oracle, W, O, O + 3)
    seq = s.seq
    max_raw = max(r.shape[0] for r in seq.raw)
    sa = StageA(seq.sensor, max_raw)
    od, oh = PointOdometry(0.1, 1, 25, max_full_points=max_raw), PointOdometry(0.1, 1, 25, max_full_points=max_raw)
    md, mh = PointMapping(max_points=1 << 17), PointMapping(max_points=1 << 17)
    for m in (md, mh):
        m.EnablePublish(0.6, max_raw)
    keep = []
    for k in range(W):
        raw = np.ascontiguousarray(seq.raw[k], np.float32)
        ptrs = sa.run(raw)
        td, _, idv = od.ProcessDev(ptrs, sa.n_dev, [1 << 17] * 4 + [max_raw])
        th, _, ih = oh.Process(*sa.host())
        assert np.array_equal(th, td) and ih == idv
        if idv["published"]:
            cptr, cn_dev, cn = od.clouds_dev()
            a = md.ProcessDev(cptr, cn_dev, cn, td)
            tf7, c, sf, full = wire.compact_decode(oh.compact_data())
            keep.append(_dev_inputs(c, sf, full))
            b = mh.ProcessDev(keep[-1][1], keep[-1][2].data_ptr(), keep[-1][3], tf7)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    _same_map(md, mh)
    eh, ed = s.eg, s.eb      # identical warm starts, local clouds on
    ed.attach_map(md)
    eh.attach_map(mh)
    idx = {name: i for i, name in enumerate(("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat",
                                               "surface_points_less_flat", "cloud_in_rings"))}
    for i in range(O + 3):
        k = W + i
        raw = np.ascontiguousarray(seq.raw[k], np.float32)
        ptrs = sa.run(raw)
        host = sa.host()
        ed.set_scan_clouds_dev(ptrs[idx["corner_points_less_sharp"]], sa.n_dev[idx["corner_points_less_sharp"]], 1 << 17,
                               ptrs[idx["cloud_in_rings"]], sa.n_dev[idx["cloud_in_rings"]], max_raw)
        eh.set_scan_clouds(host[idx["corner_points_less_sharp"]], host[idx["cloud_in_rings"]])
        for e in (ed, eh):
            s.imu(e, k)
        ed.process_scan_dev(ptrs[idx["surface_points_less_flat"]], sa.n_dev[idx["surface_points_less_flat"]], 1 << 17)
        eh.process_scan(host[idx["surface_points_less_flat"]])
        assert np.array_equal(ed.states(), eh.states()), i
        pd_, ph_ = ed.map_poses(), eh.map_poses()
        assert all(np.array_equal(a, b) for a, b in zip(pd_[:3], ph_[:3])) and pd_[3] == ph_[3], i
        assert np.array_equal(md.registered_full_cloud(), mh.registered_full_cloud()), i
        if pd_[3]["surround_published"]:
            assert np.array_equal(md.surround_map(), mh.surround_map()), i
    _same_map(md, mh)
