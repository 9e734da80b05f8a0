"""The device estimator with imu_factor = 0 fed the odometry's /compact_data clouds (lio_est_attach_mapping /
lio_est_process_compact_*): PointMapping::Process on every message, the NOT_INITED window of mapped poses with its decimation, the
start-up from the pushed laser transforms, and the INITED lidar-only solve with the map insert of each frame's saved valid list and
cube centre (Estimator.cc:430-856, :1670-1676; PointMapping.cc:765-1052)."""
import numpy as np
import pytest

from tests import helpers
from tests.test_global_map_gpu import _T, _T_state, _dev_inputs, _same_map
from tests.test_local_clouds_gpu import _stage_a

pytestmark = pytest.mark.gpu

MAX_FRAME, MAX_SCAN, MAX_CORNER = 1 << 15, 1 << 17, 1 << 14


class _Drive:
    """An HDL-64 drive with its stage-A clouds and the ground-truth lidar pose relative to the first sweep as /laser_odom_to_init
    (transform_sum_ starts at identity like the odometry's), and the ground-truth body positions in that frame."""

    def __init__(self, oracle, n):
        self.seq = seq = helpers.Sequence(oracle, "hdl64", n_total=n)
        self.corner, self.full = _stage_a(oracle, seq)
        self.max_full = max(f.shape[0] for f in self.full)
        tlb = _T(seq.tf_lb7())
        T0inv = np.linalg.inv(_T_state(seq.state16(0, None)) @ np.linalg.inv(tlb))
        self.sum7, self.gt_p = [], []
        for k in range(n):
            Tb = T0inv @ _T_state(seq.state16(k, None))
            T = Tb @ np.linalg.inv(tlb)
            self.sum7.append(np.r_[helpers.synth.rot_to_quat(T[:3, :3]), T[:3, 3]].astype(np.float32))
            self.gt_p.append(Tb[:3, 3])

    def clouds(self, k):
        return self.corner[k], self.seq.less_flat[k], self.full[k]

    def imu(self, e, k):
        if k == 0:
            return
        tt, acc, gyr = self.seq.imu[k]
        last = self.seq.t[k - 1]
        for j in range(len(tt)):
            e.process_imu(tt[j] - last, acc[j], gyr[j], tt[j])
            last = tt[j]


def _make(drive, W, O, f, **cfg):
    from lio_mapping_b200 import estimator
    from lio_mapping_b200.point_mapping import PointMapping
    e = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=MAX_FRAME, max_scan_points=MAX_SCAN, imu_factor=0,
                            init_window_factor=f, opt_extrinsic=0, **cfg)
    e.set_extrinsic(drive.seq.tf_lb7())
    e.enable_local_clouds(0.2, MAX_CORNER, drive.max_full)
    pm = PointMapping(max_points=1 << 17)
    pm.EnablePublish(0.6, drive.max_full)
    e.attach_mapping(pm)
    return e, pm


def _run(drive, W, O, f, n, dev=False, **cfg):
    """Feed n messages; returns (estimator, map, per-message status / map_poses / cube lists)."""
    e, pm = _make(drive, W, O, f, **cfg)
    log = []
    for k in range(n):
        drive.imu(e, k)
        if dev:
            keep, ptrs, nd, nn = _dev_inputs(*drive.clouds(k))
            st = e.process_compact_dev(ptrs, nd.data_ptr(), nn, drive.sum7[k])
        else:
            st = e.process_compact(*drive.clouds(k), drive.sum7[k])
        log.append((st, e.map_poses(), pm.cube_lists(), pm.centre()))
    return e, pm, log


# The drift bound is 0.2 m, except with enable_deskew alone: the scan is then de-skewed with transform_es_, which comes from IMU
# propagation with velocities that the lidar-only solve never estimates (as in the reference), and the window drifts further.
CONFIGS = [
    pytest.param(5, 4, 1, dict(enable_deskew=0, cutoff_deskew=0), 0.2, id="W5O4-f1-no_deskew"),
    pytest.param(4, 4, 2, dict(enable_deskew=0, cutoff_deskew=0), 0.2, id="W4O4-f2-no_deskew"),
    pytest.param(5, 4, 1, {}, 0.2, id="W5O4-f1-cutoff_deskew"),
    pytest.param(4, 4, 1, dict(cutoff_deskew=0), 0.5, id="W4O4-f1-enable_deskew"),
]


@pytest.mark.parametrize("W,O,f,extra,drift", CONFIGS)
def test_lidar_only_follows_the_reference(oracle, W, O, f, extra, drift):
    """(1) The decisions of ProcessLaserOdom: before initialisation only every f-th message pushes, cir_buf_count_ counts the pushes up
    to W, the (W+1)-th push solves once and initialises, then every message pushes and solves.  (2) Until and including the start-up
    message the estimator's mapping is bit-equal to a plain publishing PointMapping fed the same messages (Process in full: its poses,
    every cube).  (3) After it, no Process inserts: the replay map receives only the estimator's inserts, from the (O+1)-th INITED
    message on, each replayed bit for bit through lio_pm_update_map_database_host with the clouds the aliasing rules select from the
    device's own slots, the reported pose and THAT frame's saved valid list and centre; the surround map every 5th message counting
    all messages; the registered cloud is the message's full cloud with the final tobe; aft is live.  (4) The run repeats bit for bit.
    (5) The window's body positions stay within `drift` of ground truth."""
    from oracle import pm_publish_py as pmp
    from lio_mapping_b200.point_mapping import PointMapping
    n_inited = O + 5
    n = f * W + 1 + n_inited                      # W pushes, the start-up push, then the INITED messages
    n += (f - (f * W + 1) % f) % f                # the start-up message is a multiple of f
    drive = _Drive(oracle, n + 1)
    e, pm = _make(drive, W, O, f, **extra)
    pr = PointMapping(max_points=1 << 17)
    pr.EnablePublish(0.6, drive.max_full)
    deskew = bool(extra.get("enable_deskew", 1) or extra.get("cutoff_deskew", 1))
    pivot = W - O
    pushes, inited_msgs, start_msg = 0, 0, None
    valid_of, centre_of, pub_corner = {}, {}, {}
    own_prev = None
    for k in range(n):
        drive.imu(e, k)
        was_inited = start_msg is not None
        st = e.process_compact(*drive.clouds(k), drive.sum7[k])
        tobe, aft, ins, info = e.map_poses()
        m = k + 1
        # (1) the decisions
        push = was_inited or m % f == 0
        assert st["pushed"] == push, k
        if push:
            fid = pushes
            pushes += 1
            valid_of[fid] = pm.cube_lists()[0]
            centre_of[fid] = pm.centre()
        if not was_inited:
            startup = push and pushes == W + 1
            assert st["solved"] == startup and st["inited"] == startup, k
            assert st["cir_buf_count"] == min(pushes, W), k
            keep, ptrs, nd, nn = _dev_inputs(*drive.clouds(k))
            r_tobe, r_aft, _ = pr.ProcessDev(ptrs, nd.data_ptr(), nn, drive.sum7[k])
            # (2) Process in full, bit-equal to a plain PointMapping
            assert np.array_equal(tobe, r_tobe) and np.array_equal(aft, r_aft), k
            _same_map(pm, pr)
            assert not info["inserted"]
            if startup:
                start_msg = k
                pub_corner[fid - O + 1] = e.local_clouds()["corner"]
                own_prev = e.frame(0)
            continue
        assert st["solved"] and st["inited"] and st["cir_buf_count"] == W, k
        inited_msgs += 1
        i = inited_msgs - 1                        # 0-based INITED message, pushed as frame W + 1 + i
        # (3) the insert and the publication
        assert info["inserted"] == (i >= O), k
        if info["inserted"]:
            f_opt = W + 1 + i - O                   # opt_*.first(): its valid list and centre
            f_cloud = f_opt - (1 if deskew else 0)  # the clouds its stack entries alias (see lio_est_attach_map)
            surf = own_prev if (deskew and pivot == 0) else e.frame(pivot - 1 if deskew else pivot)
            corner = pub_corner[f_cloud]
            assert info["points"] == corner.shape[0] + surf.shape[0], k
            pr.UpdateMapDatabase(corner, surf, valid_of[f_opt], ins, centre_of[f_opt])
        _same_map(pm, pr)
        assert info["surround_published"] == (m % 5 == 1), k
        if info["surround_published"]:
            acc = np.concatenate([pm.cube(idx, w) for idx in pm.cube_lists()[1] for w in ("corner", "surf")] + [np.zeros((0, 4), np.float32)])
            assert np.array_equal(pm.surround_map(), oracle.voxel_grid(acc, 0.6)), k
        assert np.array_equal(pm.registered_full_cloud(), pmp.associate_to_map(drive.full[k], tobe)), k
        pub_corner[W + 1 + i - O + 1] = e.local_clouds()["corner"]
        own_prev = e.frame(0)
    assert start_msg == f * (W + 1) - 1 and inited_msgs == n_inited
    # (4) the same run again, bit for bit
    e2, pm2, log2 = _run(drive, W, O, f, n, **extra)
    assert np.array_equal(e.states(), e2.states())
    _same_map(pm, pm2)
    assert all(np.array_equal(a, b) for a, b in zip(e.map_poses()[:3], e2.map_poses()[:3]))
    # (5) drift: logical frame j < W holds message n - W + j
    st_ = e.states()
    gt = np.array([drive.gt_p[n - W + j] for j in range(W)])
    err = np.abs(st_[:W, 0:3] - gt).max()
    assert err < drift, err


def test_device_entry_matches_host_entry(oracle):
    """lio_est_process_compact_dev with the clouds in HBM and lio_est_process_compact_host ("upload, then the same steps") give
    bit-identical states, maps, poses, local clouds and decisions, message by message."""
    W, O, f = 5, 4, 1
    n = W + 1 + O + 3
    drive = _Drive(oracle, n + 1)
    eh, pmh, logh = _run(drive, W, O, f, n)
    ed, pmd, logd = _run(drive, W, O, f, n, dev=True)
    for (sh, mh, ch, zh), (sd, md, cd, zd) in zip(logh, logd):
        assert sh == sd and mh[3] == md[3] and zh == zd
        assert all(np.array_equal(a, b) for a, b in zip(mh[:3], md[:3]))
        assert all(np.array_equal(a, b) for a, b in zip(ch, cd))
    assert np.array_equal(eh.states(), ed.states())
    _same_map(pmh, pmd)
    lh, ld = eh.local_clouds(), ed.local_clouds()
    assert all(np.array_equal(lh[q], ld[q]) for q in lh)


def test_lidar_only_errors(oracle):
    """Every refusal of lio_est_attach_mapping (nothing changes), process_scan / init_frame on an attached estimator, attach_map
    still refusing imu_factor = 0, init_window_factor = 0, and a count above n3_max (the context is then poisoned)."""
    from lio_mapping_b200 import _lib, estimator
    from lio_mapping_b200.point_mapping import PointMapping
    W, O = 4, 4
    drive = _Drive(oracle, 2)

    def est(**cfg):
        kw = dict(window_size=W, opt_window_size=O, max_frame_points=MAX_FRAME, max_scan_points=MAX_SCAN, imu_factor=0)
        kw.update(cfg)
        return estimator.Estimator(**kw)

    def pmap(publish=True, **kw):
        p = PointMapping(max_points=1 << 17, **kw)
        if publish:
            p.EnablePublish(0.6, drive.max_full)
        return p

    with pytest.raises(_lib.LioError):
        est(init_window_factor=0)
    no_lc = est()
    with pytest.raises(_lib.LioError, match="local clouds"):
        no_lc.attach_mapping(pmap())
    imu = est(imu_factor=1)
    imu.enable_local_clouds(0.2, MAX_CORNER, drive.max_full)
    with pytest.raises(_lib.LioError, match="imu_factor"):
        imu.attach_mapping(pmap())
    e = est()
    e.enable_local_clouds(0.2, MAX_CORNER, drive.max_full)
    with pytest.raises(_lib.LioError):
        e.attach_mapping(pmap(publish=False))                     # does not publish
    with pytest.raises(_lib.LioError):
        e.attach_mapping(pmap(surf_filter_size=0.5))              # leaf sizes differ
    used = pmap()
    keep, ptrs, nd, nn = _dev_inputs(*drive.clouds(0))
    used.ProcessDev(ptrs, nd.data_ptr(), nn, drive.sum7[0])
    with pytest.raises(_lib.LioError, match="no process call"):
        e.attach_mapping(used)                                    # not fresh
    small = PointMapping(max_points=1 << 17)
    small.EnablePublish(0.6, 16)
    assert _lib.lib().lio_est_attach_mapping(e.h, small.h) == -3  # LIO_ERR_CAPACITY
    with pytest.raises(_lib.LioError):
        e.compact_status()                                        # nothing attached: the refusals changed nothing
    pm = pmap()
    e.attach_mapping(pm)
    with pytest.raises(_lib.LioError):
        e.attach_mapping(pmap())                                  # twice
    with pytest.raises(_lib.LioError):
        e.attach_map(pm)                                          # a mapping is attached
    with pytest.raises(_lib.LioError, match="mapping"):
        e.process_scan(drive.seq.less_flat[0])
    with pytest.raises(_lib.LioError):
        e.init_frame(0, drive.seq.state16(0), drive.seq.less_flat[0][:10], None)
    with pytest.raises(_lib.LioError):
        pm.Process(drive.corner[0], drive.seq.less_flat[0], drive.sum7[0])   # the attached map refuses its own calls
    e.set_extrinsic(drive.seq.tf_lb7())
    st = e.process_compact(*drive.clouds(0), drive.sum7[0])
    assert st == dict(inited=False, cir_buf_count=1, pushed=True, solved=False)
    keep, ptrs, nd, nn = _dev_inputs(*drive.clouds(1))
    with pytest.raises(_lib.LioError, match="n3_max"):
        e.process_compact_dev(ptrs, nd.data_ptr(), [nn[0] - 1, nn[1], nn[2]], drive.sum7[1])
    with pytest.raises(_lib.LioError, match="poisoned"):
        e.process_compact(*drive.clouds(1), drive.sum7[1])
    e.close()
    pm.close()
    assert pm.h is None                                           # released with the estimator


@pytest.mark.parametrize("W,O,f,extra", [
    pytest.param(5, 4, 1, dict(enable_deskew=0, cutoff_deskew=0), id="W5O4-f1-no_deskew"),
    pytest.param(4, 4, 2, {}, id="W4O4-f2-cutoff_deskew"),
])
def test_device_against_the_oracle_chain(oracle, W, O, f, extra):
    """The device against oracle/o_lidar_only.cc fed the same messages (no IMU input): every decision (push, start-up, solve, insert,
    Process and estimator publication) equal; before the start-up the mapped poses within lio_pm's parity bounds (2e-4 position,
    2e-5 quaternion); the window states after every solve within max(1e-3, 30 x the oracle's own divergence when its start-up
    positions move by 2e-4 m, the mapping's parity bound), so the bound is measured: the device's mapping is not bit-equal to the
    oracle's after its first frame, which moves the pushed laser transforms by up to that much."""
    from oracle import lidar_only_py as lo
    n = f * (W + 1) + O + 4
    drive = _Drive(oracle, n)
    e, pm = _make(drive, W, O, f, **extra)
    kw = dict(window_size=W, opt_window_size=O, opt_extrinsic=0, **extra)
    o = lo.LidarOnlyEstimator(init_window_factor=f, **kw)
    o2 = lo.LidarOnlyEstimator(init_window_factor=f, start_shift=2e-4, **kw)
    for x in (o, o2):
        x.set_extrinsic(drive.seq.tf_lb7())
    worst = []
    for k in range(n):
        sg = e.process_compact(*drive.clouds(k), drive.sum7[k])
        so = o.process_compact(*drive.clouds(k), drive.sum7[k])
        o2.process_compact(*drive.clouds(k), drive.sum7[k])
        assert sg == so, (k, sg, so)
        tg, ag, _, ig = e.map_poses()
        to, ao, _, io = o.map_poses()
        assert ig["inserted"] == io["inserted"] and ig["surround_published"] == io["surround_published"], k
        if not sg["inited"]:
            assert np.abs(ag[4:] - ao[4:]).max() <= 2e-4 and np.abs(ag[:4] - ao[:4]).max() <= 2e-5, (k, ag, ao)
            continue
        if ig["inserted"]:
            assert ig["points"] == io["points"] or abs(ig["points"] - io["points"]) <= 2 + 0.01 * io["points"], k
        s_g, s_o, s_o2 = e.states(), o.states(), o2.states()
        div = np.abs(s_o2[:, :7] - s_o[:, :7]).max()
        diff = np.abs(s_g[:, :7] - s_o[:, :7]).max()
        worst.append((diff, div))
        assert diff <= max(1e-3, 30 * div), (k, diff, div)
    assert worst


def test_compact_capacity(oracle):
    """A full-cloud bound above the local full capacity is refused with LIO_ERR_CAPACITY before anything changes."""
    from lio_mapping_b200 import _lib
    drive = _Drive(oracle, 2)
    e, pm = _make(drive, 4, 4, 1)
    big = np.zeros((drive.max_full + 1, 4), np.float32)
    assert _lib.lib().lio_est_process_compact_host(e.h, drive.corner[0], drive.corner[0].shape[0], drive.seq.less_flat[0],
                                                   drive.seq.less_flat[0].shape[0], big, big.shape[0], drive.sum7[0]) == -3
    assert e.compact_status() == dict(inited=False, cir_buf_count=0, pushed=False, solved=False)
    st = e.process_compact(*drive.clouds(0), drive.sum7[0])   # not poisoned
    assert st["pushed"] and st["cir_buf_count"] == 1
