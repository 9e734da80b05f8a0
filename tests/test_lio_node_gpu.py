"""lio_node: processor_node + estimator_node as one handle (raw sweeps and IMU messages in).  The node must equal the same inner handles
wired by hand here - stage A, PointOdometry, the estimator with its attached PointMapping, the pairing by the restatement of
tests/test_measurement_pairing.py and the /enable_odom call made by the test - bit for bit, message by message; and lio_pp_process_dev_ring
must equal lio_pp_process_host_ring."""
import dataclasses

import numpy as np
import pytest

from lio_mapping_b200 import synth
from tests.test_global_map_gpu import _same_map
from tests.test_imu_startup_gpu import _rigid_residual
from tests.test_measurement_pairing import Restated

pytestmark = pytest.mark.gpu

LIO_ERR_INVALID, LIO_ERR_CAPACITY = -2, -3
MAX_POINTS, MAX_FEAT = 1 << 18, 1 << 16
RS32 = synth.Sensor("rs32", 32, -25.0, 15.0, 1800, 100.0)   # the 320 preset's geometry (processor_node.cc:72-73)
BIAS = np.array([0.02, -0.03, 0.025])


def _rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _rings(sensor, xyzi):
    """A ring index per point from its elevation (the synthetic sensors fire rings at evenly spaced elevations)."""
    el = np.degrees(np.arctan2(xyzi[:, 2], np.hypot(xyzi[:, 0], xyzi[:, 1])))
    return np.clip(np.rint((el - sensor.lower_deg) / (sensor.upper_deg - sensor.lower_deg) * (sensor.rings - 1)), 0, sensor.rings - 1).astype(np.uint16)


class _RawDrive:
    """n motion-distorted sweeps ending at t0 + 0.1 k and one continuous 200 Hz IMU stream (gyro bias added), lidar mounted at (R_lb,
    t_lb).  arrivals(): every IMU message up to a sweep's stamp, then the sweep (what a robot's drivers deliver in time order)."""

    def __init__(self, kind, n, k=0.25, bias=BIAS, R_lb=np.eye(3), t_lb=(0.0, 0.0, -0.1), sensor=None, seed=300, t0=1.0):
        s0, scene, traj = synth.default_config(kind)
        self.sensor = sensor or s0
        self.traj = traj = dataclasses.replace(traj, k_roll=k, k_pitch=k)
        self.R_lb, self.t_lb = np.asarray(R_lb, np.float64), np.asarray(t_lb, np.float64)
        self.t = t0 + 0.1 * np.arange(n)
        self.raw = [synth.make_sweep(self.sensor, scene, traj, float(t), seed=seed + i, R_lb=self.R_lb, t_lb=self.t_lb, distort=True)
                    for i, t in enumerate(self.t)]
        self.max_raw = max(r.shape[0] for r in self.raw)
        self.imu_t, acc, gyr = synth.make_imu(traj, t0 - 0.1, float(self.t[-1]) + 0.2, 200.0)
        self.imu_acc, self.imu_gyr = acc, gyr + np.asarray(bias, np.float64)

    def tf_lb7(self):
        return np.r_[synth.rot_to_quat(self.R_lb), self.t_lb].astype(np.float32)

    def arrivals(self):
        out, j = [], 0
        for i, t in enumerate(self.t):
            while j < len(self.imu_t) and self.imu_t[j] <= t:
                out.append(("imu", float(self.imu_t[j]), tuple(self.imu_acc[j]), tuple(self.imu_gyr[j])))
                j += 1
            out.append(("sweep", float(t), i))
        return out

    def gt_positions(self, stamps):
        return self.traj.state(np.asarray(stamps))[0]


_DRIVES = {}


def _drive(name, n):
    key = (name, n)
    if key not in _DRIVES:
        if name == "hdl64":
            _DRIVES[key] = _RawDrive("hdl64", n)
        elif name == "hdl64_rot":   # test_extrinsic_calibration_gpu's mounting, amplitude 0.75 so that calibration succeeds
            _DRIVES[key] = _RawDrive("hdl64", n, k=0.75, R_lb=_rot_x(0.15))
        else:
            _DRIVES[key] = _RawDrive("vlp16", n, k=0.03, bias=np.zeros(3))
    return _DRIVES[key]


# (drive, sweeps, sensor_type, odom_io, delay, estimator config, extrinsic guess)
SHAPES = {
    "outdoor_64": ("hdl64", 66, 64, 3, 0.0, dict(window_size=7, opt_window_size=5, init_window_factor=1, enable_deskew=0, cutoff_deskew=1,
                                                 prior_factor=1, imu_factor=1, estimate_extrinsic=1, opt_extrinsic=0, keep_features=0), None),
    "indoor": ("hdl64_rot", 96, 64, 2, 0.05, dict(window_size=12, opt_window_size=7, init_window_factor=2, enable_deskew=1, cutoff_deskew=0,
                                                 prior_factor=0, imu_factor=1, estimate_extrinsic=2, opt_extrinsic=1, keep_features=1), "identity"),
    "vlp16_imu0": ("vlp16", 30, 16, 2, 0.0, dict(window_size=5, opt_window_size=4, init_window_factor=1, enable_deskew=0, cutoff_deskew=0,
                                                 prior_factor=0, imu_factor=0, estimate_extrinsic=0, opt_extrinsic=0, keep_features=0), None),
}
COMMON = dict(acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5, g_norm=9.805, min_match_sq_dis=1.0, min_plane_dis=0.2, surf_filter_size=0.4,
              max_frame_points=1 << 15, max_scan_points=1 << 17)


def _shape(name):
    dname, n, st, io, delay, est, guess = SHAPES[name]
    drive = _drive(dname, n)
    tf = drive.tf_lb7()
    if guess == "identity":
        tf = np.r_[0.0, 0.0, 0.0, 1.0, drive.t_lb].astype(np.float32)
    return drive, dict(sensor_type=st, odom_io=io, msg_time_delay=delay, tf_lb7=tf, max_points=MAX_POINTS, max_feature_points=MAX_FEAT,
                       **COMMON, **est)


def _node(kw, **over):
    from lio_mapping_b200 import LioNode
    return LioNode(**dict(kw, **over))


class _HandWired:
    """The same handles wired by hand: stage A from host clouds, lio_po_process_dev on stage A's outputs, the published clouds downloaded
    and kept until the restated pairing releases them, then the ProcessImu calls and the stamped host compact entry; the test makes the
    /enable_odom call."""

    def __init__(self, kw):
        from lio_mapping_b200 import estimator
        from lio_mapping_b200.point_mapping import PointMapping
        from lio_mapping_b200.point_odometry import PointOdometry
        from lio_mapping_b200.point_processor import PointProcessor
        st = kw["sensor_type"]
        lo, hi, R = {16: (-15.0, 15.0, 16), 32: (-30.67, 10.67, 32), 64: (-24.9, 2.0, 64), 320: (-25.0, 15.0, 32)}[st]
        self.ring = st == 320
        self.pp = PointProcessor(lo, hi, R, max_points=kw["max_points"])
        self.po = PointOdometry(0.1, kw["odom_io"], 25, kw["max_feature_points"], kw["max_points"])
        self.pm = PointMapping(max_points=kw["max_feature_points"], corner_filter_size=0.2, surf_filter_size=0.4, min_match_sq_dis=1.0,
                               min_plane_dis=0.2, max_iterations=10)
        self.pm.EnablePublish(0.6, kw["max_points"])
        est = {k: v for k, v in kw.items() if k in dict(estimator._lib.EstConfig._fields_)}
        self.e = estimator.Estimator(**est)
        self.e.set_extrinsic(kw["tf_lb7"])
        self.e.enable_local_clouds(0.2, kw["max_feature_points"], kw["max_points"])
        if est["imu_factor"] and est["estimate_extrinsic"] == 2:
            self.e.enable_extrinsic_calibration()
        (self.e.attach_imu_mapping if est["imu_factor"] else self.e.attach_mapping)(self.pm)
        self.pairing = Restated(kw["msg_time_delay"])
        self.F, self.N = kw["max_feature_points"], kw["max_points"]
        self.deskew = bool(est["enable_deskew"] or est["cutoff_deskew"])
        self.imu_factor = bool(est["imu_factor"])
        self.pending, self.inited, self.odom_on, self.odom_off_at = {}, False, True, None
        self.sweeps = 0
        self.processed = []

    def push(self, i, a, rings=None):
        if a[0] == "sweep":
            self.pp.SetInputCloud(a[3])
            if self.ring:
                self.pp.ProcessWithRingField(rings)
            else:
                self.pp.Process()
            names = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")
            ts, _, info = self.po.ProcessDev([self.pp.cloud_dev(n) for n in names], [self.pp.cloud_count_dev(n) for n in names],
                                             [self.F] * 4 + [self.N])
            self.sweeps += 1
            if not info["published"]:
                return
            self.pending[i] = (self.po.cloud("last_corner"), self.po.cloud("last_surf"), self.po.cloud("full"), ts.copy(), a[1])
            a = ("msg", a[1])
        for idx, processed, calls in self.pairing.push(i, a):
            c, s, f, ts, stamp = self.pending.pop(idx)
            if not processed:
                continue
            for dt, ax, ay, az, rx, ry, rz, t in calls:
                self.e.process_imu(dt, np.array([ax, ay, az]), np.array([rx, ry, rz]), t)
            st = self.e.process_compact(c, s, f, ts, stamp=stamp)
            if self.imu_factor and not self.inited and st["inited"] and self.deskew:
                self.po.EnableOdom(False)
                self.odom_on, self.odom_off_at = False, self.sweeps
            self.inited = st["inited"]
            self.processed.append(stamp)


def _snapshot(e):
    s = e.imu_init_status()
    c = e.extrinsic_calib_status()
    tobe, aft, ins, info = e.map_poses()
    return (e.states().copy(), s["attempts"], s["outcome"], s["inited"], s["g_vec"].copy(), s["R_WI"].copy(), c["runs"], c["result"],
            e.extrinsic().copy(), tobe.copy(), aft.copy(), ins.copy(), tuple(sorted(info.items())))


def _same_snapshot(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert np.array_equal(x, y, equal_nan=True)
        else:
            assert x == y


def _run_node(drive, kw, arrivals=None, dev=False):
    """Feeds the node; returns (node, snapshots after every arrival that processed a message, sweep index of the odometry switch)."""
    import torch
    node = _node(kw)
    snaps, off_at, done = [], None, 0
    for a in arrivals or drive.arrivals():
        if a[0] == "imu":
            node.push_imu(a[1], a[2], a[3])
        elif dev:
            t = torch.from_numpy(np.ascontiguousarray(drive.raw[a[2]], np.float32)).cuda()
            node.push_sweep_dev(t.data_ptr(), t.shape[0], a[1])
            torch.cuda.synchronize()
        else:
            node.push_sweep(drive.raw[a[2]], a[1])
        st = node.status()
        if off_at is None and not st["odom_enabled"]:
            off_at = st["sweeps"]
        if st["processed"] != done:
            done = st["processed"]
            snaps.append(_snapshot(node.estimator))
    return node, snaps, off_at


@pytest.mark.parametrize("shape", list(SHAPES))
def test_node_equals_the_hand_wired_chain(shape):
    """Every estimator state, imu_init_status, the extrinsic, its calibration and map_poses after every processed message, then the cube
    map, the surround map and /cloud_registered: the node against the hand-wired chain, bit for bit; the run repeats bit for bit; the
    odometry goes to pass-through exactly once, on the sweep after the initialising message, only with imu_factor = 1 and a de-skew flag;
    and the window stays near ground truth after a rigid alignment."""
    drive, kw = _shape(shape)
    hw = _HandWired(kw)
    ref, done = [], 0
    for i, a in enumerate(drive.arrivals()):
        if a[0] == "sweep":
            hw.push(i, ("sweep", a[1], a[2], drive.raw[a[2]]))
        else:
            hw.push(i, a)
        if len(hw.processed) != done:
            done = len(hw.processed)
            ref.append(_snapshot(hw.e))
    node, snaps, off_at = _run_node(drive, kw)
    st = node.status()
    assert st["processed"] == len(hw.processed) and st["sweeps"] == hw.sweeps
    assert len(snaps) == len(ref) and len(snaps) > 0
    for a, b in zip(snaps, ref):
        _same_snapshot(a, b)
    _same_map(node.mapping, hw.pm)
    assert np.array_equal(node.mapping.surround_map(), hw.pm.surround_map())
    assert np.array_equal(node.mapping.registered_full_cloud(), hw.pm.registered_full_cloud())
    assert st["last_stamp"] == hw.processed[-1]
    # the /enable_odom switch
    want_switch = kw["imu_factor"] == 1 and bool(kw["enable_deskew"] or kw["cutoff_deskew"])
    assert st["inited"], shape
    assert (off_at is not None) == want_switch and st["odom_enabled"] == (not want_switch)
    if want_switch:
        assert off_at == hw.odom_off_at   # switched during the push that processed the initialising message: the next sweep runs without
    # repeatability
    node2, snaps2, off2 = _run_node(drive, kw)
    assert off2 == off_at and len(snaps2) == len(snaps)
    for a, b in zip(snaps, snaps2):
        _same_snapshot(a, b)
    _same_map(node.mapping, node2.mapping)
    # ground truth: the window's W + 1 frames are the last W + 1 processed messages
    W = kw["window_size"]
    err = _rigid_residual(node.states()[:, 0:3], drive.gt_positions(hw.processed[-(W + 1):]))
    calib = node.extrinsic_calib_status()
    print(f"{shape}: {st}; window position error after rigid alignment {err:.3f} m; calibration {calib['runs']} run(s), result {calib['result']}")
    assert err < GT_BOUND[shape]


# Largest window position error (m) after a rigid alignment at the end of each drive.  Measured on an H100 80GB HBM3 at 700 W: 1.178 m
# (outdoor_64), 0.756 m (indoor, one calibration, successful) and 0.059 m (vlp16_imu0).  The raw sweeps here are motion-distorted and the
# messages come every odom_io sweeps, so the imu_factor = 1 drives sit above the 0.33-0.41 m of test_imu_startup_gpu's undistorted,
# every-sweep messages.
GT_BOUND = {"outdoor_64": 1.5, "indoor": 1.0, "vlp16_imu0": 0.1}


def test_sweeps_ahead_of_their_imu_and_the_queue_bound():
    """A second of sweeps pushed before their IMU gives what time-ordered pushing gives; one sweep past max_pending returns
    LIO_ERR_CAPACITY and changes nothing."""
    from lio_mapping_b200 import _lib
    drive, kw = _shape("outdoor_64")
    arr = drive.arrivals()
    sweeps_first = [a for a in arr if a[0] == "sweep" and a[1] <= drive.t[0] + 1.0]
    ahead = [a for a in arr if a[0] == "imu" and a[1] <= drive.t[0]] + sweeps_first + \
        [a for a in arr if not (a[0] == "imu" and a[1] <= drive.t[0]) and a not in sweeps_first]
    _, ordered, _ = _run_node(drive, kw, arr)
    node, early, _ = _run_node(drive, kw, ahead)
    assert len(ordered) == len(early)
    for a, b in zip(ordered, early):
        _same_snapshot(a, b)
    # max_pending 2 with odom_io 1: the third published sweep ahead of the IMU is refused
    n = _node(kw, odom_io=1, max_pending=2)
    n.push_imu(*arr[0][1:])
    for k in range(3):
        n.push_sweep(drive.raw[k], drive.t[k])
    before = n.status()
    assert before["pending"] == 2 and before["sweeps"] == 3
    rc = _lib.lib().lio_node_push_sweep_host(n.h, np.ascontiguousarray(drive.raw[3]), None, drive.raw[3].shape[0], float(drive.t[3]))
    assert rc == LIO_ERR_CAPACITY
    assert n.status() == before


def test_host_and_device_sweep_entries_agree():
    drive, kw = _shape("vlp16_imu0")
    _, a, _ = _run_node(drive, kw, dev=False)
    _, b, _ = _run_node(drive, kw, dev=True)
    assert len(a) == len(b) > 0
    for x, y in zip(a, b):
        _same_snapshot(x, y)


def test_refusals():
    from lio_mapping_b200 import _lib
    L = _lib.lib()
    drive, kw = _shape("vlp16_imu0")
    n = _node(kw)
    raw = np.ascontiguousarray(drive.raw[0])
    rings = _rings(drive.sensor, raw)
    assert L.lio_node_push_sweep_host(n.h, raw, rings.ctypes.data, raw.shape[0], 1.0) == LIO_ERR_INVALID   # rings on a 16-ring sensor
    big = np.zeros((kw["max_points"] + 1, 4), np.float32)
    assert L.lio_node_push_sweep_host(n.h, big, None, big.shape[0], 1.0) == LIO_ERR_CAPACITY
    r = _node(dict(kw, sensor_type=320))
    assert L.lio_node_push_sweep_host(r.h, raw, None, raw.shape[0], 1.0) == LIO_ERR_INVALID                # 320 without rings
    assert n.status()["sweeps"] == 0 and r.status()["sweeps"] == 0
    n.push_imu(1.0, np.zeros(3), np.zeros(3))
    n.push_imu(1.0, np.zeros(3), np.zeros(3))                                                               # not later: dropped
    n.push_imu(0.5, np.zeros(3), np.zeros(3))
    s = n.status()
    assert s["imu_dropped"] == 2 and not s["poisoned"]
    # inner refusals come back as their status
    import ctypes as C
    cfg = _lib.NodeConfig()
    L.lio_node_default_config(C.byref(cfg))
    cfg.surf_filter_size = 0.3                                                   # map leaf != the estimator's surf_filter_size
    h = C.c_void_p()
    assert L.lio_node_create(C.byref(cfg), 0, None, C.byref(h)) == LIO_ERR_INVALID and not h.value
    cfg.surf_filter_size, cfg.sensor_type = 0.4, 17
    assert L.lio_node_create(C.byref(cfg), 0, None, C.byref(h)) == LIO_ERR_INVALID
    with pytest.raises(_lib.LioError):
        _node(dict(kw, imu_factor=1, window_size=4, opt_window_size=4))          # an IMU mapping needs W >= 5


def test_zero_step_leaves_the_estimator_state_unchanged():
    """A sample integrated twice reaches lio_est_process_imu with dt = 0 at the next message: Ps, Rs and Vs stay bit for bit."""
    drive, kw = _shape("vlp16_imu0")
    n = _node(kw)
    arr = drive.arrivals()
    for a in arr[:200]:
        if a[0] == "imu":
            n.push_imu(a[1], a[2], a[3])
        else:
            n.push_sweep(drive.raw[a[2]], a[1])
    e = n.estimator
    before = e.states().copy()
    e.process_imu(0.0, np.array([0.1, 0.2, 9.8]), np.array([0.01, 0.02, 0.03]), 99.0)
    assert np.array_equal(before, e.states())


def test_dev_ring_equals_host_ring():
    """lio_pp_process_dev_ring against lio_pp_process_host_ring on a 32-ring sweep of the 320 preset: every cloud, index set and count, with
    n = 0, ring ids >= R, non-finite points and the capacity refusal; each case twice."""
    import ctypes as C
    import torch
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.point_processor import CLOUDS, INDICES, PointProcessor
    _, scene, traj = synth.default_config("vlp16")
    sw = synth.make_sweep(RS32, scene, traj, 2.0, seed=5, distort=True)
    rings = _rings(RS32, sw)
    bad = sw.copy()
    bad[::97, 0] = np.nan
    bad[5::131, 2] = np.inf
    wild = rings.copy()
    wild[::53] = 32
    wild[7::211] = 65535
    cases = [(sw, rings), (sw[:0], rings[:0]), (sw, wild), (bad, rings), (sw[:5000], rings[:5000])]

    def outputs(pp):
        sizes = pp.sizes()
        return sizes, {k: pp.cloud(k) for k in CLOUDS}, {k: pp.index(k) for k in INDICES}, pp.scan_ranges(), pp.start_ori()

    ph = PointProcessor(-25.0, 15.0, 32, max_points=sw.shape[0])
    pd = PointProcessor(-25.0, 15.0, 32, max_points=sw.shape[0])
    L = _lib.lib()
    for xyz, rg in cases:
        for _ in range(2):
            ph.SetInputCloud(xyz)
            ph.ProcessWithRingField(rg)
            tx = torch.from_numpy(np.ascontiguousarray(xyz, np.float32).reshape(-1, 4)).cuda()
            tr = torch.from_numpy(rg.astype(np.int16).view(np.int16)).cuda()
            _lib.check(L.lio_pp_process_dev_ring(pd._h, C.c_void_p(tx.data_ptr() if xyz.shape[0] else 0),
                                                  C.c_void_p(tr.data_ptr() if xyz.shape[0] else 0), xyz.shape[0]), "dev_ring")
            assert pd.last_launches() == ph.last_launches() == 6
            a, b = outputs(ph), outputs(pd)
            assert a[0] == b[0]
            for k in CLOUDS:
                assert np.array_equal(a[1][k], b[1][k], equal_nan=True), k
            for k in INDICES:
                assert np.array_equal(a[2][k], b[2][k]), k
            assert np.array_equal(a[3], b[3]) and (a[4] == b[4] or (np.isnan(a[4]) and np.isnan(b[4])))
    big = torch.zeros((sw.shape[0] + 1, 4), dtype=torch.float32, device="cuda")
    rb = torch.zeros(sw.shape[0] + 1, dtype=torch.int16, device="cuda")
    assert L.lio_pp_process_dev_ring(pd._h, C.c_void_p(big.data_ptr()), C.c_void_p(rb.data_ptr()), big.shape[0]) == LIO_ERR_CAPACITY
    assert L.lio_pp_process_dev_ring(pd._h, None, None, 3) == LIO_ERR_INVALID
