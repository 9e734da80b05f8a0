"""The node's odometry topics (lio_node_enable_odometry, lio_node_take_odometry): every row bit-equal to the row the hand-wired chain of
tests/test_lio_node_gpu.py builds from its own handles at the moment the reference publishes; the publication rules (counts, stamps,
seq); /predict_laser_odom and /local_laser_odom against the float64 restatement of tests/test_odometry_topics.py; a node with the topics
on bit-equal to one without; the queue's drop-oldest rule and its refusals; and the accuracy of the published trajectories."""
import ctypes as C

import numpy as np
import pytest

from lio_mapping_b200.node import TOPICS
from tests.test_global_map_gpu import _same_map
from tests.test_imu_startup_gpu import _rigid_residual
from tests.test_lio_node_gpu import SHAPES, _HandWired, _same_snapshot, _shape, _snapshot
from tests.test_odometry_topics import lidar_pose, quat_to_matrix

pytestmark = pytest.mark.gpu

LIO_ERR_INVALID = -2


def _row(stamp, tf7, extras=()):
    r = np.zeros(16)
    r[0], r[1:8] = stamp, tf7
    r[8:8 + len(extras)] = extras
    return r


class _OdomTap:
    """The hand-wired PointOdometry seen through ProcessDev: PublishResults of every call but the first (PointOdometry.cc:302-310,
    :681-721)."""

    def __init__(self, hw):
        self.hw, self.po, self.calls = hw, hw.po, 0

    def __getattr__(self, name):
        return getattr(self.po, name)

    def ProcessDev(self, *args):
        ts, es, info = self.po.ProcessDev(*args)
        if self.calls:
            self.hw.rows["/laser_odom_to_init"].append(_row(self.hw.sweep_stamp, ts.astype(np.float64), es.astype(np.float64)))
        self.calls += 1
        return ts, es, info


class _EstTap:
    """The hand-wired estimator seen through process_imu and process_compact."""

    def __init__(self, hw):
        self.hw, self.e = hw, hw.e

    def __getattr__(self, name):
        return getattr(self.e, name)

    def process_imu(self, dt, acc, gyr, stamp):
        self.e.process_imu(dt, acc, gyr, stamp)
        if self.hw.inited:   # the stage the message arrived in (_HandWired updates it after process_compact)
            s = self.e.states()[-1]
            self.hw.rows["/predict_odom"].append(_row(stamp, np.r_[s[3:7], s[0:3]], s[7:13]))
            self.hw.msg_calls.append(stamp)

    def process_compact(self, *args, **kw):
        st = self.e.process_compact(*args, **kw)
        self.hw.after_message(kw["stamp"])
        return st


class _HandWiredOdom(_HandWired):
    """_HandWired plus each publication built from the handles' own getters: ProcessDev's ts / es per sweep, states()[W] after each
    process_imu of an INITED message, map_poses()'s aft, extrinsic() after each solve, laser_odom() after each INITED message, and the
    Headers_ of the estimator's pushes.  msgs: per processed message (stamp, arrived INITED, solved, its INITED ProcessImu stamps)."""

    def __init__(self, kw):
        super().__init__(kw)
        self.W, self.O = kw["window_size"], kw["opt_window_size"]
        self.rows = {name: [] for name in TOPICS}
        self.headers, self.msgs, self.formula, self.msg_calls = [], [], [], []
        self.raw_e = self.e
        self.e = _EstTap(self)
        self.po = _OdomTap(self)

    def push(self, i, a, rings=None):
        if a[0] == "sweep":
            self.sweep_stamp = a[1]
        super().push(i, a, rings)

    def after_message(self, stamp):
        e = self.raw_e
        cs = e.compact_status()
        if cs["pushed"]:
            self.headers = (self.headers + [stamp])[-(self.W + 1):]
        self.rows["/aft_mapped_to_init"].append(_row(stamp, e.map_poses()[1].astype(np.float64)))
        if cs["solved"]:
            self.rows["/extrinsic_lb"].append(_row(self.headers[-1], e.extrinsic().astype(np.float64)))
        if self.inited:
            predict, local = e.laser_odom()
            self.rows["/predict_laser_odom"].append(_row(stamp, predict))
            self.rows["/local_laser_odom"].append(_row(self.headers[-self.O], local))
            self.formula.append((e.states().copy(), e.extrinsic().copy(), e.local_laser_odom().copy()))
        self.msgs.append((stamp, self.inited, cs["solved"], self.msg_calls))
        self.msg_calls = []

    def table(self, name):
        r = np.array(self.rows[name]).reshape(-1, 16)
        r[:, 15] = np.arange(1, r.shape[0] + 1)
        return r


def _rows(node, name, cap=None):
    """A take of topic name as (n, 16) rows, the C-ABI's layout."""
    t = node.take_odometry(name, cap)
    out = np.zeros((t["stamp"].shape[0], 16))
    out[:, 0], out[:, 1:8], out[:, 15] = t["stamp"], t["tf7"], t["seq"]
    col = 8
    for key in ("es", "v", "ba"):
        if key in t:
            out[:, col:col + t[key].shape[1]] = t[key]
            col += t[key].shape[1]
    return out


def _run(drive, kw, capacity=1 << 16, map_4d=True, chunks=None):
    """The node fed with the drive's arrivals, the map builder on (map_4d) and the odometry topics on (capacity, or None for off).
    Returns (node, per processed message (stamp, arrived INITED, snapshot), sweep stamps, rows taken during the run when chunks gives
    the take sizes to cycle through after every arrival, then one take of what is left)."""
    from lio_mapping_b200 import LioNode
    node = LioNode(**kw)
    if map_4d:
        node.enable_map_builder()
    if capacity is not None:
        node.enable_odometry(capacity)
    recs, sweeps, taken, k = [], [], {name: [] for name in TOPICS}, 0
    for a in drive.arrivals():
        before = node.status()
        if a[0] == "imu":
            node.push_imu(a[1], a[2], a[3])
        else:
            node.push_sweep(drive.raw[a[2]], a[1])
            sweeps.append(a[1])
        st = node.status()
        if st["processed"] != before["processed"]:
            assert st["processed"] == before["processed"] + 1
            recs.append((st["last_stamp"], before["inited"], _snapshot(node.estimator)))
        if chunks:
            for name in TOPICS:
                taken[name].append(_rows(node, name, chunks[k % len(chunks)]))
                k += 1
    if chunks:
        for name in TOPICS:
            taken[name].append(_rows(node, name))
    return node, recs, np.array(sweeps), taken


@pytest.fixture(scope="module", params=list(SHAPES))
def runs(request):
    """One shape: the hand-wired chain with its publications, the node with the topics on and its rows, the node without them; both
    nodes run the map builder (its poses give the /local_laser_odom stamps)."""
    shape = request.param
    drive, kw = _shape(shape)
    hw = _HandWiredOdom(kw)
    for i, a in enumerate(drive.arrivals()):
        hw.push(i, ("sweep", a[1], a[2], drive.raw[a[2]]) if a[0] == "sweep" else a)
    on = _run(drive, kw)
    rows = {name: _rows(on[0], name) for name in TOPICS}
    off = _run(drive, kw, capacity=None)
    return shape, drive, kw, hw, on, rows, off


def test_rows_equal_the_hand_wired_chain(runs):
    """Every row of every topic bit-equal to the hand-wired chain's, in order; the queues are empty after the take."""
    shape, _, _, hw, (node, _, _, _), rows, _ = runs
    for name in TOPICS:
        want = hw.table(name)
        assert rows[name].shape == want.shape and want.shape[0] > 0, (shape, name)
        assert np.array_equal(rows[name], want), (shape, name)
        assert node.take_odometry(name)["left"] == 0


def test_publication_rules(runs):
    """Counts, stamps and seq of each topic from what is observed outside the node: the sweeps, the processed messages and the stage
    each arrived in, the map builder's rows; /predict_odom against the ProcessImu calls of the restated pairing."""
    shape, _, kw, hw, (node, recs, sweeps, _), rows, _ = runs
    stamps = np.array([r[0] for r in recs])
    arrived = np.array([r[1] for r in recs])
    first_inited = int(np.argmax(arrived))   # the message before it is the start-up message
    assert first_inited > 0 and arrived[first_inited:].all() and not arrived[:first_inited].any(), shape
    assert len(recs) == len(hw.msgs) and [m[0] for m in hw.msgs] == list(stamps)
    r = rows["/laser_odom_to_init"]
    assert np.array_equal(r[:, 0], sweeps[1:])
    assert np.array_equal(rows["/aft_mapped_to_init"][:, 0], stamps)
    inited_calls = [t for m in hw.msgs if m[1] for t in m[3]]
    assert np.array_equal(rows["/predict_odom"][:, 0], inited_calls) and len(inited_calls) > 0
    assert sum(len(m[3]) for m in hw.msgs if not m[1]) == 0   # none recorded before INITED
    assert np.array_equal(rows["/predict_laser_odom"][:, 0], stamps[arrived])
    assert rows["/local_laser_odom"].shape[0] == arrived.sum()
    assert np.array_equal(rows["/local_laser_odom"][:, 0], node.map_builder_poses()["stamp"])
    assert np.all(rows["/local_laser_odom"][:, 0] < stamps[arrived])
    assert np.array_equal(rows["/extrinsic_lb"][:, 0], np.r_[stamps[first_inited - 1], stamps[arrived]])
    assert all(m[2] == (m[1] or k == first_inited - 1) for k, m in enumerate(hw.msgs))   # the estimator solved exactly there
    for name in TOPICS:
        assert np.array_equal(rows[name][:, 15], np.arange(1, rows[name].shape[0] + 1)), (shape, name)
    print(f"{shape}: rows {', '.join(f'{n} {rows[n].shape[0]}' for n in TOPICS)}; {len(sweeps)} sweeps, {len(recs)} processed, "
          f"{int(arrived.sum())} INITED")


def test_laser_odom_formulas(runs):
    """/predict_laser_odom and /local_laser_odom within 1e-12 of lidar_pose on the window states and extrinsic the hand-wired chain
    reads after each INITED message; /local_laser_odom rounded to float bit-equal to lio_est_local_laser_odom."""
    shape, _, kw, hw, _, rows, _ = runs
    W, O = kw["window_size"], kw["opt_window_size"]
    pred, loc = rows["/predict_laser_odom"], rows["/local_laser_odom"]
    assert len(hw.formula) == pred.shape[0] == loc.shape[0] > 0
    worst = 0.0
    for k, (states, tlb, local_f) in enumerate(hw.formula):
        for row, slot in ((pred[k], W), (loc[k], W - O)):
            s = states[slot]
            want = lidar_pose(s[0:3], quat_to_matrix(s[3:7]), tlb)
            worst = max(worst, float(np.abs(row[1:8] - want).max()))
        assert np.array_equal(loc[k, 1:8].astype(np.float32), local_f), (shape, k)
    assert worst <= 1e-12, (shape, worst)


def test_topics_change_nothing(runs):
    """The node with the topics on against the node without them: every snapshot after every processed message, the cube map, the
    surround map, /cloud_registered and the map builder's poses, bit for bit."""
    shape, _, _, _, (node, recs, _, _), _, (node0, recs0, _, _) = runs
    assert len(recs) == len(recs0) > 0
    for a, b in zip(recs, recs0):
        assert a[0] == b[0] and a[1] == b[1]
        _same_snapshot(a[2], b[2])
    _same_map(node.mapping, node0.mapping)
    assert np.array_equal(node.mapping.surround_map(), node0.mapping.surround_map())
    assert np.array_equal(node.mapping.registered_full_cloud(), node0.mapping.registered_full_cloud())
    p, p0 = node.map_builder_poses(), node0.map_builder_poses()
    for key in p:
        assert np.array_equal(p[key], p0[key]), key
    assert node.status() == node0.status()


def test_uneven_takes_and_a_small_queue(runs):
    """Rows taken in uneven chunks after every arrival (a node without the map builder) concatenate to the one take of the fixture's node;
    capacity 3 keeps each topic's newest 3 rows with their seq, the gap before them showing the drops."""
    shape, drive, kw, _, _, rows, _ = runs
    if shape != "vlp16_imu0":
        pytest.skip("one shape suffices for the queue rules")
    _, _, _, taken = _run(drive, kw, map_4d=False, chunks=(1, 3, 0, 7, 2, 5))
    small, _, _, _ = _run(drive, kw, capacity=3, map_4d=False)
    for name in TOPICS:
        got = np.concatenate(taken[name])
        assert np.array_equal(got, rows[name]), name
        last = _rows(small, name)
        n = rows[name].shape[0]
        assert last.shape[0] == min(3, n) and np.array_equal(last, rows[name][n - last.shape[0]:]), name
        assert last[0, 15] == n - last.shape[0] + 1


def test_refusals():
    """Enable twice, after the first sweep, with capacity < 1, on a poisoned node; take with an unknown topic, cap < 0 or without
    enable: LIO_ERR_INVALID, nothing changes.  A poisoned node's rows stay takeable."""
    from lio_mapping_b200 import LioNode, _lib
    L = _lib.lib()
    drive, kw = _shape("vlp16_imu0")
    n, left = C.c_int(), C.c_int()
    buf = np.zeros((4, 16))
    p = buf.ctypes.data_as(C.c_void_p)
    a = LioNode(**kw)
    assert L.lio_node_take_odometry(a.h, 0, p, 4, C.byref(n), C.byref(left)) == LIO_ERR_INVALID and n.value == 0
    assert L.lio_node_enable_odometry(a.h, 0) == LIO_ERR_INVALID and L.lio_node_enable_odometry(a.h, -5) == LIO_ERR_INVALID
    a.enable_odometry(8)
    assert L.lio_node_enable_odometry(a.h, 8) == LIO_ERR_INVALID
    for topic in (-1, 6, 99):
        assert L.lio_node_take_odometry(a.h, topic, p, 4, C.byref(n), C.byref(left)) == LIO_ERR_INVALID
    assert L.lio_node_take_odometry(a.h, 0, p, -1, C.byref(n), C.byref(left)) == LIO_ERR_INVALID
    assert L.lio_node_take_odometry(a.h, 0, p, 4, None, C.byref(left)) == LIO_ERR_INVALID
    assert L.lio_node_take_odometry(a.h, 0, None, 0, C.byref(n), None) == 0 and n.value == 0
    with pytest.raises(_lib.LioError):
        a.take_odometry("/odom")
    # after the first sweep
    b = LioNode(**kw)
    arr = drive.arrivals()
    first = next(k for k, x in enumerate(arr) if x[0] == "sweep")
    for x in arr[:first]:
        b.push_imu(x[1], x[2], x[3])
    b.push_sweep(drive.raw[0], drive.t[0])
    before = b.status()
    assert L.lio_node_enable_odometry(b.h, 8) == LIO_ERR_INVALID and b.status() == before
    assert L.lio_node_take_odometry(b.h, 0, p, 4, C.byref(n), C.byref(left)) == LIO_ERR_INVALID
    # the refused calls changed nothing: a drives on and gives the rows of a node that never saw them
    ref = LioNode(**kw)
    ref.enable_odometry(8)
    for node in (a, ref):
        for x in arr:
            if x[0] == "imu":
                node.push_imu(x[1], x[2], x[3])
            else:
                node.push_sweep(drive.raw[x[2]], x[1])
    for name in TOPICS:
        assert np.array_equal(_rows(a, name), _rows(ref, name)), name
    # poisoned: a map builder whose corner leaf overflows its voxel index fails a call (test_lio_node_map_gpu); rows stay takeable
    c = LioNode(**kw)
    c.enable_map_builder(corner_filter_size=1e-3)
    c.enable_odometry(1 << 12)
    with pytest.raises(_lib.LioError):
        for x in arr:
            if x[0] == "imu":
                c.push_imu(x[1], x[2], x[3])
            else:
                c.push_sweep(drive.raw[x[2]], x[1])
    st = c.status()
    assert st["poisoned"]
    assert L.lio_node_enable_odometry(c.h, 8) == LIO_ERR_INVALID and c.status() == st
    got = c.take_odometry("/aft_mapped_to_init")
    assert got["stamp"].shape[0] == st["processed"] and np.array_equal(got["seq"], np.arange(1, st["processed"] + 1))


# Largest position error (m) after a rigid alignment against the drive's ground-truth lidar positions at the rows' stamps: the
# /predict_laser_odom trajectory (every message that arrived INITED) and the /aft_mapped_to_init rows published before INITED (the
# start-up's scan-to-map poses, lidar only).  Measured on an H100 80GB HBM3 at 700 W: /predict_laser_odom 0.248 m (outdoor_64, 14 poses),
# 1.348 m (indoor, 21) and 0.015 m (vlp16_imu0, 8); pre-init /aft_mapped_to_init 0.471 m (outdoor_64, 8 poses), 4.174 m (indoor, 26) and
# 0.036 m (vlp16_imu0, 6).  The indoor drive rolls and pitches with three times the outdoor_64 amplitude; its pre-init error is not
# explained here.  The bounds leave about 25 % above the metre-scale numbers and about twice the centimetre-scale ones.
PREDICT_GT_BOUND = {"outdoor_64": 0.35, "indoor": 1.7, "vlp16_imu0": 0.03}
PREINIT_GT_BOUND = {"outdoor_64": 0.6, "indoor": 5.2, "vlp16_imu0": 0.07}


def _gt_lidar(drive, stamps):
    gt_p, gt_R = drive.traj.state(np.asarray(stamps))[:2]
    return gt_p + np.einsum("nij,j->ni", gt_R, drive.t_lb)


def test_trajectory_accuracy(runs):
    shape, drive, _, _, (_, recs, _, _), rows, _ = runs
    pred = rows["/predict_laser_odom"]
    err = _rigid_residual(pred[:, 5:8], _gt_lidar(drive, pred[:, 0]))
    aft = rows["/aft_mapped_to_init"]
    pre = aft[[not r[1] for r in recs]]
    err0 = _rigid_residual(pre[:, 5:8], _gt_lidar(drive, pre[:, 0]))
    print(f"{shape}: /predict_laser_odom ({pred.shape[0]} poses) position error after rigid alignment {err:.3f} m; "
          f"pre-init /aft_mapped_to_init ({pre.shape[0]} poses) {err0:.3f} m")
    assert err < PREDICT_GT_BOUND[shape] and err0 < PREINIT_GT_BOUND[shape]
