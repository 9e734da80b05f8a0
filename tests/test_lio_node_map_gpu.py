"""map_4D*.launch inside the node (lio_node_enable_map_builder, lio_node_map_builder_poses, lio_node_attach_registered_map): the node
against the chain of tests/test_lio_node_gpu.py wired by hand plus MapBuilder.ProcessMapDev on the estimator's /local/* clouds after every
message that arrived INITED, bit for bit; the map builder changes nothing of the estimator; its calls follow the rule of the header; its
poses follow the oracle's MapBuilder fed with the node's own clouds; the drive maps of both /cloud_registered sources equal maps filled
by hand; and the refusals change nothing."""
import ctypes as C

import numpy as np
import pytest

from tests.test_global_map_gpu import _same_map
from tests.test_imu_startup_gpu import _rigid_residual
from tests.test_lio_node_gpu import SHAPES, _HandWired, _node, _same_snapshot, _shape, _snapshot
from tests.test_map_builder_gpu import POS_TOL, QUAT_TOL

pytestmark = pytest.mark.gpu

LIO_ERR_INVALID, LIO_ERR_CAPACITY = -2, -3
LEAVES = (0.0, 0.2)
CAPACITY = {0.0: 1 << 24, 0.2: 1 << 22}   # points (raw) / voxels
SOURCES = ("estimator", "map_builder")
ROW_KEYS = ("iterations", "optimised", "corner_from_map", "surf_from_map", "surround_published", "surround_size")


def _maps():
    from lio_mapping_b200.registered_map import RegisteredMap
    return {(src, leaf): RegisteredMap(leaf=leaf, capacity=CAPACITY[leaf]) for src in SOURCES for leaf in LEAVES}


class _Tap:
    """The hand-wired estimator seen through its process_compact: after each message, what the node does after it."""

    def __init__(self, hw):
        self.hw, self.e = hw, hw.e

    def __getattr__(self, name):
        return getattr(self.e, name)

    def process_compact(self, *args, **kw):
        st = self.e.process_compact(*args, **kw)
        self.hw.after_message(kw["stamp"])
        return st


class _HandWiredMap(_HandWired):
    """_HandWired plus map_builder_node by hand: ProcessMapDev(local_clouds_dev(), local_laser_odom()) on the same stream after every
    message that arrived INITED, the set's header stamp from the estimator's pushes (Headers_), and RegisteredMaps filled per publication."""

    def __init__(self, kw):
        from lio_mapping_b200.map_builder import MapBuilder
        super().__init__(kw)
        _, _, n_max = self.e.local_clouds_dev()
        self.mb = MapBuilder(max_points=int(max(n_max[0], n_max[1])), max_full_points=int(n_max[2]))
        self.maps = _maps()
        self.W, self.O = kw["window_size"], kw["opt_window_size"]
        self.headers, self.rows = [], []
        self.e = _Tap(self)

    def after_message(self, stamp):
        e = self.e.e
        if e.compact_status()["pushed"]:
            self.headers = (self.headers + [stamp])[-(self.W + 1):]
        for leaf in LEAVES:
            self.maps[("estimator", leaf)].insert_dev(*self.pm.registered_full_cloud_dev())
        if not self.inited:          # updated after this call: the stage the message arrived in
            return
        ptrs, n_dev, n_max = e.local_clouds_dev()
        tobe, info = self.mb.ProcessMapDev(ptrs, n_dev, n_max, e.local_laser_odom())
        self.rows.append((self.headers[-self.O], tobe, self.mb.transform_aft_mapped.copy(), info))
        for leaf in LEAVES:
            self.maps[("map_builder", leaf)].insert_dev(*self.mb.registered_full_cloud_dev())


def _cubes(pm):
    return pm.centre(), pm.cube_sizes("corner"), pm.cube_sizes("surf")


def _same_cubes(a, b):
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def _run(drive, kw, map_4d, oracle_mb=None):
    """The node fed with the drive's arrivals; per processed message (one per push here): the estimator snapshot, its cube directory,
    the stage at entry, and with the map builder the downloads the checks need.  Returns (node, per-message records, maps, waits0)."""
    node = _node(kw)
    maps, waits0 = {}, {}
    if map_4d:
        node.enable_map_builder()
        maps = _maps()
        for (src, leaf), rm in maps.items():
            node.attach_registered_map(rm, src)
            waits0[(src, leaf)] = rm.stats()["waits"]
    recs = []
    for a in drive.arrivals():
        before = node.status()
        if a[0] == "imu":
            node.push_imu(a[1], a[2], a[3])
        else:
            node.push_sweep(drive.raw[a[2]], a[1])
        st = node.status()
        if st["processed"] == before["processed"]:
            continue
        assert st["processed"] == before["processed"] + 1   # per-message observation from outside the node
        r = dict(inited_at_entry=before["inited"], stamp=st["last_stamp"], snap=_snapshot(node.estimator), cubes=_cubes(node.mapping))
        if map_4d:
            r["rows"] = len(node.map_builder_poses()["stamp"])
            r["est_cloud"] = node.mapping.registered_full_cloud()
            if before["inited"]:
                r["mb_cloud"] = node.map_builder.registered_full_cloud()
                if oracle_mb is not None:
                    lc = node.estimator.local_clouds()
                    r["oracle"] = oracle_mb.process_map(lc["corner"], lc["surf"], lc["full"], node.estimator.local_laser_odom())
                    r["oracle_aft"] = oracle_mb.transform_aft_mapped.copy()
        recs.append(r)
    return node, recs, maps, waits0


@pytest.fixture(scope="module", params=list(SHAPES))
def drive_runs(request):
    """One shape: the hand-wired chain with its map builder, the node with it (and the oracle fed from the node), the node without it."""
    from oracle import map_builder_py as mbo
    from oracle import oracle_py
    oracle_py.build()
    shape = request.param
    drive, kw = _shape(shape)
    hw = _HandWiredMap(kw)
    for i, a in enumerate(drive.arrivals()):
        hw.push(i, ("sweep", a[1], a[2], drive.raw[a[2]]) if a[0] == "sweep" else a)
    mo = mbo.MapBuilderOracle()
    on = _run(drive, kw, True, mo)
    off = _run(drive, kw, False)
    return shape, drive, kw, hw, on, off


def _rows(node):
    p = node.map_builder_poses()
    return [(p["stamp"][k], p["tobe"][k], p["aft"][k], {name: (bool if name in ("optimised", "surround_published") else int)(p[name][k])
                                                          for name in ROW_KEYS}) for k in range(len(p["stamp"]))]


def test_node_map_builder_equals_the_hand_wired_chain(drive_runs):
    """Every map builder row (stamp, tobe, aft, info) bit-equal to the hand-wired chain's, call by call; at the end the map builder's
    cube centre, every cube, the surround map and the registered cloud."""
    shape, _, _, hw, (node, recs, _, _), _ = drive_runs
    rows = _rows(node)
    assert len(rows) == len(hw.rows) > 0, shape
    for k, (a, b) in enumerate(zip(rows, hw.rows)):
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and a[3] == b[3], (shape, k)
    _same_map(node.map_builder, hw.mb)
    assert np.array_equal(node.map_builder.surround_map(), hw.mb.surround_map())
    assert np.array_equal(node.map_builder.registered_full_cloud(), hw.mb.registered_full_cloud())


def test_map_builder_changes_nothing_else(drive_runs):
    """States, imu_init_status, the extrinsic, map_poses and the estimator's cube directory after every message, and its whole cube map at
    the end: bit-equal with and without the map builder."""
    shape, _, _, _, (node, recs, _, _), (node0, recs0, _, _) = drive_runs
    assert len(recs) == len(recs0) > 0
    for a, b in zip(recs, recs0):
        assert a["stamp"] == b["stamp"] and a["inited_at_entry"] == b["inited_at_entry"]
        _same_snapshot(a["snap"], b["snap"])
        _same_cubes(a["cubes"], b["cubes"])
    _same_map(node.mapping, node0.mapping)
    assert node.status()["odom_enabled"] == node0.status()["odom_enabled"]


def test_map_builder_call_rule(drive_runs):
    """One call for each message that arrived INITED, none on the start-up message or before it; each row's stamp is the header stamp of
    the set (Headers_[pivot + 1]) and precedes the message that made the call."""
    shape, _, kw, _, (node, recs, _, _), _ = drive_runs
    rows, prev = 0, 0
    first_inited = next(k for k, r in enumerate(recs) if r["inited_at_entry"])
    assert first_inited > 0 and all(not r["inited_at_entry"] for r in recs[:first_inited])
    for r in recs:
        assert r["rows"] - prev == (1 if r["inited_at_entry"] else 0)
        prev = r["rows"]
        rows += r["inited_at_entry"]
    assert rows == len(node.map_builder_poses()["stamp"]) == sum(r["inited_at_entry"] for r in recs)
    p = node.map_builder_poses()
    made_by = [r["stamp"] for r in recs if r["inited_at_entry"]]
    assert np.all(p["stamp"] < np.array(made_by)) and np.all(np.diff(p["stamp"]) > 0)
    assert p["surround_published"][0] and list(np.nonzero(p["surround_published"])[0]) == list(range(0, rows, 5))


# Over a whole drive the two sides' float Gauss-Newton reduction orders compound: every pose seeds the next call's association and the
# map it inserts.  The first PINNED calls keep test_map_builder_gpu's POS_TOL / QUAT_TOL; over the whole drive the bounds are about three
# times the largest difference measured on an H100 (indoor: 1.1e-3 m and 1.0e-5 at its 21st call; the first 10 calls stay below 1.5e-5 m;
# DESIGN §7).
PINNED = 10
DRIVE_POS_TOL, DRIVE_QUAT_TOL = 3e-3, 3e-5


def test_map_builder_against_the_oracle(drive_runs):
    """MapBuilderOracle fed the node's downloaded /local/* clouds and /local_laser_odom message by message: the first call bit-exact,
    then the same gate and publishing decisions, tobe and aft within POS_TOL / QUAT_TOL for the first PINNED calls and within the drive
    tolerances after them."""
    shape, _, _, _, (node, recs, _, _), _ = drive_runs
    rows = _rows(node)
    calls = [r for r in recs if r["inited_at_entry"]]
    assert len(calls) == len(rows) > 0
    dp, dq = [0.0], [0.0]
    for k, (r, row) in enumerate(zip(calls, rows)):
        to, io = r["oracle"]
        ao = r["oracle_aft"]
        if k == 0:
            assert np.array_equal(row[1], to) and np.array_equal(row[2], ao) and row[3] == io, shape
            continue
        assert row[3]["optimised"] == io["optimised"] and row[3]["surround_published"] == io["surround_published"], (shape, k)
        dp.append(max(float(np.abs(g[4:] - o[4:]).max()) for g, o in ((row[1], to), (row[2], ao))))
        dq.append(max(float(np.abs(g[:4] - o[:4]).max()) for g, o in ((row[1], to), (row[2], ao))))
    print(f"{shape}: {len(rows)} map builder calls; difference to the oracle per call: position (m) "
          f"{' '.join(f'{v:.1e}' for v in dp)}; quaternion {' '.join(f'{v:.1e}' for v in dq)}")
    assert max(dp[:PINNED]) <= POS_TOL and max(dq[:PINNED]) <= QUAT_TOL, shape
    assert max(dp) <= DRIVE_POS_TOL and max(dq) <= DRIVE_QUAT_TOL, shape


def test_drive_maps_of_both_sources(drive_runs):
    """The node's drive maps (both sources, leaf 0 and 0.2) bit-equal to maps the hand-wired chain filled per publication; at leaf 0 the
    concatenation of the per-message registered clouds; the inserts added no host wait; one copy per insert at leaf 0, 17 stream operations
    at leaf 0.2; one insert per processed message (estimator) or per map builder call."""
    shape, _, _, hw, (node, recs, maps, waits0), _ = drive_runs
    n_calls = sum(r["inited_at_entry"] for r in recs)
    for (src, leaf), rm in maps.items():
        s = rm.stats()
        assert s["waits"] == waits0[(src, leaf)] + 1, (shape, src, leaf)   # this stats call's own wait only
        assert s["inserts"] == (len(recs) if src == "estimator" else n_calls)
        assert s["launches"] == (1 if leaf == 0 else 17) and not s["overflow"]
    for key, rm in maps.items():
        got = rm.download()
        assert np.array_equal(got, hw.maps[key].download(), equal_nan=True), (shape, key)
        if key[1] == 0:
            parts = [r["est_cloud"] if key[0] == "estimator" else r["mb_cloud"] for r in recs if key[0] == "estimator" or r["inited_at_entry"]]
            assert np.array_equal(got, np.concatenate(parts), equal_nan=True), (shape, key)


# Largest position error (m) of the map builder's trajectory (tobe, the lidar position) against the drive's ground-truth lidar positions
# at the rows' stamps, after a rigid alignment.  Measured on an H100 80GB HBM3 at 700 W: 0.428 m (outdoor_64, 14 poses), 1.296 m (indoor,
# 21 poses) and 0.016 m (vlp16_imu0, 8 poses), next to window errors of 1.178, 0.756 and 0.059 m.  The bounds leave about 25 % (indoor,
# outdoor_64) and 90 % (vlp16_imu0, a few cm) above them.
MAP_GT_BOUND = {"outdoor_64": 0.55, "indoor": 1.6, "vlp16_imu0": 0.03}


def test_map_builder_trajectory_accuracy(drive_runs):
    shape, drive, kw, _, (node, recs, _, _), _ = drive_runs
    p = node.map_builder_poses()
    gt_p, gt_R = drive.traj.state(p["stamp"])[:2]
    gt = gt_p + np.einsum("nij,j->ni", gt_R, drive.t_lb)
    err = _rigid_residual(p["tobe"][:, 4:].astype(np.float64), gt)
    W = kw["window_size"]
    win = _rigid_residual(node.states()[:, 0:3], drive.gt_positions([r["stamp"] for r in recs][-(W + 1):]))
    print(f"{shape}: map builder trajectory ({len(p['stamp'])} poses) position error after rigid alignment {err:.3f} m; "
          f"window {win:.3f} m")
    assert err < MAP_GT_BOUND[shape]


def test_refusals_change_nothing():
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.registered_map import RegisteredMap
    import torch
    L = _lib.lib()
    drive, kw = _shape("vlp16_imu0")
    n = _node(kw)
    rm = RegisteredMap(leaf=0.0, capacity=1 << 20)
    # the map builder's source without a map builder; an unknown source
    assert L.lio_node_attach_registered_map(n.h, rm.h, 1) == LIO_ERR_INVALID
    assert L.lio_node_attach_registered_map(n.h, rm.h, 7) == LIO_ERR_INVALID
    assert L.lio_node_attach_registered_map(n.h, rm.h, -1) == LIO_ERR_INVALID
    assert n.map_builder is None
    mb = C.c_void_p()
    assert L.lio_node_map_builder(n.h, C.byref(mb)) == LIO_ERR_INVALID and not mb.value
    # an rm on another stream
    s = torch.cuda.Stream()
    other = RegisteredMap(leaf=0.0, capacity=1 << 20, stream=s.cuda_stream)
    assert L.lio_node_attach_registered_map(n.h, other.h, 0) == LIO_ERR_INVALID
    # enabling twice
    n.enable_map_builder()
    first = n.map_builder.h.value
    cfg = _lib.MBConfig()
    L.lio_mb_default_config(C.byref(cfg))
    assert L.lio_node_enable_map_builder(n.h, C.byref(cfg)) == LIO_ERR_INVALID
    assert L.lio_node_map_builder(n.h, C.byref(mb)) == 0 and mb.value == first
    # the same rm twice
    n.attach_registered_map(rm, "map_builder")
    assert L.lio_node_attach_registered_map(n.h, rm.h, 0) == LIO_ERR_INVALID
    with pytest.raises(_lib.LioError):
        n.attach_registered_map(rm, "elsewhere")
    # enabling after a sweep
    m = _node(kw)
    arr = drive.arrivals()
    first_sweep = next(k for k, a in enumerate(arr) if a[0] == "sweep")
    for a in arr[:first_sweep]:
        m.push_imu(a[1], a[2], a[3])
    m.push_sweep(drive.raw[0], drive.t[0])
    before = m.status()
    assert L.lio_node_enable_map_builder(m.h, C.byref(cfg)) == LIO_ERR_INVALID
    assert L.lio_node_map_builder(m.h, C.byref(mb)) == LIO_ERR_INVALID and m.status() == before
    # poses: refused without a map builder; *n rows otherwise
    k = C.c_int()
    z = (np.zeros(1), np.zeros((1, 7), np.float32), np.zeros((1, 7), np.float32), np.zeros((1, 6), np.int32))
    assert L.lio_node_map_builder_poses(m.h, *z, 1, C.byref(k)) == LIO_ERR_INVALID
    assert L.lio_node_map_builder_poses(n.h, *z, 1, C.byref(k)) == 0 and k.value == 0
    # the drive runs on with the refused calls behind it: the same map builder rows and drive map as a node that never saw them
    for a in arr:
        if a[0] == "imu":
            n.push_imu(a[1], a[2], a[3])
        else:
            n.push_sweep(drive.raw[a[2]], a[1])
    assert L.lio_node_map_builder_poses(n.h, *z, 1, C.byref(k)) == LIO_ERR_CAPACITY and k.value > 1
    ref = _node(kw)
    ref.enable_map_builder()
    ref_rm = RegisteredMap(leaf=0.0, capacity=1 << 20)
    ref.attach_registered_map(ref_rm, "map_builder")
    for a in arr:
        if a[0] == "imu":
            ref.push_imu(a[1], a[2], a[3])
        else:
            ref.push_sweep(drive.raw[a[2]], a[1])
    assert len(_rows(n)) > 0
    for a, b in zip(_rows(n), _rows(ref)):
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and a[3] == b[3]
    assert np.array_equal(rm.download(), ref_rm.download())
    assert other.stats()["inserts"] == 0


def test_map_builder_failure_poisons_the_node():
    """A map builder whose corner leaf is far too small for the 2^24-voxel index of its cube down-sampling: a map builder call returns
    LIO_ERR_CAPACITY, the push that made it fails with that status, the failed call keeps no row, and the node is poisoned."""
    from lio_mapping_b200 import _lib
    drive, kw = _shape("vlp16_imu0")
    n = _node(kw)
    n.enable_map_builder(corner_filter_size=1e-3)
    err, calls = None, 0
    for a in drive.arrivals():
        before = n.status()
        try:
            if a[0] == "imu":
                n.push_imu(a[1], a[2], a[3])
            else:
                n.push_sweep(drive.raw[a[2]], a[1])
        except _lib.LioError as e:
            err = e
            break
        calls += n.status()["processed"] > before["processed"] and before["inited"]
    assert err is not None and "CAPACITY" in str(err)
    st = n.status()
    assert st["poisoned"] and st["inited"] and len(n.map_builder_poses()["stamp"]) == calls
    rc = _lib.lib().lio_node_push_imu(n.h, 1e6, np.zeros(3), np.zeros(3))
    assert rc == LIO_ERR_INVALID and n.status() == st


def test_shipped_map_4d_keyword():
    from lio_mapping_b200 import LioNode
    from lio_mapping_b200.map_builder import default_config
    a = LioNode.shipped("outdoor_64", max_points=1 << 17, max_feature_points=1 << 15, max_frame_points=1 << 14, max_scan_points=1 << 16)
    b = LioNode.shipped("outdoor_64", map_4d=True, max_points=1 << 17, max_feature_points=1 << 15, max_frame_points=1 << 14,
                        max_scan_points=1 << 16)
    assert a.map_builder is None and b.map_builder.config == default_config()
    assert b.map_builder.config["map_filter_size"] == pytest.approx(0.2) and b.map_builder.config["enable_4d"] == 1
