"""Ownership of the library's CUDA resources (lio_live_resources): every handle returns what it allocated when it is destroyed, a
refused enable / attach call leaves nothing behind and the handle usable, an attached map outlives a refused lio_pm_destroy until its
estimator goes, an estimator destroyed with map and local-cloud work in flight frees everything, and the scans of the bench's
estimator allocate nothing after warm-up."""
import gc

import numpy as np
import pytest

from tests.test_global_map_gpu import _Setup

pytestmark = pytest.mark.gpu


@pytest.fixture
def live():
    """lio_live_resources() with the garbage of earlier tests collected and the collector off, so that only this test moves it."""
    from lio_mapping_b200 import _lib
    gc.collect()
    gc.disable()
    try:
        yield _lib.lib().lio_live_resources
    finally:
        gc.enable()


def _scan(s, e, k):
    e.set_scan_clouds(s.corner[k], s.full[k])
    s.imu(e, k)
    e.process_scan(s.less_flat(k))


def _close(*objs):
    for o in objs:
        o.close()


def _pp():
    from lio_mapping_b200.point_processor import PointProcessor
    return [PointProcessor(max_points=1 << 14)]


def _po():
    from lio_mapping_b200.point_odometry import PointOdometry
    return [PointOdometry(max_feature_points=1 << 12, max_full_points=1 << 14)]


def _pm(publish):
    from lio_mapping_b200.point_mapping import PointMapping
    pm = PointMapping(max_points=1 << 12)
    if publish:
        pm.EnablePublish(0.6, 1 << 14)
    return [pm]


def _mb():
    from lio_mapping_b200.map_builder import MapBuilder
    return [MapBuilder(max_points=1 << 12, max_full_points=1 << 14)]


def _rm(leaf):
    from lio_mapping_b200.registered_map import RegisteredMap
    return [RegisteredMap(leaf=leaf, capacity=1 << 16)]


def _est_local_clouds():
    from lio_mapping_b200.estimator import Estimator
    e = Estimator(window_size=4, opt_window_size=4, max_frame_points=1 << 12, max_scan_points=1 << 14)
    e.enable_local_clouds(0.2, 1 << 12, 1 << 14)
    return [e]


def _node_map_builder():
    from lio_mapping_b200.node import LioNode
    from lio_mapping_b200.registered_map import RegisteredMap
    node = LioNode(max_points=1 << 14, max_feature_points=1 << 12, max_pending=4)
    node.enable_map_builder()
    rm = RegisteredMap(leaf=0.2, capacity=1 << 16)
    node.attach_registered_map(rm, "map_builder")
    return [node, rm]   # the node goes first: it inserts into rm


HANDLES = {
    "pp": _pp, "po": _po, "pm": lambda: _pm(False), "pm_publish": lambda: _pm(True), "mb": _mb, "rm_raw": lambda: _rm(0.0),
    "rm_voxel": lambda: _rm(0.2), "est_local_clouds": _est_local_clouds, "node_map_builder_drive_map": _node_map_builder,
}


@pytest.mark.parametrize("kind", list(HANDLES))
def test_create_destroy_returns_every_resource(live, kind):
    n0 = live()
    objs = HANDLES[kind]()
    assert live() > n0
    _close(*objs)
    assert live() == n0


def test_attached_map_released_with_its_estimator(oracle, live):
    """Create, warm start, attach and destroy: the estimator's and both maps' resources all return."""
    n0 = live()
    s = _Setup(oracle, 4, 4, 1)
    n1 = live()
    s.eg.attach_map(s.pm)
    assert live() > n1                          # the map step's events, the grown insert buffers
    _close(s.eg, s.pm, s.eb, s.pr)
    assert live() == n0


def test_refused_attach_leaves_nothing(oracle, live):
    """A map whose leaf sizes differ is refused before anything is allocated; the estimator then still runs a scan (whose first solve
    captures its graph), like its twin that was never offered a map."""
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.point_mapping import PointMapping
    from tests.test_global_map_gpu import _dev_inputs
    n0 = live()
    s = _Setup(oracle, 4, 4, 1)
    leaf = PointMapping(max_points=1 << 15, surf_filter_size=0.5)
    leaf.EnablePublish(0.6, 1 << 18)
    keep, ptrs, n, nn = _dev_inputs(s.corner[0], s.less_flat(0), s.full[0])
    leaf.ProcessDev(ptrs, n.data_ptr(), nn, np.array([0, 0, 0, 1, 0, 0, 0], np.float32))
    n1 = live()
    with pytest.raises(_lib.LioError):
        s.eg.attach_map(leaf)
    assert live() == n1
    _scan(s, s.eg, 4)
    n2 = live()
    _scan(s, s.eb, 4)
    assert live() - n2 == n2 - n1                         # the same first-solve allocations as the twin's
    assert np.array_equal(s.eg.states(), s.eb.states())   # as if the attach had not been tried
    _close(s.eg, s.eb, s.pm, s.pr, leaf)
    assert live() == n0


def test_refused_pm_destroy_frees_nothing(oracle, live):
    """lio_pm_destroy of an attached map is refused and frees nothing, before and after a scan; once the estimator is destroyed the
    map's destroy frees it."""
    from lio_mapping_b200 import _lib
    n0 = live()
    s = _Setup(oracle, 4, 4, 1)
    s.eg.attach_map(s.pm)
    n1 = live()
    assert _lib.lib().lio_pm_destroy(s.pm.h) == -2       # LIO_ERR_INVALID: attached
    assert live() == n1
    _scan(s, s.eg, 4)
    n2 = live()
    assert _lib.lib().lio_pm_destroy(s.pm.h) == -2
    assert live() == n2
    s.eg.close()
    n3 = live()
    assert n3 < n2
    assert _lib.lib().lio_pm_destroy(s.pm.h) == 0
    s.pm.h = None
    assert live() < n3
    _close(s.eb, s.pr)
    assert live() == n0


def test_destroy_in_the_middle_of_a_drive(oracle, live):
    """W == O with de-skew: from scan O on every scan inserts on the map's stream and runs local-cloud work on its own; the estimator
    is destroyed right after a scan returns, with that work still queued."""
    n0 = live()
    W = O = 4
    s = _Setup(oracle, W, O, O + 2)
    s.eg.attach_map(s.pm)
    for i in range(O + 2):
        _scan(s, s.eg, W + i)
    assert s.eg.map_poses()[3]["inserted"]
    s.eg.close()
    _close(s.pm, s.eb, s.pr)
    assert live() == n0


def test_bench_estimator_allocates_nothing_after_warm_up(live):
    """The bench's hdl64 estimator fed by the point processor: after the first solve (graph capture) and three warm-up scans the
    timed scans allocate and free nothing."""
    import ctypes as C
    from lio_mapping_b200 import _lib, estimator, ops, scenario
    from lio_mapping_b200.point_processor import PointProcessor
    kind, warmup, steps = "hdl64", 3, 3
    W, cfg = scenario.WINDOWS[kind], dict(scenario.EST_CFG[kind])
    scn = scenario.Scenario(kind, n_total=W + warmup + steps + 1)
    max_pts = max(r.shape[0] for r in scn.raw)
    n0 = live()
    pp = PointProcessor(scn.sensor.lower_deg, scn.sensor.upper_deg, scn.sensor.rings, max_points=max_pts)
    est = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 16, max_scan_points=max_pts, **cfg)

    def surf_ds_of(k):
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        return ops.voxel_grid(pp.cloud("surface_points_less_flat"), cfg["surf_filter_size"])

    scenario.warm_start(est, scn, W, surf_ds_of,
                        lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=cfg["acc_n"], gyr_n=cfg["gyr_n"],
                                                   acc_w=cfg["acc_w"], gyr_w=cfg["gyr_w"], g_norm=cfg["g_norm"]))
    lf_ptr = pp.cloud_dev("surface_points_less_flat")
    nptr = C.c_void_p()
    _lib.check(_lib.lib().lio_pp_cloud_count_dev(pp._h, 5, C.byref(nptr)), "lio_pp_cloud_count_dev")

    def step(k):
        est.begin_scan()
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        scenario.feed_imu(est, scn, k)
        est.process_scan_dev(lf_ptr, nptr.value, max_pts)

    for k in range(W, W + warmup):
        step(k)
    n1 = live()
    for k in range(W + warmup, W + warmup + steps):
        step(k)
        assert live() == n1, k
    _close(est, pp)
    assert live() == n0
