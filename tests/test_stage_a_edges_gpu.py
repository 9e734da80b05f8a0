"""Stage A on the device against the plain PointProcessor statement (tests/pp_ref.py) at its edges: the configuration range of
lio_pp_config, pick walks that skip whole 32-candidate chunks or stop early, curvature ties, bucket edges, scatter order across
classify blocks, ring sizes around the skip and the shared-memory limit, and the ring-field variant.  Every case runs twice on
fresh handles and must give the same bits both times."""
import numpy as np
import pytest

from tests import pp_ref as R

pytestmark = pytest.mark.gpu

CLOUDS = ("laser_scans", "cloud_in_rings", "corner_points_sharp", "corner_points_less_sharp", "surface_points_flat",
          "surface_points_less_flat")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _run_once(cloud, cfg, rings=None, max_points=None):
    from lio_mapping_b200.point_processor import PointProcessor
    lo, hi, nr = cfg["lower_bound"], cfg["upper_bound"], cfg["num_rings"]
    rest = {k: v for k, v in cfg.items() if k not in ("lower_bound", "upper_bound", "num_rings")}
    pp = PointProcessor(lo, hi, nr, max_points=max_points or max(cloud.shape[0], 1), **rest)
    try:
        pp.SetInputCloud(cloud)
        pp.Process() if rings is None else pp.ProcessWithRingField(rings)
        g = {k: pp.cloud(k) for k in CLOUDS}
        for k in ("sharp", "less_sharp", "flat", "orig"):
            g["idx_" + k] = pp.index(k)
        g["scan_ranges"] = pp.scan_ranges()
        g["mask"], g["labels"] = pp.mask_labels()
        g["start_ori"] = np.float32(pp.start_ori())
        g["sizes"] = pp.sizes()
        return g
    finally:
        pp.close()


def run(cloud, cfg, rings=None):
    """Two runs on fresh handles, bit-identical; returns one."""
    a, b = _run_once(cloud, cfg, rings), _run_once(cloud, cfg, rings)
    for k in a:
        if isinstance(a[k], np.ndarray) and a[k].dtype == np.float32:
            assert np.array_equal(_bits(a[k]), _bits(b[k])), k
        elif k == "sizes":
            assert a[k] == b[k]
        else:
            assert np.array_equal(a[k], b[k]), k
    return a


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))


def check(cloud, cfg, rings=None):
    """Device against the statement; returns the statement's result."""
    s = R.process(cloud, cfg, rings)
    g = run(cloud, cfg, rings)
    n = cloud.shape[0]
    assert all(v >= 0 for v in g["sizes"].values()), g["sizes"]
    g_orig = g["idx_orig"].astype(np.int64)
    g_ring = np.full(n, -1)
    starts = g["scan_ranges"][:, 0].astype(np.int64)
    g_ring[g_orig] = np.repeat(np.arange(cfg["num_rings"]), np.diff(np.append(starts, g_orig.shape[0])))
    amb = np.zeros(n, bool)
    amb[s["idx_orig_index"]] = s["ambiguous"]
    moved = g_ring != s["ring"]
    if moved.any():
        # only ambiguous points may move, and only to a ring one float32 ulp of elevation away
        alt = R.point_alternatives(cloud, cfg, g["start_ori"], rings, s.get("end_ori"))
        for i in np.flatnonzero(moved):
            assert amb[i] and g_ring[i] in alt["ring"][:, i], (i, cloud[i], g_ring[i], s["ring"][i])
        return s
    assert g["start_ori"].tobytes() == np.float32(s["start_ori"]).tobytes()
    assert np.array_equal(g_orig, s["idx_orig_index"])
    assert np.array_equal(g["scan_ranges"], s["scan_ranges"])
    assert np.array_equal(g["mask"], s["mask"])
    assert np.array_equal(g["labels"], s["labels"])
    for k in ("sharp", "less_sharp", "flat"):
        assert np.array_equal(g["idx_" + k], s["idx_" + k]), k
    assert np.array_equal(_bits(g["laser_scans"][:, :3]), _bits(s["laser_scans"][:, :3]))
    assert np.array_equal(_bits(g["cloud_in_rings"][:, :3]), _bits(s["cloud_in_rings"][:, :3]))
    ring_amb = s["ambiguous"]
    for k in ("laser_scans", "cloud_in_rings"):
        same = _same(g[k][:, 3], s[k][:, 3])
        assert same[~ring_amb].all(), (k, np.flatnonzero(~same & ~ring_amb)[:8])
    for gk, sk in (("corner_points_sharp", "sharp"), ("corner_points_less_sharp", "less_sharp"), ("surface_points_flat", "flat")):
        assert np.array_equal(_bits(g[gk][:, :3]), _bits(s[sk][:, :3])), gk
    lf_g, lf_s = g["surface_points_less_flat"], s["less_flat"]
    assert lf_g.shape == lf_s.shape
    assert np.array_equal(_bits(lf_g[:, :3]), _bits(lf_s[:, :3]))
    defined = ~np.isnan(lf_s[:, 3])          # int(NaN) of a range_ori = 0 centroid is undefined in C++
    assert np.array_equal(_bits(lf_g[defined, 3]), _bits(lf_s[defined, 3]))
    return s


# ---- configurations -----------------------------------------------------------------------------------------------------------
def _sweep_with_pick_ring():
    from lio_mapping_b200 import synth
    sensor, scene, traj = synth.default_config("vlp16")
    sw = synth.make_sweep(sensor, scene, traj, 1.3, seed=2)
    return np.concatenate([sw, R.pick_ring(8, seed=1)])


CAPS = {"caps0": (0, 0, 0), "caps1": (1, 1, 1), "caps_max": (20, 64, 16)}
GRID = ([(16, 32, c, 0.1) for c in CAPS] + [(16, 32, "caps_max", th) for th in (0.0, 1e30)]
        + [(1, 1, "caps0", 0.1), (2, 7, "caps1", 0.1), (8, 32, "caps_max", 0.1), (1, 7, "caps_max", 0.1), (2, 1, "caps_max", 0.0),
           (8, 1, "caps1", 0.1), (16, 7, "caps0", 0.1), (16, 1, "caps_max", 0.1), (1, 32, "caps1", 1e30), (2, 32, "caps_max", 0.1)])


def test_default_configuration():
    check(_sweep_with_pick_ring(), R.config())


@pytest.mark.parametrize("d,S,caps,th", GRID, ids=["d%d-S%d-%s-th%g" % g for g in GRID])
def test_configuration_grid(d, S, caps, th):
    sharp, less, flat = CAPS[caps]
    cfg = R.config(num_curvature_regions=d, num_scan_subregions=S, max_corner_sharp=sharp, max_corner_less_sharp=less,
                   max_surf_flat=flat, surf_curv_th=th)
    check(_sweep_with_pick_ring(), cfg)


# ---- pick walks and ties ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,S", [(5, 8), (16, 8), (5, 1)])
def test_pick_walks_skip_whole_chunks_and_stop(d, S):
    cfg = R.config(num_curvature_regions=d, num_scan_subregions=S)
    s = check(R.pick_ring(8), cfg)
    assert R.chunk_skips(s, "corner"), "no corner pick after a 32-candidate masked chunk"
    if (d, S) != (16, 8):
        assert R.chunk_skips(s, "flat"), "no flat pick after a 32-candidate masked chunk"
    if S == 8:
        assert R.stop_breaks(s, "corner")
    if d == 16:
        assert R.stop_breaks(s, "flat")


def test_ties_duplicates_and_occlusion():
    cfg = R.config()
    s = check(R.pick_ring(2, seed=4), cfg)
    st, en = s["scan_ranges"][8]
    assert (R.curvature(s["laser_scans"][st:en + 1], 5)[5:-5] == 0).sum() > 50
    s = check(R.plane_ring(900, seed=2), cfg)
    assert R.chunk_skips(s, "flat")


# ---- buckets ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rings", [16, 32, 64, 128])
def test_bucket_edges_azimuth_wrap_and_first_point(rings):
    cfg = R.preset_config(rings)
    s = check(R.bucket_edge_cloud(rings), cfg)
    assert s["ambiguous"].sum() >= rings
    check(R.azimuth_wrap_cloud(rings), cfg)
    for _, cloud in R.first_point_cases(rings):
        check(cloud, cfg)


# ---- scatter order ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025])
def test_scatter_order_small(n):
    cfg = R.preset_config(16)
    per = np.random.default_rng(n).multinomial(n, np.full(16, 1 / 16))
    check(R.interleaved_rings(cfg, per, seed=n), cfg)


def test_scatter_order_one_million_points():
    cfg = R.preset_config(128)
    per = np.random.default_rng(9).integers(7800, 8150, 128)
    check(R.interleaved_rings(cfg, per, seed=9), cfg)


# ---- ring sizes -----------------------------------------------------------------------------------------------------------------
def test_ring_of_8192_points_in_one_subregion():
    cfg = R.config(num_scan_subregions=1)
    check(R.centre_ring_cloud(cfg, 3, 8192, seed=1), cfg)


def test_ring_of_8193_points_is_refused_and_the_handle_recovers():
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.point_processor import PointProcessor
    cfg = R.config()
    big = R.centre_ring_cloud(cfg, 3, 8193, seed=1)
    ok = np.concatenate([R.centre_ring_cloud(cfg, 3, 8192, seed=2), R.plane_ring(700, seed=3)])
    pp = PointProcessor(max_points=big.shape[0] + ok.shape[0])
    try:
        pp.SetInputCloud(big)
        with pytest.raises(_lib.LioError, match="LIO_ERR_CAPACITY"):
            pp.Process()
        pp.SetInputCloud(ok)
        pp.Process()
        s = R.process(ok, cfg)
        assert np.array_equal(pp.index("orig"), s["idx_orig_index"])
        m, lab = pp.mask_labels()
        assert np.array_equal(m, s["mask"]) and np.array_equal(lab, s["labels"])
        for k in ("sharp", "less_sharp", "flat"):
            assert np.array_equal(pp.index(k), s["idx_" + k]), k
        assert np.array_equal(_bits(pp.cloud("surface_points_less_flat")), _bits(s["less_flat"]))
    finally:
        pp.close()


@pytest.mark.parametrize("d", [1, 5, 16])
def test_rings_around_the_skip(d):
    cfg = R.config(num_curvature_regions=d)
    for n in (2 * d + 1, 2 * d + 2):
        cloud = R.plane_ring(n, seed=n, occlusion=False)
        cloud[:, 1] *= 40.0                  # far-apart points: PrepareRing would mask them if the ring were processed
        s = check(cloud, cfg)
        assert s["mask"].any() == (n == 2 * d + 2)


# ---- ring-field variant -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ids", "start_near_2pi", "equal_azimuths"])
def test_ring_field_edges(name):
    [(_, cloud, rings)] = [c for c in R.ring_field_cases() if c[0] == name]
    check(cloud, R.config(), rings)


# ---- configuration limits -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", ["max_corner_sharp", "max_corner_less_sharp", "max_surf_flat"])
def test_negative_pick_budgets_are_refused(field):
    """A negative budget used to be accepted: with max_corner_sharp < 0 the sharp count that lio_pp_cloud_sizes and
    lio_pp_cloud_count_dev hand on became negative."""
    from lio_mapping_b200 import _lib
    from lio_mapping_b200.point_processor import PointProcessor
    cfg = {field: -1}
    if field == "max_corner_less_sharp":
        cfg["max_corner_sharp"] = -1
    with pytest.raises(_lib.LioError, match="LIO_ERR_INVALID"):
        PointProcessor(max_points=16, **cfg)
