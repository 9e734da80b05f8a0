"""The plain PointProcessor statement (tests/pp_ref.py) against the oracle on stage A's edge inputs: ring order, mask, labels and
index sets element for element, xyz bit for bit, and both intensity encodings bit for bit except where the oracle's atan2f
rounds an angle differently; every such difference must be one of the statement's one-ulp alternatives."""
import numpy as np
import pytest

from tests import pp_ref as R

SETS = ("idx_orig_index", "scan_ranges", "mask", "labels", "idx_sharp", "idx_less_sharp", "idx_flat")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    """float32 arrays equal bit for bit, any NaN matching any NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))


def _ring_of(o, R_):
    starts = o["scan_ranges"][:, 0].astype(np.int64)
    counts = np.diff(np.append(starts, o["laser_scans"].shape[0]))
    return np.repeat(np.arange(R_), counts)


def compare(oracle, cloud, cfg, rings=None):
    """Asserts the statement equals the oracle; returns (points that differ, of which ambiguous, whether rings moved)."""
    s = R.process(cloud, cfg, rings)
    o = oracle.stage_a(cloud, cfg["lower_bound"], cfg["upper_bound"], cfg["num_rings"], cfg["scan_period"], ring_field=rings)
    n = cloud.shape[0]
    o_orig = o["idx_orig_index"].astype(np.int64)
    # start_ori_: the first accepted point's azimuth, up to one float32 ulp of its atan2
    o_first = int(o_orig.min()) if o_orig.size else -1
    alt0 = R.point_alternatives(cloud, cfg, o["start_ori"], rings, s.get("end_ori"))
    if o_first >= 0:
        assert o_first == int(s["idx_orig_index"].min())
        cand = {float(R.azimuth(R._ulp_shift(np.float32(np.arctan2(np.float64(cloud[o_first, 1]), np.float64(cloud[o_first, 0]))), k)))
                for k in (-1, 0, 1)}
        assert float(o["start_ori"]) in cand
    if rings is not None and o_orig.size:
        # the ring-field alternatives take the statement's end_ori_, so they hold only for the statement's start_ori_
        assert np.float32(o["start_ori"]) == s["start_ori"]
    # per point, keyed by the input index
    o_ring = np.full(n, -1)
    o_ring[o_orig] = _ring_of(o, cfg["num_rings"])
    o_laser = np.full(n, np.nan, np.float32)
    o_full = np.full(n, np.nan, np.float32)
    o_laser[o_orig], o_full[o_orig] = o["laser_scans"][:, 3], o["cloud_in_rings"][:, 3]
    s_ring = s["ring"]
    s_laser = np.full(n, np.nan, np.float32)
    s_full = np.full(n, np.nan, np.float32)
    s_laser[s["idx_orig_index"]], s_full[s["idx_orig_index"]] = s["laser_scans"][:, 3], s["cloud_in_rings"][:, 3]
    differ = (o_ring != s_ring) | ~_same(o_laser, s_laser) | ~_same(o_full, s_full)
    for i in np.flatnonzero(differ):
        ok = [(alt0["ring"][c, i] == o_ring[i]) and (o_ring[i] < 0 or (_same(alt0["laser"][c, i], o_laser[i])
                                                                         and _same(alt0["full"][c, i], o_full[i])))
              for c in range(9)]
        assert any(ok), (i, cloud[i], o_ring[i], s_ring[i], o_laser[i], s_laser[i])
    amb_in = np.zeros(n, bool)
    amb_in[s["idx_orig_index"]] = s["ambiguous"]
    # xyz of every ring-ordered point is its input point, bit for bit
    assert np.array_equal(_bits(o["laser_scans"][:, :3]), _bits(cloud[o_orig, :3]))
    assert np.array_equal(_bits(o["cloud_in_rings"][:, :3]), _bits(cloud[o_orig, :3]))
    moved = bool(np.any(o_ring != s_ring))
    if not moved:
        for k in SETS:
            assert np.array_equal(np.asarray(s[k], np.int64), np.asarray(o[k], np.int64)), k
        assert np.array_equal(_bits(s["laser_scans"][:, :3]), _bits(o["laser_scans"][:, :3]))
        for k in ("sharp", "less_sharp", "flat"):
            assert np.array_equal(_bits(s[k][:, :3]), _bits(o[k][:, :3])), k
        assert s["less_flat"].shape == o["less_flat"].shape
        assert np.array_equal(_bits(s["less_flat"][:, :3]), _bits(o["less_flat"][:, :3]))
        # the less-flat intensity is int(I) + rel_time of the centroid's own atan2: one float32 ulp of the azimuth either way.
        # With range_ori = 0 the centroid's I is NaN and int(NaN) is undefined in C++: those points are not compared.
        keep = ~np.isnan(s["less_flat"][:, 3])
        a, b = s["less_flat"][keep, 3], o["less_flat"][keep, 3]
        tol = 2 * cfg["scan_period"] * np.spacing(np.float32(2 * np.pi)) / (2 * np.pi) + 2 * np.spacing(np.abs(b))
        assert np.all(_same(a, b) | (np.abs(a.astype(np.float64) - b) <= tol))
    return int(differ.sum()), int((differ & amb_in).sum()), moved


@pytest.mark.parametrize("rings", [16, 32, 64, 128])
def test_bucket_edges_match_oracle(oracle, rings):
    cfg = R.preset_config(rings)
    cloud = R.bucket_edge_cloud(rings)
    s = R.point_to_ring(cloud, cfg)
    # the input really sits on the edges: some points change ring one ulp away, some lie half a bucket below ring 0
    assert s["ambiguous_in"].sum() >= rings
    v_below = (s["ring"] == 0) & (R.elevation_to_ring(R.raw_angles(cloud)[0].astype(np.float32), cfg) == 0)
    assert v_below.any()
    compare(oracle, cloud, cfg)


def test_truncation_accepts_points_below_ring_0():
    cfg = R.preset_config(16)
    factor = float(R._factor(cfg))
    below = np.radians(cfg["lower_bound"] - 1.0 / factor)     # v = -0.5: ring 0 by truncation toward zero
    far = np.radians(cfg["lower_bound"] - 1.6 / factor)       # v = -1.1: rejected
    xyz = R._points_at(np.array([below, far], np.float32), np.array([0.3, 0.3]), np.array([5.0, 5.0]))
    s = R.point_to_ring(np.concatenate([xyz, np.ones((2, 1), np.float32)], 1), cfg)
    assert list(s["ring"]) == [0, -1]


@pytest.mark.parametrize("rings", [16, 32, 64, 128])
def test_azimuth_wrap_and_first_point_match_oracle(oracle, rings):
    cfg = R.preset_config(rings)
    compare(oracle, R.azimuth_wrap_cloud(rings), cfg)
    for name, cloud in R.first_point_cases(rings):
        s = R.point_to_ring(cloud, cfg)
        assert s["idx_orig_index"].min() > 0, name            # start_ori_ comes from a later point
        compare(oracle, cloud, cfg)


def test_pick_loops_ties_and_occlusion_match_oracle(oracle):
    cfg = R.config()
    cloud = R.pick_ring(8)
    s = R.process(cloud, cfg)
    # the pick walks really pass a whole 32-candidate chunk of masked candidates, and meet candidates failing the threshold
    assert R.chunk_skips(s, "corner") and R.chunk_skips(s, "flat")
    assert R.stop_breaks(s, "corner")
    # curvature ties at exactly 0 among the flat candidates
    st, en = s["scan_ranges"][8]
    assert (R.curvature(s["laser_scans"][st:en + 1], 5)[5:-5] == 0).sum() > 100
    assert compare(oracle, cloud, cfg)[2] is False
    assert compare(oracle, R.plane_ring(600), cfg)[2] is False


@pytest.mark.parametrize("d", [5])
def test_ring_sizes_around_the_skip_match_oracle(oracle, d):
    cfg = R.config()
    for n in (2 * d + 1, 2 * d + 2, 2 * d + 3):
        cloud = R.plane_ring(n, seed=n, occlusion=False)
        cloud[:, 1] *= 40.0                                   # far-apart points: PrepareRing masks them
        s = R.process(cloud, cfg)
        assert compare(oracle, cloud, cfg)[2] is False
        if n == 2 * d + 1:
            assert not s["mask"].any()


def test_scatter_order_matches_oracle(oracle):
    cfg = R.preset_config(128)
    per = np.random.default_rng(3).integers(0, 40, 128)
    compare(oracle, R.interleaved_rings(cfg, per, seed=3), cfg)


@pytest.mark.parametrize("name", ["ids", "start_near_2pi", "equal_azimuths"])
def test_ring_field_matches_oracle(oracle, name):
    cfg = R.config()
    [(_, cloud, rings)] = [c for c in R.ring_field_cases() if c[0] == name]
    s = R.process(cloud, cfg, rings)
    if name == "equal_azimuths":
        assert np.isnan(s["laser_scans"][:, 3]).all()          # range_ori = 0: rel_time is 0 / 0
    if name == "start_near_2pi":
        assert s["start_ori"] > np.float32(6.28)
    assert compare(oracle, cloud, cfg, rings)[2] is False


def test_synthetic_sweeps_match_oracle(oracle):
    from lio_mapping_b200 import synth
    for kind, seed in [("vlp16", 1), ("hdl64", 3)]:
        sensor, scene, traj = synth.default_config(kind)
        sw = synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * seed, seed=seed)
        cfg = R.config(lower_bound=sensor.lower_deg, upper_bound=sensor.upper_deg, num_rings=sensor.rings)
        compare(oracle, sw, cfg)
