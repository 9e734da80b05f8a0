"""PointMapping::UpdateMapDatabase on the device (csrc/cubemap.cu pm_update, csrc/voxel.cu SegVoxelGrid) through its own entry,
lio_pm_update_map_database_host, against the oracle's CubeMap::UpdateMapDatabase (orc_cm_update) bit for bit: a few cubes, every
cube of the 5 x 5 x 5 block, a margin centre that differs from the current centre, and valid cubes holding more points than the
handle's max_points.  lio_pm_process_* and lio_mb_process_map_* run the same code; their parity tests cover those paths."""
import numpy as np
import pytest

from lio_mapping_b200 import _lib

pytestmark = pytest.mark.gpu

CEN = (10, 10, 5)


def _cloud(rng, n, lo, hi):
    xyz = rng.uniform(lo, hi, (n, 3))
    return np.concatenate([xyz, rng.uniform(0, 5, (n, 1))], 1).astype(np.float32)


def _tf(yaw, t):
    return np.array([0, 0, np.sin(yaw / 2), np.cos(yaw / 2), *t], np.float32)


def _block(centre):
    i0, j0, k0 = centre
    return np.array([i + 21 * j + 441 * k for i in range(i0 - 2, i0 + 3) for j in range(j0 - 2, j0 + 3) for k in range(k0 - 2, k0 + 3)], np.int64)


def _assert_same_cubes(pg, cm):
    nonempty = 0
    for w, which in enumerate(("corner", "surf")):
        sg = pg.cube_sizes(which)
        so = np.array([cm.L.orc_cm_cube_size(cm.h, i, w) for i in range(21 * 21 * 11)])
        assert np.array_equal(sg, so), (which, np.nonzero(sg != so)[0][:10])
        for idx in np.nonzero(so)[0]:
            assert np.array_equal(pg.cube(idx, which), cm.cube(idx, which)), (which, idx)
        nonempty += int((so > 0).sum())
    return nonempty


def _run(oracle, rounds, max_points=1 << 17):
    from lio_mapping_b200.point_mapping import PointMapping
    pg = PointMapping(max_points=max_points, corner_filter_size=0.2, surf_filter_size=0.4)
    cm = oracle.CubeMap()
    stats = []
    for corner, surf, valid, tf7, margin in rounds:
        cm.update(corner, surf, valid, tf7, margin)
        stats.append(pg.UpdateMapDatabase(corner, surf, valid, tf7, margin))
    return pg, cm, stats


def test_few_cubes_bit_exact(oracle):
    """Clouds around the sensor's cube, three inserts (the second and third land in non-empty cubes and grow segments)."""
    rng = np.random.default_rng(7)
    valid = _block(CEN)[::7]
    rounds = [(_cloud(rng, 900, -30, 30), _cloud(rng, 5000, -30, 30), valid, _tf(0.1 * r, (1.0 * r, -0.5, 0.2)), CEN) for r in range(3)]
    pg, cm, stats = _run(oracle, rounds)
    assert _assert_same_cubes(pg, cm) >= 8
    assert all(s["points"] == 5900 for s in stats) and all(1 <= s["jobs"] < 20 for s in stats)
    assert stats[0]["waits"] == 2          # the first insert only allocates: the run list and, later, the re-filtered sizes


def test_every_cube_of_the_block_bit_exact(oracle):
    """Points over the whole 5 x 5 x 5 block and every block cube valid: 250 jobs in one segmented VoxelGrid, with the same launch
    count as an update that re-filters a handful of cubes.  A few points fall outside the cube array and are dropped."""
    rng = np.random.default_rng(11)
    far = np.array([[1e4, 0, 0, 1], [0, -2e4, 0, 2], [0, 0, 600, 3]], np.float32)
    valid = _block(CEN)
    rounds = [(np.concatenate([_cloud(rng, 20000, -124, 124), far]), _cloud(rng, 60000, -124, 124), valid, _tf(0.05 * r, (0.3 * r, 0.1, 0)), CEN)
              for r in range(2)]
    few = (_cloud(rng, 500, -20, 20), _cloud(rng, 2000, -20, 20), valid[:3], _tf(0.0, (0, 0, 0)), CEN)
    pg, cm, stats = _run(oracle, rounds + [few])
    assert _assert_same_cubes(pg, cm) > 250                 # the rotated clouds also reach cubes around the block
    assert stats[0]["jobs"] == 250 and stats[1]["jobs"] == 250 and 1 <= stats[2]["jobs"] <= 6
    assert stats[2]["launches"] == stats[0]["launches"] == stats[1]["launches"]


def test_margin_centre_differs_from_current_centre(oracle):
    """valid computed with an older centre (the estimator's margin centre): the indices move to the current centre, and those that
    leave the array are skipped (PointMapping.cc:1173-1183)."""
    rng = np.random.default_rng(5)
    rounds = []
    for r, margin in enumerate([(11, 9, 5), (8, 12, 6)]):
        rounds.append((_cloud(rng, 3000, -110, 110), _cloud(rng, 12000, -110, 110), _block(margin), _tf(0.2, (2.0, 1.0 * r, 0.5)), margin))
    # a block around cube (14, 10, 5) of the centre (4, 10, 5): its x columns 12..16 move to 18..22, so two leave the array
    far = [np.concatenate([rng.uniform(300, 530, (n, 1)), rng.uniform(-110, 110, (n, 2)), rng.uniform(0, 5, (n, 1))], 1).astype(np.float32)
           for n in (3000, 12000)]
    valid3 = np.array([i + 21 * j + 441 * k for i in range(12, 17) for j in range(8, 13) for k in range(3, 8)], np.int64)
    rounds.append((far[0], far[1], valid3, _tf(0.0, (0, 0, 0)), (4, 10, 5)))
    pg, cm, stats = _run(oracle, rounds)
    assert _assert_same_cubes(pg, cm) > 40
    moved = [v + 6 for v in valid3 if v % 21 + 6 < 21]
    assert len(moved) == 75
    assert stats[2]["jobs"] == sum(cm.L.orc_cm_cube_size(cm.h, int(v), w) > 0 for v in moved for w in (0, 1)) > 0


def test_valid_cubes_beyond_max_points(oracle):
    """The re-filter's workspace grows past max_points: the valid cubes hold more points than one call may insert."""
    rng = np.random.default_rng(9)
    valid = _block(CEN)
    rounds = [(_cloud(rng, 1000, -24, 24), _cloud(rng, 4000, -24, 24), valid, _tf(0.0, (0.0, 0.0, 0.0)), CEN) for _ in range(6)]
    pg, cm, _ = _run(oracle, rounds, max_points=4096)
    _assert_same_cubes(pg, cm)
    assert pg.cube(21 * 21 * 5 + 21 * 10 + 10, "surf").shape[0] > 4096


def test_update_map_database_errors():
    from lio_mapping_b200.point_mapping import PointMapping
    pg = PointMapping(max_points=1024)
    c = np.zeros((10, 4), np.float32)
    tf = _tf(0.0, (0, 0, 0))
    for valid in ([5, 5], [-1], [21 * 21 * 11]):
        with pytest.raises(_lib.LioError, match="INVALID"):
            pg.UpdateMapDatabase(c, c, np.array(valid), tf, CEN)
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        pg.UpdateMapDatabase(c, c, np.arange(126), tf, CEN)
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        pg.UpdateMapDatabase(np.zeros((1025, 4), np.float32), c, [], tf, CEN)
    assert pg.cube_sizes("surf").sum() == 0 and pg.cube_sizes("corner").sum() == 0


def test_voxel_bound_error_is_sticky():
    """A leaf too small for a full cube (0.1 m over 50 m: 500^3 voxels > 2^24) makes the re-filter's key overflow: the next reader
    of the cubes reports LIO_ERR_CAPACITY, and so does every later call, instead of handing out wrong centroids."""
    from lio_mapping_b200.point_mapping import PointMapping
    pg = PointMapping(max_points=1 << 14, corner_filter_size=0.2, surf_filter_size=0.1)
    surf = np.array([[-24.9, -24.9, -24.9, 1.0], [24.9, 24.9, 24.9, 1.0], [0.0, 0.0, 0.0, 1.0]], np.float32)
    tf = _tf(0.0, (0, 0, 0))
    centre = 21 * 21 * 5 + 21 * 10 + 10
    pg.UpdateMapDatabase(np.zeros((0, 4), np.float32), surf, [centre], tf, CEN)
    for _ in range(2):
        with pytest.raises(_lib.LioError, match="CAPACITY"):
            pg.cube(centre, "surf")
    with pytest.raises(_lib.LioError, match="CAPACITY"):
        pg.UpdateMapDatabase(np.zeros((0, 4), np.float32), surf, [centre], tf, CEN)
    # a leaf of 0.2 m keeps a full cube inside the bound
    ok = PointMapping(max_points=1 << 14, corner_filter_size=0.2, surf_filter_size=0.2)
    ok.UpdateMapDatabase(np.zeros((0, 4), np.float32), surf, [centre], tf, CEN)
    assert ok.cube(centre, "surf").shape[0] == 3
