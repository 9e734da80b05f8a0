"""The device VoxelGrid copies and the radix sort under them against the plain statement of tests/pcl_voxel_ref.py, at their
structural edges: sort tiles (2048 keys) and emit tiles (256), look-back chains over hundreds of tiles, one run over every
tile, odd pass counts (result in the second buffer pair), top-byte keys, voxel faces, and PCL's index-overflow fallback.
Every case runs twice and the two results must agree bit for bit: nothing may depend on the order tiles are scheduled in."""
import numpy as np
import pytest

from lio_mapping_b200 import synth
from tests import pcl_voxel_ref as ref

pytestmark = pytest.mark.gpu

SORT_SIZES = (1, 255, 256, 257, 2047, 2048, 2049, 2048 * 32 - 1, 2048 * 32 + 1, 2048 * 33, 1 << 20, 4_000_001)
KEY_BITS = (8, 14, 24, 32)
PATTERNS = ("constant", "one_different", "ascending", "descending", "random", "one_digit", "top_byte", "duplicates")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def sort_keys(pattern: str, n: int, key_bits: int, rng) -> np.ndarray:
    passes = -(-key_bits // 8)
    if pattern == "constant":
        return np.full(n, 0x5AC3961E, np.uint32)
    if pattern == "one_different":                       # one key unlike the rest in every byte, in the last tile
        k = np.full(n, 0x80808080, np.uint32)
        k[n - 1 - rng.integers(0, min(n, 2048))] = 0x7F017F01
        return k
    if pattern in ("ascending", "descending"):
        k = np.linspace(0, 2 ** 32 - 1, n).astype(np.uint64).astype(np.uint32)
        return k if pattern == "ascending" else k[::-1].copy()
    if pattern == "random":
        return rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    if pattern == "one_digit":                           # every other pass sees all keys in one bin
        shift = 8 * (passes // 2)
        return (np.uint32(0x3C3C3C3C) & ~np.uint32(0xFF << shift)) | (rng.integers(0, 256, n).astype(np.uint32) << shift)
    if pattern == "top_byte":                            # SegVoxelGrid's job ids >= 128
        return (rng.integers(0, 256, n).astype(np.uint32) << 24) | np.uint32(0x00ABCDEF)
    if pattern == "duplicates":                          # few distinct keys: stability across tiles decides the order
        return (rng.integers(0, 5, n).astype(np.uint32) * np.uint32(0x01010101)) ^ np.uint32(0x00FF00FF)
    raise ValueError(pattern)


@pytest.mark.parametrize("key_bits", KEY_BITS)
@pytest.mark.parametrize("n", SORT_SIZES)
def test_radix_sort_pairs_matches_stable_argsort(n, key_bits):
    from lio_mapping_b200 import ops
    rng = np.random.default_rng(n * 64 + key_bits)
    vals = np.arange(n, dtype=np.uint32)                 # value = input index: the permutation itself is compared
    for pattern in PATTERNS:
        keys = sort_keys(pattern, n, key_bits, rng)
        ek, ev = ref.radix_sort_pairs(keys, vals, key_bits)
        k1, v1 = ops.radix_sort_pairs(keys, vals, key_bits)
        k2, v2 = ops.radix_sort_pairs(keys, vals, key_bits)
        assert np.array_equal(k1, k2) and np.array_equal(v1, v2), f"{pattern}: two runs differ"
        assert np.array_equal(v1, ev), f"{pattern}: permutation differs from the stable argsort"
        assert np.array_equal(k1, ek), pattern


def test_radix_sort_pairs_rejects_bad_arguments():
    from lio_mapping_b200 import _lib
    k = np.zeros(4, np.uint32)
    for bad_bits in (0, 33):
        assert _lib.lib().lio_radix_sort_pairs_host(k, k, 4, bad_bits, k, k, 0) == -2
    assert _lib.lib().lio_radix_sort_pairs_host(k, k, 0, 32, k, k, 0) == 0


def _device_voxel_grid(cloud, leaf):
    from lio_mapping_b200 import ops
    g1 = ops.voxel_grid(cloud, leaf)
    g2 = ops.voxel_grid(cloud, leaf)
    assert g1.shape == g2.shape and np.array_equal(bits(g1), bits(g2)), "two runs differ"
    return g1


@pytest.mark.parametrize("case", ref.VOXEL_CASES, ids=ref.case_id)
def test_voxel_grid_matches_reference(case):
    kind, n, leaf = case
    cloud = ref.edge_cloud(kind, n, leaf)
    g = _device_voxel_grid(cloud, leaf)
    r = ref.voxel_grid(cloud, leaf)
    assert g.shape == r.shape and np.array_equal(bits(g), bits(r))
    if kind == "overflow":
        assert np.array_equal(bits(g), bits(cloud))


@pytest.mark.parametrize("name,cloud,leaf,overflow", ref.overflow_boundary_clouds(), ids=lambda v: v if isinstance(v, str) else "")
def test_voxel_grid_overflow_boundary(name, cloud, leaf, overflow):
    g = _device_voxel_grid(cloud, leaf)
    assert np.array_equal(bits(g), bits(ref.voxel_grid(cloud, leaf)))
    assert np.array_equal(bits(g), bits(cloud)) == overflow


# ---- SegVoxelGrid ---------------------------------------------------------------------------------------------------------
def _seg_jobs(njobs: int, seed: int):
    """Jobs of one point, whole-voxel runs that cross the 256- and 2048-point tiles of the concatenation, lattice and
    face points, clouds around zero and one point per voxel, each with a leaf of its own."""
    kinds = [("one_point", 1), ("one_voxel", 3000), ("lattice", 700), ("straddle", 300), ("own_voxel", 257), ("one_voxel", 5)]
    clouds, leaves = [], []
    for j in range(njobs):
        kind, n = kinds[j % len(kinds)]
        leaf = ref.LEAVES[(j // len(kinds) + j) % len(ref.LEAVES)]
        c = ref.edge_cloud("straddle" if kind == "one_point" else kind, n, leaf, seed=seed + j)
        clouds.append(c[:1] if kind == "one_point" else c)
        leaves.append(leaf)
    return clouds, leaves


def _device_seg(clouds, leaves):
    from lio_mapping_b200 import ops
    a, err_a = ops.seg_voxel_grid(clouds, leaves)
    b, err_b = ops.seg_voxel_grid(clouds, leaves)
    assert err_a == err_b
    if not err_a:
        assert all(x.shape == y.shape and np.array_equal(bits(x), bits(y)) for x, y in zip(a, b)), "two runs differ"
    return a, err_a


@pytest.mark.parametrize("njobs", [1, 2, 255, 256])
def test_seg_voxel_grid_matches_voxel_grid_per_job(njobs):
    from lio_mapping_b200 import ops
    clouds, leaves = _seg_jobs(njobs, seed=njobs)
    outs, err = _device_seg(clouds, leaves)
    assert not err and len(outs) == njobs
    for j, (c, leaf, g) in enumerate(zip(clouds, leaves, outs)):
        r = ref.voxel_grid(c, leaf)
        assert g.shape == r.shape and np.array_equal(bits(g), bits(r)), f"job {j} vs the reference"
        assert np.array_equal(bits(g), bits(ops.voxel_grid(c, leaf))), f"job {j} vs VoxelGrid::run"


def _grid_job(extent, n, seed):
    """Leaf 1, floor-space grid of exactly extent[0] x extent[1] x extent[2] voxels, points spread over all of it."""
    rng = np.random.default_rng(seed)
    far = np.asarray(extent, np.float32) - np.float32(0.5)
    xyz = np.concatenate([[[0.5, 0.5, 0.5], far], rng.uniform(0, 1, (n, 3)) * (np.asarray(extent) - 0.01)]).astype(np.float32)
    return np.concatenate([xyz, rng.uniform(0, 100, (xyz.shape[0], 1)).astype(np.float32)], 1)


def test_seg_voxel_grid_index_bound():
    """A job of exactly 2^24 voxels fills the 24-bit voxel field of the key and is accepted; one of 2^24 + 1 voxels
    (97 * 257 * 673) sets the error flag and returns cleanly, and the next call works."""
    small, _ = _seg_jobs(3, seed=9)
    full = _grid_job((4096, 4096, 1), 6000, seed=1)
    jobs = [small[0], full, small[1], small[2]]
    leaves = [0.2, 1.0, 0.4, 0.3]
    outs, err = _device_seg(jobs, leaves)
    assert not err
    assert ref.voxel_index(full[:, :3], 1.0)[0].max() >= 1 << 23
    for j, (c, leaf) in enumerate(zip(jobs, leaves)):
        assert np.array_equal(bits(outs[j]), bits(ref.voxel_grid(c, leaf))), j
    over = _grid_job((97, 257, 673), 6000, seed=2)
    outs, err = _device_seg([small[0], over], [0.2, 1.0])
    assert err and outs is None
    outs, err = _device_seg(jobs, leaves)
    assert not err and np.array_equal(bits(outs[1]), bits(ref.voxel_grid(full, 1.0)))


# ---- stage A's per-ring VoxelGrid ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,leaf,seed", [("vlp16", 0.005, 3), ("hdl64", 0.01, 3), ("hdl64", 0.02, 5)])
def test_stage_a_less_flat_rings_match_reference(kind, leaf, seed):
    """A less_flat_filter_size small enough that PCL's index-overflow check fires on some rings (output = the ring's members)
    and not on others.  The members are rebuilt from the processor's own ring-ordered cloud, labels and scan ranges."""
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config(kind)
    sw = synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * seed, seed=seed)
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=sw.shape[0], less_flat_filter_size=leaf)
    try:
        runs = []
        for _ in range(2):
            pp.SetInputCloud(sw)
            pp.Process()
            runs.append(pp.cloud("surface_points_less_flat"))
        assert runs[0].shape == runs[1].shape and np.array_equal(bits(runs[0]), bits(runs[1])), "two runs differ"
        laser = pp.cloud("laser_scans")
        _, labels = pp.mask_labels()
        cfg = pp.cfg
        exp, overflowed = ref.less_flat_cloud(laser, pp.scan_ranges(), labels, cfg.num_curvature_regions, cfg.num_scan_subregions,
                                              np.float32(cfg.less_flat_filter_size), pp.start_ori(), cfg.scan_period)
    finally:
        pp.close()
    assert any(overflowed) and not all(overflowed), overflowed
    g = runs[0]
    assert g.shape == exp.shape
    assert np.array_equal(bits(g[:, :3]), bits(exp[:, :3]))
    assert np.allclose(g[:, 3], exp[:, 3], atol=1e-4, rtol=0)
