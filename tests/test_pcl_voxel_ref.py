"""The plain VoxelGrid statement (tests/pcl_voxel_ref.py) pinned bit for bit against the oracle on every edge input the GPU
tests feed the device copies, so that a GPU failure against it points at the device and not at the yardstick."""
import numpy as np
import pytest

from lio_mapping_b200 import synth
from tests import pcl_voxel_ref as ref


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("case", ref.VOXEL_CASES, ids=ref.case_id)
def test_reference_matches_oracle(oracle, case):
    kind, n, leaf = case
    cloud = ref.edge_cloud(kind, n, leaf)
    r = ref.voxel_grid(cloud, leaf)
    o = oracle.voxel_grid(cloud, leaf)
    assert r.shape == o.shape and np.array_equal(bits(r), bits(o))
    overflow = ref.voxel_index(cloud[:, :3], leaf)[1]
    assert overflow == (kind == "overflow")
    if kind == "overflow":
        assert np.array_equal(bits(r), bits(cloud))
    if kind == "one_voxel":
        assert r.shape[0] == 1
    if kind == "own_voxel":
        assert r.shape[0] == n


@pytest.mark.parametrize("name,cloud,leaf,overflow", ref.overflow_boundary_clouds(), ids=lambda v: v if isinstance(v, str) else "")
def test_overflow_boundary_matches_oracle(oracle, name, cloud, leaf, overflow):
    assert ref.voxel_index(cloud[:, :3], leaf)[1] == overflow
    r = ref.voxel_grid(cloud, leaf)
    assert np.array_equal(bits(r), bits(oracle.voxel_grid(cloud, leaf)))
    assert np.array_equal(bits(r), bits(cloud)) == overflow


def test_segment_sums_are_left_folds():
    """Both branches of the segmented sum (rank by rank, and np.add.accumulate for long runs) equal a float32 loop."""
    rng = np.random.default_rng(2)
    counts = np.array([1, 3, 64, 65, 1000, 2, 5000])
    vals = (rng.standard_normal((counts.sum(), 4)) * 10.0 ** rng.integers(-3, 6, (counts.sum(), 1))).astype(np.float32)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    got = ref.sequential_segment_sums(vals, starts, counts)
    for v, (s, c) in enumerate(zip(starts, counts)):
        acc = np.zeros(4, np.float32)
        for row in vals[s:s + c]:
            acc = acc + row
        assert np.array_equal(bits(got[v]), bits(acc)), v


def test_radix_reference_is_stable_by_whole_bytes():
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 1 << 32, 3000, dtype=np.uint64).astype(np.uint32)
    keys[::3] = keys[0]
    vals = np.arange(keys.shape[0], dtype=np.uint32)
    for key_bits, mask in [(8, 0xFF), (14, 0xFFFF), (24, 0xFFFFFF), (32, 0xFFFFFFFF)]:
        order = sorted(range(keys.shape[0]), key=lambda i: (int(keys[i]) & mask, i))
        ko, vo = ref.radix_sort_pairs(keys, vals, key_bits)
        assert np.array_equal(vo, np.array(order, np.uint32)) and np.array_equal(ko, keys[order])


def test_less_flat_rebuild_matches_oracle(oracle):
    """The per-ring member sets and the ring-by-ring VoxelGrid rebuilt from stage A's own ring-ordered outputs reproduce the
    oracle's pre-voxel index list and its surface_points_less_flat."""
    sensor, scene, traj = synth.default_config("vlp16")
    sw = synth.make_sweep(sensor, scene, traj, 1.3, seed=3)
    o = oracle.stage_a(sw, sensor.lower_deg, sensor.upper_deg, sensor.rings)
    d, S = 5, 8                                     # lio_pp_default_config / PointProcessorConfig defaults
    members = ref.less_flat_members(o["scan_ranges"], o["labels"], d, S)
    assert np.array_equal(np.concatenate(members), o["idx_less_flat_prevoxel"])
    got, overflowed = ref.less_flat_cloud(o["laser_scans"], o["scan_ranges"], o["labels"], d, S, 0.2, o["start_ori"])
    assert not any(overflowed)
    assert got.shape == o["less_flat"].shape
    assert np.array_equal(bits(got[:, :3]), bits(o["less_flat"][:, :3]))
    assert np.allclose(got[:, 3], o["less_flat"][:, 3], atol=1e-4, rtol=0)
