"""Plain float32 numpy statement of pcl::VoxelGrid<PointXYZI>::applyFilter (PCL 1.8) and of the stable radix sort under the
device copies, written in the operation order the kernels document.  Imports nothing from the package or the oracle: it is
the independent yardstick the device VoxelGrid copies (VoxelGrid, SegVoxelGrid, stage A's per-ring grid) and the radix
sort are compared with.

VoxelGrid, step by step:
  inv = float32(1) / leaf; bounding box min / max per axis in float32;
  PCL's index-overflow check: int64((max - min) * inv) + 1 per axis, product > INT_MAX -> the output is the input;
  min_b = floor(min * inv); ijk = int(floor(p * inv) - float32(min_b)); index = i + j * div_x + k * div_x * div_y in int32
  arithmetic (wrapping), read as uint32;
  stable sort by index (input order inside a voxel); per voxel a sequential float32 sum in input order, then one float32
  division by the count.
"""
from __future__ import annotations

import numpy as np

INT32_MAX = 2 ** 31 - 1
_SEQ_RANK_LIMIT = 64   # voxels with more points are summed by np.add.accumulate (sequential) one at a time


def voxel_index(xyz: np.ndarray, leaf: float):
    """PCL's voxel index of every point (uint32) and whether the index-overflow check fires (then the index is None)."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    inv = np.float32(1) / np.float32(leaf)
    mn, mx = xyz.min(0), xyz.max(0)
    d = [int(np.float32(mx[a] - mn[a]) * inv) + 1 for a in range(3)]      # float32 product, truncation toward zero
    assert d[0] * d[1] * d[2] < 2 ** 63, "PCL's int64 product itself would overflow: outside what this statement covers"
    if d[0] * d[1] * d[2] > INT32_MAX:
        return None, True
    min_b = [int(np.floor(mn[a] * inv)) for a in range(3)]
    max_b = [int(np.floor(mx[a] * inv)) for a in range(3)]
    div = [max_b[a] - min_b[a] + 1 for a in range(3)]
    ijk = [(np.floor(xyz[:, a] * inv) - np.float32(min_b[a])).astype(np.int64) for a in range(3)]
    idx = ijk[0] + ijk[1] * div[0] + ijk[2] * ((div[0] * div[1]) & 0xFFFFFFFF)
    return (idx & 0xFFFFFFFF).astype(np.uint32), False


def sequential_segment_sums(vals: np.ndarray, starts: np.ndarray, counts: np.ndarray) -> np.ndarray:
    """Float32 sums of vals[starts[v] : starts[v] + counts[v]] (rows of 4 channels), each accumulated left to right from 0."""
    acc = np.zeros((starts.shape[0], vals.shape[1]), np.float32)
    small = counts <= _SEQ_RANK_LIMIT
    for r in range(int(counts[small].max(initial=0))):         # rank by rank: every small voxel adds its r-th point
        sel = np.nonzero(small & (counts > r))[0]
        acc[sel] += vals[starts[sel] + r]
    for v in np.nonzero(~small)[0]:                             # np.add.accumulate is a strict left fold (np.sum is pairwise)
        acc[v] = np.add.accumulate(vals[starts[v]:starts[v] + counts[v]], axis=0, dtype=np.float32)[-1]
    return acc


def voxel_grid(cloud: np.ndarray, leaf: float) -> np.ndarray:
    """pcl::VoxelGrid<PointXYZI> with setLeafSize(leaf, leaf, leaf): centroids (x, y, z, intensity) in ascending voxel-index
    order, or the input unchanged when PCL's index-overflow check fires."""
    cloud = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    if cloud.shape[0] == 0:
        return cloud.copy()
    idx, overflow = voxel_index(cloud[:, :3], leaf)
    if overflow:
        return cloud.copy()
    order = np.argsort(idx, kind="stable")
    sk = idx[order]
    starts = np.flatnonzero(np.concatenate([[True], sk[1:] != sk[:-1]]))
    counts = np.diff(np.append(starts, sk.shape[0]))
    sums = sequential_segment_sums(cloud[order], starts, counts)
    return sums / counts.astype(np.float32)[:, None]


def radix_sort_pairs(keys: np.ndarray, vals: np.ndarray, key_bits: int):
    """Stable sort of (key, value) pairs by the low key_bits bits rounded up to whole bytes (one 8-bit pass per byte)."""
    keys = np.asarray(keys, np.uint32)
    mask = np.uint32((1 << (8 * -(-key_bits // 8))) - 1)
    order = np.argsort(keys & mask, kind="stable")
    return keys[order], np.asarray(vals, np.uint32)[order]


# ---- edge inputs of the VoxelGrid copies (shared by the CPU pinning test and the GPU tests) --------------------------------
LEAVES = (0.1, 0.2, 0.3, 0.4, 5.0)
SIZES = (1, 255, 256, 257, 2047, 2049, 2_000_000)


def _with_intensity(xyz, rng):
    return np.concatenate([np.asarray(xyz, np.float32), rng.uniform(0, 100, (len(xyz), 1)).astype(np.float32)], 1)


def edge_cloud(kind: str, n: int, leaf: float, seed: int = 0) -> np.ndarray:
    """one_voxel     every point inside one voxel: one run across all emit / sort tiles
       own_voxel     every point in its own voxel, in shuffled order, on both sides of zero
       lattice       coordinates k * leaf in float32 (and the float32 of the decimal product) plus one ulp either side, k of
                     both signs, each point repeated so that voxels hold several points in shuffled order
       straddle      uniform over a box around the origin on every axis
       overflow      a leaf far too small for the extent: PCL's index-overflow check fires, the output is the input"""
    rng = np.random.default_rng(seed)
    lf = np.float32(leaf)
    if kind == "one_voxel":
        inv = np.float32(1) / lf
        lo = np.float32(7) * lf
        centre = lo + np.float32(0.5) * lf
        xyz = lo + rng.uniform(0.05, 0.95, (n, 3)).astype(np.float32) * lf
        xyz = xyz[np.all(np.floor(xyz * inv) == np.floor(centre * inv), 1)]
        xyz = np.concatenate([xyz, np.full((n - xyz.shape[0], 3), centre, np.float32)])
        return _with_intensity(xyz, rng)
    if kind == "own_voxel":
        side = int(np.ceil(n ** (1 / 3))) + 1
        cells = rng.permutation(side ** 3)[:n]
        ijk = np.stack([cells % side, cells // side % side, cells // (side * side)], 1) - side // 2
        return _with_intensity((ijk.astype(np.float32) + np.float32(0.5)) * lf, rng)
    if kind == "lattice":
        k = rng.integers(-12, 13, (max(n // 4, 1), 3))
        base = np.where(rng.uniform(size=k.shape) < 0.5, k.astype(np.float32) * lf, (k * float(leaf)).astype(np.float32))
        step = rng.integers(-1, 2, base.shape)
        xyz = np.where(step < 0, np.nextafter(base, np.float32(-np.inf)), np.where(step > 0, np.nextafter(base, np.float32(np.inf)), base))
        xyz = xyz[rng.integers(0, xyz.shape[0], n)]
        return _with_intensity(xyz, rng)
    if kind == "straddle":
        return _with_intensity(rng.uniform(-3.0, 3.0, (n, 3)) * max(1.0, leaf), rng)
    if kind == "overflow":
        return _with_intensity(rng.uniform(-50.0, 50.0, (n, 3)), rng)
    raise ValueError(kind)


VOXEL_CASES = ([("one_voxel", n, 0.4) for n in SIZES] + [("own_voxel", n, 0.2) for n in SIZES]
               + [("lattice", 4096, leaf) for leaf in LEAVES] + [("lattice", 2049, 0.3)]
               + [("straddle", n, leaf) for n in (255, 257, 2049) for leaf in LEAVES]
               + [("overflow", n, 1e-3) for n in SIZES if n > 1])


def case_id(case) -> str:
    return "%s-%d-%g" % case


def overflow_boundary_clouds():
    """Two-axis and three-axis clouds on either side of PCL's dx * dy * dz > INT_MAX check at leaf 1 (46341^2 and 1291^3
    exceed INT_MAX, 46340 * 46341 and 1290^3 do not): (name, cloud, leaf, overflows)."""
    rng = np.random.default_rng(5)
    out = []
    for name, far, ovf in [("2axis_below", (46339.5, 46340.5, 0.5), False), ("2axis_above", (46340.5, 46340.5, 0.5), True),
                           ("3axis_below", (1289.5, 1289.5, 1289.5), False), ("3axis_above", (1290.5, 1290.5, 1290.5), True),
                           ("1axis_near_int_max", (2147483520.0, 0.0, 0.0), False)]:
        xyz = np.concatenate([[[0.25, 0.25, 0.25], far], rng.uniform(0, 1, (2047, 3)) * np.asarray(far)]).astype(np.float32)
        out.append((name, _with_intensity(xyz, rng), 1.0, ovf))
    return out


# ---- stage A's less-flat cloud (PointProcessor.cc:647-783) rebuilt from the processor's own ring-ordered outputs ----------
def subregions(scan_size: int, d: int, S: int):
    """The (sp, ep) ranges ExtractFeaturePoints processes in one ring (PointProcessor.cc:672-675, size_t arithmetic), with the
    rings the reference skips (:660) giving none."""
    if scan_size <= 2 * d + 1:
        return []
    out = []
    for j in range(S):
        sp = (d * (S - j) + (scan_size - d) * j) // S
        ep = (d * (S - 1 - j) + (scan_size - d) * (j + 1)) // S - 1
        if ep > sp:
            out.append((sp, ep))
    return out


def less_flat_members(scan_ranges: np.ndarray, labels: np.ndarray, d: int, S: int):
    """Per ring, the ring-ordered indices of the points that enter the ring's VoxelGrid: label <= 0 inside a processed
    subregion.  Points outside every processed subregion also carry label 0, so the label alone does not decide."""
    rings = []
    for start, end in np.asarray(scan_ranges, np.int64):
        size = int(end - start + 1) if end >= start else 0
        mem = [np.arange(sp, ep + 1) for sp, ep in subregions(size, d, S)]
        mem = np.concatenate(mem) if mem else np.zeros(0, np.int64)
        rings.append(int(start) + mem[labels[int(start) + mem] <= 0])
    return rings


def _rel_time(xy: np.ndarray, start_ori: float, scan_period: float) -> np.ndarray:
    """:758-776: azimuth of the point, its offset from start_ori_ and the relative time (float, double atan2)."""
    f64 = lambda a: np.asarray(a, np.float64)
    atan = np.arctan2(f64(xy[:, 1]), f64(xy[:, 0])).astype(np.float32)
    azi = (2 * np.pi - f64(atan)).astype(np.float32)
    azi = np.where(f64(azi) >= 2 * np.pi, (f64(azi) - 2 * np.pi).astype(np.float32), azi)
    rel = azi - np.float32(start_ori)
    rel = np.where(rel < 0, (f64(rel) + 2 * np.pi).astype(np.float32), rel)
    return (scan_period * f64(rel) / (2 * np.pi)).astype(np.float32)


def less_flat_cloud(laser_scans, scan_ranges, labels, d, S, leaf, start_ori, scan_period=0.1):
    """surface_points_less_flat_: every ring's members through VoxelGrid(leaf), rings in order, then intensity =
    int(intensity) + relative time of the output point.  Also returns, per ring, whether its index-overflow check fired."""
    parts, overflowed = [], []
    for mem in less_flat_members(scan_ranges, labels, d, S):
        if mem.shape[0] == 0:
            overflowed.append(False)
            continue
        ring = np.ascontiguousarray(laser_scans[mem], np.float32)
        overflowed.append(voxel_index(ring[:, :3], leaf)[1])
        parts.append(voxel_grid(ring, leaf))
    out = np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)
    out[:, 3] = np.trunc(out[:, 3]) + _rel_time(out[:, :2], start_ori, scan_period)
    return out, overflowed
