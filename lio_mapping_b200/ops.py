"""Thin Python wrappers over the host-array C-ABI entry points (used by the parity tests)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib


def voxel_grid(cloud: np.ndarray, leaf: float, device: int = 0) -> np.ndarray:
    """pcl::VoxelGrid<PointXYZI> on the GPU (lio_voxel_grid_host)."""
    _lib.require_device()
    cloud = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    out = np.zeros((max(cloud.shape[0], 1), 4), np.float32)
    n = C.c_int()
    _lib.check(_lib.lib().lio_voxel_grid_host(cloud, cloud.shape[0], leaf, out, out.shape[0], C.byref(n), device),
               "lio_voxel_grid_host")
    return out[:n.value].copy()


def radix_sort_pairs(keys: np.ndarray, vals: np.ndarray, key_bits: int, device: int = 0):
    """The device's stable radix sort of (key, value) pairs by the low key_bits bits in whole bytes (lio_radix_sort_pairs_host)."""
    _lib.require_device()
    keys = np.ascontiguousarray(keys, np.uint32)
    vals = np.ascontiguousarray(vals, np.uint32)
    ko, vo = np.zeros_like(keys), np.zeros_like(vals)
    _lib.check(_lib.lib().lio_radix_sort_pairs_host(keys, vals, keys.shape[0], key_bits, ko, vo, device), "lio_radix_sort_pairs_host")
    return ko, vo


def seg_voxel_grid(clouds, leaves, device: int = 0):
    """The segmented VoxelGrid (lio_seg_voxel_grid_host): one pcl::VoxelGrid per cloud with its own leaf, in one pass.
    Returns (the filtered clouds, False), or (None, True) when a cloud's grid exceeds the 2^24-voxel index bound."""
    _lib.require_device()
    clouds = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in clouds]
    n = np.array([c.shape[0] for c in clouds], np.int32)
    cat = np.ascontiguousarray(np.concatenate(clouds), np.float32)
    out = np.zeros_like(cat)
    n_out = np.zeros_like(n)
    err = C.c_int()
    rc = _lib.lib().lio_seg_voxel_grid_host(cat, n, np.asarray(leaves, np.float32), n.shape[0], out, n_out, C.byref(err), device)
    if rc == -3 and err.value:
        return None, True
    _lib.check(rc, "lio_seg_voxel_grid_host")
    off = np.concatenate([[0], np.cumsum(n)])
    return [out[off[j]:off[j] + n_out[j]].copy() for j in range(n.shape[0])], False


def cell_hash_build(map_pts, cell_size, n_max=None, cap_points=None, prev_map=None, device: int = 0):
    """CellHash::build on explicit arrays (lio_cell_hash_build_host), optionally after an earlier build over prev_map.
    Returns (keys, count, start) of the eff_size slots in use and cellpts (n x 4: xyz + bit-cast map index)."""
    _lib.require_device()
    m = np.ascontiguousarray(map_pts, np.float32).reshape(-1, 4)
    prev = np.ascontiguousarray(prev_map if prev_map is not None else np.zeros((0, 4)), np.float32).reshape(-1, 4)
    n = m.shape[0]
    n_max = n if n_max is None else n_max
    cap = max(n_max, prev.shape[0], 1) if cap_points is None else cap_points
    table = 1024
    while table < 2 * cap:
        table <<= 1
    keys, count, start = np.zeros(table, np.uint64), np.zeros(table, np.int32), np.zeros(table, np.int32)
    cellpts = np.zeros((max(n, 1), 4), np.float32)
    eff = C.c_int()
    pad = [x if x.shape[0] else np.zeros((1, 4), np.float32) for x in (m, prev)]
    _lib.check(_lib.lib().lio_cell_hash_build_host(pad[0], n, n_max, cap, cell_size, pad[1], prev.shape[0], C.byref(eff), keys, count,
                                                   start, cellpts, device), "lio_cell_hash_build_host")
    return keys[:eff.value].copy(), count[:eff.value].copy(), start[:eff.value].copy(), cellpts[:n].copy()


def calculate_features_batch(map_pts, frames, tf7s, fit=0, min_match_sq_dis=1.0, min_plane_dis=0.2, cell_size=None, n_bound=None,
                             append=None, initial_count=None, out_cap=None, zaxis=None, done_flag=None, work_queries=None,
                             sentinel=np.float32(-7.5), device: int = 0):
    """calculate_features_batch on explicit arrays (lio_calculate_features_batch_host): every frame of `frames` against one map in
    one launch.  Output buffers and counts go in pre-filled (`sentinel`, src = -7, count = initial_count) and come back whole:
    returns the raw status code and, per frame, (pts, coef, src, count) with pts / coef / src of the frame's full out_cap length."""
    _lib.require_device()
    m = np.ascontiguousarray(map_pts, np.float32).reshape(-1, 4)
    frames = [np.ascontiguousarray(f, np.float32).reshape(-1, 4) for f in frames]
    nf = len(frames)
    per = 2 if fit == 1 else 1
    n = np.array([f.shape[0] for f in frames], np.int32)
    n_bound = n.copy() if n_bound is None else np.asarray(n_bound, np.int32)
    append = np.zeros(nf, np.int32) if append is None else np.asarray(append, np.int32)
    count = np.zeros(nf, np.int32) if initial_count is None else np.asarray(initial_count, np.int32).copy()
    out_cap = (np.where(append != 0, count, 0) + per * n + 8).astype(np.int32) if out_cap is None else np.asarray(out_cap, np.int32)
    cat = np.ascontiguousarray(np.concatenate(frames + [np.zeros((1, 4), np.float32)]), np.float32)
    tot = int(out_cap.sum())
    pts = np.full((max(tot, 1), 4), sentinel, np.float32)
    coef = np.full((max(tot, 1), 4), sentinel, np.float32)
    src = np.full(max(tot, 1), -7, np.int32)
    if cell_size is None:   # the production choice: the search radius plus a 2^-10 margin, in float32
        cell_size = np.sqrt(np.float32(min_match_sq_dis)) * (np.float32(1) + np.float32(1) / np.float32(1024))
    z = None if zaxis is None else np.ascontiguousarray(zaxis, np.float32)
    rc = _lib.lib().lio_calculate_features_batch_host(
        m if m.shape[0] else np.zeros((1, 4), np.float32), m.shape[0], cell_size, min_match_sq_dis, min_plane_dis, nf, cat, n, n_bound,
        np.ascontiguousarray(tf7s, np.float32).reshape(nf, 7), append, None if z is None else z.ctypes.data, fit,
        -1 if done_flag is None else int(done_flag), int(n_bound.sum()) if work_queries is None else work_queries, out_cap, pts, coef,
        src, count, device)
    off = np.concatenate([[0], np.cumsum(out_cap)])
    return rc, [(pts[off[k]:off[k + 1]], coef[off[k]:off[k + 1]], src[off[k]:off[k + 1]], int(count[k])) for k in range(nf)]


def calculate_features(map_pts, surf, tf7, min_match_sq_dis=1.0, min_plane_dis=0.2, device: int = 0):
    """Estimator::CalculateFeatures on explicit arrays (lio_calculate_features_host)."""
    _lib.require_device()
    m = np.ascontiguousarray(map_pts, np.float32).reshape(-1, 4)
    s = np.ascontiguousarray(surf, np.float32).reshape(-1, 4)
    cap = max(s.shape[0], 1)
    pts = np.zeros((cap, 4), np.float32)
    coef = np.zeros((cap, 4), np.float32)
    src = np.zeros(cap, np.int32)
    n = C.c_int()
    _lib.check(_lib.lib().lio_calculate_features_host(m, m.shape[0], s, s.shape[0], np.ascontiguousarray(tf7, np.float32),
                                                      min_match_sq_dis, min_plane_dis, pts, coef, src, C.byref(n), device),
               "lio_calculate_features_host")
    return pts[:n.value].copy(), coef[:n.value].copy(), src[:n.value].copy()


def laser_odom(map_pts, surf, tf7, min_match_sq_dis=1.0, min_plane_dis=0.2, keep_features=False, max_iter=10, device: int = 0):
    """Estimator::CalculateLaserOdom on explicit arrays (lio_laser_odom_host).

    Returns (tf7, pts, coef, src, iterations)."""
    _lib.require_device()
    m = np.ascontiguousarray(map_pts, np.float32).reshape(-1, 4)
    s = np.ascontiguousarray(surf, np.float32).reshape(-1, 4)
    cap = max(s.shape[0] * (max_iter if keep_features else 1), 1)
    pts = np.zeros((cap, 4), np.float32)
    coef = np.zeros((cap, 4), np.float32)
    src = np.zeros(cap, np.int32)
    tf = np.ascontiguousarray(tf7, np.float32).copy()
    n, it = C.c_int(), C.c_int()
    _lib.check(_lib.lib().lio_laser_odom_host(m, m.shape[0], s, s.shape[0], tf, min_match_sq_dis, min_plane_dis,
                                              1 if keep_features else 0, max_iter, pts, coef, src, C.byref(n), C.byref(it), device),
               "lio_laser_odom_host")
    return tf, pts[:n.value].copy(), coef[:n.value].copy(), src[:n.value].copy(), it.value


def transform_to_end(cloud, tf7_es, time_factor=10.0, device: int = 0):
    """TransformToEnd (lio_transform_to_end_host): returns the motion-compensated copy of `cloud`."""
    _lib.require_device()
    c = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4).copy()
    _lib.check(_lib.lib().lio_transform_to_end_host(c, c.shape[0], np.ascontiguousarray(tf7_es, np.float32), time_factor, device),
               "lio_transform_to_end_host")
    return c


def calculate_line_features(corner_map, corner, tf7, min_match_sq_dis=1.0, device: int = 0):
    """Point-to-line matching (lio_calculate_line_features_host): two half-weight features per accepted corner point."""
    _lib.require_device()
    m = np.ascontiguousarray(corner_map, np.float32).reshape(-1, 4)
    s = np.ascontiguousarray(corner, np.float32).reshape(-1, 4)
    cap = max(2 * s.shape[0], 1)
    pts = np.zeros((cap, 4), np.float32)
    coef = np.zeros((cap, 4), np.float32)
    src = np.zeros(cap, np.int32)
    n = C.c_int()
    _lib.check(_lib.lib().lio_calculate_line_features_host(m, m.shape[0], s, s.shape[0], np.ascontiguousarray(tf7, np.float32),
                                                           min_match_sq_dis, pts, coef, src, C.byref(n), device),
               "lio_calculate_line_features_host")
    return pts[:n.value].copy(), coef[:n.value].copy(), src[:n.value].copy()


def scan_to_map(corner_map, surf_map, corner, surf, tf7, min_match_sq_dis=1.0, min_plane_dis=0.2, max_iter=10,
                delta_r_abort=0.05, delta_t_abort=0.05, variant: int = 0, device: int = 0):
    """PointMapping::OptimizeTransformTobeMapped (lio_scan_to_map_host; variant 1 = MapBuilder::OptimizeMap):
    returns (tf7, pts, coef, src, iterations)."""
    _lib.require_device()
    a = [np.ascontiguousarray(x, np.float32).reshape(-1, 4) for x in (corner_map, surf_map, corner, surf)]
    pad = [x if x.shape[0] else np.zeros((1, 4), np.float32) for x in a]
    cap = max(a[2].shape[0] + a[3].shape[0], 1)
    pts = np.zeros((cap, 4), np.float32)
    coef = np.zeros((cap, 4), np.float32)
    src = np.zeros(cap, np.int32)
    tf = np.ascontiguousarray(tf7, np.float32).copy()
    n, it = C.c_int(), C.c_int()
    _lib.check(_lib.lib().lio_scan_to_map_host(pad[0], a[0].shape[0], pad[1], a[1].shape[0], pad[2], a[2].shape[0], pad[3], a[3].shape[0],
                                               tf, min_match_sq_dis, min_plane_dis, max_iter, delta_r_abort, delta_t_abort, variant, pts, coef, src,
                                               C.byref(n), C.byref(it), device), "lio_scan_to_map_host")
    return tf, pts[:n.value].copy(), coef[:n.value].copy(), src[:n.value].copy(), it.value


def odom_normal_equations(pts, coef, tf7, kernel: int, blocks: int = 0, device: int = 0):
    """A^T A (6 x 6) and A^T b (6) of the features as one production reduction stores them (lio_odom_normal_equations_host):
    kernel 0..2 = k_odom_reduce mode 0..2 on `blocks` CTAs (0 = the callers' grid), 3 = the fused single-CTA k_odom_round."""
    _lib.require_device()
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    c = np.ascontiguousarray(coef, np.float32).reshape(-1, 4)
    pad = [x if x.shape[0] else np.zeros((1, 4), np.float32) for x in (p, c)]
    AtA, AtB = np.zeros(36), np.zeros(6)
    _lib.check(_lib.lib().lio_odom_normal_equations_host(pad[0], pad[1], p.shape[0], np.ascontiguousarray(tf7, np.float32), kernel, blocks,
                                                         AtA, AtB, device), "lio_odom_normal_equations_host")
    return AtA.reshape(6, 6), AtB


def odom_step(AtA, AtB, n_feat, tf7, variant: int, delta_r_abort=0.05, delta_t_abort=0.05, device: int = 0):
    """One chain of odom_solve_step rounds on given normal equations (lio_odom_step_host; variant 0 CalculateLaserOdom,
    1 PointMapping, 2 MapBuilder, 3 PointOdometry).  Returns (tf7, tf7 after each round, {degenerate, done, iter}, matP)."""
    _lib.require_device()
    A = np.ascontiguousarray(AtA, np.float64).reshape(-1, 36)
    rounds = A.shape[0]
    b = np.ascontiguousarray(AtB, np.float64).reshape(rounds, 6)
    n = np.ascontiguousarray(n_feat, np.int32).reshape(rounds)
    tf = np.ascontiguousarray(tf7, np.float32).copy()
    per = np.zeros((max(rounds, 1), 7), np.float32)
    st = np.zeros(3, np.int32)
    matP = np.zeros(36, np.float32)
    pad = [x if rounds else np.zeros(k, x.dtype) for x, k in ((A, 36), (b, 6), (n, 1))]
    _lib.check(_lib.lib().lio_odom_step_host(rounds, pad[0], pad[1], pad[2], variant, delta_r_abort, delta_t_abort, tf, per, st, matP, device),
               "lio_odom_step_host")
    return tf, per[:rounds].copy(), dict(degenerate=int(st[0]), done=int(st[1]), iter=int(st[2])), matP.reshape(6, 6)
