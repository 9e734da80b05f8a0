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
