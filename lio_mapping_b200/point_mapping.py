"""Host-side mirror of lio::PointMapping (pre-initialisation scan-to-map path) over the C-ABI: the rolling cube map
lives in HBM inside the library (csrc/cubemap.cu), the Python layer only moves arrays.

Method names follow the reference (include/point_processor/PointMapping.h): Process, and accessors for the cube arrays
laser_cloud_corner_array_ / laser_cloud_surf_array_."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

NUM_CUBES = 21 * 21 * 11


class PointMapping:
    def __init__(self, max_points: int = 1 << 17, corner_filter_size: float = 0.2, surf_filter_size: float = 0.4,
                 min_match_sq_dis: float = 1.0, min_plane_dis: float = 0.2, max_iterations: int = 10, device: int = 0, stream: int = 0):
        _lib.require_device()
        self.h = C.c_void_p()
        _lib.check(_lib.lib().lio_pm_create(int(max_points), corner_filter_size, surf_filter_size, min_match_sq_dis, min_plane_dis,
                                            int(max_iterations), device, C.c_void_p(stream), C.byref(self.h)), "lio_pm_create")

    def close(self):
        # an attached map (Estimator.attach_map) is refused until its estimator is closed; the handle is kept for then
        if getattr(self, "h", None) and _lib.lib().lio_pm_destroy(self.h) == 0:
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def Process(self, corner_last, surf_last, transform_sum7):
        """PointMapping::Process: returns (transform_tobe_mapped tf7, info dict)."""
        c = np.ascontiguousarray(corner_last, np.float32).reshape(-1, 4); s = np.ascontiguousarray(surf_last, np.float32).reshape(-1, 4)
        tobe = np.zeros(7, np.float32); info = np.zeros(3, np.int32)
        _lib.check(_lib.lib().lio_pm_process_host(self.h, c if c.shape[0] else np.zeros((1, 4), np.float32), c.shape[0],
                                                  s if s.shape[0] else np.zeros((1, 4), np.float32), s.shape[0],
                                                  np.ascontiguousarray(transform_sum7, np.float32), tobe, info), "lio_pm_process_host")
        return tobe, dict(iterations=int(info[0]), corner_from_map=int(info[1]), surf_from_map=int(info[2]))

    def EnablePublish(self, map_filter_size: float = 0.6, max_full_points: int = 1 << 18):
        """PointMapping::PublishResults (PointMapping.cc:1210-1270) on every ProcessDev: the surround map on calls 1, 6, 11, ...
        through VoxelGrid(map_filter_size) (0.6, :123) and the registered full cloud.  Once, before the first Process / ProcessDev;
        a publishing mapper takes ProcessDev only."""
        _lib.check(_lib.lib().lio_pm_enable_publish(self.h, float(map_filter_size), int(max_full_points)), "lio_pm_enable_publish")

    def ProcessDev(self, ptrs, n_dev_ptr: int, n_max, transform_sum7):
        """Process with the clouds in HBM: ptrs = device pointers {corner, surf, full} of float4 arrays (full may be 0 without
        EnablePublish), n_dev_ptr = device pointer of their int[3] counts, n_max = host bounds of the counts - exactly what
        PointOdometry.clouds_dev() returns.  Returns (transform_tobe_mapped tf7, transform_aft_mapped tf7, info dict); info has
        Process's keys plus surround_published and surround_size.  Stream rule: share the producer's stream or order the streams."""
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); info = np.zeros(5, np.int32)
        _lib.check(_lib.lib().lio_pm_process_dev(self.h, C.c_void_p(ptrs[0]), C.c_void_p(ptrs[1]), C.c_void_p(ptrs[2]), C.c_void_p(n_dev_ptr),
                                                 np.ascontiguousarray(n_max, np.int32), np.ascontiguousarray(transform_sum7, np.float32),
                                                 tobe, aft, info), "lio_pm_process_dev")
        return tobe, aft, dict(iterations=int(info[0]), corner_from_map=int(info[1]), surf_from_map=int(info[2]),
                               surround_published=bool(info[3]), surround_size=int(info[4]))

    def UpdateMapDatabase(self, corner_ds, surf_ds, valid, tf7, margin_centre):
        """PointMapping::UpdateMapDatabase (PointMapping.cc:1112-1208) on its own: insert the down-sampled sensor-frame clouds with the
        pose tf7, then VoxelGrid the valid cubes (indices computed with the cube-array centre margin_centre).  Returns the update's
        statistics: cube jobs re-filtered, kernel launches, host waits, points inserted."""
        c = np.ascontiguousarray(corner_ds, np.float32).reshape(-1, 4); s = np.ascontiguousarray(surf_ds, np.float32).reshape(-1, 4)
        v = np.ascontiguousarray(valid, np.int64).reshape(-1)
        _lib.check(_lib.lib().lio_pm_update_map_database_host(self.h, c if c.shape[0] else np.zeros((1, 4), np.float32), c.shape[0],
                                                              s if s.shape[0] else np.zeros((1, 4), np.float32), s.shape[0],
                                                              v if v.shape[0] else np.zeros(1, np.int64), v.shape[0],
                                                              np.ascontiguousarray(tf7, np.float32),
                                                              np.ascontiguousarray(margin_centre, np.int32)), "lio_pm_update_map_database_host")
        return self.update_stats()

    def update_stats(self):
        """The last UpdateMapDatabase of this mapper (from any entry): jobs, launches, waits, points."""
        out = np.zeros(4, np.int32)
        _lib.check(_lib.lib().lio_pm_update_stats(self.h, out), "lio_pm_update_stats")
        return dict(jobs=int(out[0]), launches=int(out[1]), waits=int(out[2]), points=int(out[3]))

    def centre(self):
        out = np.zeros(3, np.int32)
        _lib.check(_lib.lib().lio_pm_map_centre(self.h, out), "lio_pm_map_centre")
        return tuple(out.tolist())

    def cube_lists(self):
        """(laser_cloud_valid_idx_, laser_cloud_surround_idx_) of the last process call as int64 arrays."""
        v = np.zeros(125, np.int64); s = np.zeros(125, np.int64); n = np.zeros(2, np.int32)
        _lib.check(_lib.lib().lio_pm_cube_lists(self.h, v, s, n), "lio_pm_cube_lists")
        return v[:n[0]].copy(), s[:n[1]].copy()

    def cube_sizes(self, which):
        w = 0 if which == "corner" else 1
        n = C.c_int()
        out = np.zeros(NUM_CUBES, np.int64)
        L = _lib.lib()
        for i in range(NUM_CUBES):
            L.lio_pm_cube_size(self.h, i, w, C.byref(n))
            out[i] = n.value
        return out

    def cube(self, index, which):
        w = 0 if which == "corner" else 1
        n = C.c_int()
        _lib.check(_lib.lib().lio_pm_cube_size(self.h, int(index), w, C.byref(n)), "lio_pm_cube_size")
        out = np.zeros((max(n.value, 1), 4), np.float32)
        _lib.check(_lib.lib().lio_pm_cube_download(self.h, int(index), w, out, out.shape[0]), "lio_pm_cube_download")
        return out[:n.value]

    def _download(self, fn, count):
        n = C.c_int()
        out = np.zeros((max(count, 1), 4), np.float32)
        _lib.check(fn(self.h, out, out.shape[0], C.byref(n)), fn.__name__)
        return out[:n.value]

    def surround_map(self):
        """laser_cloud_surround_downsampled_ of the last publishing call (calls 1, 6, 11, ...), (n, 4) float32.  Needs a publishing
        mapper (EnablePublish) or a MapBuilder."""
        return self._download(_lib.lib().lio_mb_surround_download, self.surround_map_dev()[1])

    def registered_full_cloud(self):
        """The last full cloud in the map frame (/cloud_registered), (n, 4) float32."""
        return self._download(_lib.lib().lio_mb_full_download, self.registered_full_cloud_dev()[1])

    def surround_map_dev(self):
        """(device pointer, count) of the surround map: float4 in HBM, valid until the next process call."""
        n, p = C.c_int(), C.c_void_p()
        _lib.check(_lib.lib().lio_mb_surround_dev(self.h, C.byref(p), C.byref(n)), "lio_mb_surround_dev")
        return p.value, n.value

    def registered_full_cloud_dev(self):
        """(device pointer, count) of the registered full cloud, valid until the next process call."""
        n, p = C.c_int(), C.c_void_p()
        _lib.check(_lib.lib().lio_mb_full_dev(self.h, C.byref(p), C.byref(n)), "lio_mb_full_dev")
        return p.value, n.value
