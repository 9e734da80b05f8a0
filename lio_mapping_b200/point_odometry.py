"""Host-side mirror of lio::PointOdometry (scan-to-scan odometry of the pre-initialisation phase and the /compact_data
pass-through) over the C-ABI: clouds, matching and the 6 x 6 Gauss-Newton live in the library (csrc/podom.cu).

Method names follow the reference (include/point_processor/PointOdometry.h): Process, EnableOdom; the topic handlers
collapse into the arguments of Process (one synchronised set of the five feature topics)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

_WHICH = {"last_corner": 0, "last_surf": 1, "full": 2}


class PointOdometry:
    def __init__(self, scan_period: float = 0.1, io_ratio: int = 2, num_max_iterations: int = 25, max_feature_points: int = 1 << 17,
                 max_full_points: int = 1 << 20, device: int = 0, stream: int = 0):
        _lib.require_device()
        self.h = C.c_void_p()
        _lib.check(_lib.lib().lio_po_create(scan_period, int(io_ratio), int(num_max_iterations), int(max_feature_points), int(max_full_points),
                                            device, C.c_void_p(stream), C.byref(self.h)), "lio_po_create")

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lio_po_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def EnableOdom(self, enable: bool):
        """The /enable_odom service (PointOdometry.cc:126-131)."""
        _lib.check(_lib.lib().lio_po_set_enable_odom(self.h, int(bool(enable))), "lio_po_set_enable_odom")

    def Process(self, corner_points_sharp, corner_points_less_sharp, surf_points_flat, surf_points_less_flat, full_cloud):
        """PointOdometry::Process + PublishResults: returns (transform_sum tf7, transform_es tf7, info dict)."""
        args = []
        for c in (corner_points_sharp, corner_points_less_sharp, surf_points_flat, surf_points_less_flat, full_cloud):
            c = np.ascontiguousarray(c, np.float32).reshape(-1, 4)
            args += [c if c.shape[0] else np.zeros((1, 4), np.float32), c.shape[0]]
        ts = np.zeros(7, np.float32); te = np.zeros(7, np.float32); info = np.zeros(4, np.int32)
        _lib.check(_lib.lib().lio_po_process_host(self.h, *args, ts, te, info), "lio_po_process_host")
        return ts, te, dict(iterations=int(info[0]), published=int(info[1]), frame_count=int(info[2]), matches=int(info[3]))

    def ProcessDev(self, ptrs, n_dev_ptrs, n_max):
        """Process with the five clouds in HBM: ptrs / n_dev_ptrs = device pointers of the float4 clouds {sharp, less_sharp, flat,
        less_flat, full} and of one int count each (PointProcessor.cloud_dev / cloud_count_dev), n_max = host bounds of the counts.
        Same return value as Process; less_sharp, less_flat and full are copied, sharp and flat are read during the call.  Stream
        rule: share the producer's stream or order the two streams."""
        clouds = (C.c_void_p * 5)(*[C.c_void_p(int(p)) for p in ptrs])
        counts = (C.c_void_p * 5)(*[C.c_void_p(int(p)) for p in n_dev_ptrs])
        ts = np.zeros(7, np.float32); te = np.zeros(7, np.float32); info = np.zeros(4, np.int32)
        _lib.check(_lib.lib().lio_po_process_dev(self.h, clouds, counts, np.ascontiguousarray(n_max, np.int32), ts, te, info),
                   "lio_po_process_dev")
        return ts, te, dict(iterations=int(info[0]), published=int(info[1]), frame_count=int(info[2]), matches=int(info[3]))

    def clouds_dev(self):
        """(device pointers {last_corner, last_surf, full}, device pointer of their int[3] counts, host counts): the published clouds in
        HBM, what PointMapping.ProcessDev takes.  The pointers are valid until the next process call; the count pointer is stable."""
        ptr = (C.c_void_p * 3)(); n_dev = C.c_void_p(); n = np.zeros(3, np.int32)
        _lib.check(_lib.lib().lio_po_clouds_dev(self.h, ptr, C.byref(n_dev), n), "lio_po_clouds_dev")
        return [p or 0 for p in ptr], n_dev.value, n.tolist()

    def cloud(self, which: str):
        w = _WHICH[which]
        n = C.c_int()
        _lib.check(_lib.lib().lio_po_cloud_size(self.h, w, C.byref(n)), "lio_po_cloud_size")
        out = np.zeros((max(n.value, 1), 4), np.float32)
        _lib.check(_lib.lib().lio_po_cloud_download(self.h, w, out, out.shape[0]), "lio_po_cloud_download")
        return out[:n.value]

    def compact_data(self):
        """The /compact_data payload of the sweep just processed as (3 + nc + ns + nf, 4) float32."""
        n = sum(self.cloud_size(w) for w in _WHICH) + 3
        out = np.zeros((n, 4), np.float32)
        m = C.c_int()
        _lib.check(_lib.lib().lio_po_compact_data(self.h, out, n, C.byref(m)), "lio_po_compact_data")
        return out[:m.value]

    def cloud_size(self, which: str) -> int:
        n = C.c_int()
        _lib.check(_lib.lib().lio_po_cloud_size(self.h, _WHICH[which], C.byref(n)), "lio_po_cloud_size")
        return n.value

    def matches(self, kind: str, n_queries: int):
        k = 0 if kind == "corner" else 1
        out = np.zeros((max(n_queries, 1), 2 + k), np.int32)
        _lib.check(_lib.lib().lio_po_matches(self.h, k, out, n_queries), "lio_po_matches")
        return out[:n_queries]

    def last_launches(self) -> int:
        return int(_lib.lib().lio_po_last_launches(self.h))
