"""ctypes bindings of the estimator's /local/* publication in oracle/liboracle.so (o_local_clouds.cc) — TEST INFRASTRUCTURE ONLY.

Only tests/ and scripts/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, f64p = oracle_py.f32p, np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")

LOCAL_CLOUDS = ("corner", "surf", "full")


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_lc_bound", False):
        L.orc_lc_create.restype = C.c_void_p
        L.orc_lc_create.argtypes = [C.c_void_p, C.c_float]
        L.orc_lc_destroy.argtypes = [C.c_void_p]
        L.orc_lc_set_scan_clouds.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int]
        L.orc_lc_init_frame.argtypes = [C.c_void_p, C.c_int]
        L.orc_lc_process_scan.argtypes = [C.c_void_p, f32p, C.c_int]
        L.orc_lc_cloud_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_lc_cloud_copy.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_lc_transform_es.argtypes = [C.c_void_p, f32p]
        L.orc_lc_local_laser_odom.argtypes = [C.c_void_p, f32p]
        L.orc_local_laser_odom_of.argtypes = [f64p, f32p, f32p]
        L.orc_transform_to_end_keep.argtypes = [f32p, C.c_int, f32p, C.c_float, C.c_int]
        for fn in ("orc_lc_destroy", "orc_lc_set_scan_clouds", "orc_lc_init_frame", "orc_lc_process_scan", "orc_lc_cloud_copy",
                   "orc_lc_transform_es", "orc_lc_local_laser_odom", "orc_local_laser_odom_of", "orc_transform_to_end_keep"):
            getattr(L, fn).restype = None
        L._lc_bound = True
    return L


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return (a if a.shape[0] else np.zeros((1, 4), np.float32)), a.shape[0]


class LocalCloudsEstimator(oracle_py.Estimator):
    """oracle_py.Estimator plus corner_stack_ / full_stack_ and the /local/* publication (Estimator.cc:474-482, :628-693,
    :2355-2375, :2416).  Stage the corner / full cloud with set_scan_clouds before every init_frame and process_scan."""

    def __init__(self, corner_filter_size=0.2, **cfg):
        super().__init__(**cfg)
        self.LL = _lib()
        self.lc = self.LL.orc_lc_create(self.h, float(corner_filter_size))

    def set_scan_clouds(self, corner, full):
        (c, nc), (f, nf) = _cloud(corner), _cloud(full)
        self.LL.orc_lc_set_scan_clouds(self.lc, c, nc, f, nf)

    def init_frame(self, k, state16, surf_ds, pim):
        super().init_frame(k, state16, surf_ds, pim)
        self.LL.orc_lc_init_frame(self.lc, k)

    def process_scan(self, surf_last):
        s, n = _cloud(surf_last)
        self.LL.orc_lc_process_scan(self.lc, s, n)

    def local_clouds(self):
        out = {}
        for w, name in enumerate(LOCAL_CLOUDS):
            n = self.LL.orc_lc_cloud_size(self.lc, w)
            a = np.zeros((max(n, 1), 4), np.float32)
            if n:
                self.LL.orc_lc_cloud_copy(self.lc, w, a)
            out[name] = a[:n]
        return out

    def transform_es(self):
        """transform_es_ used by the last scan's pushes, tf7 (qx qy qz qw px py pz)."""
        t = np.zeros(7, np.float32)
        self.LL.orc_lc_transform_es(self.lc, t)
        return t

    def local_laser_odom(self):
        t = np.zeros(7, np.float32)
        self.LL.orc_lc_local_laser_odom(self.lc, t)
        return t

    def __del__(self):
        try:
            self.LL.orc_lc_destroy(self.lc)
        except Exception:
            pass
        super().__del__()


def local_laser_odom_of(state16, tlb7):
    """/local_laser_odom (Estimator.cc:725-742) of an explicit state16 and float extrinsic tf7, rounded to float."""
    out = np.zeros(7, np.float32)
    _lib().orc_local_laser_odom_of(np.ascontiguousarray(state16, np.float64), np.ascontiguousarray(tlb7, np.float32), out)
    return out


def transform_to_end(cloud, tf7, time_factor=10.0, keep_intensity=False):
    """TransformToEnd (Estimator.cc:62-103) with the keep_intensity argument, on a copy."""
    c = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4).copy()
    _lib().orc_transform_to_end_keep(c if c.shape[0] else np.zeros((1, 4), np.float32), c.shape[0],
                                     np.ascontiguousarray(tf7, np.float32), float(time_factor), int(bool(keep_intensity)))
    return c
