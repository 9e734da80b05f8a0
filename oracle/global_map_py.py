"""ctypes bindings of the estimator's global cube map after initialisation in oracle/liboracle.so (o_global_map.cc) — TEST
INFRASTRUCTURE ONLY.

Only tests/ and scripts/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py, pm_publish_py

f32p, i32p, f64p = oracle_py.f32p, oracle_py.i32p, np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
CLOUDS = ("corner", "surf", "surround", "registered")


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_gm_bound", False):
        pm_publish_py._lib()
        L.orc_gm_create.restype = C.c_void_p
        L.orc_gm_create.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_float]
        L.orc_gm_destroy.argtypes = [C.c_void_p]
        L.orc_gm_set_scan_clouds.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int]
        L.orc_gm_pre_init_process.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int, f32p, C.c_int, f32p, i32p]
        L.orc_gm_init_frame.argtypes = [C.c_void_p, C.c_int, f32p, C.c_int]
        L.orc_gm_process_scan.argtypes = [C.c_void_p, f32p, C.c_int]
        L.orc_gm_poses.argtypes = [C.c_void_p, f32p, f32p, f32p, i32p]
        L.orc_gm_cloud_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_gm_cloud_copy.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_gm_valid.argtypes = [C.c_void_p, i64p]
        L.orc_gm_predict.argtypes = [f32p, f64p, f64p, f32p, f32p]
        for fn in ("orc_gm_destroy", "orc_gm_set_scan_clouds", "orc_gm_pre_init_process", "orc_gm_init_frame", "orc_gm_process_scan",
                   "orc_gm_poses", "orc_gm_cloud_copy", "orc_gm_predict"):
            getattr(L, fn).restype = None
        L._gm_bound = True
    return L


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return (a if a.shape[0] else np.zeros((1, 4), np.float32)), a.shape[0]


class GlobalMapEstimator:
    """oracle_py.Estimator + a PointMappingPublishOracle that the pre-initialisation calls build, continued after initialisation the
    way lio::Estimator (a PointMapping) does.  Same method names as the GPU estimator: set_scan_clouds before every init_frame /
    process_scan, pre_init_process for the mapper's calls before the warm start ends; process_scan runs the estimator's scan itself."""

    def __init__(self, corner_filter_size=0.2, map_filter_size=0.6, **cfg):
        self.L = _lib()
        self.est = oracle_py.Estimator(**cfg)
        self.pm = pm_publish_py.PointMappingPublishOracle(map_filter_size=map_filter_size)
        self.h = self.L.orc_gm_create(self.est.h, self.pm.h, float(corner_filter_size), float(map_filter_size))
        self.cfg = self.est.cfg

    def __getattr__(self, name):   # set_extrinsic, finish_init, process_imu, states, extrinsic, frame, ...
        return getattr(self.__dict__["est"], name)

    def set_scan_clouds(self, corner, full):
        (c, nc), (f, nf) = _cloud(corner), _cloud(full)
        self.L.orc_gm_set_scan_clouds(self.h, c, nc, f, nf)

    def pre_init_process(self, corner, surf, full, transform_sum7):
        (c, nc), (s, ns), (f, nf) = _cloud(corner), _cloud(surf), _cloud(full)
        info = np.zeros(5, np.int32)
        self.L.orc_gm_pre_init_process(self.h, c, nc, s, ns, f, nf, np.ascontiguousarray(transform_sum7, np.float32), info)
        return info

    def init_frame(self, k, state16, surf_ds, pim):
        self.est.init_frame(k, state16, surf_ds, pim)
        s, n = _cloud(surf_ds)
        self.L.orc_gm_init_frame(self.h, k, s, n)

    def process_scan(self, surf_last):
        s, n = _cloud(surf_last)
        self.L.orc_gm_process_scan(self.h, s, n)

    def map_poses(self):
        tobe, aft, ins = (np.zeros(7, np.float32) for _ in range(3))
        info = np.zeros(4, np.int32)
        self.L.orc_gm_poses(self.h, tobe, aft, ins, info)
        return tobe, aft, ins, dict(inserted=bool(info[0]), points=int(info[1]), surround_published=bool(info[2]), surround_size=int(info[3]))

    def cloud(self, which):
        """'corner' / 'surf': the clouds the last insert took; 'surround': the last surround map; 'registered': /cloud_registered."""
        w = CLOUDS.index(which)
        n = self.L.orc_gm_cloud_size(self.h, w)
        a = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_gm_cloud_copy(self.h, w, a)
        return a[:n]

    def valid(self):
        out = np.zeros(125, np.int64)
        return out[:self.L.orc_gm_valid(self.h, out)].copy()

    def cube(self, index, which):
        return self.pm.cube(index, which)

    def cube_sizes(self, which):
        return self.pm.cube_sizes(which)

    def __del__(self):
        try:
            self.L.orc_gm_destroy(self.h)
        except Exception:
            pass


def predict(tobe7, state_prev16, state_curr16, tlb7):
    """ProcessCompactData's prediction (Estimator.cc:776-809) on explicit states, float Twist as the reference evaluates it."""
    out = np.zeros(7, np.float32)
    _lib().orc_gm_predict(np.ascontiguousarray(tobe7, np.float32), np.ascontiguousarray(state_prev16, np.float64),
                          np.ascontiguousarray(state_curr16, np.float64), np.ascontiguousarray(tlb7, np.float32), out)
    return out
