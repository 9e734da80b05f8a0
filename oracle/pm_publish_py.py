"""ctypes bindings of PointMapping::Process + PublishResults in oracle/liboracle.so (o_pm_publish.cc) — TEST INFRASTRUCTURE ONLY.

Only tests/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, i32p = oracle_py.f32p, oracle_py.i32p
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")

PMP_CFG_DEFAULT = dict(map_filter_size=0.6, min_match_sq_dis=1.0, min_plane_dis=0.2, max_iterations=10)
PMP_CFG_ORDER = ["map_filter_size", "min_match_sq_dis", "min_plane_dis", "max_iterations"]


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_pmp_bound", False):
        L.orc_pmp_create.restype = C.c_void_p
        L.orc_pmp_create.argtypes = [f32p]
        L.orc_pmp_destroy.argtypes = [C.c_void_p]
        L.orc_pmp_process.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int, f32p, C.c_int, f32p, f32p, f32p, i32p]
        L.orc_pmp_cloud_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_pmp_cloud_copy.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_pmp_surround_idx.argtypes = [C.c_void_p, i64p]
        L.orc_pmp_cube_size.argtypes = [C.c_void_p, C.c_longlong, C.c_int]
        L.orc_pmp_cube_copy.argtypes = [C.c_void_p, C.c_longlong, C.c_int, f32p]
        L.orc_pmp_centre.argtypes = [C.c_void_p, i32p]
        L.orc_associate_to_map.argtypes = [f32p, C.c_int, f32p, f32p]
        L.orc_associate_to_map.restype = None
        L._pmp_bound = True
    return L


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return (a if a.shape[0] else np.zeros((1, 4), np.float32)), a.shape[0]


class PointMappingPublishOracle:
    """PointMapping::Process + PublishResults (PointMapping.cc:765-1052, :1210-1270) around the cube map (oracle only): the
    PointMappingOracle steps plus /laser_cloud_surround, /cloud_registered and /aft_mapped_to_init."""

    def __init__(self, **cfg):
        self.L = _lib()
        c = dict(PMP_CFG_DEFAULT)
        for k, v in cfg.items():
            if k not in c:
                raise AttributeError(f"PointMappingPublishOracle has no parameter {k}")
            c[k] = v
        self.h = self.L.orc_pmp_create(np.array([c[k] for k in PMP_CFG_ORDER], np.float32))

    def __del__(self):
        try:
            self.L.orc_pmp_destroy(self.h)
        except Exception:
            pass

    def process(self, corner, surf, full, transform_sum7):
        """Returns (transform_tobe_mapped tf7, transform_aft_mapped tf7, info dict) with the keys of PointMapping.ProcessDev."""
        (c, nc), (s, ns), (f, nf) = _cloud(corner), _cloud(surf), _cloud(full)
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); info = np.zeros(5, np.int32)
        self.L.orc_pmp_process(self.h, c, nc, s, ns, f, nf, np.ascontiguousarray(transform_sum7, np.float32), tobe, aft, info)
        return tobe, aft, dict(iterations=int(info[0]), corner_from_map=int(info[1]), surf_from_map=int(info[2]),
                               surround_published=bool(info[3]), surround_size=int(info[4]))

    def _cloud(self, which):
        n = self.L.orc_pmp_cloud_size(self.h, which)
        out = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_pmp_cloud_copy(self.h, which, out)
        return out[:n]

    def surround_map(self):
        return self._cloud(0)

    def registered_full_cloud(self):
        return self._cloud(1)

    def surround_idx(self):
        out = np.zeros(125, np.int64)
        n = self.L.orc_pmp_surround_idx(self.h, out)
        return out[:n].copy()

    def centre(self):
        out = np.zeros(3, np.int32)
        self.L.orc_pmp_centre(self.h, out)
        return tuple(out.tolist())

    def cube(self, index, which):
        w = 0 if which == "corner" else 1
        n = self.L.orc_pmp_cube_size(self.h, int(index), w)
        out = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_pmp_cube_copy(self.h, int(index), w, out)
        return out[:n]

    def cube_sizes(self, which):
        w = 0 if which == "corner" else 1
        return np.array([self.L.orc_pmp_cube_size(self.h, i, w) for i in range(21 * 21 * 11)], np.int64)


def associate_to_map(cloud, tf7):
    """PointMapping::PointAssociateToMap (PointMapping.cc:303-314) of every point with one float tf7 (qx qy qz qw px py pz)."""
    L = _lib()
    c = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    out = np.zeros_like(c)
    if c.shape[0]:
        L.orc_associate_to_map(c, c.shape[0], np.ascontiguousarray(tf7, np.float32), out)
    return out
