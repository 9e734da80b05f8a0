"""ctypes bindings of the map-builder part of oracle/liboracle.so (o_mapbuilder.cc) — TEST INFRASTRUCTURE ONLY.

Only tests/ and scripts/map_builder_bench.py import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, i32p = oracle_py.f32p, oracle_py.i32p

MB_CFG_DEFAULT = dict(map_filter_size=0.2, min_match_sq_dis=1.0, min_plane_dis=0.2, enable_4d=1, skip_count=2, max_iterations=10)
MB_CFG_ORDER = ["map_filter_size", "min_match_sq_dis", "min_plane_dis", "enable_4d", "skip_count", "max_iterations"]


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_mb_bound", False):
        L.orc_mb_create.restype = C.c_void_p
        L.orc_mb_create.argtypes = [f32p]
        L.orc_mb_destroy.argtypes = [C.c_void_p]
        L.orc_mb_process.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int, f32p, C.c_int, f32p, f32p, f32p, i32p]
        L.orc_mb_cloud_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_mb_cloud_copy.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_mb_cube_size.argtypes = [C.c_void_p, C.c_longlong, C.c_int]
        L.orc_mb_cube_copy.argtypes = [C.c_void_p, C.c_longlong, C.c_int, f32p]
        L.orc_mb_centre.argtypes = [C.c_void_p, i32p]
        L.orc_mb_associate.argtypes = [f32p, f32p, f32p, C.c_int, f32p]
        L.orc_mb_associate.restype = None
        L.orc_matrix_to_quat.argtypes = [f32p, f32p]
        L.orc_matrix_to_quat.restype = None
        L._mb_bound = True
    return L


class MapBuilderOracle:
    """MapBuilder::ProcessMap + PublishMapBuilderResults (src/map_builder/MapBuilder.cc:144-622) around the cube map (oracle only).
    The cube leaves are the node's 0.2 / 0.4; cfg takes the other MapBuilder parameters (MB_CFG_DEFAULT)."""

    def __init__(self, **cfg):
        self.L = _lib()
        c = dict(MB_CFG_DEFAULT)
        for k, v in cfg.items():
            if k not in c:
                raise AttributeError(f"MapBuilderOracle has no parameter {k}")
            c[k] = v
        self.h = self.L.orc_mb_create(np.array([c[k] for k in MB_CFG_ORDER], np.float32))
        self.transform_aft_mapped = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)

    def __del__(self):
        try:
            self.L.orc_mb_destroy(self.h)
        except Exception:
            pass

    def process_map(self, corner, surf, full, transform_sum7):
        args = []
        for a in (corner, surf, full):
            a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
            args += [a if a.shape[0] else np.zeros((1, 4), np.float32), a.shape[0]]
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); info = np.zeros(6, np.int32)
        self.L.orc_mb_process(self.h, *args, np.ascontiguousarray(transform_sum7, np.float32), tobe, aft, info)
        self.transform_aft_mapped = aft
        return tobe, dict(iterations=int(info[0]), optimised=bool(info[1]), corner_from_map=int(info[2]), surf_from_map=int(info[3]),
                          surround_published=bool(info[4]), surround_size=int(info[5]))

    def _cloud(self, which):
        n = self.L.orc_mb_cloud_size(self.h, which)
        out = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_mb_cloud_copy(self.h, which, out)
        return out[:n]

    def surround_map(self):
        return self._cloud(0)

    def registered_full_cloud(self):
        return self._cloud(1)

    def centre(self):
        out = np.zeros(3, np.int32)
        self.L.orc_mb_centre(self.h, out)
        return tuple(out.tolist())

    def cube(self, index, which):
        w = 0 if which == "corner" else 1
        n = self.L.orc_mb_cube_size(self.h, int(index), w)
        out = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_mb_cube_copy(self.h, int(index), w, out)
        return out[:n]

    def cube_sizes(self, which):
        w = 0 if which == "corner" else 1
        return np.array([self.L.orc_mb_cube_size(self.h, i, w) for i in range(21 * 21 * 11)], np.int64)


def associate_to_map(tobe7, bef7, sum7, enable_4d=True):
    """MapBuilder::Transform4DAssociateToMap (MapBuilder.cc:55-75), or with enable_4d=False PointMapping::TransformAssociateToMap
    (PointMapping.cc:755-758), on explicit float tf7 transforms: the new tobe."""
    L = _lib()
    out = np.zeros(7, np.float32)
    L.orc_mb_associate(*[np.ascontiguousarray(a, np.float32) for a in (tobe7, bef7, sum7)], int(bool(enable_4d)), out)
    return out


def matrix_to_quat(R):
    """Eigen 3.3's Matrix3f -> Quaternionf assignment (quaternion_assign_impl<Other,3,3>) as the oracle states it: (x, y, z, w)."""
    L = _lib()
    q = np.zeros(4, np.float32)
    L.orc_matrix_to_quat(np.ascontiguousarray(R, np.float32).reshape(9), q)
    return q
