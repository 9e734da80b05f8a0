"""ctypes bindings of the imu_factor = 0 estimator fed /compact_data messages in oracle/liboracle.so (o_lidar_only.cc) — TEST
INFRASTRUCTURE ONLY.

Only tests/ and scripts/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, i32p, f64p = oracle_py.f32p, oracle_py.i32p, np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_lo_bound", False):
        L.orc_lo_create.restype = C.c_void_p
        L.orc_lo_create.argtypes = [C.c_void_p, C.c_int, C.c_double]
        L.orc_lo_destroy.argtypes = [C.c_void_p]
        L.orc_lo_process_compact.argtypes = [C.c_void_p, f32p, C.c_int, f32p, C.c_int, f32p, C.c_int, f32p, i32p]
        L.orc_lo_poses.argtypes = [C.c_void_p, f32p, f32p, f32p, i32p]
        L.orc_lo_startup_states.argtypes = [C.c_void_p, f64p]
        L.orc_lo_prediction.argtypes = [C.c_void_p, f64p]
        L.orc_lo_centre.argtypes = [C.c_void_p, i32p]
        L.orc_lo_cube_size.argtypes = [C.c_void_p, C.c_longlong, C.c_int]
        L.orc_lo_cube_copy.argtypes = [C.c_void_p, C.c_longlong, C.c_int, f32p]
        L.orc_lo_predict.argtypes = [f32p, f32p, f32p, f64p, f64p, f64p]
        for fn in ("orc_lo_destroy", "orc_lo_process_compact", "orc_lo_poses", "orc_lo_prediction", "orc_lo_centre", "orc_lo_cube_copy",
                   "orc_lo_predict"):
            getattr(L, fn).restype = None
        L._lo_bound = True
    return L


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return (a if a.shape[0] else np.zeros((1, 4), np.float32)), a.shape[0]


class LidarOnlyEstimator:
    """oracle_py.Estimator (imu_factor = 0) driven the way lio::Estimator::ProcessCompactData drives it, with its own PointMapping.
    start_shift (m) is added to every start-up position: the probe of the chain's own divergence."""

    def __init__(self, init_window_factor=1, start_shift=0.0, **cfg):
        self.L = _lib()
        self.est = oracle_py.Estimator(imu_factor=0, **cfg)
        self.h = self.L.orc_lo_create(self.est.h, int(init_window_factor), float(start_shift))
        self.cfg = self.est.cfg
        self.W = self.est.W

    def __getattr__(self, name):   # set_extrinsic, states, frame, ...
        return getattr(self.__dict__["est"], name)

    def process_compact(self, corner, surf, full, transform_sum7):
        (c, nc), (s, ns), (f, nf) = _cloud(corner), _cloud(surf), _cloud(full)
        info = np.zeros(4, np.int32)
        self.L.orc_lo_process_compact(self.h, c, nc, s, ns, f, nf, np.ascontiguousarray(transform_sum7, np.float32), info)
        return dict(inited=bool(info[0]), cir_buf_count=int(info[1]), pushed=bool(info[2]), solved=bool(info[3]))

    def map_poses(self):
        tobe, aft, ins = (np.zeros(7, np.float32) for _ in range(3))
        info = np.zeros(5, np.int32)
        self.L.orc_lo_poses(self.h, tobe, aft, ins, info)
        return tobe, aft, ins, dict(inserted=bool(info[0]), points=int(info[1]), surround_published=bool(info[2]),
                                    process_published=bool(info[3]), surround_size=int(info[4]))

    def startup_states(self):
        out = np.zeros((self.W + 1) * 16)
        n = self.L.orc_lo_startup_states(self.h, out)
        return out.reshape(-1, 16) if n else None

    def prediction(self):
        """The last state-W overwrite: (P_{W-1}, R_{W-1}, incre tf7 (float values), P_W, R_W)."""
        p = np.zeros(31)
        self.L.orc_lo_prediction(self.h, p)
        return p[0:3], p[3:12].reshape(3, 3), p[12:19].astype(np.float32), p[19:22], p[22:31].reshape(3, 3)

    def centre(self):
        out = np.zeros(3, np.int32)
        self.L.orc_lo_centre(self.h, out)
        return tuple(int(v) for v in out)

    def cube(self, index, which):
        w = ("corner", "surf").index(which)
        n = self.L.orc_lo_cube_size(self.h, int(index), w)
        a = np.zeros((max(n, 1), 4), np.float32)
        if n:
            self.L.orc_lo_cube_copy(self.h, int(index), w, a)
        return a[:n]

    def cube_sizes(self, which):
        w = ("corner", "surf").index(which)
        return np.array([self.L.orc_lo_cube_size(self.h, i, w) for i in range(21 * 21 * 11)], np.int32)

    def __del__(self):
        try:
            self.L.orc_lo_destroy(self.h)
        except Exception:
            pass


def predict(t_prev7, t_curr7, tlb7, p_prev3, r_prev9):
    """SolveOptimization's state-W overwrite (Estimator.cc:1670-1676) on explicit inputs: (P_W, R_W)."""
    out = np.zeros(12)
    _lib().orc_lo_predict(*(np.ascontiguousarray(a, np.float32) for a in (t_prev7, t_curr7, tlb7)),
                          np.ascontiguousarray(p_prev3, np.float64), np.ascontiguousarray(r_prev9, np.float64).reshape(9), out)
    return out[:3], out[3:].reshape(3, 3)
