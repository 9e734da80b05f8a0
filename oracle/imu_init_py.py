"""ctypes binding of the oracle's RunInitialization (oracle/o_imu_init.cc) — TEST INFRASTRUCTURE ONLY.

Only tests/ and scripts/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, f64p = oracle_py.f32p, np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_ii_bound", False):
        L.orc_imu_run_initialization.restype = C.c_int
        L.orc_imu_run_initialization.argtypes = [C.c_int, f32p, C.POINTER(C.c_void_p), f32p, C.c_double, f64p, f64p, f64p, f64p, f64p,
                                                 f64p, f64p]
        L._ii_bound = True
    return L


def run_initialization(laser_tf7, pims, tlb7, g_norm, bas, bgs, vs, R_WI):
    """Estimator::RunInitialization on oracle_py.Pim objects (repropagated in place); the same dict as
    lio_mapping_b200.estimator.run_initialization."""
    tf = np.ascontiguousarray(laser_tf7, np.float32).reshape(-1, 7)
    W = tf.shape[0] - 1
    bgs = np.array(bgs, np.float64).reshape(W + 1, 3); vs = np.array(vs, np.float64).reshape(W + 1, 3)
    R = np.array(R_WI, np.float64).reshape(3, 3).copy()
    ps = np.zeros((W + 1, 3)); rs = np.zeros((W + 1, 3, 3)); g = np.zeros(3)
    handles = (C.c_void_p * (W + 1))(*[p.h for p in pims])
    out = _lib().orc_imu_run_initialization(W, tf, handles, np.ascontiguousarray(tlb7, np.float32), float(g_norm),
                                            np.ascontiguousarray(bas, np.float64).reshape(-1), bgs, vs, R, ps, rs, g)
    return dict(outcome=int(out), Ps=ps, Rs=rs, Vs=vs, Bgs=bgs, g_vec=g, R_WI=R)
