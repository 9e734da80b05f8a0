"""ctypes binding of the oracle's EstimateExtrinsicRotation (oracle/o_extrinsic_rotation.cc) — TEST INFRASTRUCTURE ONLY.

Only tests/ and scripts/ import this module; the product package (lio_mapping_b200/) never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle_py

f32p, f64p = oracle_py.f32p, np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def _lib():
    L = oracle_py.lib()
    if not getattr(L, "_er_bound", False):
        L.orc_imu_estimate_extrinsic_rotation.restype = C.c_int
        L.orc_imu_estimate_extrinsic_rotation.argtypes = [C.c_int, f32p, C.POINTER(C.c_void_p), f32p, f64p]
        L._er_bound = True
    return L


def estimate_extrinsic_rotation(laser_tf7, pims, tlb7):
    """ImuInitializer::EstimateExtrinsicRotation on oracle_py.Pim objects; the same (ok, tlb7, singular values) as
    lio_mapping_b200.estimator.estimate_extrinsic_rotation."""
    tf = np.ascontiguousarray(laser_tf7, np.float32).reshape(-1, 7)
    W = tf.shape[0] - 1
    t = np.array(tlb7, np.float32).reshape(7).copy()
    sv = np.zeros(4)
    handles = (C.c_void_p * (W + 1))(*[p.h for p in pims])
    ok = _lib().orc_imu_estimate_extrinsic_rotation(W, tf, handles, t, sv)
    return bool(ok), t, sv
