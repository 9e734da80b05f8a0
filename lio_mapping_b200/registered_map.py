"""The map of a whole drive over the C-ABI (csrc/regmap.cu, lio_rm_*): the registered clouds (/cloud_registered) of every
publishing step accumulated in HBM, as the reference's src/save_bag_to_pcd.cc accumulates them from a bag, and written as one
binary PCD.

leaf == 0 keeps every point in insert order (the reference tool); leaf > 0 keeps one fp64-averaged point per float32 voxel,
numbered in the order voxels are first seen.  Feed it PointMapping.registered_full_cloud_dev() after each publishing call:

    rm = RegisteredMap(leaf=0.2, capacity=1 << 22)
    ...
    rm.insert_dev(*pm.registered_full_cloud_dev())
    ...
    rm.write_pcd("drive.pcd")
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

STATS = ("inserts", "offered", "size", "overflow", "accepted", "dropped", "waits", "launches")


def write_pcd(path, xyzi):
    """A binary PCD v0.7 of an (n, 4) float32 x, y, z, intensity array (pcl::PointXYZI through PCDWriter::writeBinary).  Needs
    no device."""
    a = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    _lib.check(_lib.lib().lio_pcd_write_xyzi(str(path).encode(), a if a.shape[0] else np.zeros((1, 4), np.float32), a.shape[0]),
               "lio_pcd_write_xyzi")


class RegisteredMap:
    def __init__(self, leaf: float = 0.0, capacity: int = 1 << 22, device: int = 0, stream: int = 0):
        """capacity counts points when leaf == 0 and voxels when leaf > 0.  stream: the CUDA stream of the mapping whose clouds
        are inserted (or order the two streams with an event)."""
        _lib.require_device()
        self.leaf, self.capacity = float(leaf), int(capacity)
        self.h = C.c_void_p()
        _lib.check(_lib.lib().lio_rm_create(self.leaf, self.capacity, int(device), C.c_void_p(stream), C.byref(self.h)),
                   "lio_rm_create")

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lio_rm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def insert(self, xyzi):
        """Insert an (n, 4) float32 host cloud; it is copied before the call returns."""
        a = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
        _lib.check(_lib.lib().lio_rm_insert_host(self.h, a if a.shape[0] else np.zeros((1, 4), np.float32), a.shape[0]),
                   "lio_rm_insert_host")

    def insert_dev(self, ptr: int, n: int):
        """Insert n float4 points at a device pointer, stream-ordered, without a host wait."""
        _lib.check(_lib.lib().lio_rm_insert_dev(self.h, C.c_void_p(ptr), int(n)), "lio_rm_insert_dev")

    def stats(self) -> dict:
        """Synchronises.  inserts / offered count every insert call; size is in points (raw) or voxels; accepted and dropped are
        the points the map took or dropped; waits counts the handle's host waits (this call's included); launches is the number
        of stream operations of the last insert."""
        out = np.zeros(8, np.int64)
        _lib.check(_lib.lib().lio_rm_stats(self.h, out), "lio_rm_stats")
        return {k: int(v) for k, v in zip(STATS, out)}

    def export_dev(self):
        """(device pointer, n) of the map as float4, valid until the next insert or reset."""
        p, n = C.c_void_p(), C.c_longlong()
        _lib.check(_lib.lib().lio_rm_export_dev(self.h, C.byref(p), C.byref(n)), "lio_rm_export_dev")
        return p.value, n.value

    def download(self):
        """The map as an (n, 4) float32 array."""
        n = self.export_dev()[1]
        out = np.zeros((max(n, 1), 4), np.float32)
        got = C.c_longlong()
        _lib.check(_lib.lib().lio_rm_download(self.h, out, out.shape[0], C.byref(got)), "lio_rm_download")
        return out[:got.value]

    def reset(self):
        """Empty the map and clear the overflow flag."""
        _lib.check(_lib.lib().lio_rm_reset(self.h), "lio_rm_reset")

    def write_pcd(self, path):
        """The map as a binary PCD (see write_pcd)."""
        _lib.check(_lib.lib().lio_rm_write_pcd(self.h, str(path).encode()), "lio_rm_write_pcd")
