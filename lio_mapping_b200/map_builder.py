"""Host-side mirror of lio::MapBuilder, the global 4-D mapper (src/map_builder/MapBuilder.cc, map_builder_node.cc), over the
C-ABI: a PointMapping context in map-builder mode (csrc/cubemap.cu, lio_mb_*).  The cube map, the surround map and the
registered full cloud stay in HBM; the Python layer only moves arrays.

Feed it what the node subscribes to, one matched set per call: /laser_cloud_corner_last, /laser_cloud_surf_last,
/full_odom_cloud and the /laser_odom_to_init pose as a float tf7 (qx qy qz qw px py pz).  In the LIO pipeline these are the
estimator's local clouds and Estimator.local_laser_odom()."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .point_mapping import PointMapping


def default_config() -> dict:
    """The node's values: map_filter_size 0.2, corner 0.2, surf 0.4, enable_4d, skip_count 2, 10 iterations."""
    c = _lib.MBConfig()
    _lib.lib().lio_mb_default_config(C.byref(c))
    return {name: getattr(c, name) for name, _ in c._fields_}


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return (a if a.shape[0] else np.zeros((1, 4), np.float32)), a.shape[0]


class MapBuilder(PointMapping):
    """lio::MapBuilder : PointMapping.  centre(), cube_sizes(), cube(), surround_map(_dev) and registered_full_cloud(_dev) of
    PointMapping apply unchanged; Process(), ProcessDev() and EnablePublish() do not (the library rejects them on a map-builder
    context)."""

    def __init__(self, max_points: int = 1 << 17, max_full_points: int = 1 << 18, device: int = 0, stream: int = 0, **cfg):
        _lib.require_device()
        c = _lib.MBConfig()
        _lib.lib().lio_mb_default_config(C.byref(c))
        for k, v in cfg.items():
            if not hasattr(c, k):
                raise AttributeError(f"MapBuilderConfig has no field {k}")
            setattr(c, k, v)
        self.config = {name: getattr(c, name) for name, _ in c._fields_}
        self.h = C.c_void_p()
        _lib.check(_lib.lib().lio_mb_create(C.byref(c), int(max_points), int(max_full_points), device, C.c_void_p(stream),
                                            C.byref(self.h)), "lio_mb_create")
        self.transform_aft_mapped = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)

    def ProcessMap(self, corner, surf, full, transform_sum7):
        """MapBuilder::ProcessMap + PublishMapBuilderResults: returns (transform_tobe_mapped tf7, info dict).  info: iterations,
        optimised (the skip_count gate chose OptimizeMap), corner_from_map, surf_from_map, surround_published, surround_size."""
        (c, nc), (s, ns), (f, nf) = _cloud(corner), _cloud(surf), _cloud(full)
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); info = np.zeros(6, np.int32)
        _lib.check(_lib.lib().lio_mb_process_map_host(self.h, c, nc, s, ns, f, nf, np.ascontiguousarray(transform_sum7, np.float32),
                                                      tobe, aft, info), "lio_mb_process_map_host")
        self.transform_aft_mapped = aft
        return tobe, dict(iterations=int(info[0]), optimised=bool(info[1]), corner_from_map=int(info[2]), surf_from_map=int(info[3]),
                          surround_published=bool(info[4]), surround_size=int(info[5]))

    def ProcessMapDev(self, ptrs, n_dev_ptr: int, n_max, transform_sum7):
        """ProcessMap with the clouds in HBM: ptrs = device pointers {corner, surf, full} of float4 arrays, n_dev_ptr = device pointer
        of their int[3] counts, n_max = host bounds of the counts - exactly what Estimator.local_clouds_dev() returns.  Stream rule:
        share the producer's stream or order the two streams."""
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); info = np.zeros(6, np.int32)
        _lib.check(_lib.lib().lio_mb_process_map_dev(self.h, C.c_void_p(ptrs[0]), C.c_void_p(ptrs[1]), C.c_void_p(ptrs[2]),
                                                     C.c_void_p(n_dev_ptr), np.ascontiguousarray(n_max, np.int32),
                                                     np.ascontiguousarray(transform_sum7, np.float32), tobe, aft, info),
                   "lio_mb_process_map_dev")
        self.transform_aft_mapped = aft
        return tobe, dict(iterations=int(info[0]), optimised=bool(info[1]), corner_from_map=int(info[2]), surf_from_map=int(info[3]),
                          surround_published=bool(info[4]), surround_size=int(info[5]))
