"""The reference's launch/test_*.launch graph - lio_processor_node + lio_estimator_node (src/processor_node.cc, src/estimator_node.cc) - as
one device-resident handle over the C-ABI (lio_node_*): raw sweeps and IMU messages in; stage A, the odometry, MeasurementManager's pairing,
the estimator's start-up and window solve, and its PointMapping inside the library.

SHIPPED holds the three shipped configurations: config/indoor_test_config.yaml, config/outdoor_test_config.yaml and
config/outdoor_test_config_64.yaml (the values below cite file:line), with the processor_node parameters of the launch file that starts
each of them.  LioNode.shipped(name, ...) builds a node from one; the capacities and anything else can be given as keyword arguments.

The second line of the reference's example, launch/map_4D*.launch (map_builder_node on the estimator's /local/* clouds), runs inside the
node after enable_map_builder() (or shipped(name, map_4d=True)): one MapBuilder::ProcessMap per message that reaches the estimator
INITED, on the node's stream.  map_builder_poses() is the drive's 4-D trajectory; attach_registered_map() feeds a RegisteredMap (the
save_bag_to_pcd tool) from the estimator's or the map builder's /cloud_registered.

enable_odometry() (or shipped(name, odometry=True)) keeps the pose topics the two nodes publish, one row per publication, in queues the
caller drains with take_odometry(topic): TOPICS maps the reference's topic names to the C-ABI's ids.  write_tum() writes a trajectory
in the TUM format that trajectory-evaluation tools read."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib, synth
from .estimator import Estimator
from .map_builder import MapBuilder
from .point_mapping import PointMapping
from .point_odometry import PointOdometry
from .point_processor import PointProcessor

_I3 = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]

# Lines are the same in the two 70-line files (indoor_test_config.yaml, outdoor_test_config.yaml); outdoor_test_config_64.yaml has one line
# more ("# KITTI 00", :23), so its lines from extrinsic_rotation on are one later.  min_plane_dis :3, min_match_sq_dis :5,
# corner_filter_size :7, surf_filter_size :8, map_filter_size :9, window_size :12, opt_window_size :13, init_window_factor :15,
# estimate_extrinsic :18, opt_extrinsic :21 in all three.
SHIPPED = {
    "indoor": dict(
        yaml="config/indoor_test_config.yaml",
        launch="launch/test_indoor.launch",       # sensor_type left at 16; launch/test_indoor_rs32.launch:6 runs the same YAML with 320
        sensor_type=16, no_deskew=False,
        min_plane_dis=0.2, min_match_sq_dis=1.0, corner_filter_size=0.2, surf_filter_size=0.4, map_filter_size=0.6,
        window_size=12, opt_window_size=7, init_window_factor=2, estimate_extrinsic=2, opt_extrinsic=1,
        extrinsic_rotation=_I3,                   # :23-30
        extrinsic_translation=[0.0, 0.0, -0.081939],   # :32-36
        imu_factor=1, point_distance_factor=1,    # :46, :47
        prior_factor=0, marginalization_factor=1,  # :49, :51
        odom_io=2,                                # :53
        acc_n=0.2, gyr_n=0.02, acc_w=0.0002, gyr_w=2.0e-5, g_norm=9.805,   # :58-62
        enable_deskew=1, cutoff_deskew=0,         # :65, :66
        keep_features=1,                          # :68
        msg_time_delay=0.05),                     # :70
    "outdoor": dict(
        yaml="config/outdoor_test_config.yaml",
        launch="launch/test_outdoor.launch",      # sensor_type left at 16
        sensor_type=16, no_deskew=False,
        min_plane_dis=0.2, min_match_sq_dis=1.0, corner_filter_size=0.2, surf_filter_size=0.4, map_filter_size=0.6,
        window_size=7, opt_window_size=5, init_window_factor=1, estimate_extrinsic=1, opt_extrinsic=1,
        extrinsic_rotation=_I3,                   # :23-30
        extrinsic_translation=[-2.4, 0.0, 0.7],   # :32-36
        imu_factor=1, point_distance_factor=1,    # :46, :47
        prior_factor=0, marginalization_factor=1,  # :49, :51
        odom_io=3,                                # :53
        acc_n=0.2, gyr_n=0.02, acc_w=0.0002, gyr_w=2.0e-5, g_norm=9.80,    # :58-62
        enable_deskew=1, cutoff_deskew=0,         # :65, :66
        keep_features=0,                          # :68
        msg_time_delay=0.05),                     # :70
    "outdoor_64": dict(
        yaml="config/outdoor_test_config_64.yaml",
        launch="launch/test_outdoor_64.launch",   # sensor_type 64 (:6); no_deskew true (:11), a parameter estimator_node.cc never reads
        sensor_type=64, no_deskew=True,
        min_plane_dis=0.2, min_match_sq_dis=1.0, corner_filter_size=0.2, surf_filter_size=0.4, map_filter_size=0.6,
        window_size=7, opt_window_size=5, init_window_factor=1, estimate_extrinsic=1, opt_extrinsic=1,
        extrinsic_rotation=[[9.999976e-01, 7.553071e-04, -2.035826e-03],     # :24-31 (KITTI 00)
                            [-7.854027e-04, 9.998898e-01, -1.482298e-02],
                            [2.024406e-03, 1.482454e-02, 9.998881e-01]],
        extrinsic_translation=[-8.086759e-01, 3.195559e-01, -7.997231e-01],  # :33-37
        imu_factor=1, point_distance_factor=1,    # :47, :48
        prior_factor=1, marginalization_factor=1,  # :50, :52
        odom_io=3,                                # :54
        acc_n=0.2, gyr_n=0.02, acc_w=0.0002, gyr_w=2.0e-5, g_norm=9.80,    # :59-63
        enable_deskew=1, cutoff_deskew=1,         # :66, :67
        keep_features=0,                          # :69
        msg_time_delay=0.0),                      # :71
}

_EST_KEYS = ("min_plane_dis", "min_match_sq_dis", "surf_filter_size", "window_size", "opt_window_size", "init_window_factor",
             "estimate_extrinsic", "opt_extrinsic", "imu_factor", "point_distance_factor", "prior_factor", "marginalization_factor",
             "acc_n", "gyr_n", "acc_w", "gyr_w", "g_norm", "enable_deskew", "cutoff_deskew", "keep_features")


# The odometry topics of lio_node_enable_odometry (include/lio_b200.h: LIO_NODE_ODOM_*), by the reference's topic names
TOPICS = {"/laser_odom_to_init": 0, "/aft_mapped_to_init": 1, "/predict_odom": 2, "/predict_laser_odom": 3, "/local_laser_odom": 4,
          "/extrinsic_lb": 5}
# The named extras of a topic's row (columns 8..14): /laser_odom_to_init carries transform_es_ (/laser_odom_to_last), /predict_odom
# Vs_.last() and Bas_.last()
_EXTRAS = {"/laser_odom_to_init": (("es", 7),), "/predict_odom": (("v", 3), ("ba", 3))}


def write_tum(path, stamp, tf7):
    """One pose per line, "stamp tx ty tz qx qy qz qw" (the TUM trajectory format): stamp (n,), tf7 (n, 7) in the repository's order
    qx qy qz qw px py pz (take_odometry(topic)["tf7"])."""
    t = np.asarray(stamp, np.float64).reshape(-1)
    p = np.asarray(tf7, np.float64).reshape(-1, 7)
    if p.shape[0] != t.shape[0]:
        raise ValueError("one tf7 row per stamp")
    np.savetxt(path, np.column_stack([t, p[:, 4:7], p[:, 0:4]]), fmt="%.9f")


def shipped_tf_lb7(name):
    """transform_lb_ of a shipped configuration as estimator_node.cc:90-97 builds it (Quaternionf of the float rotation), tf7."""
    s = SHIPPED[name]
    q = synth.rot_to_quat(np.array(s["extrinsic_rotation"], np.float32).astype(np.float64))
    return np.array([*q, *s["extrinsic_translation"]], np.float32)


class _Borrowed:
    """A wrapper object over an inner handle of a node: its getters work, closing it does nothing (the node owns the handle)."""

    def close(self):
        pass


class _EstimatorView(_Borrowed, Estimator):
    def __init__(self, h, c):
        self.h, self.c, self.W, self._cb = h, c, c.window_size, None
        self.cfg = {name: getattr(c, name) for name, _ in c._fields_}


class _MappingView(_Borrowed, PointMapping):
    def __init__(self, h):
        self.h = h


class _MapBuilderView(_Borrowed, MapBuilder):
    def __init__(self, h, config):
        self.h, self.config = h, config   # transform_aft_mapped: see LioNode.map_builder_poses()

    def ProcessMap(self, *args):
        raise TypeError("the node runs its map builder; ProcessMap is not available on the view")

    ProcessMapDev = ProcessMap


class _OdometryView(_Borrowed, PointOdometry):
    def __init__(self, h):
        self.h = h


class _ProcessorView(_Borrowed, PointProcessor):
    def __init__(self, h, cfg):
        self._h, self.cfg, self._cloud = h, cfg, None


class LioNode:
    """lio_node: push_imu / push_imu_batch and push_sweep (host arrays) / push_sweep_dev (device pointers) in any order the sensors deliver
    them; every message that MeasurementManager's pairing releases is processed at once.  status() reports the counters; estimator,
    mapping, odometry and processor are read-only views of the inner handles (their getters only: the node owns the handles)."""

    def __init__(self, sensor_type=16, odom_io=2, msg_time_delay=0.0, tf_lb7=None, corner_filter_size=0.2, surf_filter_size=0.4,
                 map_filter_size=0.6, max_points=1 << 18, max_feature_points=1 << 16, max_pending=16, pp=None, device=0, stream=0, **est):
        L = _lib.lib()
        _lib.require_device()
        c = _lib.NodeConfig()
        L.lio_node_default_config(C.byref(c))
        c.sensor_type, c.odom_io, c.msg_time_delay = int(sensor_type), int(odom_io), float(msg_time_delay)
        c.corner_filter_size, c.surf_filter_size, c.map_filter_size = corner_filter_size, surf_filter_size, map_filter_size
        c.est.surf_filter_size = surf_filter_size   # one YAML key for the Estimator and the PointMapping it is
        c.max_points, c.max_feature_points, c.max_pending = int(max_points), int(max_feature_points), int(max_pending)
        if tf_lb7 is not None:
            c.tf_lb7[:] = [float(v) for v in np.asarray(tf_lb7, np.float32)]
        for k, v in (pp or {}).items():
            if not hasattr(c.pp, k):
                raise AttributeError(f"PointProcessorConfig has no field {k}")
            setattr(c.pp, k, v)
        for k, v in est.items():
            if not hasattr(c.est, k):
                raise AttributeError(f"EstimatorConfig has no field {k}")
            setattr(c.est, k, v)
        self.cfg = c
        self.h = C.c_void_p()
        _lib.check(L.lio_node_create(C.byref(c), device, C.c_void_p(stream), C.byref(self.h)), "lio_node_create")
        pp_h, po_h, est_h, pm_h = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        _lib.check(L.lio_node_handles(self.h, C.byref(pp_h), C.byref(po_h), C.byref(est_h), C.byref(pm_h)), "lio_node_handles")
        self.estimator = _EstimatorView(est_h, c.est)
        self.mapping = _MappingView(pm_h)
        self.odometry = _OdometryView(po_h)
        self.processor = _ProcessorView(pp_h, c.pp)
        self.map_builder = None
        self._maps = []   # attached RegisteredMaps: the node inserts into them, so it keeps them alive

    @classmethod
    def shipped(cls, name, map_4d=False, odometry=False, **overrides):
        """A node with the values of SHIPPED[name]; keyword arguments (capacities, tf_lb7, any config field) take precedence.  map_4d=True
        also runs map_4D*.launch's map builder with its defaults (enable_map_builder()); odometry=True keeps the odometry topics
        (enable_odometry() with its default capacity)."""
        s = SHIPPED[name]
        kw = dict(sensor_type=s["sensor_type"], odom_io=s["odom_io"], msg_time_delay=s["msg_time_delay"], tf_lb7=shipped_tf_lb7(name),
                  corner_filter_size=s["corner_filter_size"], surf_filter_size=s["surf_filter_size"], map_filter_size=s["map_filter_size"])
        kw.update({k: s[k] for k in _EST_KEYS if k != "surf_filter_size"})
        kw.update(overrides)
        node = cls(**kw)
        if map_4d:
            node.enable_map_builder()
        if odometry:
            node.enable_odometry()
        return node

    def enable_map_builder(self, **cfg):
        """map_builder_node inside the node (lio_node_enable_map_builder): MBConfig fields as keyword arguments over the defaults of
        map_4D.launch / map_4D_indoor.launch (map_builder.default_config()).  Once, before the first sweep.  Afterwards map_builder is a
        read-only MapBuilder view of it."""
        c = _lib.MBConfig()
        _lib.lib().lio_mb_default_config(C.byref(c))
        for k, v in cfg.items():
            if not hasattr(c, k):
                raise AttributeError(f"MapBuilderConfig has no field {k}")
            setattr(c, k, v)
        _lib.check(_lib.lib().lio_node_enable_map_builder(self.h, C.byref(c)), "lio_node_enable_map_builder")
        mb = C.c_void_p()
        _lib.check(_lib.lib().lio_node_map_builder(self.h, C.byref(mb)), "lio_node_map_builder")
        self.map_builder = _MapBuilderView(mb, {name: getattr(c, name) for name, _ in c._fields_})

    def map_builder_poses(self):
        """The map builder's trajectory, one row per call: dict of stamp (n,) float64 (the set's header stamp), tobe and aft (n, 7) float32
        tf7 (transform_tobe_mapped_, transform_aft_mapped_), and the per-call iterations, optimised, corner_from_map, surf_from_map,
        surround_published and surround_size as (n,) arrays."""
        L = _lib.lib()
        n = C.c_int()
        one = (np.zeros(1), np.zeros((1, 7), np.float32), np.zeros((1, 7), np.float32), np.zeros((1, 6), np.int32))
        rc = L.lio_node_map_builder_poses(self.h, *one, 0, C.byref(n))
        if rc != -3:   # LIO_ERR_CAPACITY: *n rows do not fit in 0, as asked
            _lib.check(rc, "lio_node_map_builder_poses")
        cap = max(n.value, 1)
        stamp, tobe, aft, info = np.zeros(cap), np.zeros((cap, 7), np.float32), np.zeros((cap, 7), np.float32), np.zeros((cap, 6), np.int32)
        _lib.check(L.lio_node_map_builder_poses(self.h, stamp, tobe, aft, info, cap, C.byref(n)), "lio_node_map_builder_poses")
        k = n.value
        out = dict(stamp=stamp[:k], tobe=tobe[:k], aft=aft[:k])
        for j, name in enumerate(("iterations", "optimised", "corner_from_map", "surf_from_map", "surround_published", "surround_size")):
            out[name] = info[:k, j].astype(bool) if name in ("optimised", "surround_published") else info[:k, j].copy()
        return out

    def enable_odometry(self, capacity=1 << 16):
        """Keep every publication of the TOPICS (lio_node_enable_odometry): one queue of capacity rows per topic, the oldest row dropped
        when a queue is full.  Once, before the first sweep."""
        _lib.check(_lib.lib().lio_node_enable_odometry(self.h, int(capacity)), "lio_node_enable_odometry")

    def take_odometry(self, topic, cap=None):
        """Removes and returns the oldest queued rows of topic (a name of TOPICS or its id), all of them unless cap is given: dict of
        stamp (n,), tf7 (n, 7) {qx qy qz qw px py pz}, the topic's extras (/laser_odom_to_init: es (n, 7); /predict_odom: v and ba
        (n, 3)), seq (n,) int64 (the publication count from 1: a gap is a dropped row) and left, the rows still queued.  float64."""
        name = topic if isinstance(topic, str) else next((k for k, v in TOPICS.items() if v == topic), None)
        tid = TOPICS.get(name, -1) if isinstance(topic, str) else int(topic)
        L = _lib.lib()
        n, left = C.c_int(), C.c_int()
        if cap is None:   # how many are queued: a take of none
            _lib.check(L.lio_node_take_odometry(self.h, tid, None, 0, C.byref(n), C.byref(left)), "lio_node_take_odometry")
            cap = left.value
        rows = np.zeros((max(int(cap), 1), 16))
        _lib.check(L.lio_node_take_odometry(self.h, tid, rows.ctypes.data_as(C.c_void_p), int(cap), C.byref(n), C.byref(left)),
                   "lio_node_take_odometry")
        rows = rows[:n.value]
        out = dict(stamp=rows[:, 0].copy(), tf7=rows[:, 1:8].copy())
        col = 8
        for key, width in _EXTRAS.get(name, ()):
            out[key] = rows[:, col:col + width].copy()
            col += width
        out["seq"] = rows[:, 15].astype(np.int64)
        out["left"] = left.value
        return out

    def attach_registered_map(self, rm, source="estimator"):
        """Insert every /cloud_registered of source ("estimator": the estimator's PointMapping, once per processed message;
        "map_builder": once per map builder call) into the RegisteredMap rm, stream-ordered.  rm must be on the node's device and stream;
        the node keeps a reference to it."""
        code = {"estimator": 0, "map_builder": 1}.get(source, -1)
        _lib.check(_lib.lib().lio_node_attach_registered_map(self.h, rm.h, code), "lio_node_attach_registered_map")
        self._maps.append(rm)

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lio_node_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push_imu(self, stamp, acc, gyr):
        _lib.check(_lib.lib().lio_node_push_imu(self.h, float(stamp), np.ascontiguousarray(acc, np.float64),
                                                np.ascontiguousarray(gyr, np.float64)), "lio_node_push_imu")

    def push_imu_batch(self, stamps, acc, gyr):
        """n IMU messages: stamps (n,), acc / gyr (n, 3)."""
        t = np.ascontiguousarray(stamps, np.float64).reshape(-1)
        a = np.ascontiguousarray(acc, np.float64).reshape(-1, 3)
        g = np.ascontiguousarray(gyr, np.float64).reshape(-1, 3)
        if a.shape[0] != t.shape[0] or g.shape[0] != t.shape[0]:
            raise ValueError("one acc and one gyr row per stamp")
        _lib.check(_lib.lib().lio_node_push_imu_batch(self.h, t.shape[0], t, a if t.shape[0] else np.zeros((1, 3)),
                                                      g if t.shape[0] else np.zeros((1, 3))), "lio_node_push_imu_batch")

    def push_sweep(self, xyzi, stamp, rings=None):
        """One raw sweep from host arrays: (n, 4) float32 x y z intensity, optional (n,) ring ids (sensor_type 320 only)."""
        x = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
        r = None if rings is None else np.ascontiguousarray(rings, np.uint16).reshape(-1)
        if r is not None and r.shape[0] != x.shape[0]:
            raise ValueError("one ring index per point")
        _lib.check(_lib.lib().lio_node_push_sweep_host(self.h, x if x.shape[0] else np.zeros((1, 4), np.float32),
                                                       None if r is None else r.ctypes.data_as(C.c_void_p), x.shape[0], float(stamp)),
                   "lio_node_push_sweep_host")

    def push_sweep_dev(self, xyzi_ptr: int, n: int, stamp, rings_ptr: int | None = None):
        """One raw sweep already in HBM (float4 array, optional uint16 ring array); stream-ordered on the node's stream."""
        _lib.check(_lib.lib().lio_node_push_sweep_dev(self.h, C.c_void_p(xyzi_ptr), None if rings_ptr is None else C.c_void_p(rings_ptr),
                                                      int(n), float(stamp)), "lio_node_push_sweep_dev")

    def status(self):
        s = _lib.NodeInfo()
        _lib.check(_lib.lib().lio_node_status(self.h, C.byref(s)), "lio_node_status")
        out = {name: getattr(s, name) for name, _ in s._fields_}
        for k in ("odom_enabled", "inited", "poisoned"):
            out[k] = bool(out[k])
        return out

    # ---- read-only views of the estimator
    def states(self):
        return self.estimator.states()

    def map_poses(self):
        return self.estimator.map_poses()

    def imu_init_status(self):
        return self.estimator.imu_init_status()

    def extrinsic_calib_status(self):
        return self.estimator.extrinsic_calib_status()

    def extrinsic(self):
        return self.estimator.extrinsic()


def measure_replay(msg_time_delay, arrivals):
    """The node's pairing on a replayed arrival sequence (lio_measure_replay; no device needed).  arrivals: list of ("imu", stamp, acc3,
    gyr3) or ("msg", stamp).  Returns (calls (m, 8) float64 {dt, acc xyz, gyr xyz, stamp}, events [(arrival index, processed, first call)],
    out-of-order IMU messages dropped)."""
    n = len(arrivals)
    kind = np.array([0 if a[0] == "imu" else 1 for a in arrivals] or [0], np.int32)
    stamp = np.array([a[1] for a in arrivals] or [0.0], np.float64)
    acc = np.zeros((max(n, 1), 3)); gyr = np.zeros((max(n, 1), 3))
    for i, a in enumerate(arrivals):
        if a[0] == "imu":
            acc[i], gyr[i] = a[2], a[3]
    cap = 2 * n + 2
    calls = np.zeros((cap, 8)); ev = np.zeros((cap, 3), np.int32)
    nc, ne, nd = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib().lio_measure_replay(float(msg_time_delay), n, kind, stamp, acc, gyr, calls, cap, C.byref(nc), ev, cap,
                                             C.byref(ne), C.byref(nd)), "lio_measure_replay")
    return calls[:nc.value].copy(), [tuple(int(v) for v in e) for e in ev[:ne.value]], nd.value
