"""Host-side mirror of lio::Estimator (steady state) over the C-ABI (stages B, C, D).

Method names follow the reference (include/imu_processor/Estimator.h:110-170): ProcessImu,
ProcessLaserOdom (via process_scan), SolveOptimization and SlideWindow run inside the library; the
Python layer only moves arrays.  IntegrationBase / ImuFactor / PivotPointPlaneFactor operators are
exposed as Pim / ppp_evaluate.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

SUMMARY_KEYS = ["iterations", "successful", "termination", "initial_cost", "final_cost", "cost_pim", "cost_ppp", "cost_marg",
                "turn_off", "convergence_flag", "map_size", "num_features", "odom_iters", "t_build_map", "t_features",
                "t_solve", "t_marg", "t_total", "has_prior", "linearizations", "cost_evals", "launches", "t_lin_wait", "t_lin_host",
                "t_lin_lidar", "t_marg_wait"]


def _d(a):
    return np.ascontiguousarray(a, np.float64)


def ppp_evaluate(point, coeff, pose_pivot, pose_i, pose_ex):
    """PivotPointPlaneFactor::Evaluate for one factor (host analytic operator)."""
    r = np.zeros(1)
    J = [np.zeros(7) for _ in range(3)]
    _lib.check(_lib.lib().lio_ppp_evaluate(_d(point), _d(coeff), _d(pose_pivot), _d(pose_i), _d(pose_ex), r, J[0], J[1], J[2]),
               "lio_ppp_evaluate")
    return float(r[0]), J


def ppp_evaluate_batch(pts4, coef4, pose_pivot, pose_i, pose_ex, device=0):
    """The same operator for N factors on the GPU: residuals (N,), Jacobian rows (N, 18)."""
    _lib.require_device()
    p = np.ascontiguousarray(pts4, np.float32).reshape(-1, 4)
    c = np.ascontiguousarray(coef4, np.float32).reshape(-1, 4)
    n = p.shape[0]
    r = np.zeros(max(n, 1))
    J = np.zeros((max(n, 1), 18))
    _lib.check(_lib.lib().lio_ppp_evaluate_batch_host(p, c, n, _d(pose_pivot), _d(pose_i), _d(pose_ex), r, J, device),
               "lio_ppp_evaluate_batch_host")
    return r[:n], J[:n]


def asm_ppp(pts4, coef4, R, t, device=0):
    """Stage C reduction of one frame on the GPU: (S 7x7, sum rho)."""
    _lib.require_device()
    p = np.ascontiguousarray(pts4, np.float32).reshape(-1, 4)
    c = np.ascontiguousarray(coef4, np.float32).reshape(-1, 4)
    out = np.zeros(32)
    _lib.check(_lib.lib().lio_asm_ppp_host(p, c, p.shape[0], _d(R).reshape(9), _d(t), out, device), "lio_asm_ppp_host")
    S = np.zeros((7, 7))
    S[np.triu_indices(7)] = out[:28]
    S = S + S.T - np.diag(np.diag(S))
    return S, out[28]


def asm_stream_bench(n_features: int, iters: int = 10, device: int = 0):
    """Streaming rate of the fused stage-C kernel on a synthetic stream (choose n*32 B > L2 for the HBM rate)."""
    _lib.require_device()
    o = np.zeros(4)
    _lib.check(_lib.lib().lio_asm_stream_bench(int(n_features), int(iters), device, o), "lio_asm_stream_bench")
    return dict(avg_ms=o[0], min_ms=o[1], bytes=o[2], launches=int(o[3]), gbs=o[2] / (o[0] * 1e-3) / 1e9)


class Pim:
    """IntegrationBase (include/imu_processor/IntegrationBase.h) + ImuFactor operator."""

    def __init__(self, acc0, gyr0, ba, bg, acc_n=0.1, gyr_n=0.01, acc_w=2e-4, gyr_w=2e-5, g_norm=9.805):
        self.h = C.c_void_p()
        _lib.check(_lib.lib().lio_pim_create(_d(acc0), _d(gyr0), _d(ba), _d(bg), _d([acc_n, gyr_n, acc_w, gyr_w, g_norm]),
                                             C.byref(self.h)), "lio_pim_create")
        self.owned = True

    def push_back(self, dt, acc, gyr):
        _lib.check(_lib.lib().lio_pim_push_back(self.h, float(dt), _d(acc), _d(gyr)), "lio_pim_push_back")

    def get(self):
        s = np.zeros(11); J = np.zeros(225); P = np.zeros(225)
        _lib.check(_lib.lib().lio_pim_get(self.h, s, J, P), "lio_pim_get")
        return dict(delta_p=s[0:3], delta_q=s[3:7], delta_v=s[7:10], sum_dt=s[10], jacobian=J.reshape(15, 15),
                    covariance=P.reshape(15, 15))

    def imu_factor(self, pose_i, sb_i, pose_j, sb_j):
        r = np.zeros(15)
        J = [np.zeros(15 * 7), np.zeros(15 * 9), np.zeros(15 * 7), np.zeros(15 * 9)]
        _lib.check(_lib.lib().lio_imu_factor_evaluate(self.h, _d(pose_i), _d(sb_i), _d(pose_j), _d(sb_j), r, *J),
                   "lio_imu_factor_evaluate")
        return r, [J[0].reshape(15, 7), J[1].reshape(15, 9), J[2].reshape(15, 7), J[3].reshape(15, 9)]

    def __del__(self):
        try:
            if self.owned and self.h:
                _lib.lib().lio_pim_destroy(self.h)
        except Exception:
            pass


class Estimator:
    def __init__(self, device: int = 0, stream: int = 0, **cfg):
        L = _lib.lib()
        _lib.require_device()
        c = _lib.EstConfig()
        L.lio_est_default_config(C.byref(c))
        for k, v in cfg.items():
            if not hasattr(c, k):
                raise AttributeError(f"EstimatorConfig has no field {k}")
            setattr(c, k, v)
        self.c = c
        self.cfg = {name: getattr(c, name) for name, _ in c._fields_}
        self.W = c.window_size
        self.h = C.c_void_p()
        _lib.check(L.lio_est_create(C.byref(c), device, C.c_void_p(stream), C.byref(self.h)), "lio_est_create")
        self._cb = None

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lio_est_destroy(self.h)
            self.h = None
        self._map = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_extrinsic(self, tf7):
        _lib.check(_lib.lib().lio_est_set_extrinsic(self.h, np.ascontiguousarray(tf7, np.float32)), "set_extrinsic")

    def extrinsic(self):
        t = np.zeros(7, np.float32)
        _lib.check(_lib.lib().lio_est_get_extrinsic(self.h, t), "get_extrinsic")
        return t

    def init_frame(self, k, state16, surf_ds, pim: "Pim | None"):
        s = np.ascontiguousarray(surf_ds, np.float32).reshape(-1, 4)
        h = None
        if pim is not None:
            h = pim.h
            pim.owned = False   # ownership passes to the estimator
        _lib.check(_lib.lib().lio_est_init_frame(self.h, k, _d(state16), s, s.shape[0], h), "lio_est_init_frame")

    def finish_init(self, acc_last, gyr_last):
        _lib.check(_lib.lib().lio_est_finish_init(self.h, _d(acc_last), _d(gyr_last)), "lio_est_finish_init")

    def process_imu(self, dt, acc, gyr, stamp):
        _lib.check(_lib.lib().lio_est_process_imu(self.h, float(dt), _d(acc), _d(gyr), float(stamp)), "lio_est_process_imu")

    def process_imu_batch(self, dt, acc, gyr, stamp):
        """n consecutive ProcessImu calls in one C-ABI crossing (arrays of n, n x 3, n x 3, n)."""
        dt = np.ascontiguousarray(dt, np.float64)
        _lib.check(_lib.lib().lio_est_process_imu_batch(self.h, dt.shape[0], dt, np.ascontiguousarray(acc, np.float64),
                                                        np.ascontiguousarray(gyr, np.float64), np.ascontiguousarray(stamp, np.float64)),
                   "lio_est_process_imu_batch")

    def process_scan(self, surf_last):
        s = np.ascontiguousarray(surf_last, np.float32).reshape(-1, 4)
        _lib.check(_lib.lib().lio_est_process_scan_host(self.h, s, s.shape[0]), "lio_est_process_scan_host")

    # ---- stepwise API (Estimator::ProcessLaserOdom / SolveOptimization phase by phase)
    def open_scan(self, surf_last):
        s = np.ascontiguousarray(surf_last, np.float32).reshape(-1, 4)
        _lib.check(_lib.lib().lio_est_open_scan_host(self.h, s, s.shape[0]), "lio_est_open_scan_host")

    def parameters(self):
        O = self.c.opt_window_size
        pose = np.zeros((O + 1, 7)); sb = np.zeros((O + 1, 9)); ex = np.zeros(7)
        _lib.check(_lib.lib().lio_est_get_parameters(self.h, pose, sb, ex), "lio_est_get_parameters")
        return pose, sb, ex

    def assemble(self, pose=None, sb=None, ex=None):
        """(H, g, cost) of the open window's ceres problem at the given parameter blocks (None: the estimator's own)."""
        nmax = 15 * (self.c.opt_window_size + 1) + 6
        H = np.zeros((nmax, nmax)); g = np.zeros(nmax); cost = C.c_double(); n = C.c_int()
        keep = [None if a is None else np.ascontiguousarray(a, np.float64) for a in (pose, sb, ex)]
        ptr = [None if a is None else a.ctypes.data_as(C.c_void_p) for a in keep]
        _lib.check(_lib.lib().lio_est_assemble(self.h, ptr[0], ptr[1], ptr[2], H, g, C.byref(cost), C.byref(n)), "lio_est_assemble")
        n = n.value
        return H.reshape(-1)[:n * n].reshape(n, n).copy(), g[:n].copy(), cost.value

    def solve(self, pose, sb, ex, max_iter=None):
        pose = np.ascontiguousarray(pose, np.float64).copy(); sb = np.ascontiguousarray(sb, np.float64).copy()
        ex = np.ascontiguousarray(ex, np.float64).copy()
        summ = np.zeros(8)
        _lib.check(_lib.lib().lio_est_solve(self.h, pose, sb, ex, self.c.max_num_iterations if max_iter is None else int(max_iter), summ),
                   "lio_est_solve")
        keys = ["iterations", "successful", "termination", "initial_cost", "final_cost", "evaluations", "convergence_flag", "ex_constant"]
        return pose, sb, ex, dict(zip(keys, summ.tolist()))

    def close_scan(self, pose=None, sb=None, ex=None):
        keep = [None if a is None else np.ascontiguousarray(a, np.float64) for a in (pose, sb, ex)]
        ptr = [None if a is None else a.ctypes.data_as(C.c_void_p) for a in keep]
        _lib.check(_lib.lib().lio_est_close_scan(self.h, ptr[0], ptr[1], ptr[2]), "lio_est_close_scan")

    def begin_scan(self):
        """Announce the next sweep (starts the previous scan's background marginalisation algebra)."""
        _lib.check(_lib.lib().lio_est_begin_scan(self.h), "lio_est_begin_scan")

    def process_scan_dev(self, dev_ptr: int, n_dev_ptr: int, n_max: int):
        _lib.check(_lib.lib().lio_est_process_scan_dev(self.h, C.c_void_p(dev_ptr), C.c_void_p(n_dev_ptr), n_max),
                   "lio_est_process_scan_dev")

    def set_shard(self, rank, world, fn):
        """fn(buf_dev_ptr:int, count:int) -> int must sum-allreduce `count` doubles in place on the device."""
        if fn is None:
            cb = _lib.ALLREDUCE_FN()
        else:
            cb = _lib.ALLREDUCE_FN(lambda user, buf, count: int(fn(buf, count)))
        self._cb = cb
        _lib.check(_lib.lib().lio_est_set_shard(self.h, rank, world, cb, None), "lio_est_set_shard")

    def exchange_buffer(self) -> int:
        """Device pointer of this rank's exchange buffer (peer-memory exchange of the S blocks)."""
        p = C.c_void_p()
        _lib.check(_lib.lib().lio_est_exchange_buffer(self.h, C.byref(p), None), "lio_est_exchange_buffer")
        return p.value

    def exchange_handle(self) -> np.ndarray:
        """64-byte CUDA IPC handle of the exchange buffer, to be all-gathered across ranks."""
        h = np.zeros(64, np.uint8)
        _lib.check(_lib.lib().lio_ipc_export(C.c_void_p(self.exchange_buffer()), h), "lio_ipc_export")
        return h

    def set_peers(self, rank, world, ptrs=None, handles=None):
        """Switch the sharded solve to the fused peer-memory exchange.  ptrs: device pointers of every rank's exchange
        buffer valid in this process (same-process contexts), or handles: (world, 64) uint8 IPC handles (one per rank)."""
        self.set_shard(rank, world, None)
        self._peer_open = []
        arr = self._peer_array(rank, world, self.exchange_buffer(), ptrs, handles, self._peer_open)
        _lib.check(_lib.lib().lio_est_set_peers(self.h, world, arr), "lio_est_set_peers")

    def feature_slab(self):
        p = C.c_void_p(); n = C.c_size_t()
        _lib.check(_lib.lib().lio_est_feature_slab(self.h, C.byref(p), C.byref(n)), "lio_est_feature_slab")
        return p.value

    def feature_slab_handle(self):
        h = np.zeros(64, np.uint8)
        _lib.check(_lib.lib().lio_ipc_export(C.c_void_p(self.feature_slab()), h), "lio_ipc_export")
        return h

    def set_feature_peers(self, rank, world, ptrs=None, handles=None):
        """Sharded matching with a per-scan exchange of the features themselves (lio_est_set_feature_peers): ptrs = every rank's
        feature slab as a device pointer valid in this process, or handles = (world, 64) uint8 IPC handles."""
        self.set_shard(rank, world, None)
        self._fpeer_open = []
        arr = self._peer_array(rank, world, self.feature_slab(), ptrs, handles, self._fpeer_open)
        _lib.check(_lib.lib().lio_est_set_feature_peers(self.h, world, arr), "lio_est_set_feature_peers")

    @staticmethod
    def _peer_array(rank, world, own, ptrs, handles, opened):
        """Every rank's buffer as a device pointer valid in this process: `own` for this rank, ptrs[r] or the IPC handle
        handles[r] opened here (its pointer appended to `opened`) for the others."""
        arr = (C.c_void_p * world)()
        for r in range(world):
            if r == rank:
                arr[r] = own
            elif ptrs is not None:
                arr[r] = int(ptrs[r])
            else:
                p = C.c_void_p()
                _lib.check(_lib.lib().lio_ipc_open(np.ascontiguousarray(handles[r], np.uint8), C.byref(p)), "lio_ipc_open")
                opened.append(p.value)
                arr[r] = p.value
        return arr

    def kernel_profile(self, reset=False):
        o = np.zeros(8)
        _lib.check(_lib.lib().lio_est_kernel_profile(self.h, o, 1 if reset else 0), "kernel_profile")
        return dict(asm_ms=o[0], asm_launches=int(o[1]), asm_features=int(o[2]), bytes_per_feature=o[3],
                    knn_ms=o[4], knn_launches=int(o[5]), knn_queries=int(o[6]), bytes_per_query=o[7])

    def solver_trace(self):
        """Phase timestamps of the device solver's step kernel, (24, 16) int64 (see lio_est_solver_trace)."""
        out = np.zeros(24 * 16 + 4 * 28 + 4, np.int64)
        _lib.check(_lib.lib().lio_est_solver_trace(self.h, out, out.size), "lio_est_solver_trace")
        self.chol_profile = out[24 * 16:]
        return out[:24 * 16].reshape(24, 16)

    def states(self):
        out = np.zeros((self.W + 1, 16))
        _lib.check(_lib.lib().lio_est_get_states(self.h, out), "lio_est_get_states")
        return out

    def local_laser_odom(self):
        """/local_laser_odom (Estimator.cc:725-742) after process_scan, as the float tf7 (qx qy qz qw px py pz) that the map
        builder's LaserOdometryHandler (PointMapping.cc:267-282) keeps: the lidar pose of window slot W - O, i.e. of the scan
        received O - 1 scans before the newest, rot = R q_lb^-1 and pos = P - rot p_lb.  The clouds that go with it are that
        scan's: local_clouds() / local_clouds_dev() once enable_local_clouds() is on."""
        t = np.zeros(7, np.float32)
        _lib.check(_lib.lib().lio_est_local_laser_odom(self.h, t), "lio_est_local_laser_odom")
        return t

    # ---- /local/* publication (lio_est_enable_local_clouds): the map builder's input
    LOCAL_CLOUDS = ("corner", "surf", "full")

    def enable_local_clouds(self, corner_filter_size=0.2, max_corner_points=1 << 16, max_full_points=1 << 18):
        """Keep corner_stack_ / full_stack_ and publish /local/* (call before the first init_frame)."""
        _lib.check(_lib.lib().lio_est_enable_local_clouds(self.h, float(corner_filter_size), int(max_corner_points), int(max_full_points)),
                   "lio_est_enable_local_clouds")

    def set_scan_clouds(self, corner, full):
        """Stage /laser_cloud_corner_last and the full cloud of the next pushed frame (host arrays, copied before return)."""
        c = np.ascontiguousarray(corner, np.float32).reshape(-1, 4)
        f = np.ascontiguousarray(full, np.float32).reshape(-1, 4)
        nc, nf = c.shape[0], f.shape[0]
        c = c if nc else np.zeros((1, 4), np.float32)
        f = f if nf else np.zeros((1, 4), np.float32)
        _lib.check(_lib.lib().lio_est_set_scan_clouds_host(self.h, c, nc, f, nf), "lio_est_set_scan_clouds_host")

    def set_scan_clouds_dev(self, corner_ptr: int, nc_dev_ptr: int, nc_max: int, full_ptr: int, nf_dev_ptr: int, nf_max: int):
        """The same from device float4 arrays and device counts (stream-ordered on the estimator's stream)."""
        _lib.check(_lib.lib().lio_est_set_scan_clouds_dev(self.h, C.c_void_p(corner_ptr), C.c_void_p(nc_dev_ptr), int(nc_max),
                                                          C.c_void_p(full_ptr), C.c_void_p(nf_dev_ptr), int(nf_max)),
                   "lio_est_set_scan_clouds_dev")

    def local_clouds_dev(self):
        """(ptrs {corner, surf, full} as ints, device pointer of their int[3] counts, their capacities as n_max) of /local/*:
        valid until the next scan entry, stream-ordered on the estimator's stream."""
        ptrs = (C.c_void_p * 3)(); n_dev = C.c_void_p(); n_max = np.zeros(3, np.int32)
        _lib.check(_lib.lib().lio_est_local_clouds_dev(self.h, ptrs, C.byref(n_dev), n_max), "lio_est_local_clouds_dev")
        return [int(p or 0) for p in ptrs], n_dev.value, n_max

    def local_clouds(self):
        """/local/corner_points, /local/surf_points and /local/full_points of the last scan as a dict of (n, 4) float32 arrays."""
        _, _, cap = self.local_clouds_dev()
        out = {}
        for w, name in enumerate(self.LOCAL_CLOUDS):
            a = np.zeros((max(int(cap[w]), 1), 4), np.float32); n = C.c_int()
            _lib.check(_lib.lib().lio_est_local_clouds_download(self.h, w, a, a.shape[0], C.byref(n)), "lio_est_local_clouds_download")
            out[name] = a[:n.value].copy()
        return out

    # ---- the global cube map after initialisation (lio_est_attach_map)
    def attach_map(self, pm):
        """Hand a publishing PointMapping (EnablePublish, at least one ProcessDev, same device) that built the pre-initialisation map
        to the estimator: after finish_init, before the first scan, with local clouds on.  From then on every scan predicts
        transform_tobe_mapped_, inserts the oldest optimised frame from the (O+1)-th scan on and publishes the surround map and the
        registered full cloud on pm (pm.surround_map(), pm.registered_full_cloud(), pm.cube(...)).  pm refuses its own process
        calls and close() until this estimator is closed; the estimator keeps a reference to it."""
        _lib.check(_lib.lib().lio_est_attach_map(self.h, pm.h), "lio_est_attach_map")
        self._map = pm

    def map_poses(self):
        """After a scan with an attached map: (tobe tf7 = transform_tobe_mapped_, aft tf7 = the frozen transform_aft_mapped_,
        insert tf7 = the pose of the last insert, info dict)."""
        tobe = np.zeros(7, np.float32); aft = np.zeros(7, np.float32); ins = np.zeros(7, np.float32); info = np.zeros(4, np.int32)
        _lib.check(_lib.lib().lio_est_map_poses(self.h, tobe, aft, ins, info), "lio_est_map_poses")
        return tobe, aft, ins, dict(inserted=bool(info[0]), points=int(info[1]), surround_published=bool(info[2]), surround_size=int(info[3]))

    def summary(self):
        s = np.zeros(32)
        _lib.check(_lib.lib().lio_est_summary(self.h, s), "lio_est_summary")
        return dict(zip(SUMMARY_KEYS, s.tolist()))

    def features(self, frame):
        n = C.c_int()
        _lib.check(_lib.lib().lio_est_feature_count(self.h, frame, C.byref(n)), "feature_count")
        n = n.value
        p = np.zeros((max(n, 1), 4), np.float32); c = np.zeros((max(n, 1), 4), np.float32); s = np.zeros(max(n, 1), np.int32)
        _lib.check(_lib.lib().lio_est_get_features(self.h, frame, p, c, s, max(n, 1)), "get_features")
        return p[:n], c[:n], s[:n]

    def local_map(self):
        n = C.c_int()
        _lib.check(_lib.lib().lio_est_map_size(self.h, C.byref(n)), "map_size")
        m = np.zeros((max(n.value, 1), 4), np.float32)
        _lib.check(_lib.lib().lio_est_get_map(self.h, m, m.shape[0]), "get_map")
        return m[:n.value]

    def frame(self, k):
        n = C.c_int()
        _lib.check(_lib.lib().lio_est_frame_size(self.h, k, C.byref(n)), "frame_size")
        m = np.zeros((max(n.value, 1), 4), np.float32)
        _lib.check(_lib.lib().lio_est_get_frame(self.h, k, m, m.shape[0]), "get_frame")
        return m[:n.value]

    def local_transform(self, k):
        t = np.zeros(7, np.float32)
        _lib.check(_lib.lib().lio_est_get_local_transform(self.h, k, t), "get_local_transform")
        return t

    def prior(self):
        n = C.c_int()
        _lib.check(_lib.lib().lio_est_prior_dim(self.h, C.byref(n)), "prior_dim")
        n = n.value
        H = np.zeros((max(n, 1), max(n, 1))); b = np.zeros(max(n, 1))
        if n:
            _lib.check(_lib.lib().lio_est_get_prior(self.h, H, b), "get_prior")
        return H[:n, :n], b[:n]

    def normal_equations(self):
        nmax = 15 * (self.c.opt_window_size + 1) + 6
        n = C.c_int(); cost = C.c_double()
        H = np.zeros((nmax, nmax)); g = np.zeros(nmax)
        _lib.check(_lib.lib().lio_est_last_normal_equations(self.h, H, g, C.byref(cost), C.byref(n)), "normal_eq")
        n = n.value
        return H.reshape(-1)[:n * n].reshape(n, n).copy(), g[:n].copy(), cost.value
