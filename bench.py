#!/usr/bin/env python
"""bench.py — scans/sec of the steady-state LIO hot path (stage A on the new sweep + stage B for the O
window frames + <= 10 Gauss-Newton/dogleg iterations of stage C + stage D marginalisation) on synthetic
HDL-64 sweeps + IMU, window 10/10 (BASELINE.json configs[2], the configuration the metric is quoted on).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--workload hdl64|vlp16|stress128]
                  [--dump-outputs DIR]

One "step" = one scan through the whole path.  `value` times the path with the raw sweep already resident
in HBM; `e2e` times the same call chain through the C-ABI with HOST buffers (pinned host -> device copy of the
sweep and the result read-back inside the timed region).  `--impl reference` times the CPU restatement of
the reference path (oracle/, the reference itself cannot be built here: no Eigen/PCL/Ceres/ROS) on the box's
host cores.  Multi-GPU (torchrun, one rank per GPU): the window's frames are sharded one-per-rank, the
packed S blocks are sum-allreduced over NCCL once per evaluation (strong scaling of one window solve).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "scans/sec + GN-iter ms, HDL-64 window=10 at 1/2/4/8 H100 vs CPU Ceres ref"
DUMP_LIMIT_BYTES = 64 << 20


def env_int(name, default):
    try:
        return int(os.environ.get(name, default))
    except ValueError:
        return default


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.p = None
        self.gpu = gpu_index
        self.path = "/tmp/lio_bench_clocks_%d.csv" % os.getpid()

    def start(self):
        try:
            self.f = open(self.path, "w")
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                                       "-lms", "100"], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def stop(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        if self.p is None:
            return out
        try:
            for _ in range(20):          # a run shorter than the first sampling period: wait for one sample rather than report none
                if os.path.getsize(self.path) > 0:
                    break
                time.sleep(0.05)
            self.p.terminate(); self.p.wait(timeout=5); self.f.close()
            sm, smax, reasons = [], [], set()
            for line in open(self.path):
                v = [x.strip() for x in line.split(",")]
                if len(v) < 9:
                    continue
                try:
                    sm.append(float(v[1])); smax.append(float(v[2]))
                except ValueError:
                    continue
                for name, val in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], v[5:9]):
                    if val.lower().startswith("active"):
                        reasons.add(name)
            if sm:
                out = {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(np.max(smax)), "reasons": sorted(reasons), "samples": len(sm),
                       "window": "warm-up + timed steps (nvidia-smi -lms 100)"}
        except Exception:
            pass
        return out


def load_peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
    except Exception:
        return 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s HBM3)"


# ------------------------------------------------------------------------------------------------
def run_reference(args, scn, W, est_cfg):
    """CPU restatement of the reference path on the host cores (oracle/): the reference arm and cpu_baseline."""
    from oracle import oracle_py as O
    from lio_mapping_b200 import scenario
    O.build()
    sensor = scn.sensor
    eo = O.Estimator(window_size=W, opt_window_size=W, **est_cfg)
    lf = {}

    def stage_a(k):
        if k not in lf:
            lf[k] = O.stage_a(scn.raw[k], sensor.lower_deg, sensor.upper_deg, sensor.rings)["less_flat"]
        return lf[k]

    scenario.warm_start(eo, scn, W, lambda k: O.voxel_grid(stage_a(k), est_cfg["surf_filter_size"]),
                        lambda a, g: O.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=est_cfg["acc_n"], gyr_n=est_cfg["gyr_n"],
                                           acc_w=est_cfg["acc_w"], gyr_w=est_cfg["gyr_w"], g_norm=est_cfg["g_norm"]))
    times, iters, solve_t, states = [], [], [], {}
    k0 = W
    for s in range(args.warmup + args.steps):
        k = k0 + s
        t0 = time.perf_counter()
        r = O.stage_a(scn.raw[k], sensor.lower_deg, sensor.upper_deg, sensor.rings)      # stage A (timed)
        scenario.feed_imu(eo, scn, k)
        eo.process_scan(r["less_flat"])
        dt = time.perf_counter() - t0
        states[k] = eo.states()
        if s >= args.warmup:
            times.append(dt)
            sm = eo.summary()
            iters.append(sm["iterations"]); solve_t.append(sm["t_solve"])
    total = float(np.sum(times))
    return dict(scans_per_s=len(times) / total, ms_per_step=1e3 * total / len(times),
                gn_iter_ms=1e3 * float(np.sum(solve_t)) / max(1.0, float(np.sum(iters))), steps=len(times), states=states)


def host_cores():
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


def dump_outputs(out_dir, arrays):
    """Writes the arrays as out_dir/<name>.npy (float32 stays float32, everything else float64).  Above DUMP_LIMIT_BYTES in
    all, the larger arrays are cut to a fixed, seeded sample of their rows (kept in order) so that two runs stay comparable."""
    os.makedirs(out_dir, exist_ok=True)
    arrays = {k: np.asarray(v, np.float32 if np.asarray(v).dtype == np.float32 else np.float64) for k, v in arrays.items()}
    total = sum(a.nbytes for a in arrays.values())
    for name, a in arrays.items():
        if total > DUMP_LIMIT_BYTES and a.ndim >= 1 and a.shape[0] > 1:
            keep = max(1, int(a.shape[0] * DUMP_LIMIT_BYTES / total))
            rows = np.sort(np.random.default_rng(0).choice(a.shape[0], keep, replace=False))
            a = a[rows]
        np.save(os.path.join(out_dir, name + ".npy"), a)


def asm_traffic(kind):
    """dram__bytes_read+write per asm_ppp launch from the committed `ncu --set full` capture of the SAME workload
    (profiles/asm_ppp_traffic.json), else None."""
    try:
        t = json.load(open(os.path.join(ROOT, "profiles", "asm_ppp_traffic.json")))
        return t.get(kind, {}).get("traffic_bytes_per_launch")
    except Exception:
        return None


# ------------------------------------------------------------------------------------------------
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="hdl64", choices=["hdl64", "vlp16", "stress128"])
    ap.add_argument("--overlap-marginalization", type=int, default=1, choices=[0, 1],
                    help="0: marginalisation algebra inline (reference order); 1: on a worker thread beside the next scan's front end")
    ap.add_argument("--exchange", default="peer", choices=["peer", "rows", "nccl"],
                    help="multi-GPU: peer = per-scan exchange of the features over peer memory (default); rows = S blocks stored from the "
                         "stage-C kernel tail at every evaluation; nccl = allreduce callback of the S blocks")
    ap.add_argument("--cpu-sample", type=int, default=4, help="scans of the cpu_baseline sample (rank 0, N=1 only)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed scan computed as DIR/<name>.npy (rank 0)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else max(args.warmup, 1)

    rank, world, local_rank = env_int("RANK", 0), env_int("WORLD_SIZE", 1), env_int("LOCAL_RANK", 0)
    from lio_mapping_b200 import scenario
    kind = args.workload
    W = scenario.WINDOWS[kind]
    est_cfg = dict(scenario.EST_CFG[kind])
    workload = {"hdl64": "HDL-64 outdoor_test_config_64 synthetic, 64x2032 sweep, window=10/10, prior_factor=1",
                "vlp16": "VLP-16 indoor synthetic, 16x1800 sweep, window=10/10",
                "stress128": "synthetic 128x4096 sweep, window=15/15"}[kind]
    n_total = W + args.warmup + args.steps + 1

    if args.impl == "reference":
        if rank != 0:
            return 0
        scn = scenario.Scenario(kind, n_total=n_total)
        r = run_reference(args, scn, W, est_cfg)
        cores = 4   # threads the restatement actually uses: 1 (front end, kNN, dogleg: Ceres num_threads = 1) + 4 only inside ThreadsConstructA
        line = {"impl": "reference", "metric": METRIC, "value": r["scans_per_s"], "unit": "scans/s", "n_gpus": args.gpus,
                "steps": args.steps, "warmup": args.warmup, "ms_per_step": r["ms_per_step"], "higher_is_better": True,
                "scaling": "strong", "vs_baseline": None, "dtype": "f32 features / f64 solve", "data": "synthetic",
                "gn_iter_ms": r["gn_iter_ms"],
                "config": {"workload": workload, "window": W, "opt_window": W, "points_per_scan": int(scn.raw[W].shape[0])},
                "cpu_baseline": {"value": r["scans_per_s"], "unit": "scans/s", "cores": cores, "host_cores": host_cores(), "kind": "port",
                                 "sample": "%d scans of the same workload (oracle/: CPU restatement; the reference needs Eigen/PCL/Ceres/ROS, absent here); 1 thread + 4 marginalisation threads" % r["steps"]},
                "e2e": {"value": r["scans_per_s"], "unit": "scans/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return 0

    # ---------------- our arm ----------------
    import torch
    import torch.distributed as dist
    from lio_mapping_b200 import _lib, estimator, ops
    from lio_mapping_b200.point_processor import PointProcessor
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (lio_mapping_b200 has no CPU fallback)")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    stream = torch.cuda.current_stream().cuda_stream
    scn = scenario.Scenario(kind, n_total=n_total)
    sensor = scn.sensor
    max_pts = max(s.shape[0] for s in scn.raw)
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_pts, device=local_rank, stream=stream)
    est = estimator.Estimator(device=local_rank, stream=stream, window_size=W, opt_window_size=W,
                              max_frame_points=1 << 16 if kind != "stress128" else 1 << 18,
                              max_scan_points=max_pts, overlap_marginalization=args.overlap_marginalization, **est_cfg)
    if world > 1:
        class _Arr:
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 3}

        def allreduce(ptr, count):
            t = torch.as_tensor(_Arr(ptr, count), device=dev)
            dist.all_reduce(t)
            return 0

        exchange = {"kind": "nccl allreduce (torch.distributed) of O x 32 doubles per evaluation"}

        def attach(e):
            """Preferred: per-scan exchange of the features over peer memory (every rank then solves like a single GPU);
            --exchange rows: S rows stored from the stage-C kernel tail at every evaluation; fallback: NCCL allreduce callback."""
            if args.exchange == "nccl":
                e.set_shard(rank, world, allreduce)
                return
            try:
                feat = args.exchange != "rows"
                mine = torch.from_numpy(e.feature_slab_handle() if feat else e.exchange_handle()).to(dev)
                allh = [torch.zeros(64, dtype=torch.uint8, device=dev) for _ in range(world)]
                dist.all_gather(allh, mine)
                if feat:
                    e.set_feature_peers(rank, world, handles=[h.cpu().numpy() for h in allh])
                else:
                    e.set_peers(rank, world, handles=[h.cpu().numpy() for h in allh])
                ok = torch.ones(1, device=dev)
            except Exception as exc:   # no P2P / IPC on this box
                print(f"[bench] peer exchange unavailable on rank {rank}: {exc!r}", file=sys.stderr)
                ok = torch.zeros(1, device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
            if float(ok.item()) < 0.5:
                e.set_shard(rank, world, allreduce)
            elif feat:
                exchange["kind"] = ("matching sharded by frame; once per scan every rank stores the features of its frames into every rank's feature slab "
                                    "(P2P stores + epoch flags over CUDA-IPC peer memory), then each rank runs the complete solve like a single GPU")
            else:
                exchange["kind"] = "fused into the stage-C kernel tail: P2P stores of the owned S blocks into every rank's buffer + epoch flags (CUDA IPC peer memory)"
        attach(est)

    def surf_ds_of(k):
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        return ops.voxel_grid(pp.cloud("surface_points_less_flat"), est_cfg["surf_filter_size"], device=local_rank)

    scenario.warm_start(est, scn, W, surf_ds_of,
                        lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=est_cfg["acc_n"], gyr_n=est_cfg["gyr_n"],
                                                   acc_w=est_cfg["acc_w"], gyr_w=est_cfg["gyr_w"], g_norm=est_cfg["g_norm"]))
    L = _lib.lib()
    lf_ptr = pp.cloud_dev("surface_points_less_flat")
    nptr = C.c_void_p()
    _lib.check(L.lio_pp_cloud_count_dev(pp._h, 5, C.byref(nptr)), "lio_pp_cloud_count_dev")
    # raw sweeps resident in HBM for the device-timed value; pinned host copies for e2e
    dev_raw = {k: torch.from_numpy(scn.raw[k]).to(dev) for k in range(W, n_total - 1)}
    pin_raw = {k: torch.from_numpy(np.ascontiguousarray(scn.raw[k], np.float32)).pin_memory() for k in range(W, n_total - 1)}
    pin_np = {k: v.numpy() for k, v in pin_raw.items()}       # numpy views of the page-locked buffers
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)   # > 50 MB L2

    def step_dev(k):
        t = dev_raw[k]
        est.begin_scan()                                     # sweep k arrived: background marginalisation of scan k-1 starts here
        pp.process_device(t.data_ptr(), t.shape[0])
        scenario.feed_imu(est, scn, k)
        est.process_scan_dev(lf_ptr, nptr.value, max_pts)

    def step_host(k):
        est.begin_scan()
        pp.SetInputCloud(pin_np[k]); pp.Process()            # H2D of the sweep (pinned host memory) inside
        scenario.feed_imu(est, scn, k)
        est.process_scan_dev(lf_ptr, nptr.value, max_pts)
        return est.states()                                  # result read-back (host state after the solve)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # The window is stateful, so the device-timed and e2e passes each consume their own scans:
    #   warmup scans -> K device-timed scans (value) ; the e2e pass re-runs a fresh estimator on the same scans.
    k = W
    barrier()   # ranks leave the (CPU-heavy, unequal) set-up together: the device-side exchange waits are bounded
    # nvidia-smi needs ~100 ms for its first sample and the timed region is K x 2 ms: the sampler starts with the warm-up steps
    # (the same load) so that it is running when the timed steps begin; samples = warm-up + timed region
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    for _ in range(args.warmup):
        step_dev(k); k += 1
    est.kernel_profile(reset=True)
    barrier()
    profiling = os.environ.get("LIO_BENCH_PROFILE") == "1"   # ncu --profile-from-start off: capture the timed steps only
    if profiling:
        torch.cuda.cudart().cudaProfilerStart()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    launches, iters, solve_t, feats = 0, [], [], []
    brk = {"t_build_map": [], "t_features": [], "t_solve": [], "t_marg": [], "t_total": [], "t_lin_wait": [], "t_lin_host": [],
           "t_lin_lidar": [], "t_marg_wait": []}
    for s in range(args.steps):
        flush.fill_(1.0)                                      # flush L2 between timed steps (outside the event pair)
        barrier()
        ev[s][0].record()
        step_dev(k)
        ev[s][1].record()
        torch.cuda.synchronize()
        launches += pp.last_launches() + int(L.lio_est_last_launches(est.h))
        sm = est.summary()
        iters.append(sm["iterations"]); solve_t.append(sm["t_solve"]); feats.append(sm["num_features"])
        for kk in brk:
            brk[kk].append(sm[kk])
        k += 1
    barrier()
    if profiling:
        torch.cuda.cudart().cudaProfilerStop()
    clocks = sampler.stop() if rank == 0 else None
    if os.environ.get("LIO_BENCH_TRACE") == "1" and rank == 0:
        # device-side timeline of the last solve (%globaltimer stamps, ns): per evaluation the gap kernels between two k_step launches
        tr = est.solver_trace()
        n_ev = int((tr[:12, 0] > 0).sum())
        print("[trace] eval: k_step in..out | gap to next k_step | asm in/out, k_factors in/out, k_hpart out (all relative to the previous k_step's exit)", file=sys.stderr)
        for e_ in range(1, n_ev):
            t0 = int(tr[e_ - 1, 11])
            rel = lambda v: (int(v) - t0) / 1000.0 if v else float("nan")
            print("[trace] ev %2d  k_step %6.1f us | gap %5.1f | asm %5.1f..%5.1f  k_factors %5.1f..%5.1f  k_hpart ..%5.1f | phases(cyc) %s" % (
                e_, (int(tr[e_, 11]) - int(tr[e_, 0])) / 1000.0, rel(tr[e_, 0]), rel(tr[13, e_]), rel(tr[14, e_]), rel(tr[e_, 12]), rel(tr[e_, 13]),
                rel(tr[e_, 14]), np.diff(tr[e_, 1:11]).tolist()), file=sys.stderr)
        print("[trace] lidar_blocks marks (cycles from entry, eval 2): %s" % (tr[16, 1:4] - tr[16, 0]).tolist(), file=sys.stderr)
        cp = est.chol_profile
        NBp = (15 * (W + 1) + 6 + 7) // 8
        pp_ = cp[:4 * NBp].reshape(NBp, 4)
        print("[trace] in-kernel Cholesky (eval 1) per panel [solve, own_update, diag, update_total] cycles: %s backsub %d total %d" % (
            pp_.tolist(), int(cp[4 * NBp]), int(pp_[:, 0].sum() + pp_[:, 3].sum() + cp[4 * NBp])), file=sys.stderr)
        print("[trace] chol %%globaltimer ns: entry->loop %d, loop %d, backsub %d, total %d" % (
            cp[4 * NBp + 2] - cp[4 * NBp + 1], cp[4 * NBp + 3] - cp[4 * NBp + 2], cp[4 * NBp + 4] - cp[4 * NBp + 3], cp[4 * NBp + 4] - cp[4 * NBp + 1]), file=sys.stderr)
    ms = [a.elapsed_time(b) for a, b in ev]
    total_ms = float(np.sum(ms))
    if world > 1:
        t = torch.tensor([total_ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        total_ms = float(t.item())
    prof = est.kernel_profile()
    final_states = est.states()
    if args.dump_outputs and rank == 0:
        # what a caller of the timed path receives for the last timed scan: stage A's clouds, the newest frame's matched
        # features (stage B), the local map and the solved window (stages C + D)
        p_new, c_new, _ = est.features(W)
        sm = est.summary()
        dump_outputs(args.dump_outputs, dict(
            {"pp_" + name: pp.cloud(name) for name in ("laser_scans", "corner_points_sharp", "corner_points_less_sharp",
                                                       "surface_points_flat", "surface_points_less_flat")},
            features_points=p_new, features_coef=c_new, local_map=est.local_map(), states=final_states,
            extrinsic=est.extrinsic(),
            solve=np.array([sm[kk] for kk in ("iterations", "initial_cost", "final_cost", "map_size", "num_features", "has_prior")])))

    if profiling:
        print(json.dumps({"profiling_run": True, "ms_per_step_under_profiler": total_ms / args.steps}))
        return 0
    # ---- e2e pass (host buffers, fresh estimator, same scans) --------------------------------------
    est2 = estimator.Estimator(device=local_rank, stream=stream, window_size=W, opt_window_size=W,
                               max_frame_points=1 << 16 if kind != "stress128" else 1 << 18, max_scan_points=max_pts,
                               overlap_marginalization=args.overlap_marginalization, **est_cfg)
    if world > 1:
        attach(est2)
    est_saved, est = est, est2
    scenario.warm_start(est, scn, W, surf_ds_of,
                        lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=est_cfg["acc_n"], gyr_n=est_cfg["gyr_n"],
                                                   acc_w=est_cfg["acc_w"], gyr_w=est_cfg["gyr_w"], g_norm=est_cfg["g_norm"]))
    k = W
    barrier()
    e2e_states = {}
    for _ in range(args.warmup):
        e2e_states[k] = step_host(k); k += 1
    e2e_t = 0.0
    h2d = d2h = 0
    for s in range(args.steps):
        flush.fill_(1.0)
        barrier()
        t0 = time.perf_counter()
        st = step_host(k)
        torch.cuda.synchronize()
        e2e_t += time.perf_counter() - t0
        e2e_states[k] = st
        sm = est.summary()
        h2d += scn.raw[k].shape[0] * 16 + (W + 1) * 28 + 4
        d2h += int(sm["linearizations"] + 2) * W * 32 * 8 + (W + 8) * 4 + 28
        k += 1
    if world > 1:
        t = torch.tensor([e2e_t], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_t = float(t.item())
    # both passes processed the same scans from the same start: their trajectories must agree
    drift = float(np.abs(st[:, :3] - final_states[:, :3]).max())

    if rank == 0:
        peak, peak_src = load_peaks()
        value = args.steps / (total_ms * 1e-3)
        asm_launches = max(1, prof["asm_launches"])
        avg_ms = prof["asm_ms"] / asm_launches
        bytes_per_launch = prof["bytes_per_feature"] * prof["asm_features"] / asm_launches
        achieved = bytes_per_launch / (avg_ms * 1e-3) / 1e9 if avg_ms > 0 else 0.0
        line = {"metric": METRIC, "value": value, "unit": "scans/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": total_ms / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                "dtype": "f32 features / f64 solve", "data": "synthetic",
                "gn_iter_ms": 1e3 * float(np.sum(solve_t)) / max(1.0, float(np.sum(iters))),
                "config": {"workload": workload, "window": W, "opt_window": W, "points_per_scan": int(scn.raw[W].shape[0]),
                           "features_per_solve": float(np.mean(feats)), "gn_iterations_per_scan": float(np.mean(iters)),
                           "l2": "flushed between timed steps (256 MB write outside the event pair)",
                           "parallelism": "frames sharded 1..O over %d rank(s)%s" % (world, ("; exchange: " + exchange["kind"]) if world > 1 else ""),
                           "e2e_vs_device_pass_max_pos_diff_m": drift,
                           "overlap_marginalization": args.overlap_marginalization,
                           "timing": "value: CUDA events around each scan (device-resident sweep); e2e: host perf_counter around the C-ABI calls; the bench host is shared, runs differ by about +-10 %; host_wall keys with the device solver: t_lin_host = host time from the start of the solve to the end of the graph launch call, t_lin_lidar = re-parameterising the asm_ppp graph nodes, t_marg_wait = joining the previous scan's marginalisation algebra (overlapped with the GPU front end)",
                           "ms_per_timed_step": [round(float(v), 3) for v in ms],
                           "host_wall_ms_per_scan": {kk: 1e3 * float(np.mean(v)) for kk, v in brk.items()}},
                "roofline": {"kernel": "asm_ppp (fused PivotPointPlane residual+Jacobian+JtJ reduction)", "bound": "hbm",
                             "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                             "traffic": asm_traffic(kind),
                             "avg_launch_us": avg_ms * 1e3, "bytes_per_launch": bytes_per_launch, "launches": prof["asm_launches"],
                             "peak_source": peak_src,
                             "note": "32 B/feature x features of the solve (3.9 MB per launch on HDL-64): launch-latency bound, ~12 us fixed cost; traffic = dram__bytes_read+write per launch from the committed ncu --set full capture of this workload (profiles/asm_ppp_traffic.json; null when there is none); the streaming rate of the same kernel is in roofline_stream"},
                "roofline_knn": {"kernel": "knn_plane (frame-batched 5-NN + plane fit, the largest share of kernel time)", "bound": "hbm",
                                 "achieved": (prof["bytes_per_query"] * prof["knn_queries"] / max(1, prof["knn_launches"])) /
                                             (max(prof["knn_ms"], 1e-9) / max(1, prof["knn_launches"]) * 1e-3) / 1e9,
                                 "peak": peak, "unit": "GB/s", "traffic": None,
                                 "avg_launch_us": 1e3 * prof["knn_ms"] / max(1, prof["knn_launches"]),
                                 "queries_per_launch": prof["knn_queries"] / max(1, prof["knn_launches"]),
                                 "note": "128 B/query algorithmic (query + 5 neighbours + feature out); an L2-gather + ALU kernel, not HBM bound"},
                "e2e": {"value": args.steps / e2e_t, "unit": "scans/s", "h2d_bytes_per_step": h2d // args.steps,
                        "d2h_bytes_per_step": d2h // args.steps},
                "gpu_launches": launches, "clocks": clocks}
        line["roofline_knn"]["frac"] = line["roofline_knn"]["achieved"] / peak
        if world == 1:
            try:   # the same kernel on a stream larger than L2 (512 MB): its HBM-resident streaming rate
                sb = estimator.asm_stream_bench(1 << 26, 10, local_rank)
                line["roofline_stream"] = {"kernel": "asm_ppp", "features": 1 << 26, "bytes_per_launch": sb["bytes"],
                                           "avg_launch_ms": sb["avg_ms"], "achieved": sb["gbs"], "peak": peak, "unit": "GB/s",
                                           "frac": sb["gbs"] / peak,
                                           "note": "the same kernel on a synthetic 67 M-feature stream (2 GB >> 50 MB L2, 8 frames, centimetre residuals like a converged window); CUDA events per launch"}
            except Exception as exc:
                line["roofline_stream"] = {"error": repr(exc)}
            try:
                ra = argparse.Namespace(warmup=1, steps=min(args.cpu_sample, n_total - W - 2))
                r = run_reference(ra, scn, W, est_cfg)
                line["cpu_baseline"] = {"value": r["scans_per_s"], "unit": "scans/s", "cores": 4, "host_cores": host_cores(), "kind": "port",
                                        "gn_iter_ms": r["gn_iter_ms"],
                                        "sample": "%d scans of the same workload through oracle/ (CPU restatement of the reference; 1 thread + 4 marginalisation threads)" % r["steps"]}
                # parity of THIS run: the oracle consumed the same scans from the same start as the e2e pass
                common = sorted(set(r["states"]) & set(e2e_states))
                perr, qerr = 0.0, 0.0
                for kk in common:
                    xo, xg = r["states"][kk], e2e_states[kk]
                    perr = max(perr, float(np.abs(xg[:, :3] - xo[:, :3]).max() / max(1.0, np.abs(xo[:, :3]).max())))
                    qerr = max(qerr, float(np.abs(xg[:, 3:7] - xo[:, 3:7]).max()))
                line["parity"] = {"max_rel_pos_err": perr, "max_quat_err": qerr, "scans": len(common), "tolerance": 1e-4,
                                  "ok": bool(common) and perr <= 1e-4 and qerr <= 1e-4,
                                  "against": "oracle/ (CPU restatement of the reference) on the same scans, window states after every scan"}
            except Exception as exc:  # the baseline leg must not take the bench line down
                line["cpu_baseline"] = {"value": None, "unit": "scans/s", "cores": 0, "kind": "port", "sample": "failed: %r" % (exc,)}
        print(json.dumps(line))
        if "parity" in line and not line["parity"]["ok"]:
            print("[bench] PARITY FAILED: %r" % (line["parity"],), file=sys.stderr)
            if world > 1:
                dist.destroy_process_group()
            return 3
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
