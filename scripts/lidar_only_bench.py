"""Cost of the device estimator with imu_factor = 0 fed the odometry's clouds (lio_est_attach_mapping / lio_est_process_compact_*);
print one JSON line.

HDL-64 drive, device stage A (less-sharp corner, less-flat surf, cloud_in_rings full cloud, the clouds /compact_data carries), the
ground-truth lidar pose relative to the first sweep as transform_sum_, init_window_factor 2, windows 10 / 10 and 7 / 5.  Per message:
host time of process_compact_dev plus a device synchronise, split into NOT_INITED pushes, decimated NOT_INITED messages (Process
only) and INITED messages; the first --warmup INITED messages are not timed.  For INITED messages also the estimator's kernel
launches (summary "launches", the scan's own launches without the mapping's) and its front-end / solve / marginalisation host times.

    python scripts/lidar_only_bench.py [--scans 30] [--warmup 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.map_builder_bench import card  # noqa: E402


def run_shape(W, O, f, scans, warmup):
    import torch
    from lio_mapping_b200 import estimator, synth
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_processor import PointProcessor
    n = f * (W + 1) + warmup + scans
    sensor, scene, traj = synth.default_config("hdl64")
    sweeps = [synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * k, seed=40 + k, distort=False) for k in range(n)]
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max(s.shape[0] for s in sweeps))
    p, R, _, _, _ = traj.state(1.0 + 0.1 * np.arange(n))
    tlb = np.array([0, 0, 0, 1, 0, 0, -0.1], np.float32)
    msgs = []
    for k in range(n):
        pp.SetInputCloud(sweeps[k]); pp.Process()
        clouds = [np.ascontiguousarray(pp.cloud(c), np.float32) for c in ("corner_points_less_sharp", "surface_points_less_flat", "cloud_in_rings")]
        sum7 = np.array([*synth.rot_to_quat(R[0].T @ R[k]), *(R[0].T @ (p[k] - p[0]))], np.float32)
        msgs.append((clouds, sum7))
    max_full = max(m[0][2].shape[0] for m in msgs)
    e = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 16, max_scan_points=1 << 18, imu_factor=0,
                            init_window_factor=f, opt_extrinsic=0, enable_deskew=0, cutoff_deskew=0)
    e.set_extrinsic(tlb)
    e.enable_local_clouds(0.2, 1 << 16, max_full)
    pm = PointMapping(max_points=1 << 18)
    pm.EnablePublish(0.6, max_full)
    e.attach_mapping(pm)
    t = {"not_inited_push": [], "decimated": [], "inited": []}
    launches, t_build, t_solve, t_marg = [], [], [], []
    inited_seen = 0
    for clouds, sum7 in msgs:
        dev = [torch.from_numpy(c).cuda() for c in clouds]
        nd = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        was_inited = e.compact_status()["inited"]   # the state the last call left
        t0 = time.perf_counter()
        st = e.process_compact_dev([d.data_ptr() for d in dev], nd.data_ptr(), [c.shape[0] for c in clouds], sum7)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) * 1e3
        if was_inited:
            inited_seen += 1
            if inited_seen > warmup:
                t["inited"].append(dt)
                s = e.summary()
                launches.append(s["launches"]); t_build.append(s["t_build_map"] + s["t_features"]); t_solve.append(s["t_solve"]); t_marg.append(s["t_marg"])
        elif st["pushed"]:
            t["not_inited_push"].append(dt)
        else:
            t["decimated"].append(dt)
    med = lambda v: float(np.median(v)) if v else None
    e.close(); pm.close()
    return dict(W=W, O=O, init_window_factor=f, ms_not_inited_push=med(t["not_inited_push"]), ms_decimated=med(t["decimated"]),
                ms_inited=med(t["inited"]), ms_inited_p90=float(np.percentile(t["inited"], 90)), inited_timed=len(t["inited"]),
                est_launches_per_inited=med(launches), ms_front_end=med(t_build) * 1e3, ms_solve=med(t_solve) * 1e3, ms_marg=med(t_marg) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lidar_only_bench: no CUDA device")
    name, power = card()
    res = dict(bench="lidar_only", gpu=name, power_limit=power,
               shapes=[run_shape(10, 10, 2, a.scans, a.warmup), run_shape(7, 5, 2, a.scans, a.warmup)])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
