"""Cost of the imu_factor = 1 estimator starting itself from /compact_data messages and the IMU (Estimator.attach_imu_mapping,
process_compact_dev with stamps), with and without the extrinsic-rotation calibration of estimate_extrinsic = 2; print one JSON line.

HDL-64 drive with roll / pitch amplitude k, device stage A (less-sharp corner, less-flat surf, cloud_in_rings full cloud), the
ground-truth lidar pose relative to the first sweep as transform_sum_, 200 Hz IMU samples fed before each message.  Two shapes:
  indoor   W 12 / O 7, init_window_factor 2, enable_deskew, keep_features, prior_factor 0, estimate_extrinsic 2 with
           enable_extrinsic_calibration, the lidar mounted at rot_x(0.15) and the identity as the configured rotation.  A k = 0.25 leg
           keeps failing its calibrations (sigma_2 < 0.25); a k = 0.75 leg calibrates, starts and runs INITED.
  outdoor  W 7 / O 5, init_window_factor 1, cutoff_deskew, estimate_extrinsic 1, k = 0.25, the lidar mounted at the identity.
Per message: host time of process_compact_dev plus a device synchronise (median, p90), split into NOT_INITED pushes before the window
is full, decimated messages (Process only), full-window messages that calibrate and fail, the start-up message (calibration,
RunInitialization and the first solve) and INITED messages (the first --warmup not timed), with the estimator's kernel launches per
INITED message.  Also the host time of one lio_imu_estimate_extrinsic_rotation_host call on a W 12 window of the drive.

    python scripts/imu_startup_bench.py [--scans 20] [--warmup 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.map_builder_bench import card  # noqa: E402

T_LB = np.array([0.0, 0.0, -0.1])
NOISE = dict(acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5)


def rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def make_drive(n, k, R_lb):
    """n messages: (clouds, transform_sum7, stamp, IMU samples (dt, acc, gyr, t) since the previous message)."""
    from lio_mapping_b200 import synth
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config("hdl64")
    traj = dataclasses.replace(traj, k_roll=k, k_pitch=k)
    t = 1.0 + 0.1 * np.arange(n)
    sweeps = [synth.make_sweep(sensor, scene, traj, float(t[i]), seed=40 + i, R_lb=R_lb, t_lb=T_LB, distort=False) for i in range(n)]
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max(s.shape[0] for s in sweeps))
    p, R, _, _, _ = traj.state(t)
    Tlb = np.eye(4); Tlb[:3, :3] = R_lb; Tlb[:3, 3] = T_LB
    T_l = []
    for i in range(n):
        Tb = np.eye(4); Tb[:3, :3] = R[i]; Tb[:3, 3] = p[i]
        T_l.append(Tb @ np.linalg.inv(Tlb))
    msgs = []
    for i in range(n):
        pp.SetInputCloud(sweeps[i]); pp.Process()
        clouds = [np.ascontiguousarray(pp.cloud(c), np.float32) for c in ("corner_points_less_sharp", "surface_points_less_flat", "cloud_in_rings")]
        T = np.linalg.inv(T_l[0]) @ T_l[i]
        sum7 = np.array([*synth.rot_to_quat(T[:3, :3]), *T[:3, 3]], np.float32)
        samples = []
        if i > 0:
            tt, acc, gyr = synth.make_imu(traj, float(t[i - 1]), float(t[i]), 200.0)
            last = t[i - 1]
            for j in range(len(tt)):
                samples.append((tt[j] - last, acc[j], gyr[j], tt[j]))
                last = tt[j]
        msgs.append((clouds, sum7, float(t[i]), samples))
    return msgs


def run_leg(msgs, W, O, f, warmup, calib, **cfg):
    import torch
    from lio_mapping_b200 import estimator
    from lio_mapping_b200.point_mapping import PointMapping
    max_full = max(m[0][2].shape[0] for m in msgs)
    e = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 16, max_scan_points=1 << 18, imu_factor=1,
                            init_window_factor=f, **NOISE, **cfg)
    e.set_extrinsic(np.r_[0.0, 0.0, 0.0, 1.0, T_LB].astype(np.float32))
    e.enable_local_clouds(0.2, 1 << 16, max_full)
    pm = PointMapping(max_points=1 << 18)
    pm.EnablePublish(0.6, max_full)
    if calib:
        e.enable_extrinsic_calibration()
    e.attach_imu_mapping(pm)
    t = {k: [] for k in ("not_inited_push", "decimated", "calib_failed", "startup", "inited")}
    launches, inited_seen = [], 0
    for clouds, sum7, stamp, samples in msgs:
        for dt, a, g, ts in samples:
            e.process_imu(dt, a, g, ts)
        dev = [torch.from_numpy(c).cuda() for c in clouds]
        nd = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        was_inited = e.compact_status()["inited"]
        t0 = time.perf_counter()
        st = e.process_compact_dev([d.data_ptr() for d in dev], nd.data_ptr(), [c.shape[0] for c in clouds], sum7, stamp=stamp)
        torch.cuda.synchronize()
        dt_ms = (time.perf_counter() - t0) * 1e3
        calibrated = calib and e.extrinsic_calib_status()["ran"]
        if was_inited:
            inited_seen += 1
            if inited_seen > warmup:
                t["inited"].append(dt_ms)
                launches.append(e.summary()["launches"])
        elif st["inited"]:
            t["startup"].append(dt_ms)
        elif calibrated:
            t["calib_failed"].append(dt_ms)
        elif st["pushed"]:
            t["not_inited_push"].append(dt_ms)
        else:
            t["decimated"].append(dt_ms)
    e.close(); pm.close()
    return t, launches


def stats(v):
    return dict(median=float(np.median(v)), p90=float(np.percentile(v, 90)), n=len(v)) if v else None


def calib_call_us(msgs, W, f, reps=2000):
    """Host time of one lio_imu_estimate_extrinsic_rotation_host call (through ctypes) on W + 1 pushes f messages apart."""
    from lio_mapping_b200 import estimator
    pushes = list(range(f - 1, f * (W + 1), f))
    tf = np.array([msgs[i][1] for i in pushes])
    pims = [estimator.Pim(np.zeros(3), np.zeros(3), np.zeros(3), np.zeros(3), **NOISE)]
    for a, b in zip(pushes[:-1], pushes[1:]):
        first = msgs[a][3][-1]
        p = estimator.Pim(first[1], first[2], np.zeros(3), np.zeros(3), **NOISE)
        for i in range(a + 1, b + 1):
            for dt, acc, gyr, _ in msgs[i][3]:
                p.push_back(dt, acc, gyr)
        pims.append(p)
    tlb = np.r_[0.0, 0.0, 0.0, 1.0, T_LB].astype(np.float32)
    out = []
    for _ in range(5):
        t0 = time.perf_counter()
        for _ in range(reps):
            estimator.estimate_extrinsic_rotation(tf, pims, tlb)
        out.append((time.perf_counter() - t0) / reps * 1e6)
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("imu_startup_bench: no CUDA device")
    name, power = card()
    indoor = dict(enable_deskew=1, cutoff_deskew=0, keep_features=1, prior_factor=0, estimate_extrinsic=2, opt_extrinsic=1)
    W, O, f = 12, 7, 2
    fail = make_drive(f * (W + 1) + 2 * a.scans, 0.25, rot_x(0.15))
    t_fail, _ = run_leg(fail, W, O, f, a.warmup, True, **indoor)
    ok = make_drive(f * (W + 1) + a.warmup + a.scans, 0.75, rot_x(0.15))
    t_ok, l_ok = run_leg(ok, W, O, f, a.warmup, True, **indoor)
    merged = {k: t_fail[k] + t_ok[k] for k in t_ok}
    shapes = [dict(shape="indoor", W=W, O=O, init_window_factor=f, **{f"ms_{k}": stats(v) for k, v in merged.items()},
                   launches_per_inited=float(np.median(l_ok)), calib_call_us=calib_call_us(ok, W, f))]
    W, O, f = 7, 5, 1
    out = make_drive(f * (W + 1) + a.warmup + a.scans, 0.25, np.eye(3))
    t_out, l_out = run_leg(out, W, O, f, a.warmup, False, enable_deskew=0, cutoff_deskew=1, estimate_extrinsic=1, opt_extrinsic=0)
    shapes.append(dict(shape="outdoor", W=W, O=O, init_window_factor=f, **{f"ms_{k}": stats(v) for k, v in t_out.items()},
                       launches_per_inited=float(np.median(l_out))))
    res = dict(bench="imu_startup", gpu=name, power_limit=power, shapes=shapes)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
