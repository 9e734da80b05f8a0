"""Time the map builder inside lio_node (lio_node_enable_map_builder, map_4D*.launch's map_builder_node) on HDL-64 drives in the
outdoor_64 and indoor shapes of tests/test_lio_node_gpu.py; print one JSON line.

Legs, on fresh nodes, alternated `--rounds` times after one warm-up round:
  plain      the node as test_*.launch runs it
  map        the node with enable_map_builder() (map_4D*.launch defaults)
  map_drive  the same plus a leaf-0.2 drive map (RegisteredMap) attached to the map builder's /cloud_registered

Each sweep is timed with a host clock from push_sweep_dev to the end of the IMU messages up to the next sweep, closed by a device
synchronise.  The sweeps that processed a message that reached the estimator INITED (the map builder's calls) give `ms per INITED message`.
The map builder call alone is timed inside the node: the difference of the map and plain legs per INITED message is reported beside a
direct timing of the same calls on a hand-driven MapBuilder fed with the same inputs (ProcessMapDev, host clock + synchronise).  Launches
and host waits per INITED message come from one extra round of each leg under torch.profiler (CUDA runtime calls: kernel launches and
memory operations; stream, event and device synchronisations and synchronous copies as waits).  identical_states: every leg of every
round ends in bit-identical estimator states.

    python scripts/lio_node_map_bench.py [--rounds 2] [--out FILE]
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

COMMON = dict(acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5, g_norm=9.805, min_match_sq_dis=1.0, min_plane_dis=0.2, surf_filter_size=0.4,
              max_frame_points=1 << 15, max_scan_points=1 << 17, max_points=1 << 18, max_feature_points=1 << 16, sensor_type=64)
# (sweeps, roll / pitch amplitude, lidar mounting roll, node configuration); the indoor drive is the calibration drive of the tests
SHAPES = {
    "outdoor_64": (66, 0.25, 0.0, dict(odom_io=3, msg_time_delay=0.0, window_size=7, opt_window_size=5, init_window_factor=1, enable_deskew=0,
                                       cutoff_deskew=1, prior_factor=1, imu_factor=1, estimate_extrinsic=1, opt_extrinsic=0, keep_features=0)),
    "indoor": (96, 0.75, 0.15, dict(odom_io=2, msg_time_delay=0.05, window_size=12, opt_window_size=7, init_window_factor=2, enable_deskew=1,
                                    cutoff_deskew=0, prior_factor=0, imu_factor=1, estimate_extrinsic=2, opt_extrinsic=1, keep_features=1)),
}
WAITS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize", "cudaMemcpy", "cudaMemcpy2D")
LAUNCHES = ("cudaLaunchKernel", "cudaLaunchKernelExC", "cudaMemcpyAsync", "cudaMemsetAsync", "cudaMemset", "cudaMemcpy")


def make_drive(n, k, roll):
    """n motion-distorted HDL-64 sweeps at 10 Hz and the 200 Hz IMU (gyro bias added) between them."""
    from lio_mapping_b200 import synth
    sensor, scene, traj = synth.default_config("hdl64")
    traj = dataclasses.replace(traj, k_roll=k, k_pitch=k)
    c, s = np.cos(roll), np.sin(roll)
    R_lb = np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    t_lb = np.array([0.0, 0.0, -0.1])
    t = 1.0 + 0.1 * np.arange(n)
    raw = [synth.make_sweep(sensor, scene, traj, float(tk), seed=300 + i, R_lb=R_lb, t_lb=t_lb, distort=True) for i, tk in enumerate(t)]
    it, acc, gyr = synth.make_imu(traj, 0.9, float(t[-1]) + 0.2, 200.0)
    gyr = gyr + np.array([0.02, -0.03, 0.025])
    spans = []
    for j in range(n):
        hi = t[j + 1] if j + 1 < n else np.inf
        sel = (it > t[j]) & (it <= hi)
        spans.append((it[sel], acc[sel], gyr[sel]))
    first = it <= t[0]
    return t, raw, (it[first], acc[first], gyr[first]), spans, np.r_[0.0, 0.0, 0.0, 1.0, t_lb].astype(np.float32)


def run_leg(leg, shape, drive, dev, profile=False):
    import torch
    from lio_mapping_b200 import LioNode
    from lio_mapping_b200.registered_map import RegisteredMap
    t, raw, imu0, spans, tf = drive
    node = LioNode(tf_lb7=tf, **COMMON, **SHAPES[shape][3])
    rm = None
    if leg != "plain":
        node.enable_map_builder()
    if leg == "map_drive":
        rm = RegisteredMap(leaf=0.2, capacity=1 << 22)
        node.attach_registered_map(rm, "map_builder")
    node.push_imu_batch(*imu0)
    times, inited = [], []
    prof = None
    if profile:
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA])
        prof.__enter__()
    for j in range(len(t)):
        before = node.status()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        node.push_sweep_dev(dev[j].data_ptr(), dev[j].shape[0], float(t[j]))
        node.push_imu_batch(*spans[j])
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        s = node.status()
        inited.append(s["processed"] > before["processed"] and before["inited"])
    counts = None
    if prof is not None:
        prof.__exit__(None, None, None)
        names = [e.name for e in prof.events()]
        counts = dict(launches=sum(names.count(n) for n in LAUNCHES), waits=sum(names.count(n) for n in WAITS))
    out = dict(times=times, inited=inited, states=node.states(), counts=counts)
    if leg != "plain":
        p = node.map_builder_poses()
        out["calls"] = len(p["stamp"])
        out["surround"] = int(p["surround_published"].sum())
    if rm is not None:
        out["drive_map_voxels"] = rm.stats()["size"]
    return out


def map_builder_alone(shape, drive, dev):
    """The same map builder calls on a hand-driven MapBuilder: the node's /local/* clouds and /local_laser_odom, timed per call."""
    import torch
    from lio_mapping_b200 import LioNode
    from lio_mapping_b200.map_builder import MapBuilder
    t, raw, imu0, spans, tf = drive
    node = LioNode(tf_lb7=tf, **COMMON, **SHAPES[shape][3])
    e = node.estimator
    _, _, n_max = e.local_clouds_dev()
    mb = MapBuilder(max_points=int(max(n_max[0], n_max[1])), max_full_points=int(n_max[2]))
    node.push_imu_batch(*imu0)
    out = []
    for j in range(len(t)):
        before = node.status()
        node.push_sweep_dev(dev[j].data_ptr(), dev[j].shape[0], float(t[j]))
        node.push_imu_batch(*spans[j])
        s = node.status()
        if s["processed"] > before["processed"] and before["inited"]:
            ptrs, n_dev, nm = e.local_clouds_dev()
            odom = e.local_laser_odom()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mb.ProcessMapDev(ptrs, n_dev, nm, odom)
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lio_node_map_bench: no CUDA device")
    name, power = card()
    res = dict(metric="lio_node_map_builder_ms_per_inited_message", gpu=name, power_limit=power, rounds=a.rounds)
    same = True
    for shape, (n, k, roll, _) in SHAPES.items():
        drive = make_drive(n, k, roll)
        dev = [torch.from_numpy(np.ascontiguousarray(r, np.float32)).cuda() for r in drive[1]]
        legs = ("plain", "map", "map_drive")
        for leg in legs:                 # warm-up round
            run_leg(leg, shape, drive, dev)
        runs = {leg: [] for leg in legs}
        ref = None
        for _ in range(a.rounds):
            for leg in legs:
                r = run_leg(leg, shape, drive, dev)
                runs[leg].append(r)
                ref = r["states"] if ref is None else ref
                same = same and np.array_equal(ref, r["states"])
        for leg in legs:
            v = [x for r in runs[leg] for x, i in zip(r["times"], r["inited"]) if i]
            res[f"{shape}_{leg}_ms_median"] = round(float(np.median(v)), 3)
            res[f"{shape}_{leg}_ms_p90"] = round(float(np.percentile(v, 90)), 3)
            prof = run_leg(leg, shape, drive, dev, profile=True)
            m = sum(prof["inited"])
            if prof["counts"] is not None and m:
                res[f"{shape}_{leg}_launches_per_inited_message"] = round(prof["counts"]["launches"] / m, 1)
                res[f"{shape}_{leg}_waits_per_inited_message"] = round(prof["counts"]["waits"] / m, 1)
        res[f"{shape}_inited_messages"] = sum(runs["plain"][0]["inited"])
        res[f"{shape}_map_builder_calls"] = runs["map"][0]["calls"]
        res[f"{shape}_surround_publications"] = runs["map"][0]["surround"]
        res[f"{shape}_drive_map_voxels"] = runs["map_drive"][0]["drive_map_voxels"]
        res[f"{shape}_map_minus_plain_ms_median"] = round(res[f"{shape}_map_ms_median"] - res[f"{shape}_plain_ms_median"], 3)
        alone = map_builder_alone(shape, drive, dev)
        res[f"{shape}_map_builder_call_ms_median"] = round(float(np.median(alone)), 3)
        res[f"{shape}_map_builder_call_ms_p90"] = round(float(np.percentile(alone, 90)), 3)
    res["identical_states"] = bool(same)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
