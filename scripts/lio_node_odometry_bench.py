"""What the node's odometry topics (lio_node_enable_odometry) cost: the outdoor_64 drive of tests/test_lio_node_gpu.py with the topics off
and on; print one JSON line.

Legs, on fresh nodes, alternated `--rounds` times after one warm-up round:
  off   the node as test_outdoor_64.launch runs it
  on    the same with enable_odometry() (default capacity), nothing taken during the drive

Each sweep is timed with a host clock from push_sweep_dev to the end of the IMU messages up to the next sweep, closed by a device
synchronise (`ms per sweep`, median and p90 over every sweep of every round).  CUDA runtime calls per sweep come from one extra run of
each leg under torch.profiler (kernel launches and memory operations; stream, event and device synchronisations and synchronous copies
as waits): recording reads host state only, so the two legs must make the same calls.  After each on leg: the rows per topic, and the
host time of taking the whole drive's rows, every topic once through LioNode.take_odometry.  identical_states: every leg of every round
ends in bit-identical estimator states.

    python scripts/lio_node_odometry_bench.py [--rounds 2] [--out FILE]
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

from scripts.lio_node_map_bench import COMMON, LAUNCHES, SHAPES, WAITS, make_drive  # noqa: E402
from scripts.map_builder_bench import card  # noqa: E402

SHAPE = "outdoor_64"


def run_leg(leg, drive, dev, profile=False):
    import torch
    from lio_mapping_b200 import TOPICS, LioNode
    t, raw, imu0, spans, tf = drive
    node = LioNode(tf_lb7=tf, **COMMON, **SHAPES[SHAPE][3])
    if leg == "on":
        node.enable_odometry()
    node.push_imu_batch(*imu0)
    times = []
    prof = None
    if profile:
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA])
        prof.__enter__()
    for j in range(len(t)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        node.push_sweep_dev(dev[j].data_ptr(), dev[j].shape[0], float(t[j]))
        node.push_imu_batch(*spans[j])
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    counts = None
    if prof is not None:
        prof.__exit__(None, None, None)
        names = [e.name for e in prof.events()]
        counts = dict(launches=sum(names.count(n) for n in LAUNCHES), waits=sum(names.count(n) for n in WAITS))
    out = dict(times=times, states=node.states(), counts=counts)
    if leg == "on":
        t0 = time.perf_counter()
        taken = {name: node.take_odometry(name) for name in TOPICS}
        out["take_us"] = (time.perf_counter() - t0) * 1e6
        out["rows"] = {name: int(v["stamp"].shape[0]) for name, v in taken.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lio_node_odometry_bench: no CUDA device")
    name, power = card()
    n, k, roll, _ = SHAPES[SHAPE]
    drive = make_drive(n, k, roll)
    dev = [torch.from_numpy(np.ascontiguousarray(r, np.float32)).cuda() for r in drive[1]]
    legs = ("off", "on")
    for leg in legs:                     # warm-up round
        run_leg(leg, drive, dev)
    runs = {leg: [] for leg in legs}
    ref, same = None, True
    for _ in range(a.rounds):
        for leg in legs:
            r = run_leg(leg, drive, dev)
            runs[leg].append(r)
            ref = r["states"] if ref is None else ref
            same = same and np.array_equal(ref, r["states"])
    res = dict(metric="lio_node_odometry_ms_per_sweep", shape=SHAPE, sweeps=n, gpu=name, power_limit=power, rounds=a.rounds)
    for leg in legs:
        v = [x for r in runs[leg] for x in r["times"]]
        res[f"{leg}_ms_median"] = round(float(np.median(v)), 3)
        res[f"{leg}_ms_p90"] = round(float(np.percentile(v, 90)), 3)
    res["on_minus_off_ms_median"] = round(res["on_ms_median"] - res["off_ms_median"], 3)
    for leg in legs:
        prof = run_leg(leg, drive, dev, profile=True)
        res[f"{leg}_runtime_calls_per_sweep"] = round(prof["counts"]["launches"] / n, 2)
        res[f"{leg}_waits_per_sweep"] = round(prof["counts"]["waits"] / n, 2)
    res["same_runtime_calls"] = (res["on_runtime_calls_per_sweep"] == res["off_runtime_calls_per_sweep"]
                                 and res["on_waits_per_sweep"] == res["off_waits_per_sweep"])
    res["rows"] = runs["on"][0]["rows"]
    res["take_whole_drive_us"] = [round(r["take_us"], 1) for r in runs["on"]]
    res["identical_states"] = bool(same)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
