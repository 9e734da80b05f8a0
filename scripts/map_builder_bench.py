"""Time lio::MapBuilder::ProcessMap (lio_mb_process_map_host) over an HDL-64 drive on the GPU and the oracle's CPU restatement
on the same frames; print one JSON line.

Frames are split by what ProcessMap does on them: the skip_count gate's two branches (OptimizeMap or Transform4DUpdate) and
whether PublishMapBuilderResults builds the surround map.  The first frame (empty map, first allocations) is reported apart.
The GPU time is a host clock around ProcessMap followed by a device synchronise.

    python scripts/map_builder_bench.py [--frames 31] [--kind hdl64] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def drive(kind, n, seed0=40):
    """Stage A on the GPU for n sweeps of the synthetic drive; the odometry is the ground-truth pose relative to frame 0."""
    from lio_mapping_b200 import ops, synth
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config(kind)
    sweeps = [synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * f, seed=seed0 + f, distort=False) for f in range(n)]
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max(s.shape[0] for s in sweeps))
    p, R, _, _, _ = traj.state(1.0 + 0.1 * np.arange(n))
    frames = []
    for f in range(n):
        pp.SetInputCloud(sweeps[f]); pp.Process()
        Rr = R[0].T @ R[f]
        t = R[0].T @ (p[f] - p[0])
        q = synth.rot_to_quat(Rr)
        frames.append((ops.voxel_grid(pp.cloud("corner_points_less_sharp"), 0.2), ops.voxel_grid(pp.cloud("surface_points_less_flat"), 0.4),
                       pp.cloud("cloud_in_rings"), np.array([*q, *t], np.float32)))
    return frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=31)
    ap.add_argument("--kind", default="hdl64")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("map_builder_bench: no CUDA device")
    from lio_mapping_b200.map_builder import MapBuilder
    from oracle import map_builder_py, oracle_py
    oracle_py.build()
    frames = drive(a.kind, a.frames)
    max_full = max(f[2].shape[0] for f in frames)
    warm = MapBuilder(max_points=1 << 17, max_full_points=max_full)       # module load, first allocations
    for c, s, full, tf in frames[:6]:
        warm.ProcessMap(c, s, full, tf)
    warm.close()
    torch.cuda.synchronize()
    mg = MapBuilder(max_points=1 << 17, max_full_points=max_full)
    mo = map_builder_py.MapBuilderOracle()
    rows = []
    for c, s, full, tf in frames:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, ig = mg.ProcessMap(c, s, full, tf)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        _, io = mo.process_map(c, s, full, tf)
        t2 = time.perf_counter()
        rows.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3, ig["optimised"], ig["surround_published"], ig["iterations"], io["iterations"]))

    def stats(sel):
        g = [r[0] for r in sel]; o = [r[1] for r in sel]
        if not g:
            return None
        return dict(frames=len(g), gpu_ms_median=round(float(np.median(g)), 3), gpu_ms_mean=round(float(np.mean(g)), 3),
                    oracle_cpu_ms_median=round(float(np.median(o)), 3), iterations_mean=round(float(np.mean([r[4] for r in sel])), 2))
    steady = rows[1:]
    name, power = card()
    res = dict(metric="map_builder_process_map_ms", kind=a.kind, frames=len(rows), gpu=name, power_limit=power,
               mean_points=dict(corner=int(np.mean([f[0].shape[0] for f in frames])), surf=int(np.mean([f[1].shape[0] for f in frames])),
                                full=int(np.mean([f[2].shape[0] for f in frames]))),
               first_frame=dict(gpu_ms=round(rows[0][0], 3), oracle_cpu_ms=round(rows[0][1], 3)),
               all=stats(steady),
               optimised=stats([r for r in steady if r[2]]), skipped=stats([r for r in steady if not r[2]]),
               publishing=stats([r for r in steady if r[3]]), not_publishing=stats([r for r in steady if not r[3]]))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
