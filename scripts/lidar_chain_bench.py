"""Time the reference's lidar-only pipeline lio_processor_node -> lio_odometry_node -> lio_mapping_node (16_scans_test.launch,
64_scans_test.launch) over a motion-distorted HDL-64 drive with io_ratio 2 (the indoor config's odom_io); print one JSON line.

  device   PointProcessor.process_device -> PointOdometry.ProcessDev -> (io_ratio gate) PointOdometry.clouds_dev ->
           PointMapping.ProcessDev with EnablePublish (surround map, registered cloud), all on one stream: no cloud crosses the PCIe
           bus (only the raw sweep is resident in HBM beforehand, like a driver's DMA target)
  host     the same device stage A, then the chain through host copies: stage-A downloads, PointOdometry.Process, compact_data,
           wire.compact_decode and PointMapping.Process (the host entry, which does not publish)

Each leg runs fresh odometry and mapping contexts on the same sweeps; per sweep a host clock spans the leg's calls and a device
synchronise.  The script also checks that both chains produced identical mapped poses.

    python scripts/lidar_chain_bench.py [--sweeps 30] [--warmup 6] [--out FILE]
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

STAGE_A = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--io-ratio", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lidar_chain_bench: no CUDA device")
    from lio_mapping_b200 import synth, wire
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config("hdl64")
    n_total = a.warmup + a.sweeps
    raw = [np.ascontiguousarray(synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * f, seed=70 + f, distort=True), np.float32)
           for f in range(n_total)]
    max_raw = max(r.shape[0] for r in raw)
    dev_raw = [torch.from_numpy(r).cuda() for r in raw]
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_raw)
    n_dev = [pp.cloud_count_dev(name) for name in STAGE_A]
    n_max = [1 << 17] * 4 + [max_raw]

    def run(leg):
        od = PointOdometry(0.1, a.io_ratio, 25, max_full_points=max_raw)
        pm = PointMapping(max_points=1 << 17)
        if leg == "device":
            pm.EnablePublish(0.6, max_raw)
        times, poses, mapped = [], [], 0
        for f in range(n_total):
            t = dev_raw[f]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pp.process_device(t.data_ptr(), t.shape[0])
            tobe = None
            if leg == "device":
                ts, _, info = od.ProcessDev([pp.cloud_dev(name) for name in STAGE_A], n_dev, n_max)
                if info["published"]:
                    ptrs, cn_dev, cn = od.clouds_dev()
                    tobe, _, _ = pm.ProcessDev(ptrs, cn_dev, cn, ts)
            else:
                ts, _, info = od.Process(*[pp.cloud(name) for name in STAGE_A])
                if info["published"]:
                    tf7, c, s, _ = wire.compact_decode(od.compact_data())
                    tobe, _ = pm.Process(c, s, tf7)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if f >= a.warmup:
                times.append((t1 - t0) * 1e3)
            if tobe is not None:
                poses.append(tobe)
                mapped += f >= a.warmup
        od.close(); pm.close()
        return times, poses, mapped

    res_legs = {leg: run(leg) for leg in ("device", "host")}
    name, power = card()
    med = {leg: round(float(np.median(v[0])), 3) for leg, v in res_legs.items()}
    dp, hp = res_legs["device"][1], res_legs["host"][1]
    same = len(dp) == len(hp) and all(np.array_equal(x, y) for x, y in zip(dp, hp))
    res = dict(metric="lidar_chain_ms_per_sweep", kind="hdl64", io_ratio=a.io_ratio, sweeps=a.sweeps, warmup=a.warmup,
               mapped_sweeps=res_legs["device"][2], gpu=name, power_limit=power, chain_device_resident_ms_median=med["device"],
               chain_host_copies_ms_median=med["host"], identical_mapped_poses=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
