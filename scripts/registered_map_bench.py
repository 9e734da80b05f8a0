"""Time the map of a whole drive (RegisteredMap, csrc/regmap.cu) fed from the device lidar chain; print one JSON line.

The chain is stage A -> PointOdometry -> publishing PointMapping over a motion-distorted synthetic HDL-64 drive, all on one stream,
with io_ratio 1 so that every sweep is mapped.  Four legs run it with fresh odometry and mapping contexts on the same sweeps:

  none    the chain alone
  raw     + RegisteredMap(leaf 0).insert_dev(registered_full_cloud_dev()) after every mapped sweep (save_bag_to_pcd.cc's map)
  voxel   the same with leaf 0.2
  host    + registered_full_cloud() (lio_mb_full_download) and a host-side list of the clouds, concatenated at the end

A leg's ms per sweep is a host clock around the sweep's calls and a device synchronise.  The insert alone is timed by CUDA events
around insert_dev on the chain's stream.  The legs run twice, in the order none, raw, voxel, host and then reversed; medians and
p90 are over both rounds.  Then export_dev (with its synchronise) and write_pcd (to a temporary directory) of both final maps.

    python scripts/registered_map_bench.py [--sweeps 110] [--warmup 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.map_builder_bench import card  # noqa: E402

STAGE_A = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")
LEGS = ("none", "raw", "voxel", "host")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=110)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("registered_map_bench: no CUDA device")
    from lio_mapping_b200 import synth
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from lio_mapping_b200.point_processor import PointProcessor
    from lio_mapping_b200.registered_map import RegisteredMap
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
        od = PointOdometry(0.1, 1, 25, max_full_points=max_raw)
        pm = PointMapping(max_points=1 << 17)
        pm.EnablePublish(0.6, max_raw)
        rm = None
        if leg == "raw":
            rm = RegisteredMap(0.0, n_total * max_raw)
        elif leg == "voxel":
            rm = RegisteredMap(a.leaf, 1 << 24)
        host = []
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sweep_ms, insert_ms, launches = [], [], set()
        for f in range(n_total):
            t = dev_raw[f]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pp.process_device(t.data_ptr(), t.shape[0])
            ts, _, info = od.ProcessDev([pp.cloud_dev(name) for name in STAGE_A], n_dev, n_max)
            timed = False
            if info["published"]:
                ptrs, cn_dev, cn = od.clouds_dev()
                pm.ProcessDev(ptrs, cn_dev, cn, ts)
                if rm is not None:
                    ev0.record()
                    rm.insert_dev(*pm.registered_full_cloud_dev())
                    ev1.record()
                    timed = True
                elif leg == "host":
                    host.append(pm.registered_full_cloud())
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if f >= a.warmup:
                sweep_ms.append((t1 - t0) * 1e3)
                if timed:
                    insert_ms.append(ev0.elapsed_time(ev1))
        res = dict(sweep_ms=sweep_ms, insert_ms=insert_ms)
        if rm is not None:
            s = rm.stats()
            res.update(size=s["size"], launches=s["launches"], waits=s["waits"] - 1, accepted=s["accepted"])
            exp, pcd = [], []
            for _ in range(5):
                t0 = time.perf_counter(); rm.export_dev(); torch.cuda.synchronize(); exp.append((time.perf_counter() - t0) * 1e3)
            tmp = tempfile.mkdtemp()
            try:
                for _ in range(3):
                    t0 = time.perf_counter(); rm.write_pcd(os.path.join(tmp, "map.pcd")); pcd.append((time.perf_counter() - t0) * 1e3)
            finally:
                shutil.rmtree(tmp)
            res.update(export_ms=float(np.median(exp)), write_pcd_ms=float(np.median(pcd)))
            rm.close()
        if leg == "host":
            t0 = time.perf_counter()
            m = np.concatenate(host)
            res.update(concat_ms=(time.perf_counter() - t0) * 1e3, size=int(m.shape[0]))
        od.close(); pm.close()
        return res

    rounds = [{leg: run(leg) for leg in order} for order in (LEGS, LEGS[::-1])]
    name, power = card()

    def pooled(leg, key):
        return np.concatenate([np.asarray(r[leg][key], np.float64) for r in rounds])

    def q(x, p):
        return round(float(np.percentile(x, p)), 4)

    res = dict(metric="registered_map_ms", kind="hdl64", sweeps=a.sweeps, warmup=a.warmup, rounds=len(rounds), leaf=a.leaf,
               gpu=name, power_limit=power)
    for leg in LEGS:
        res[f"chain_{leg}_ms_per_sweep_median"] = q(pooled(leg, "sweep_ms"), 50)
    for leg in ("raw", "voxel"):
        ins = pooled(leg, "insert_ms")
        last = rounds[-1][leg]
        res.update({f"insert_{leg}_ms_median": q(ins, 50), f"insert_{leg}_ms_p90": q(ins, 90), f"inserts_{leg}_timed": int(ins.size),
                    f"launches_per_insert_{leg}": last["launches"], f"insert_host_waits_{leg}": last["waits"],
                    f"map_size_{leg}": last["size"], f"export_{leg}_ms": round(last["export_ms"], 3),
                    f"write_pcd_{leg}_ms": round(last["write_pcd_ms"], 3)})
    res["map_points_accepted_voxel"] = rounds[-1]["voxel"]["accepted"]
    res["host_concat_ms"] = round(rounds[-1]["host"]["concat_ms"], 3)
    res["same_size_raw_host"] = rounds[-1]["raw"]["size"] == rounds[-1]["host"]["size"]
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
