"""Time the reference's steady-state chain stage A -> estimator -> map builder (lio_map_builder_node fed by the estimator's /local/*
clouds and /local_laser_odom, launch/map_4D.launch) over an HDL-64 drive, window 10/10; print one JSON line.

  device   PointProcessor.process_device -> Estimator.set_scan_clouds_dev + process_scan_dev -> MapBuilder.ProcessMapDev, all on one
           stream: no cloud crosses the PCIe bus (only the raw sweep is resident in HBM beforehand, like a driver's DMA target)
  host     the same chain through host copies: stage-A downloads, set_scan_clouds (host), process_scan (host), local_clouds()
           download and ProcessMap (host)
  est_on / est_off   the estimator alone (device-resident input) with local clouds on and off

Each leg runs a fresh estimator and map builder on the same scans; per scan a host clock spans the leg's calls and a device
synchronise.  The script also checks that both chains produced identical map-builder poses.

    python scripts/lio_chain_bench.py [--scans 30] [--warmup 5] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lio_chain_bench: no CUDA device")
    from lio_mapping_b200 import estimator, ops, scenario
    from lio_mapping_b200.map_builder import MapBuilder
    from lio_mapping_b200.point_processor import PointProcessor
    W = O = scenario.WINDOWS["hdl64"]
    n_total = W + a.warmup + a.scans + 1
    scn = scenario.Scenario("hdl64", n_total=n_total)
    sensor = scn.sensor
    max_raw = max(s.shape[0] for s in scn.raw)
    cfg = dict(scenario.EST_CFG["hdl64"])
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_raw)
    names = {1: "cloud_in_rings", 3: "corner_points_less_sharp", 5: "surface_points_less_flat"}
    ptr = {w: pp.cloud_dev(name) for w, name in names.items()}
    cnt = {w: pp.cloud_count_dev(name) for w, name in names.items()}
    warm = []
    for k in range(W):   # warm-start clouds: frame k's down-sampled surf / corner and its full cloud
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        warm.append((ops.voxel_grid(pp.cloud("surface_points_less_flat"), 0.4), ops.voxel_grid(pp.cloud("corner_points_less_sharp"), 0.2),
                     pp.cloud("cloud_in_rings")))
    dev_raw = {k: torch.from_numpy(np.ascontiguousarray(scn.raw[k], np.float32)).cuda() for k in range(W, n_total)}
    max_scan, max_corner = 1 << 18, 1 << 16

    class _Staging:
        def __init__(self, est):
            self.est = est

        def __getattr__(self, name):
            return getattr(self.est, name)

        def init_frame(self, k, *args):
            self.est.set_scan_clouds(warm[k][1], warm[k][2])
            self.est.init_frame(k, *args)

    def make(local):
        est = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 16, max_scan_points=max_scan, **cfg)
        if local:
            est.enable_local_clouds(0.2, max_corner, max_raw)
        scenario.warm_start(_Staging(est) if local else est, scn, W, lambda k: warm[k][0],
                            lambda g_a, g_g: estimator.Pim(g_a, g_g, np.zeros(3), np.zeros(3), acc_n=cfg["acc_n"], gyr_n=cfg["gyr_n"],
                                                           acc_w=cfg["acc_w"], gyr_w=cfg["gyr_w"], g_norm=cfg["g_norm"]))
        return est

    def run(leg):   # "host", "est_on", "est_off"
        est = make(leg != "est_off")
        mb = MapBuilder(max_points=1 << 17, max_full_points=max_raw) if leg == "host" else None
        times, poses = [], []
        for i, k in enumerate(range(W, n_total - 1)):
            torch.cuda.synchronize()
            if leg == "host":
                t0 = time.perf_counter()
                pp.SetInputCloud(scn.raw[k]); pp.Process()
                lf, corner, full = pp.cloud(names[5]), pp.cloud(names[3]), pp.cloud(names[1])
                scenario.feed_imu(est, scn, k)
                est.set_scan_clouds(corner, full)
                est.process_scan(lf)
                lc = est.local_clouds()
                tobe, _ = mb.ProcessMap(lc["corner"], lc["surf"], lc["full"], est.local_laser_odom())
            else:   # the estimator alone: stage A runs before the clock starts
                t = dev_raw[k]
                pp.process_device(t.data_ptr(), t.shape[0])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                scenario.feed_imu(est, scn, k)
                if leg == "est_on":
                    est.set_scan_clouds_dev(ptr[3], cnt[3], max_corner, ptr[1], cnt[1], max_raw)
                est.process_scan_dev(ptr[5], cnt[5], max_scan)
                tobe = None
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if i >= a.warmup:
                times.append((t1 - t0) * 1e3)
                poses.append(tobe)
        est.close()
        return times, poses

    # the device chain's clock starts before its stage A, like the host chain's
    res_legs = {}
    for leg in ("device", "host", "est_on", "est_off"):
        if leg == "device":
            times, poses = [], []
            est = make(True)
            mb = MapBuilder(max_points=1 << 17, max_full_points=max_raw)
            pub = est.local_clouds_dev()
            for i, k in enumerate(range(W, n_total - 1)):
                t = dev_raw[k]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pp.process_device(t.data_ptr(), t.shape[0])
                scenario.feed_imu(est, scn, k)
                est.set_scan_clouds_dev(ptr[3], cnt[3], max_corner, ptr[1], cnt[1], max_raw)
                est.process_scan_dev(ptr[5], cnt[5], max_scan)
                tobe, _ = mb.ProcessMapDev(*pub, est.local_laser_odom())
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                if i >= a.warmup:
                    times.append((t1 - t0) * 1e3)
                    poses.append(tobe)
            est.close()
            res_legs[leg] = (times, poses)
        else:
            res_legs[leg] = run(leg)
    name, power = card()
    med = {leg: round(float(np.median(v[0])), 3) for leg, v in res_legs.items()}
    same = all(np.array_equal(x, y) for x, y in zip(res_legs["device"][1], res_legs["host"][1]))
    res = dict(metric="lio_chain_ms_per_scan", kind="hdl64", window=[W, O], scans=a.scans, warmup=a.warmup, gpu=name, power_limit=power,
               chain_device_resident_ms_median=med["device"], chain_host_copies_ms_median=med["host"],
               estimator_local_clouds_on_ms_median=med["est_on"], estimator_local_clouds_off_ms_median=med["est_off"],
               identical_map_builder_poses=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
