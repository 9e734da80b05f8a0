"""Cost of the estimator's global cube map after initialisation (lio_est_attach_map) on the GPU; print one JSON line.

Two estimators with the same inputs run in one process, one with the pre-initialisation map attached and one without, their scans
alternated: HDL-64 with window 10 / 10 (bench.py's workload) and one W > O shape (12 / 10, so the inserted surf cloud is an
accumulated slot).  The estimators run on the legacy default stream like bench.py; the map has a non-blocking stream of its own.
Per scan: host time of process_scan plus a device synchronise.  That time includes the map's work: the host waits inside the
insert (the run list, grown segments) and on publishing scans (the surround size) happen before process_scan returns, and the
final synchronise waits for the map's stream too.  Per insert: the map's own counts
(lio_pm_update_stats: points inserted, cube jobs re-filtered, kernel launches, host waits).  The warm-start map is a publishing
PointMapping fed the warm-start sweeps with the ground-truth pose; the first --warmup scans are not timed.

    python scripts/global_map_bench.py [--scans 24] [--warmup 4] [--out FILE]
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


def run_shape(W, O, scans, warmup, map_stream):
    import torch
    from lio_mapping_b200 import estimator, ops, scenario, synth
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_processor import PointProcessor
    scn = scenario.Scenario("hdl64", n_total=W + scans)
    pp = PointProcessor(scn.sensor.lower_deg, scn.sensor.upper_deg, scn.sensor.rings, max_points=max(r.shape[0] for r in scn.raw))
    clouds = []
    for raw in scn.raw:   # device stage A: less-sharp (corner), less-flat (surf), cloud_in_rings (full)
        pp.SetInputCloud(raw); pp.Process()
        clouds.append([pp.cloud(n) for n in ("corner_points_less_sharp", "surface_points_less_flat", "cloud_in_rings")])
    max_full = max(c[2].shape[0] for c in clouds)
    ests = []
    for _ in range(2):
        e = estimator.Estimator(window_size=W, opt_window_size=O, max_frame_points=1 << 16, max_scan_points=1 << 18)
        e.enable_local_clouds(0.2, 1 << 16, max_full)
        stage = lambda k, e=e: e.set_scan_clouds(ops.voxel_grid(clouds[k][0], 0.2), clouds[k][2])
        scenario.warm_start(_StageFirst(e, stage), scn, W, lambda k: ops.voxel_grid(clouds[k][1], 0.4),
                            lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
        ests.append(e)
    eg, eb = ests
    pm = PointMapping(max_points=1 << 17, stream=map_stream.cuda_stream)
    pm.EnablePublish(0.6, max_full)
    tlb = scn.tf_lb7()
    for k in range(W):   # the pre-initialisation map, fed the ground-truth lidar pose
        s16 = scn.state16(k)
        R = synth.quat_to_rot(s16[3:7]) @ synth.quat_to_rot(tlb[:4].astype(np.float64)).T
        sum7 = np.r_[synth.rot_to_quat(R), s16[0:3] - R @ tlb[4:].astype(np.float64)].astype(np.float32)
        dev = [torch.from_numpy(np.ascontiguousarray(c, np.float32)).cuda() for c in clouds[k]]
        n = torch.tensor([c.shape[0] for c in clouds[k]], dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        pm.ProcessDev([d.data_ptr() for d in dev], n.data_ptr(), [c.shape[0] for c in clouds[k]], sum7)
    eg.attach_map(pm)
    ms = {"map": [], "plain": []}
    ins, published = [], 0
    for i in range(scans):
        k = W + i
        for name, e in (("map", eg), ("plain", eb)) if i % 2 == 0 else (("plain", eb), ("map", eg)):
            e.set_scan_clouds(clouds[k][0], clouds[k][2])
            scenario.feed_imu(e, scn, k)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e.process_scan(clouds[k][1])
            torch.cuda.synchronize()
            if i >= warmup:
                ms[name].append(1e3 * (time.perf_counter() - t0))
        _, _, _, info = eg.map_poses()
        published += int(info["surround_published"])
        if info["inserted"]:
            ins.append(pm.update_stats())
    med = {n: float(np.median(v)) for n, v in ms.items()}
    return dict(window=W, opt_window=O, timed_scans=len(ms["map"]), ms_per_scan_median_map=med["map"], ms_per_scan_median_plain=med["plain"],
                inserts=len(ins), insert_points_median=float(np.median([r["points"] for r in ins])) if ins else 0.0,
                insert_jobs_median=float(np.median([r["jobs"] for r in ins])) if ins else 0.0,
                insert_launches=sorted({r["launches"] for r in ins}), insert_host_waits=sorted({r["waits"] for r in ins}),
                publishing_scans=published)


class _StageFirst:
    """Stages a warm-start frame's corner / full cloud before its init_frame."""

    def __init__(self, est, stage):
        self.est, self.stage = est, stage

    def __getattr__(self, name):
        return getattr(self.est, name)

    def init_frame(self, k, *args):
        self.stage(k)
        self.est.init_frame(k, *args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("global_map_bench: no CUDA device")
    map_stream = torch.cuda.Stream()   # created non-blocking by torch
    shapes = [run_shape(W, O, a.scans, a.warmup, map_stream) for W, O in ((10, 10), (12, 10))]
    name, power = card()
    line = json.dumps(dict(bench="global_map", gpu=name, power_limit=power, shapes=shapes))
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
