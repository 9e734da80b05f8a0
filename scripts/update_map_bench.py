"""Time one PointMapping::UpdateMapDatabase (lio_pm_update_map_database_host) on the GPU over an HDL-64 drive; print one JSON line.

Every frame's down-sampled corner / surf clouds (VoxelGrid 0.2 / 0.4 of stage A's less-sharp / less-flat clouds) are inserted with
the ground-truth pose, so the cube map grows like the mapping node's.  Two valid lists are timed on two fresh maps:
  fov     the cubes the reference selects for the pose (PointMapping.cc:944-1003, from the oracle's restatement)
  block   all 125 cubes of the 5 x 5 x 5 block around the sensor: every non-empty cube nearby is re-filtered
Per call: device time between two CUDA events on the map's stream around the call (this includes the clouds' upload and the
device idling while the host sizes the segments), the host time of the call plus a stream synchronise, and the code's own counts
of cube jobs, kernel launches and host waits (lio_pm_update_stats; the waits include the one the next reader of the cubes makes
for the re-filtered sizes).  The first --warmup frames are not timed.

    python scripts/update_map_bench.py [--frames 40] [--warmup 8] [--out FILE]
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

from scripts.map_builder_bench import card, drive  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("update_map_bench: no CUDA device")
    from lio_mapping_b200 import synth
    from lio_mapping_b200.point_mapping import PointMapping
    from oracle import oracle_py
    oracle_py.build()
    frames = drive("hdl64", a.frames)
    stream = torch.cuda.Stream()

    def valid_lists(tf7):
        cm = oracle_py.CubeMap()
        pos = tf7[4:].astype(np.float32)
        centre, cen = cm.recentre(pos)
        zaxis = (pos + synth.quat_to_rot(tf7[:4].astype(np.float64)) @ np.array([0, 0, 10.0])).astype(np.float32)
        valid, block = cm.select(pos, zaxis, centre)
        return dict(fov=valid, block=block), cen

    def run(which):
        pm = PointMapping(max_points=1 << 17, corner_filter_size=0.2, surf_filter_size=0.4, stream=stream.cuda_stream)
        rows = []
        for f, (c, s, _, tf) in enumerate(frames):
            lists, cen = valid_lists(tf)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            stream.synchronize()
            t0 = time.perf_counter()
            e0.record(stream)
            st = pm.UpdateMapDatabase(c, s, lists[which], tf, cen)
            e1.record(stream)
            stream.synchronize()
            t1 = time.perf_counter()
            if f >= a.warmup:
                rows.append((e0.elapsed_time(e1), (t1 - t0) * 1e3, st["jobs"], st["launches"], st["waits"], st["points"]))
        pm.close()
        r = np.array(rows)
        return dict(calls=len(rows), device_ms_median=round(float(np.median(r[:, 0])), 4), device_ms_mean=round(float(np.mean(r[:, 0])), 4),
                    host_ms_median=round(float(np.median(r[:, 1])), 4), jobs_median=float(np.median(r[:, 2])), jobs_max=int(r[:, 2].max()),
                    launches=sorted(set(int(v) for v in r[:, 3])), waits_max=int(r[:, 4].max()), waits_median=float(np.median(r[:, 4])),
                    points_mean=int(np.mean(r[:, 5])))

    res_fov = run("fov")
    res_block = run("block")
    name, power = card()
    res = dict(metric="update_map_database_ms", kind="hdl64", frames=a.frames, warmup=a.warmup, gpu=name, power_limit=power,
               fov=res_fov, block=res_block)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
