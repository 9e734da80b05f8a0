"""Time lio_node (processor_node + estimator_node as one handle) per sweep over an HDL-64 drive in the outdoor_64 shape (W 7 / O 5,
cutoff_deskew, odom_io 3, msg_time_delay 0), against the same handles wired by hand; print one JSON line.

  node        LioNode.push_sweep_dev for the sweep (already in HBM), then push_imu_batch of the IMU messages up to the next sweep
  hand_wired  PointProcessor.process_device -> PointOdometry.ProcessDev -> (pairing by lio_measure_replay's restated rules) ->
              Estimator.process_imu_batch + process_compact_dev on the odometry's clouds, EnableOdom(False) after the start-up message

A sweep's time is a host clock from its push to the end of the IMU messages that follow it, closed by a device synchronise; it includes
the message the sweep published when the pairing releases it in that span (with delay 0 the next IMU message releases it).  Sweeps are
split by what happened: not published by the io gate; published while NOT_INITED; the start-up message; INITED.  The two legs run on
fresh handles, alternated `--rounds` times; the script checks that both legs end in bit-identical window states.

    python scripts/lio_node_bench.py [--sweeps 90] [--rounds 2] [--out FILE]
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

EST = dict(window_size=7, opt_window_size=5, init_window_factor=1, enable_deskew=0, cutoff_deskew=1, prior_factor=1, imu_factor=1,
           estimate_extrinsic=1, opt_extrinsic=0, keep_features=0, acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5, g_norm=9.805,
           min_match_sq_dis=1.0, min_plane_dis=0.2, max_frame_points=1 << 15, max_scan_points=1 << 17)
F, N, IO = 1 << 16, 1 << 18, 3


def make_drive(n):
    from lio_mapping_b200 import synth
    sensor, scene, traj = synth.default_config("hdl64")
    traj = dataclasses.replace(traj, k_roll=0.25, k_pitch=0.25)   # enough excitation for RunInitialization
    t = 1.0 + 0.1 * np.arange(n)
    tlb = np.array([0.0, 0.0, -0.1])
    raw = [synth.make_sweep(sensor, scene, traj, float(tk), seed=300 + i, t_lb=tlb, distort=True) for i, tk in enumerate(t)]
    it, acc, gyr = synth.make_imu(traj, 0.9, float(t[-1]) + 0.2, 200.0)
    spans = []   # IMU messages after sweep k, up to sweep k + 1 (inclusive of its stamp)
    for k in range(n):
        hi = t[k + 1] if k + 1 < n else np.inf
        sel = (it > t[k]) & (it <= hi)
        spans.append((it[sel], acc[sel], gyr[sel]))
    first = it <= t[0]
    return t, raw, (it[first], acc[first], gyr[first]), spans, np.r_[0.0, 0.0, 0.0, 1.0, tlb].astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=90)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lio_node_bench: no CUDA device")
    from lio_mapping_b200 import LioNode, estimator
    from lio_mapping_b200.node import measure_replay
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from lio_mapping_b200.point_processor import PointProcessor
    t, raw, imu0, spans, tf = make_drive(a.sweeps)
    dev = [torch.from_numpy(np.ascontiguousarray(r, np.float32)).cuda() for r in raw]

    # the pairing of this drive, decided once and outside the clock by the node's own rules (lio_measure_replay): the io gate publishes
    # sweeps c >= 1 with c % odom_io == 1 (PointOdometry.cc:302-310, :725); with delay 0 each message is decided in its own sweep's span
    pub = [k for k in range(a.sweeps) if k >= 1 and k % IO == 1]
    arr, msg_at = [("imu", float(x), acc, gyr) for x, acc, gyr in zip(*imu0)], {}
    for k in range(a.sweeps):
        if k in pub:
            msg_at[len(arr)] = k
            arr.append(("msg", float(t[k])))
        arr += [("imu", float(x), acc, gyr) for x, acc, gyr in zip(*spans[k])]
    calls, events, _ = measure_replay(0.0, arr)
    paired = {}
    for j, (idx, processed, first) in enumerate(events):
        end = events[j + 1][2] if j + 1 < len(events) else len(calls)
        paired[msg_at[idx]] = calls[first:end] if processed else None

    def run_node():
        node = LioNode(sensor_type=64, odom_io=IO, msg_time_delay=0.0, tf_lb7=tf, max_points=N, max_feature_points=F, **EST)
        node.push_imu_batch(*imu0)
        times, kinds = [], []
        for k in range(a.sweeps):
            before = node.status()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            node.push_sweep_dev(dev[k].data_ptr(), dev[k].shape[0], float(t[k]))
            node.push_imu_batch(*spans[k])
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
            s = node.status()
            kinds.append(kind_of(before, s))
        return times, kinds, node.states(), node.processor.last_launches() + node.odometry.last_launches()

    def kind_of(before, after):
        if after["published"] == before["published"] and after["processed"] == before["processed"]:
            return "not_published"
        if after["inited"] and not before["inited"]:
            return "startup"
        return "inited" if before["inited"] else "published_not_inited"

    def run_hand():
        pp = PointProcessor(-24.9, 2.0, 64, max_points=N)
        po = PointOdometry(0.1, IO, 25, F, N)
        pm = PointMapping(max_points=F, max_iterations=10)
        pm.EnablePublish(0.6, N)
        e = estimator.Estimator(**EST)
        e.set_extrinsic(tf)
        e.enable_local_clouds(0.2, F, N)
        e.attach_imu_mapping(pm)
        names = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")
        ptrs = [pp.cloud_dev(x) for x in names]
        cnts = [pp.cloud_count_dev(x) for x in names]
        times, kinds, inited = [], [], False
        for k in range(a.sweeps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pp.process_device(dev[k].data_ptr(), dev[k].shape[0])
            ts, _, info = po.ProcessDev(ptrs, cnts, [F] * 4 + [N])
            kind = "not_published"
            assert bool(info["published"]) == (k in pub)
            c = paired.get(k)
            if c is not None:
                e.process_imu_batch(c[:, 0], c[:, 1:4], c[:, 4:7], c[:, 7])
                p, nd, nn = po.clouds_dev()
                st = e.process_compact_dev(p, nd, nn, ts, stamp=float(t[k]))
                kind = "startup" if st["inited"] and not inited else ("inited" if inited else "published_not_inited")
                if st["inited"] and not inited:
                    po.EnableOdom(False)
                inited = st["inited"]
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
            kinds.append(kind)
        return times, kinds, e.states()

    legs = {"node": [], "hand_wired": []}
    same = True
    launches = None
    for _ in range(a.rounds):
        tn, kn, sn, launches = run_node()
        th, kh, sh = run_hand()
        legs["node"].append((tn, kn))
        legs["hand_wired"].append((th, kh))
        same = same and kn == kh and np.array_equal(sn, sh)
    name, power = card()
    res = dict(metric="lio_node_ms_per_sweep", kind="hdl64", shape="outdoor_64 W7/O5 cutoff_deskew odom_io 3 delay 0", sweeps=a.sweeps,
               rounds=a.rounds, gpu=name, power_limit=power, identical_states=bool(same),
               stage_a_plus_odometry_launches_last_sweep=int(launches))
    for leg, runs in legs.items():
        for cat in ("not_published", "published_not_inited", "startup", "inited"):
            v = [x for tt, kk in runs for x, c in zip(tt[1:], kk[1:]) if c == cat]   # the first sweep of a run warms up
            if v:
                res[f"{leg}_{cat}_ms_median"] = round(float(np.median(v)), 3)
                res[f"{leg}_{cat}_ms_p90"] = round(float(np.percentile(v, 90)), 3)
                res[f"{leg}_{cat}_count"] = len(v)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
