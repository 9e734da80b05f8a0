"""Cost of one window solve by opt window size on stress128 sweeps (128 x 4096, the stress workload's sensor); prints one
JSON line.

For O = 13 the device solver runs its one-CTA step kernel (k_step); for O = 14, 15, 16 it runs the two-CTA cluster kernel
(k_step_x2), and the same windows also run under the host controller (device_solver = 0) on the same inputs.  Per scan:
the estimator's own solve time (summary t_solve: host time of the solve up to its last device synchronise), its cost
evaluations and its host waits.  A device solve waits on the device once, at its end; the host controller waits once per
cost evaluation (it reads the lidar blocks back and factors H on the CPU).  The first --warmup scans are not timed.

    python scripts/window_solve_bench.py [--scans 6] [--warmup 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.map_builder_bench import card  # noqa: E402


def run(O, device_solver, clouds, scn, scans, warmup):
    from lio_mapping_b200 import estimator, scenario
    cfg = dict(scenario.EST_CFG["stress128"], device_solver=device_solver)
    e = estimator.Estimator(window_size=O, opt_window_size=O, max_frame_points=1 << 17,
                            max_scan_points=max(c.shape[0] for c in clouds) + 16, **cfg)
    scenario.warm_start(e, scn, O, lambda k: clouds[k], lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    ms, evals = [], []
    for i, k in enumerate(range(O, O + warmup + scans)):
        scenario.feed_imu(e, scn, k)
        e.process_scan(clouds[k])
        s = e.summary()
        if i >= warmup:
            ms.append(1e3 * s["t_solve"])
            evals.append(s["cost_evals"])
    trace_nonzero = bool(np.any(e.solver_trace() != 0))
    return {"ms_per_solve": float(np.median(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)),
            "cost_evals_per_scan": float(np.mean(evals)),
            "host_waits_per_scan": 1.0 if device_solver else float(np.mean(evals)),
            "device_path": trace_nonzero}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from lio_mapping_b200 import ops, scenario
    from lio_mapping_b200.point_processor import PointProcessor
    if not torch.cuda.is_available():
        raise SystemExit("window_solve_bench.py needs a GPU")
    n = 16 + a.warmup + a.scans
    scn = scenario.Scenario("stress128", n_total=n)
    s = scn.sensor
    pp = PointProcessor(s.lower_deg, s.upper_deg, s.rings, max_points=max(r.shape[0] for r in scn.raw))
    clouds = []
    for k in range(n):
        pp.SetInputCloud(scn.raw[k]); pp.Process()
        clouds.append(np.ascontiguousarray(ops.voxel_grid(pp.cloud("surface_points_less_flat"), 0.4)))
    res = {"workload": "stress128 sweeps, W = O", "card": card(), "scans": a.scans, "warmup": a.warmup}
    res["O13_one_cta"] = run(13, 1, clouds, scn, a.scans, a.warmup)
    for O in (14, 15, 16):
        res["O%d_cluster" % O] = run(O, 1, clouds, scn, a.scans, a.warmup)
        res["O%d_host" % O] = run(O, 0, clouds, scn, a.scans, a.warmup)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
