"""Cost of BALM2's voxel outlier removal on the LiDAR handle at config C, inputs resident on the device.

Reported (median over --runs, each on a fresh handle of the same problem):
  * lvba_lidar_voxel_residuals at the handle's poses: device time between CUDA events around the call, and host wall time;
  * lvba_lidar_remove_outliers(--ratio): host wall time of the call, and of its re-plan alone (lvba_lidar_remove_voxels with the
    same mask on a twin handle).  Their difference in each run is an estimate, not a measurement, of the lambda_0 pass and the
    rule together (reported as residuals_and_rule_ms, the median of the per-run differences);
  * LM passes per second (--steps passes from the same start, stop test off) before the removal, after it, and on a fresh
    handle of the kept voxels.
Prints one JSON line with the card's name and power limit; writes nothing."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import numpy as np  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
import lidar_outlier_oracle as olo  # noqa: E402
from oracle import synth  # noqa: E402

KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def passes_per_s(P, opts, steps, warmup):
    P.reset_lm(opts); P.iterate(warmup)
    P.reset_lm(opts)
    t0 = time.perf_counter(); s = P.iterate(steps); dt = time.perf_counter() - t0
    return s["iterations"] / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--ratio", type=float, default=0.05)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config)
    args = [p[k] for k in KEYS]
    opts = pkg.lidar_default_opts(); opts.rel_tol = -1.0; opts.max_iter = a.steps
    res = {"vr_dev_ms": [], "vr_wall_ms": [], "remove_ms": [], "replan_ms": [], "residuals_and_rule_ms": [], "before": [], "after": [], "fresh": []}
    removed = None
    for _ in range(a.runs):
        P = pkg.LidarProblem(*args, device=0)
        T = pkg.LidarProblem(*args, device=0)
        P.voxel_residuals()                                            # first call uploads the voxel index of the plan
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(); t0 = time.perf_counter(); P.voxel_residuals(); t1 = time.perf_counter(); e1.record()
        torch.cuda.synchronize()
        res["vr_dev_ms"].append(e0.elapsed_time(e1)); res["vr_wall_ms"].append(1e3 * (t1 - t0))
        res["before"].append(passes_per_s(P, opts, a.steps, a.warmup))
        P.reset_state()
        t0 = time.perf_counter(); removed = P.remove_outliers(a.ratio); t1 = time.perf_counter()
        t2 = time.perf_counter(); T.remove_voxels(removed); t3 = time.perf_counter()
        res["remove_ms"].append(1e3 * (t1 - t0)); res["replan_ms"].append(1e3 * (t3 - t2))
        res["residuals_and_rule_ms"].append(res["remove_ms"][-1] - res["replan_ms"][-1])
        res["after"].append(passes_per_s(P, opts, a.steps, a.warmup))
        P.close(); T.close()
        vp, pi, cl = olo.kept_problem(p["vox_ptr"], p["pose_idx"], p["clusters"], removed)
        F = pkg.LidarProblem(vp, pi, cl, p["poses"], device=0)
        res["fresh"].append(passes_per_s(F, opts, a.steps, a.warmup))
        F.close()
    med = {k: round(float(np.median(v)), 3) for k, v in res.items()}
    print(json.dumps({"config": a.config, "V": len(p["vox_ptr"]) - 1, "ratio": a.ratio, "removed": int(removed.sum()),
                      "runs": a.runs, "steps": a.steps, "median": med, "card": card()}), flush=True)


if __name__ == "__main__":
    main()
