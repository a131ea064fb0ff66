"""Cost of the reprojection-outlier removal on the visual handle at config C, inputs resident on the device.

Reported (median over --runs, each on a fresh handle of the same problem):
  * lvba_visual_obs_residuals at the handle's state: host wall time of the call, which ends in a synchronise of the handle's
    stream (the first call, which also derives the caller index of every observation, is left out), and the device time of
    the NaN fill and visual_obs_sq_kernel from torch.profiler's CUDA activities in a separate profiled call;
  * lvba_visual_remove_outliers at a threshold that removes about --frac of the observations (the (1 - frac) quantile of the
    finite s_q, min_track_len 3): host wall time of the call, and of its re-plan alone (lvba_visual_remove_observations with the
    same mask on a twin handle);
  * visual LM passes per second (--steps passes from the same start, stop tests off) before the removal, after it, and on a
    fresh handle of the kept observations.
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
import visual_outlier_oracle as voo  # noqa: E402
from oracle import synth  # noqa: E402

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


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
    ap.add_argument("--frac", type=float, default=0.05)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config)
    args = [p[k] for k in VKEYS]
    opts = pkg.visual_default_opts()
    opts.max_iter = a.steps
    opts.function_tolerance = -1.0; opts.gradient_tolerance = -1.0; opts.parameter_tolerance = -1.0
    res = {"sq_dev_ms": [], "sq_wall_ms": [], "remove_ms": [], "replan_ms": [], "before": [], "after": [], "fresh": []}
    removed = None
    max_err = None
    for _ in range(a.runs):
        P = pkg.VisualProblem(*args, device=0)
        T = pkg.VisualProblem(*args, device=0)
        sq = P.obs_residuals()
        if max_err is None:
            max_err = float(np.sqrt(np.quantile(sq[np.isfinite(sq)], 1.0 - a.frac))) * float(p["sigma_px"])
        t0 = time.perf_counter(); P.obs_residuals(); t1 = time.perf_counter()
        res["sq_wall_ms"].append(1e3 * (t1 - t0))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            P.obs_residuals()
        dev_us = sum(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) for e in prof.events()
                     if "visual_obs_sq_kernel" in e.name or "NanFillF" in e.name)
        res["sq_dev_ms"].append(dev_us / 1e3)
        res["before"].append(passes_per_s(P, opts, a.steps, a.warmup))
        P.reset_state()
        t0 = time.perf_counter(); removed, _ = P.remove_outliers(max_err); t1 = time.perf_counter()
        t2 = time.perf_counter(); T.remove_observations(removed); t3 = time.perf_counter()
        res["remove_ms"].append(1e3 * (t1 - t0)); res["replan_ms"].append(1e3 * (t3 - t2))
        res["after"].append(passes_per_s(P, opts, a.steps, a.warmup))
        P.close(); T.close()
        tr = voo.Tracker(p)
        tr.obs_in &= ~removed
        sq_left = np.zeros(len(p["obs_ptr"]) - 1, np.int64)
        np.add.at(sq_left, np.repeat(np.arange(len(sq_left)), np.diff(p["obs_ptr"]))[tr.obs_in], 1)
        tr.lm_in &= sq_left >= 1
        k = tr.kept_problem()
        F = pkg.VisualProblem(*[k[key] for key in VKEYS], device=0)
        res["fresh"].append(passes_per_s(F, opts, a.steps, a.warmup))
        F.close()
    med = {k: round(float(np.median(v)), 3) for k, v in res.items()}
    print(json.dumps({"config": a.config, "n_obs": int(p["obs_ptr"][-1]), "max_err_px": round(max_err, 4),
                      "removed": int(removed.sum()), "runs": a.runs, "steps": a.steps, "median": med, "card": card()}), flush=True)


if __name__ == "__main__":
    main()
