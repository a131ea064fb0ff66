"""Cost of the robust losses of the visual LM (lvba_visual_opts::reproj_loss / plane_loss) at config C, inputs resident on the
device.

A plain handle and a Huber handle (the reference's HuberLoss(1.0) on the reprojection, HuberLoss(0.1) on the plane) of the same
problem run alternately, --runs times each.  A run is --steps LM passes from the same start (reset_state + reset_lm, stop tests
off), after --warmup passes.  Reported per mode: LM passes per second (host wall clock over the iterate call, which
synchronises), the build time per build from the library's CUDA events, and the wall time of one lvba_visual_cost call (median
of --cost-calls).  The card's name and power limit are read in the same call.  Prints one JSON line; writes nothing."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from oracle import synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cost-calls", type=int, default=20)
    a = ap.parse_args()
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config)
    out = {"config": a.config, "card": card(), "date": time.strftime("%Y-%m-%d"), "steps": a.steps, "runs": a.runs}

    def opts(robust):
        o = pkg.visual_default_opts(reproj_loss=pkg.LOSS_HUBER if robust else None, plane_loss=pkg.LOSS_HUBER if robust else None)
        o.function_tolerance = o.gradient_tolerance = o.parameter_tolerance = -1.0
        o.max_iter = a.steps + a.warmup
        return o

    args = [p[k] for k in ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")]
    handles = {m: pkg.VisualProblem(*args) for m in (0, 1)}
    res = {0: [], 1: []}
    for _ in range(a.runs):
        for m in (0, 1):
            P = handles[m]
            P.reset_state(); P.reset_lm(opts(m))
            if a.warmup:
                P.iterate(a.warmup)
            P.reset_state(); P.reset_lm(opts(m))
            t0 = time.perf_counter()
            s = P.iterate(a.steps)
            dt = time.perf_counter() - t0
            tc = []
            for _ in range(a.cost_calls):
                c0 = time.perf_counter(); P.cost(); tc.append(time.perf_counter() - c0)
            res[m].append(dict(it_s=s["iterations"] / dt, build_ms=s["ms_build"] / max(s["hessian_builds"], 1),
                               cost_ms=1e3 * float(np.median(tc))))
    for P in handles.values():
        P.close()
    for m, name in ((0, "plain"), (1, "huber")):
        for k in ("it_s", "build_ms", "cost_ms"):
            v = [r[k] for r in res[m]]
            out[f"{name}_{k}"] = [round(min(v), 4), round(float(np.median(v)), 4), round(max(v), 4)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
