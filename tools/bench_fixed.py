"""Cost of constant cameras in the visual LM (lvba_visual_opts::cam_fixed) at config C, inputs resident on the device.

Handles of the same problem with different constant sets run alternately, --runs times each: camera 0 constant (fixed_cam = 0,
the reference), and cameras 0 .. --many - 1 constant (fixed_cam = 0 plus a mask, set by a re-planning reset).  A run is --steps
LM passes from the same start (reset_state + reset_lm, stop tests off), after --warmup passes.  Reported per set: LM passes per
second (host wall clock over the iterate call, which synchronises), the build time per build and the solve time per pass from
the library's own CUDA events, and the system rows.  The re-plan is timed on a separate handle as the host wall time of a reset
whose mask differs from the handle's (to the many-camera mask and back to none).  Prints one JSON line with the card's name and
power limit; writes nothing."""
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

KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def mmm(v, nd=4):
    return [round(min(v), nd), round(float(np.median(v)), nd), round(max(v), nd)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--many", type=int, default=1000, help="cameras 0 .. many-1 constant in the second set")
    a = ap.parse_args()
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config, lidar=False)
    args = [p[k] for k in KEYS]
    M = len(p["q"])
    many = np.arange(M) < min(a.many, M)
    out = {"config": a.config, "card": card(), "date": time.strftime("%Y-%m-%d"), "steps": a.steps, "runs": a.runs, "cameras": M,
           "many": int(many.sum())}

    def opts():
        o = pkg.visual_default_opts()
        o.function_tolerance = o.gradient_tolerance = o.parameter_tolerance = -1.0
        o.max_iter = a.steps + a.warmup
        return o

    sets = {"cam0": None, "many": many}
    handles = {k: pkg.VisualProblem(*args, fixed_cam=0) for k in sets}
    for k, m in sets.items():
        handles[k].reset_lm(opts(), cam_fixed=m)
        out[f"rows_{k}"] = len(handles[k].structure()[0])
    res = {k: [] for k in sets}
    for _ in range(a.runs):
        for k, m in sets.items():
            P = handles[k]
            P.reset_state(); P.reset_lm(opts(), cam_fixed=m)
            if a.warmup:
                P.iterate(a.warmup)
            P.reset_state(); P.reset_lm(opts(), cam_fixed=m)
            t0 = time.perf_counter()
            s = P.iterate(a.steps)
            dt = time.perf_counter() - t0
            res[k].append(dict(it_s=s["iterations"] / dt, build_ms=s["ms_build"] / max(s["hessian_builds"], 1),
                               solve_ms=s["ms_solve"] / max(s["iterations"], 1)))
    for P in handles.values():
        P.close()
    for k in sets:
        for f in ("it_s", "build_ms", "solve_ms"):
            out[f"{k}_{f}"] = mmm([r[f] for r in res[k]])
    P = pkg.VisualProblem(*args, fixed_cam=0)
    to_many, to_none = [], []
    for _ in range(a.runs):
        for m, dst in ((many, to_many), (None, to_none)):
            t0 = time.perf_counter()
            P.reset_lm(opts(), cam_fixed=m)
            dst.append(1e3 * (time.perf_counter() - t0))
    P.close()
    out["replan_ms_to_many"] = mmm(to_many, 2)
    out["replan_ms_to_none"] = mmm(to_none, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
