"""Cost of constant poses in the LiDAR LM (lvba_lidar_opts::pose_fixed) at config C, inputs resident on the device.

Three handles of the same problem run alternately, --runs times each: no mask, pose 0 constant, and poses 0 .. --many - 1
constant (each set by a re-planning reset).  A run is --steps LM passes from the same start (reset_state + reset_lm, stop test
off), after --warmup passes.  Reported per set: LM passes per second (host wall clock over the iterate call, which synchronises),
the build time per build and the solve time per pass from the library's own CUDA events, and the system rows.  The re-plan is
timed on a separate handle as the host wall time of a reset whose mask differs from the handle's (to the many-pose mask and back
to none).  Prints one JSON line with the card's name and power limit; writes nothing."""
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

KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")


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
    ap.add_argument("--many", type=int, default=1000, help="poses 0 .. many-1 constant in the third set")
    a = ap.parse_args()
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config, visual=False)
    args = [p[k] for k in KEYS]
    W = len(p["poses"])
    many = np.arange(W) < min(a.many, W)
    out = {"config": a.config, "card": card(), "date": time.strftime("%Y-%m-%d"), "steps": a.steps, "runs": a.runs, "poses": W,
           "many": int(many.sum())}

    def opts():
        o = pkg.lidar_default_opts()
        o.rel_tol = -1.0
        o.max_iter = a.steps + a.warmup
        return o

    sets = {"none": np.zeros(W, bool), "pose0": np.arange(W) == 0, "many": many}
    handles = {k: pkg.LidarProblem(*args) for k in sets}
    for k, m in sets.items():
        handles[k].reset_lm(opts(), pose_fixed=m)
        out[f"rows_{k}"] = len(handles[k].rows())
    res = {k: [] for k in sets}
    for _ in range(a.runs):
        for k, m in sets.items():
            P = handles[k]
            P.reset_state(); P.reset_lm(opts(), pose_fixed=m)
            if a.warmup:
                P.iterate(a.warmup)
            P.reset_state(); P.reset_lm(opts(), pose_fixed=m)
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
    P = pkg.LidarProblem(*args)
    to_many, to_none = [], []
    for _ in range(a.runs):
        for m, dst in ((many, to_many), (np.zeros(W, bool), to_none)):
            t0 = time.perf_counter()
            P.reset_lm(opts(), pose_fixed=m)
            dst.append(1e3 * (time.perf_counter() - t0))
    P.close()
    out["replan_ms_to_many"] = mmm(to_many, 2)
    out["replan_ms_to_none"] = mmm(to_none, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
