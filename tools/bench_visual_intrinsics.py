"""Cost of refining the shared intrinsics in the visual LM (lvba_visual_opts::refine_intrinsics) at config C, inputs resident on
the device.

Three handles of the same problem, mask 0 (no block), LVBA_INTR_FOCAL and all eight entries, run alternately, --runs times each.
A run is --steps LM passes from the same start (reset_state + reset_lm, stop tests off), after --warmup passes.  Reported per
mask: LM passes per second (host wall clock over the iterate call, which synchronises) and the build and solve times per pass
from the library's CUDA events.  With the block, the build time includes its passes and the solve time its k + 1 camera solves,
the corner and the copy of the intrinsics step to the host.  --long N adds N tracks of --kmin..--kmax observations as
tools/bench_visual_big.py does (landmarks beyond 128 observations, whose block terms one thread each computes).  The card's name
and power limit are read in the same call.  Prints one JSON line; writes nothing."""
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

MASKS = {"none": 0, "focal": 0x03, "all": 0xFF}


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
    ap.add_argument("--long", type=int, default=0)
    ap.add_argument("--kmin", type=int, default=200)
    ap.add_argument("--kmax", type=int, default=1000)
    a = ap.parse_args()
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config)
    if a.long:
        sys.path.insert(0, str(ROOT / "tools"))
        from bench_visual_big import add_long_tracks
        p = add_long_tracks(p, a.long, a.kmin, a.kmax)
    out = {"config": a.config, "long": [a.long, a.kmin, a.kmax], "card": card(), "date": time.strftime("%Y-%m-%d"), "steps": a.steps, "runs": a.runs}

    def opts(mask):
        o = pkg.visual_default_opts()
        o.function_tolerance = o.gradient_tolerance = o.parameter_tolerance = -1.0
        o.max_iter = a.steps + a.warmup
        o.refine_intrinsics = mask
        return o

    args = [p[k] for k in ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")]
    handles = {m: pkg.VisualProblem(*args) for m in MASKS}
    res = {m: [] for m in MASKS}
    for _ in range(a.runs):
        for m, mask in MASKS.items():
            P = handles[m]
            P.reset_state(); P.reset_lm(opts(mask))
            if a.warmup:
                P.iterate(a.warmup)
            P.reset_state(); P.reset_lm(opts(mask))
            t0 = time.perf_counter()
            s = P.iterate(a.steps)
            dt = time.perf_counter() - t0
            nb = max(s["hessian_builds"], 1)
            res[m].append(dict(it_s=s["iterations"] / dt, build_ms=s["ms_build"] / nb, solve_ms=s["ms_solve"] / nb))
    for P in handles.values():
        P.close()
    for m in MASKS:
        for k in ("it_s", "build_ms", "solve_ms"):
            v = [r[k] for r in res[m]]
            out[f"{m}_{k}"] = [round(min(v), 4), round(float(np.median(v)), 4), round(max(v), 4)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
