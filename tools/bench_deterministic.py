"""Cost of the deterministic mode of both LM paths (lvba_lidar_opts / lvba_visual_opts ::deterministic) at config C, inputs
resident on the device.

For each path, default and deterministic handles of the same problem run alternately, --runs times each.  A run is --steps LM
passes from the same start (reset_state + reset_lm, stop tests off), after --warmup passes.  Reported per path and mode: LM passes
per second (host wall clock over the iterate call, which synchronises), and the build time per build and solve time per pass
from the library's own CUDA events.  The extra device memory of the mode is the drop in free device memory when a handle first
asks for it.  Prints one JSON line; writes nothing."""
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


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


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
    a = ap.parse_args()
    pkg = graft.load_package()
    pkg.load_library()
    p = synth.make_config(a.config)
    out = {"config": a.config, "card": card(), "date": time.strftime("%Y-%m-%d"), "steps": a.steps, "runs": a.runs}

    def lidar_opts(det):
        o = pkg.lidar_default_opts()
        o.rel_tol = -1.0                      # a fixed number of passes in both modes
        o.deterministic = det
        return o

    def visual_opts(det):
        o = pkg.visual_default_opts()
        o.function_tolerance = o.gradient_tolerance = o.parameter_tolerance = -1.0
        o.max_iter = a.steps + a.warmup
        o.deterministic = det
        return o

    paths = {
        "A": (lambda: pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"]), lidar_opts),
        "B": (lambda: pkg.VisualProblem(*[p[k] for k in ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr",
                                                           "sigma_px", "sigma_plane")]), visual_opts),
    }
    for path, (make, opts) in paths.items():
        handles = {}
        for det in (0, 1):
            handles[det] = make()
            f0 = free_bytes()
            handles[det].reset_lm(opts(det))
            if det:
                out[f"extra_device_bytes_{path}"] = int(f0 - free_bytes())
        res = {0: [], 1: []}
        for _ in range(a.runs):
            for det in (0, 1):
                P = handles[det]
                P.reset_state(); P.reset_lm(opts(det))
                if a.warmup:
                    P.iterate(a.warmup)
                P.reset_state(); P.reset_lm(opts(det))
                t0 = time.perf_counter()
                s = P.iterate(a.steps)
                dt = time.perf_counter() - t0
                res[det].append(dict(it_s=s["iterations"] / dt, build_ms=s["ms_build"] / max(s["hessian_builds"], 1),
                                     solve_ms=s["ms_solve"] / max(s["iterations"], 1)))
        for P in handles.values():
            P.close()
        for det, name in ((0, "default"), (1, "deterministic")):
            for k in ("it_s", "build_ms", "solve_ms"):
                v = [r[k] for r in res[det]]
                out[f"{path}_{name}_{k}"] = [round(min(v), 4), round(float(np.median(v)), 4), round(max(v), 4)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
