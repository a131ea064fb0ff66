"""The two solvers of the visual LM's reduced camera system (lvba_visual_opts::linear_solver), measured on one GPU.  Prints one
JSON line per scene and solver:

    python tools/bench_visual_pcg.py [--config C] [--long 200] [--passes 10] [--repeats 3] [--scenes config,long,loop]

Scenes: the visual problem of the bench config as bench.py builds it; the same plus `--long` tracks of 200-1000 observations
(tools/bench_visual_big.py's long-track scene, whose envelope the LDL^T fills); and a loop-closed scene of 400 cameras whose
20-observation track joins cameras 390-399 to 0-9 (tests/visual_big_scene.py), on which AUTO takes the any-width path.
Per scene and solver (DENSE_SCHUR, then ITERATIVE_SCHUR at Ceres' defaults): ms_solve and LM passes/s over `--passes` passes of
lvba_visual_iterate with the stop tests off (best of `repeats` runs after one warm-up), the CG iterations per solve (mean and
max over those passes), the cost after them, the passes to convergence with the default tolerances and the final cost, and
n_blocks_env.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import importlib.util
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
SOLVERS = (("dense_schur", 0), ("iterative_schur", 1))


def _big():
    spec = importlib.util.spec_from_file_location("bench_visual_big", ROOT / "tools" / "bench_visual_big.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def scenes(names, config, n_long):
    from oracle import synth
    import visual_big_scene as vs
    out = []
    if "config" in names or "long" in names:
        p = synth.make_config(config, lidar=False)
        if "config" in names:
            out.append((f"{config}", p))
        if "long" in names:
            out.append((f"{config} + {n_long} long tracks", _big().add_long_tracks(p, n_long, 200, 1000)))
    if "loop" in names:
        out.append(("loop-closed M=400", vs.make_scene(11, M=400, long_tracks=[(20, 390)])))
    return out


def measure(pkg, p, solver, passes, repeats):
    P = pkg.VisualProblem(*[p[k] for k in VKEYS])
    off = pkg.visual_default_opts()
    off.function_tolerance = -1.0; off.parameter_tolerance = -1.0; off.gradient_tolerance = -1.0; off.max_iter = 1 << 30
    best, cost_k = None, None
    for _ in range(repeats + 1):                                 # the first run warms up
        P.reset_lm(off, linear_solver=solver); P.reset_state()
        s = P.iterate(passes)
        if best is None or s["ms_total"] < best["ms_total"]:
            best = s
        cost_k = s["cost_last"]
    P.reset_lm(off, linear_solver=solver); P.reset_state()
    per = []
    for _ in range(passes):                                      # the iterations of every solve
        P.iterate(1)
        per.append(P.linear_stats()["cg_iters_last"])
    P.reset_lm(linear_solver=solver); P.reset_state()
    conv = P.iterate(50)
    out = {"ms_solve": best["ms_solve"] / passes, "ms_build": best["ms_build"] / passes,
           "lm_passes_per_s": 1e3 * passes / best["ms_total"], f"cost_after_{passes}": cost_k,
           "passes_to_convergence": conv["iterations"], "termination": conv["termination"], "final_cost": conv["cost_last"],
           "n_blocks_env": P.counts()["n_blocks_env"]}
    if solver:
        out["cg_iters_mean"] = sum(per) / len(per)
        out["cg_iters_max"] = max(per)
    P.close()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--long", type=int, default=200)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scenes", default="config,long,loop")
    a = ap.parse_args(argv)
    names = set(a.scenes.split(","))
    if not names <= {"config", "long", "loop"}:
        ap.error(f"--scenes: unknown {sorted(names - {'config', 'long', 'loop'})}")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    pkg.load_library()
    if pkg.device_count() < 1:
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    gpu = _big().card()
    for name, p in scenes(names, a.config, a.long):
        for sname, solver in SOLVERS:
            r = measure(pkg, p, solver, a.passes, a.repeats)
            print(json.dumps({"scene": name, "solver": sname, "gpu": gpu, **r}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
