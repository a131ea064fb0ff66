"""The two trust-region strategies of the visual LM (lvba_visual_opts::trust_region_strategy), measured on one GPU.  Prints one
JSON line per scene and strategy:

    python tools/bench_visual_dogleg.py [--config C] [--long 200] [--repeats 2] [--scenes config,long,loop]

Scenes as tools/bench_visual_pcg.py builds them: the visual problem of the bench config, the same plus `--long` tracks of
200-1000 observations, and the loop-closed scene of 400 cameras.  Per scene and strategy (LEVENBERG_MARQUARDT, then DOGLEG),
DENSE_SCHUR, Ceres' default tolerances, a solve of at most 50 passes run one pass per lvba_visual_iterate call (best of
`repeats` runs after one warm-up): LM passes/s, builds per pass, the rejected passes (not the last one), ms per pass after a
rejection (under DOGLEG the pass that reuses the linearisation), ms per pass otherwise, the passes to stop, the termination and
the final cost.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import importlib.util
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
STRATEGIES = (("levenberg_marquardt", 0), ("dogleg", 1))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, ROOT / "tools" / f"{name}.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def solve(P, strategy, max_passes=50):
    """One solve at the default tolerances, one pass per call: per-pass (ms, accepted, builds) and the last summary"""
    P.reset_lm(trust_region_strategy=strategy); P.reset_state()
    passes, last = [], None
    for _ in range(max_passes):
        s = P.iterate(1)
        if s["iterations"] == 0:
            break
        passes.append((s["ms_total"], s["accepted"], s["hessian_builds"]))
        last = s
        if s["termination"] != 0:
            break
    return passes, last


def measure(pkg, p, strategy, repeats):
    P = pkg.VisualProblem(*[p[k] for k in VKEYS])
    best = None
    for _ in range(repeats + 1):                                 # the first run warms up
        passes, last = solve(P, strategy)
        if best is None or sum(m for m, _, _ in passes) < sum(m for m, _, _ in best[0]):
            best = (passes, last)
    P.close()
    passes, last = best
    n = len(passes)
    ms = [m for m, _, _ in passes]
    after = [ms[i] for i in range(1, n) if passes[i - 1][1] == 0]
    other = [ms[i] for i in range(n) if i == 0 or passes[i - 1][1] != 0]
    return {"lm_passes_per_s": 1e3 * n / sum(ms) if n else 0.0, "builds_per_pass": sum(b for _, _, b in passes) / max(n, 1),
            "rejected": sum(1 for _, a, _ in passes[:-1] if a == 0), "ms_after_reject": sum(after) / len(after) if after else None,
            "ms_other": sum(other) / len(other) if other else None, "passes_to_stop": n,
            "termination": last["termination"] if last else None, "final_cost": last["cost_last"] if last else None}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--long", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=2)
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
    gpu = _load("bench_visual_big").card()
    for name, p in _load("bench_visual_pcg").scenes(names, a.config, a.long):
        for sname, strategy in STRATEGIES:
            r = measure(pkg, p, strategy, a.repeats)
            print(json.dumps({"scene": name, "strategy": sname, "gpu": gpu, **r}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
