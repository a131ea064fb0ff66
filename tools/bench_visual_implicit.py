"""ITERATIVE_SCHUR on the product the plan chooses (lvba_visual_schur_product: the explicit S, or the matrix-free product through
the Jacobian blocks), measured on one GPU.  Prints one JSON line per scene:

    python tools/bench_visual_implicit.py [--config C] [--long 200] [--passes 10] [--repeats 3] [--scenes config,long,loop,street]

Scenes: the three of tools/bench_visual_pcg.py (the bench config as bench.py builds it; the same plus `--long` tracks of
200-1000 observations; a loop-closed scene of 400 cameras) and a street scene of 400 cameras from tests/visual_big_scene.py with
2000 short tracks and tracks of 300, 450, 600, 800 and 1000 observations.  Per scene, at Ceres' defaults with the stop tests off,
best of `repeats` runs of `--passes` LM passes after one warm-up: the rule's choice (matrix_free), ms_build, ms_solve and
ms_residual per pass, LM passes/s, the CG iterations per solve (mean and max), the bytes of the matrix-free records, and the
plan's counts.  The long-track scene's cost stays near 1e40 (its long tracks are far off), so its passes say nothing about LM
progress, only about time.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import importlib.util
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
SCENES = ("config", "long", "loop", "street")
# the matrix-free buffers (global-lvba_b200/csrc/visual_implicit.h): per observation a record of 24 doubles; per free observation
# its row-CSR entry (int64 observation, int32 landmark); per landmark its params (16 doubles), cost, gradient max and u (5 doubles);
# per camera row 32 lanes of 39 partials and the 6x6 diagonal block
REC, FREE, TRK, ROW = 24 * 8, 12, 21 * 8, (32 * 39 + 36) * 8


def _load(name):
    spec = importlib.util.spec_from_file_location(name, ROOT / "tools" / f"{name}.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def scenes(names, config, n_long):
    import visual_big_scene as vs
    out = _load("bench_visual_pcg").scenes(names & {"config", "long", "loop"}, config, n_long)
    if "street" in names:
        out.append(("street M=400", vs.make_scene(23, M=400, n_short=2000, long_tracks=((300, 10), (450, 80), (600, 150), (800, 200), (1000, 0)))))
    return out


def record_bytes(nnz, n_free, Tv, n_rows):
    return nnz * REC + n_free * FREE + Tv * TRK + n_rows * ROW + (n_rows + 1) * 8


def measure(pkg, p, passes, repeats):
    P = pkg.VisualProblem(*[p[k] for k in VKEYS])
    off = pkg.visual_default_opts()
    off.function_tolerance = -1.0; off.parameter_tolerance = -1.0; off.gradient_tolerance = -1.0; off.max_iter = 1 << 30
    best = None
    for _ in range(repeats + 1):                                 # the first run warms up
        P.reset_lm(off, linear_solver=1); P.reset_state()
        s = P.iterate(passes)
        if best is None or s["ms_total"] < best["ms_total"]:
            best = s
    P.reset_lm(off, linear_solver=1); P.reset_state()
    per = []
    for _ in range(passes):
        P.iterate(1)
        per.append(P.linear_stats()["cg_iters_last"])
    c = P.counts()
    n_rows = len(P.structure()[0])
    n_free = int(sum(len(x) for x in _free_obs(p, n_rows)))
    out = {"matrix_free": P.schur_product(), "ms_build": best["ms_build"] / passes, "ms_solve": best["ms_solve"] / passes,
           "ms_residual": best["ms_residual"] / passes, "lm_passes_per_s": 1e3 * passes / best["ms_total"],
           "cg_iters_mean": sum(per) / len(per), "cg_iters_max": max(per),
           "record_bytes": record_bytes(c["nnz_valid"], n_free, c["n_valid_tracks"], n_rows), "nnz": c["nnz_valid"],
           "free_obs": n_free, "n_pairs": c["n_pairs"], "n_blocks_env": c["n_blocks_env"], "n_rows": n_rows}
    P.close()
    return out


def _free_obs(p, n_rows):
    """The observations of the non-constant cameras (camera 0 is constant), per landmark with a usable plane."""
    import numpy as np
    op = np.asarray(p["obs_ptr"]); cam = np.asarray(p["obs_cam"]); pl = np.asarray(p["plane_nd"])
    ok = np.linalg.norm(pl[:, :3], axis=1) > 0
    return [cam[op[a]:op[a + 1]][cam[op[a]:op[a + 1]] != 0] for a in range(len(op) - 1) if ok[a]]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--long", type=int, default=200)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scenes", default=",".join(SCENES))
    a = ap.parse_args(argv)
    names = set(a.scenes.split(","))
    if not names <= set(SCENES):
        ap.error(f"--scenes: unknown {sorted(names - set(SCENES))}")
    import __graft_entry__ as graft
    pkg = graft.load_package()
    pkg.load_library()
    if pkg.device_count() < 1:
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    gpu = _load("bench_visual_big").card()
    for name, p in scenes(names, a.config, a.long):
        r = measure(pkg, p, a.passes, a.repeats)
        print(json.dumps({"scene": name, "gpu": gpu, **r}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
