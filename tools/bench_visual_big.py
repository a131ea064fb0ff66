"""Path B with landmarks of more than 128 observations, measured on one GPU.  Prints one JSON line per problem:

    python tools/bench_visual_big.py [--config C] [--long 200] [--kmin 200] [--kmax 1000] [--iters 5] [--repeats 3]

1. the visual problem of the bench config as bench.py builds it (every track 3-8 observations: no big landmark);
2. the same problem plus `--long` tracks of kmin..kmax observations over (near-)consecutive cameras that see a point 100 m
   ahead of the middle camera (landmarks that take the passes of global-lvba_b200/csrc/visual_big.h).

Per problem: lvba_summary ms_build / ms_solve / ms_residual per LM pass (best of `repeats` runs of `iters` passes of
lvba_visual_iterate, stop tests off), ms_setup of lvba_visual_lm, lvba_visual_big_counts, the LDL^T path AUTO takes for the
reduced camera system, and the algorithmic bytes of the big passes per LM pass computed from the counts.  The card's name,
power limit and max SM clock are read in the same run."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
PATHS = {1: "one_cta", 2: "twisted", 3: "chunked", 4: "shared_window", 5: "any_width"}   # LVBA_SOLVE_*


def big_pass_bytes(n_big, n_obs, n_pairs):
    """Algorithmic bytes of the big passes per LM pass (build + back-substitution + candidate cost), from the layout of
    visual_big.h: per observation record kObs = 65 doubles, per landmark kTrkParams = 16 doubles; a pair item reads two
    observation rows (8 B), Y_x and E_y (288 B) and adds one 6x6 block (288 B) when it contributes."""
    obs_in = 4 + 4 + 8 + 32 + 24 + 24 + 24 + 48          # camera, row, uv, q, t, X, s_pt, s_cam
    per_obs = (obs_in + 29 * 8                            # ObsF: inputs -> r, J_c, J_X, J_X^T J_X, J_X^T r
               + 11 * 8                                   # TrackF: r and the stage sums
               + 20 * 8 + 4 + 16 + 36 * 8 + 54 * 8        # SlotsF: record, row, envelope row -> Y, E; 54 element REDs
               + 2 * (20 * 8 + 4 + 48)                    # BacksubF: two sweeps over record, row, y_c
               + (4 + 8 + 56))                            # CostF: camera, uv, q, t
    per_trk = (32 + 24 + 24 + 16 * 8 + 16                 # TrackF: plane, X, s_pt -> params, partial slots
               + 16 * 8 + 32 + 24 * 3 + 32                # BacksubF: params, plane, X / X_cand / pt_step, partial slot
               + 32 + 24 + 8)                             # CostF
    per_pair = 8 + 2 * 18 * 8 + 36 * 8
    return int(n_obs * per_obs + n_big * per_trk + n_pairs * per_pair)


def add_long_tracks(p, n_long, kmin, kmax, seed=5):
    """Tracks of kmin..kmax observations: a point 100 m ahead of a middle camera, seen by the nearest cameras (in index order)
    that have it in front (z > 1 m), pixel noise 0.5 px."""
    from oracle import synth, visual_oracle as vo
    rng = np.random.default_rng(seed)
    q, t = p["q_gt"], p["t_gt"]
    R = vo.quat_to_rot(q)
    M = len(q)
    cams, Xs = [], []
    for _ in range(n_long):
        K = int(rng.integers(kmin, kmax + 1))
        c = int(rng.integers(0, M))
        X = R[c].T @ (np.array([rng.uniform(-20, 20), rng.uniform(-5, 5), 100.0]) - t[c])
        z = np.einsum("nj,nj->n", R[:, 2, :], X[None]) + t[:, 2]
        ok = np.nonzero(z > 1.0)[0]
        sel = np.sort(ok[np.argsort(np.abs(ok - c), kind="stable")[:K]])
        cams.append(sel); Xs.append(X)
    obs_cam = np.concatenate(cams).astype(np.int32)
    trk = np.repeat(np.arange(n_long), [len(c) for c in cams])
    Xg = np.array(Xs)
    uv, _ = synth.project(R[obs_cam], t[obs_cam], Xg[trk])
    uv = (uv + rng.normal(0, 0.5, uv.shape)).astype(np.float32)
    n = rng.normal(size=(n_long, 3)); n /= np.linalg.norm(n, axis=1, keepdims=True)
    out = dict(p)
    nnz = p["obs_ptr"][-1]
    out["obs_ptr"] = np.concatenate([p["obs_ptr"], nnz + np.cumsum([len(c) for c in cams])]).astype(np.int64)
    out["obs_cam"] = np.concatenate([p["obs_cam"], obs_cam]).astype(np.int32)
    out["obs_uv"] = np.concatenate([p["obs_uv"], uv]).astype(np.float32)
    out["X"] = np.concatenate([p["X"], Xg + rng.normal(0, 0.05, Xg.shape)])
    out["plane_nd"] = np.concatenate([p["plane_nd"], np.concatenate([n, -np.einsum("ni,ni->n", n, Xg)[:, None]], 1)])
    return out


def card():
    try:
        import torch
        name = torch.cuda.get_device_name(0)
    except Exception:
        name = None
    info = {"name": name, "power_limit_w": None, "sm_clock_max_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = r.stdout.strip().split(",")[:2]
        info["power_limit_w"], info["sm_clock_max_mhz"] = float(pl), float(mx)
    except Exception:
        pass
    return info


def measure(pkg, p, iters, repeats):
    P = pkg.VisualProblem(*[p[k] for k in VKEYS])
    bc, cnt = P.big_counts(), P.counts()
    opts = pkg.visual_default_opts()
    opts.function_tolerance = -1.0; opts.parameter_tolerance = -1.0; opts.gradient_tolerance = -1.0; opts.max_iter = 1 << 30
    best = None
    for _ in range(repeats + 1):                                 # the first run warms up
        P.reset_lm(opts); P.reset_state()
        s = P.iterate(iters)
        per = {k: s[k] / max(s["iterations"], 1) for k in ("ms_build", "ms_solve", "ms_residual")}
        if best is None or sum(per.values()) < sum(best.values()):
            best = per
    P.reset_state()
    P.step(1e4)
    cam, rhs, br, bcol, blocks = P.get_system()
    n = len(cam)
    first = np.arange(n)
    np.minimum.at(first, br, bcol)
    _, _, info = pkg.env_solve(first, blocks, np.full(6 * n, 1.0), rhs.ravel())
    P.close()
    o1 = pkg.visual_default_opts(); o1.max_iter = 1
    setups = [pkg.visual_lm(*[p[k] for k in VKEYS], opts=o1)[3]["ms_setup"] for _ in range(repeats)]
    return {"tracks": int(len(p["obs_ptr"]) - 1), "nnz": int(p["obs_ptr"][-1]), "big_counts": bc, "n_pairs": cnt["n_pairs"],
            "ms_per_pass": best, "ms_setup": min(setups), "solve_path": PATHS.get(info["path"], info["path"]),
            "big_pass_bytes": big_pass_bytes(bc["n_big"], bc["n_big_obs"], bc["n_big_pairs"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C")
    ap.add_argument("--long", type=int, default=200)
    ap.add_argument("--kmin", type=int, default=200)
    ap.add_argument("--kmax", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as graft
    from oracle import synth
    pkg = graft.load_package()
    pkg.load_library()
    if pkg.device_count() < 1:
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    gpu = card()
    p = synth.make_config(a.config, lidar=False)
    for name, prob in (("config", p), ("config+long", add_long_tracks(p, a.long, a.kmin, a.kmax))):
        r = measure(pkg, prob, a.iters, a.repeats)
        print(json.dumps({"problem": f"{a.config} {name}", "gpu": gpu, **r}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
