"""The robust losses through the two C++ callers of the visual LM, on the H100:
- lvba_b200::solve_visual (global-lvba_b200/host/lvba_shim.hpp) with the reference's Huber losses equals lvba_visual_lm with the
  same opts, bit for bit in deterministic mode (tests/shim/visual_loss_shim.cpp);
- `lvba_offline --visual --reproj-loss huber --plane-loss huber` on the scene of tests/test_zz_offline_gpu.py: the problem its
  visual stage solved (--visual-problem) goes through the restated Ceres LM with the same losses (tests/visual_loss_oracle.py),
  which must give the tool's cameras, iterations and costs."""
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import synth
import visual_big_scene as vs
import visual_loss_oracle as vl

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


def write_problem(path, p):
    """A problem dict (visual_big_scene.KEYS) in the layout of write_visual_problem, the state after = the state before."""
    M, T, nnz = len(p["q"]), len(p["X"]), len(p["obs_cam"])
    f64 = lambda a: np.ascontiguousarray(a, np.float64).tobytes()  # noqa: E731
    state = f64(p["q"]) + f64(p["t"]) + f64(p["X"])
    Path(path).write_bytes(b"LVBAVP01" + np.array([M, T, nnz], np.int64).tobytes() + f64(p["intr"])
                           + f64([p["sigma_px"], p["sigma_plane"]]) + state + f64(p["plane_nd"])
                           + np.ascontiguousarray(p["obs_ptr"], np.int64).tobytes() + np.ascontiguousarray(p["obs_cam"], np.int32).tobytes()
                           + np.ascontiguousarray(p["obs_uv"], np.float32).tobytes() + state)


def read_problem(path):
    """write_visual_problem's file: (problem dict with the state before the solve, (q, t, X) after it)."""
    b = Path(path).read_bytes()
    assert b[:8] == b"LVBAVP01"
    M, T, nnz = np.frombuffer(b, np.int64, 3, 8)
    o = 32

    def take(dtype, n, shape):
        nonlocal o
        a = np.frombuffer(b, dtype, int(n), o).reshape(shape).copy()
        o += a.nbytes
        return a
    intr = take(np.float64, 8, (8,)); sig = take(np.float64, 2, (2,))
    p = dict(q=take(np.float64, 4 * M, (M, 4)), t=take(np.float64, 3 * M, (M, 3)), X=take(np.float64, 3 * T, (T, 3)))
    p.update(plane_nd=take(np.float64, 4 * T, (T, 4)), obs_ptr=take(np.int64, T + 1, (T + 1,)), obs_cam=take(np.int32, nnz, (nnz,)),
             obs_uv=take(np.float32, 2 * nnz, (nnz, 2)), intr=intr, sigma_px=float(sig[0]), sigma_plane=float(sig[1]))
    after = (take(np.float64, 4 * M, (M, 4)), take(np.float64, 3 * M, (M, 3)), take(np.float64, 3 * T, (T, 3)))
    assert o == len(b)
    return p, after


def test_shim_solve_visual_with_huber_equals_visual_lm(gpu_pkg, tmp_path):
    exe = tmp_path / "visual_loss_shim"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I", str(ROOT / "include"), str(ROOT / "tests" / "shim" / "visual_loss_shim.cpp"),
                        "-o", str(exe), *_link(gpu_pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    p = vl.with_outliers(synth.make_problem(30, 0, 300, seed=11, lidar=False), 0.05, 20.0, 50.0, 11)[0]
    write_problem(tmp_path / "in.bin", p)
    r = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    b = (tmp_path / "out.bin").read_bytes()
    M, T = len(p["q"]), len(p["X"])
    o = gpu_pkg.visual_default_opts(reproj_loss=gpu_pkg.LOSS_HUBER, plane_loss=gpu_pkg.LOSS_HUBER)
    o.deterministic = 1
    q, t, X, s = gpu_pkg.visual_lm(*vs.args(p), fixed_cam=0, opts=o)
    assert b[:M * 56 + T * 24] == q.tobytes() + t.tobytes() + X.tobytes()
    ints = np.frombuffer(b, np.int32, 3, M * 56 + T * 24)
    costs = np.frombuffer(b, np.float64, 2, M * 56 + T * 24 + 12)
    assert list(ints) == [s["iterations"], s["accepted"], s["termination"]] and s["accepted"] > 0
    assert costs[0] == s["cost_first"] and costs[1] == s["cost_last"]
    # it is the robust solve: cost_first is 1/2 sum rho of the reference's Huber losses, below the plain 1/2 sum r^2
    pr = vl.RobustProblem(*vs.args(p), loss_reproj=(vl.HUBER, 1.0), loss_plane=(vl.HUBER, 0.1))
    assert abs(costs[0] - pr.cost()) <= 1e-10 * pr.cost() and pr.cost() < vl.RobustProblem(*vs.args(p)).cost()


def test_offline_visual_stage_with_losses_matches_oracle(gpu_pkg, tmp_path):
    import visual_scene
    exe = tmp_path / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(gpu_pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    data = tmp_path / "data"
    visual_scene.make(data, seed=3, W=8, n_landmarks=700)
    prob = tmp_path / "visual.bin"
    r = subprocess.run([str(exe), "--data", str(data), "--config", str(data / "config.yaml"), "--visual", "--reproj-loss", "huber",
                        "--plane-loss", "huber", "--visual-problem", str(prob)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    vis = [x for x in (json.loads(ln) for ln in r.stdout.strip().splitlines()) if x.get("stage") == "visual"][0]
    p, (q1, t1, X1) = read_problem(prob)
    assert int(vl.vo.valid_tracks(p["plane_nd"]).sum()) == vis["points_kept"] and vis["points_kept"] >= 80
    pr, info = vl.ceres_lm(vl.RobustProblem(*vs.args(p), fixed_cam=0, loss_reproj=(vl.HUBER, 1.0), loss_plane=(vl.HUBER, 0.1)))
    plain = vl.RobustProblem(*vs.args(p), fixed_cam=0).cost()
    assert info["cost0"] < (1 - 1e-6) * plain                     # the losses change the cost: the flags reached the solve
    assert vis["iterations"] == info["iters"] and vis["termination"] == vl.TERM[info["term"]]
    assert abs(vis["cost_first"] - info["cost0"]) <= 1e-9 * info["cost0"]
    assert abs(vis["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    assert np.abs(q1 - pr.q).max() <= 1e-6 and np.abs(t1 - pr.t).max() <= 1e-6
