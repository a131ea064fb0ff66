"""Landmarks with more than 128 observations on the H100 (global-lvba_b200/csrc/visual_big.h): they leave the tiles and batches
and take their own passes.  Cost, step, reduced camera system and the full LM against oracle/visual_oracle.py at the tolerances
of tests/test_visual_gpu.py, the boundary 128 / 129, and the off-ROS shim call that used to refuse such a problem."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import visual_oracle as vo
import visual_big_scene as vs

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _mixed():
    """A problem_small-sized scene plus tracks of 128, 129, 300 and 1000 observations over consecutive cameras (1000 > the 400
    cameras: that track sees most cameras two or three times) and one that sees camera 3 three times."""
    p = vs.make_scene(17, M=400, n_short=300, long_tracks=((128, 5), (129, 20), (300, 60), (1000, 0)),
                      extra_tracks=([3, 3, 4, 3, 5],))
    return p


def _check_step(gpu_pkg, p, fixed_cam, n_big):
    P = gpu_pkg.VisualProblem(*vs.args(p), fixed_cam=fixed_cam)
    pr = vo.VisualProblem(*vs.args(p), fixed_cam=fixed_cam)
    K = np.diff(p["obs_ptr"])[pr.tv]
    bc = P.big_counts()
    assert bc == dict(n_big=int((K > 128).sum()), n_big_obs=int(K[K > 128].sum()), n_big_pairs=int((K[K > 128] * (K[K > 128] - 1)).sum()))
    assert bc["n_big"] == n_big
    assert abs(P.cost() - pr.cost()) <= 1e-10 * pr.cost()
    cs, ps, model, cost = P.step(1e4)
    ref = vo.single_step(pr, 1e4, True)
    assert abs(cost - ref["cost"]) <= 1e-10 * ref["cost"]
    assert abs(model - ref["model"]) <= 1e-7 * abs(ref["model"])
    assert np.abs(cs - ref["cam_step"]).max() <= 1e-6 * np.abs(ref["cam_step"]).max()
    assert np.abs(ps - ref["pt_step"]).max() <= 1e-6 * np.abs(ref["pt_step"]).max()
    cam, rhs, br, bc_, bl = P.get_system()
    S = gpu_pkg.env_blocks_to_dense(br, bc_, bl, len(cam))
    assert np.array_equal(cam, np.nonzero(pr.cam_active)[0])
    assert np.abs(S - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
    assert np.abs(rhs.ravel() - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    # the candidate cost, through lvba_visual_cost at the oracle's candidate state
    qn, tn, Xn = pr.plus(np.concatenate([ref["cam_step"][pr.cam_active].ravel(), ref["pt_step"][pr.tv].ravel()]))
    P.set_state(qn, tn, Xn)
    c2 = pr.cost(qn, tn, Xn)
    assert abs(P.cost() - c2) <= 1e-10 * c2
    P.close()


@pytest.mark.parametrize("order", ["caller", "shuffled"])
@pytest.mark.parametrize("fixed_cam", [0, -1])
def test_mixed_scene_step_matches(gpu_pkg, fixed_cam, order):
    p = _mixed()
    if order == "shuffled":
        p, _ = vs.shuffled(p, 3)
    _check_step(gpu_pkg, p, fixed_cam, n_big=3)


def test_full_lm_matches_oracle(gpu_pkg):
    """visual_lm against the restated Ceres LM; landmarks without a valid plane (a long one among them) stay untouched."""
    p = vs.make_scene(23, M=300, n_short=250, long_tracks=((129, 0), (300, 0), (700, 100), (150, 40)))
    p["plane_nd"][::13, :3] = 0.0
    p["plane_nd"][-1, :3] = 0.0                                  # the 150-observation track has no valid plane
    P = gpu_pkg.VisualProblem(*vs.args(p))
    assert P.big_counts()["n_big"] == 3
    P.close()
    q, t, X, s = gpu_pkg.visual_lm(*vs.args(p))
    pr, info = vo.ceres_lm(vo.VisualProblem(*vs.args(p)))
    assert s["iterations"] == info["iters"]
    assert s["accepted"] == info["accepted"]
    assert abs(s["cost_first"] - info["cost0"]) <= 1e-10 * info["cost0"]
    assert abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    skipped = ~vo.valid_tracks(p["plane_nd"])
    assert skipped[-1] and np.array_equal(X[skipped], p["X"][skipped])
    assert np.array_equal(q[0], p["q"][0]) and np.array_equal(t[0], p["t"][0])


def test_boundary_128_and_129_observations(gpu_pkg):
    """A longest track of exactly 128 observations takes the tiles; one more observation of that track sends it to the big
    passes.  Each problem matches its own oracle."""
    p = vs.make_scene(31, M=200, n_short=200, long_tracks=((128, 30),))
    _check_step(gpu_pkg, p, 0, n_big=0)
    a = len(p["obs_ptr"]) - 2                                     # the long track is the last landmark
    lo = p["obs_ptr"][a + 1]
    extra_cam = int(p["obs_cam"][lo - 1]) + 1
    uv = p["obs_uv"][lo - 1] + np.array([1.5, -0.5], np.float32)
    q = dict(p)
    q["obs_cam"] = np.concatenate([p["obs_cam"][:lo], [extra_cam], p["obs_cam"][lo:]]).astype(np.int32)
    q["obs_uv"] = np.concatenate([p["obs_uv"][:lo], uv[None], p["obs_uv"][lo:]]).astype(np.float32)
    q["obs_ptr"] = p["obs_ptr"].copy(); q["obs_ptr"][a + 1:] += 1
    assert np.diff(q["obs_ptr"]).max() == 129
    _check_step(gpu_pkg, q, 0, n_big=1)


def test_shim_solves_a_long_track(gpu_pkg, tmp_path):
    """lvba_b200::solve_visual with one landmark seen 300 times returns LVBA_OK (it used to refuse the whole problem)."""
    exe = tmp_path / "visual_long_track"
    cmd = ["g++", "-std=c++17", "-O1", "-I", str(ROOT / "include"), str(ROOT / "tests" / "shim" / "visual_long_track.cpp"),
           "-o", str(exe), str(gpu_pkg.LIB_PATH), f"-Wl,-rpath,{gpu_pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok:")
