"""Constant cameras in the visual LM (lvba_visual_opts::cam_fixed) on the H100: the one-shot call and the handle's re-planning reset
against the oracle with the same constant set (tests/visual_fixed_oracle.py) at the tolerances of tests/test_visual_gpu.py, the
mask {0} against fixed_cam = 0 bit for bit, constant cameras returned bit-identical, every camera constant (only the landmarks
move), landmarks of more than 128 observations, the Huber loss with a mask, and lvba_offline --fix-cameras."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_fixed_oracle as vf
import visual_loss_oracle as vl
from test_visual_big_gpu import _mixed

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
SUMMARY_KEYS = ("iterations", "accepted", "hessian_builds", "termination", "cost_first", "cost_last", "damping_last")


def _opts(pkg, deterministic=0, losses=(None, None)):
    o = pkg.visual_default_opts(reproj_loss=losses[0], plane_loss=losses[1])
    o.deterministic = deterministic
    return o


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and all(a[3][k] == b[3][k] for k in SUMMARY_KEYS)


@pytest.mark.parametrize("deterministic", [1, 0])
def test_mask_of_camera_0_equals_fixed_cam_0(gpu_pkg, problem_small, deterministic):
    """cam_fixed = {0} with fixed_cam = -1 plans the same rows as fixed_cam = 0: the same solve, bit for bit in deterministic mode."""
    args = vs.args(problem_small)
    o = _opts(gpu_pkg, deterministic)
    a = gpu_pkg.visual_lm(*args, fixed_cam=0, opts=o)
    b = gpu_pkg.visual_lm(*args, fixed_cam=-1, opts=o, cam_fixed=vf.mask_of(len(args[0]), [0]))
    if deterministic:
        assert _same(a, b)
    else:
        assert a[3]["iterations"] == b[3]["iterations"] and abs(a[3]["cost_last"] - b[3]["cost_last"]) <= 1e-9 * a[3]["cost_last"]


@pytest.mark.parametrize("cams", [(0, 5, 17), tuple(range(15))], ids=["three", "first_half"])
def test_lm_with_constant_set_matches_oracle(gpu_pkg, problem_small, cams):
    p = problem_small
    args = vs.args(p)
    M = len(p["q"])
    q, t, X, s = gpu_pkg.visual_lm(*args, fixed_cam=-1, cam_fixed=vf.mask_of(M, cams))
    pr, info = vo.ceres_lm(vf.with_constant(vo.VisualProblem(*args, fixed_cam=-1), cams))
    assert s["iterations"] == info["iters"] and s["accepted"] == info["accepted"]
    assert abs(s["cost_first"] - info["cost0"]) <= 1e-10 * info["cost0"]
    assert abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    assert np.abs(q - pr.q).max() <= 1e-6 and np.abs(t - pr.t).max() <= 1e-6 and np.abs(X - pr.X).max() <= 1e-6
    c = list(cams)
    assert np.array_equal(q[c], p["q"][c]) and np.array_equal(t[c], p["t"][c])       # constant cameras come back as they went in
    free = np.setdiff1d(np.arange(M), c)
    assert np.abs(q[free] - p["q"][free]).max() > 0


@pytest.mark.parametrize("cams", [(0, 5, 17), tuple(range(0, 400, 2))], ids=["three", "every_other"])
def test_step_and_system_with_big_landmarks(gpu_pkg, cams):
    """The mixed scene (landmarks of 128 to 1000 observations): step and reduced camera system of a handle re-planned by its reset."""
    p = _mixed()
    args = vs.args(p)
    P = gpu_pkg.VisualProblem(*args, fixed_cam=-1)
    P.reset_lm(cam_fixed=vf.mask_of(len(p["q"]), cams))
    pr = vf.with_constant(vo.VisualProblem(*args, fixed_cam=-1), cams)
    assert P.big_counts()["n_big"] == 3
    cs, ps, model, cost = P.step(1e4)
    ref = vo.single_step(pr, 1e4, True)
    assert abs(cost - ref["cost"]) <= 1e-10 * ref["cost"]
    assert abs(model - ref["model"]) <= 1e-7 * abs(ref["model"])
    assert np.abs(cs - ref["cam_step"]).max() <= 1e-6 * np.abs(ref["cam_step"]).max()
    assert np.abs(ps - ref["pt_step"]).max() <= 1e-6 * np.abs(ref["pt_step"]).max()
    assert np.all(cs[list(cams)] == 0)
    cam, rhs, br, bc, bl = P.get_system()
    assert np.array_equal(cam, np.nonzero(pr.cam_active)[0])
    S = gpu_pkg.env_blocks_to_dense(br, bc, bl, len(cam))
    assert np.abs(S - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
    assert np.abs(rhs.ravel() - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    P.close()


@pytest.mark.parametrize("deterministic", [0, 1])
def test_every_camera_constant_moves_the_landmarks_only(gpu_pkg, problem_small, deterministic):
    """No system row: lvba_visual_step writes zero camera steps and the step of the eliminated point blocks alone; the LM moves the
    landmarks as the oracle's LM on the point blocks does."""
    p = problem_small
    args = vs.args(p)
    M = len(p["q"])
    allc = np.ones(M, bool)
    P = gpu_pkg.VisualProblem(*args, fixed_cam=-1)
    P.reset_lm(_opts(gpu_pkg, deterministic), cam_fixed=allc)
    cam, br, bc = P.structure()
    assert len(cam) == 0 and len(br) == 0
    pr = vf.with_constant(vo.VisualProblem(*args, fixed_cam=-1), range(M))
    cs, ps, model, cost = P.step(1e4)
    ref = vo.single_step(pr, 1e4, True)
    assert np.all(cs == 0)
    assert abs(cost - ref["cost"]) <= 1e-10 * ref["cost"] and abs(model - ref["model"]) <= 1e-7 * abs(ref["model"])
    assert np.abs(ps - ref["pt_step"]).max() <= 1e-6 * np.abs(ref["pt_step"]).max()
    P.close()
    q, t, X, s = gpu_pkg.visual_lm(*args, fixed_cam=-1, opts=_opts(gpu_pkg, deterministic), cam_fixed=allc)
    pr, info = vo.ceres_lm(vf.with_constant(vo.VisualProblem(*args, fixed_cam=-1), range(M)))
    assert np.array_equal(q, p["q"]) and np.array_equal(t, p["t"])
    assert s["iterations"] == info["iters"] and abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    assert s["cost_last"] < s["cost_first"] and np.abs(X - pr.X).max() <= 1e-6


@pytest.mark.parametrize("deterministic", [1, 0])
def test_handle_reset_replans_to_each_mask(gpu_pkg, problem_small, deterministic):
    """Reset with mask A, then none, then B: after each, iterate equals a fresh one-shot with that mask (bit for bit in
    deterministic mode); two runs of the same handle give the same bytes."""
    p = problem_small
    args = vs.args(p)
    M = len(p["q"])
    o = _opts(gpu_pkg, deterministic)
    P = gpu_pkg.VisualProblem(*args, fixed_cam=0)
    for mask in (vf.mask_of(M, [3, 4, 20]), None, vf.mask_of(M, range(10, 30)), np.zeros(M, bool)):
        runs = []
        for _ in range(2):
            P.reset_state()
            P.reset_lm(o, cam_fixed=mask)
            s = P.iterate(o.max_iter)
            runs.append((*P.get_state(), s))
        one = gpu_pkg.visual_lm(*args, fixed_cam=0, opts=o, cam_fixed=mask)
        if deterministic:
            assert _same(runs[0], runs[1]) and _same(runs[0], one)
        else:
            assert runs[0][3]["iterations"] == one[3]["iterations"]
            assert abs(runs[0][3]["cost_last"] - one[3]["cost_last"]) <= 1e-9 * one[3]["cost_last"]
        if mask is not None and mask.any():
            assert np.array_equal(runs[0][0][mask], p["q"][mask]) and np.array_equal(runs[0][1][mask], p["t"][mask])
    P.close()


def test_huber_with_constant_set_matches_oracle(gpu_pkg):
    p = vl.with_outliers(vs.make_scene(5, M=40, n_short=300), 0.05, 20.0, 50.0, 5)[0]
    args = vs.args(p)
    cams = (0, 7, 8, 9)
    losses = ((vl.HUBER, 1.0), (vl.HUBER, 0.1))
    q, t, X, s = gpu_pkg.visual_lm(*args, fixed_cam=-1, opts=_opts(gpu_pkg, 0, losses), cam_fixed=vf.mask_of(40, cams))
    pr = vf.with_constant(vl.RobustProblem(*args, fixed_cam=-1, loss_reproj=losses[0], loss_plane=losses[1]), cams)
    pr, info = vo.ceres_lm(pr)
    assert s["iterations"] == info["iters"]
    assert abs(s["cost_first"] - info["cost0"]) <= 1e-10 * info["cost0"]
    assert abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    assert np.array_equal(q[list(cams)], p["q"][list(cams)]) and np.array_equal(t[list(cams)], p["t"][list(cams)])


def test_offline_fix_cameras(tmp_path):
    """lvba_offline --no-lidar --visual --fix-cameras 0:3: the images.txt lines of cameras 0-3 equal their input (the odometry
    cameras, images_before.txt) to the printed digits, and the other cameras move."""
    import __graft_entry__ as graft
    sys.path.insert(0, str(ROOT / "tests"))
    import visual_scene
    pkg = graft.load_package()
    exe = tmp_path / "lvba_offline"
    cmd = ["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
           str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]
    assert subprocess.run(cmd, capture_output=True, text=True).returncode == 0
    data = tmp_path / "data"
    visual_scene.make(data, seed=3, W=8, n_landmarks=700)
    r = subprocess.run([str(exe), "--data", str(data), "--config", str(data / "config.yaml"), "--no-lidar", "--visual", "--fix-cameras", "0:3"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    vis = [json.loads(x) for x in r.stdout.strip().splitlines() if '"visual"' in x][0]
    assert vis["iterations"] >= 1
    after = (data / "Colmap" / "sparse" / "images.txt").read_text().splitlines()
    before = (data / "Colmap" / "sparse" / "images_before.txt").read_text().splitlines()
    assert len(after) == len(before) == 16
    for k in range(8):
        a, b = np.array(after[2 * k].split()[1:8], float), np.array(before[2 * k].split()[1:8], float)
        if k < 4:
            assert np.abs(a - b).max() <= 2e-6, (k, after[2 * k], before[2 * k])
        else:
            assert np.abs(a - b).max() > 2e-6, k


def test_offline_fix_cameras_no_op_keeps_the_output(tmp_path):
    """--fix-cameras 0 names only the camera the reference already holds constant: with --deterministic, images.txt, points3D.txt
    and the trajectory are byte-identical to a run without the flag."""
    import __graft_entry__ as graft
    sys.path.insert(0, str(ROOT / "tests"))
    import visual_scene
    pkg = graft.load_package()
    exe = tmp_path / "lvba_offline"
    cmd = ["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
           str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]
    assert subprocess.run(cmd, capture_output=True, text=True).returncode == 0
    outs = []
    for extra in ([], ["--fix-cameras", "0"]):
        data = tmp_path / f"data{len(outs)}"
        visual_scene.make(data, seed=3, W=8, n_landmarks=700)
        r = subprocess.run([str(exe), "--data", str(data), "--config", str(data / "config.yaml"), "--visual", "--deterministic", *extra],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outs.append({f: (data / f).read_bytes() for f in ("Colmap/sparse/images.txt", "Colmap/sparse/points3D.txt",
                                                          "all_pcd_body/lidar_poses_optimized.txt")})
    assert outs[0] == outs[1]
