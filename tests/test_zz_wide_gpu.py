"""The any-width LDL^T (global-lvba_b200/csrc/envelope_wide.h) on the GPU: (1) forced onto a banded problem it must reproduce
the in-SM solvers' step; (2) a problem with loop-closure couplings (envelope columns taller than the 320 blocks the
shared-memory kernel holds — LVBA_ERR_UNSUPPORTED before this path existed) must follow the oracle's LM, which solves the
full normal equations with a sparse LU.  The arithmetic of the passes is checked without a GPU in
tests/test_wide_solver_emu.py."""
import os
import subprocess
import sys
import textwrap
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


PRELUDE = """
import os, sys
import numpy as np
sys.path.insert(0, %r)
import __graft_entry__ as graft
from oracle import synth, lidar_oracle as lo
pkg = graft.load_package(); pkg.load_library()
assert pkg.device_count() >= 1
""" % str(ROOT)


def _run(body, env=None, timeout=600):
    code = PRELUDE + textwrap.dedent(body) + "\nprint('CHILD-OK')\n"
    e = dict(os.environ); e.update(env or {})
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, cwd=str(ROOT), env=e)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    return r.stdout


@pytest.mark.gpu
def test_forced_wide_path_reproduces_the_banded_step(gpu_pkg):
    import numpy as np
    import solver_systems as ss
    from oracle import synth
    pkg = gpu_pkg
    p = synth.make_problem(60, 900, 400, seed=21)
    # LiDAR: the any-width path on the pose system against the LM step (an in-SM path)
    P = pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"]); P.build()
    g, br, bc, bl = P.get_system()
    dx = P.solve(0.01); P.close()
    first, dadd = ss.damped(br, bc, bl, P.W, 0.01)
    xw, _, info = pkg.env_solve(first, bl, dadd, -g.ravel(), path=pkg.SOLVE_ANY_WIDTH)
    assert info["path"] == pkg.SOLVE_ANY_WIDTH
    assert np.abs(xw - dx).max() <= 1e-9 * np.abs(dx).max()
    # visual: the reduced camera system at the initial state and after a few LM iterations, any-width against AUTO
    V = pkg.VisualProblem(p["q"], p["t"], p["X"], p["plane_nd"], p["obs_ptr"], p["obs_cam"], p["obs_uv"], p["intr"], p["sigma_px"], p["sigma_plane"])
    V.step(1e4)
    systems = [V.get_system()]
    V.iterate(3)
    systems.append(V.get_system())
    V.close()
    for k, (cam, rhs, br, bc, bl) in enumerate(systems):
        first, dadd = ss.damped(br, bc, bl, len(cam), 1e-4)
        xa, _, ia = pkg.env_solve(first, bl, dadd, rhs.ravel())
        xw, _, iw = pkg.env_solve(first, bl, dadd, rhs.ravel(), path=pkg.SOLVE_ANY_WIDTH)
        assert ia["path"] != pkg.SOLVE_ANY_WIDTH and iw["path"] == pkg.SOLVE_ANY_WIDTH
        assert np.abs(xw - xa).max() <= 1e-9 * np.abs(xa).max(), (k, np.abs(xw - xa).max() / np.abs(xa).max())


@pytest.mark.gpu
def test_loop_closure_problem_follows_the_oracle():
    _run("""
    p = synth.make_problem(360, 2500, 0, seed=5, visual=False, half=350)
    vp, pi = p["vox_ptr"], p["pose_idx"]
    first = np.full(360, 10 ** 9)
    for a in range(len(vp) - 1):
        s = pi[vp[a]:vp[a + 1]]; first[s] = np.minimum(first[s], s.min())
    assert ((np.arange(360) - first) > 320).any()                      # taller than the shared-memory kernel's 320 blocks
    P = pkg.LidarProblem(vp, pi, p["clusters"], p["poses"])
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(vp, pi, p["clusters"], p["poses"], 360)
    assert abs(r - r_ref) <= 1e-9 * abs(r_ref)
    dx = P.solve(0.01)
    H = lo.assemble_dense(blocks, 360)
    D = np.diag(np.diag(H))
    ref = np.linalg.solve(H + 0.01 * D, -g_ref.ravel())
    assert np.abs(dx - ref).max() <= 1e-6 * np.abs(ref).max()
    P.close()
    out, s = pkg.lidar_lm(vp, pi, p["clusters"], p["poses"])
    ref_poses, info = lo.damping_iter(vp, pi, p["clusters"], p["poses"])
    last = info["trace"][-1]                                           # the last decision sits at the rounding noise of lambda_0 when q ~ 1e-8 r1
    slack = 1 if abs(last["q"]) <= 1e-7 * last["r1"] else 0
    assert s["iterations"] == info["iters"] and abs(s["accepted"] - info["accepted"]) <= slack
    assert abs(s["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"]
    assert np.abs(out - ref_poses).max() <= 1e-6
    """, timeout=900)


@pytest.mark.gpu
def test_voxels_seen_from_hundreds_of_poses():
    """K > 128 poses per voxel (csrc/lidar_big.h) together with the any-width solver: H, g, the damped step and the LM
    against the oracle."""
    _run("""
    rng = np.random.Generator(np.random.Philox(key=77))
    W = 300
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp_b, pi_b, cl_b = synth.make_lidar(W, 5, R_gt, p_gt, rng, k_lo=200, k_hi=260, half=W - 1)       # five big voxels
    vp_s, pi_s, cl_s = synth.make_lidar(W, 1500, R_gt, p_gt, rng)                                       # and ordinary ones around them
    vp = np.concatenate([vp_s, vp_b[1:] + vp_s[-1]]); pi = np.concatenate([pi_s, pi_b]); cl = np.concatenate([cl_s, cl_b])
    order = np.random.default_rng(1).permutation(len(vp) - 1)                                           # big voxels anywhere in the list
    K = np.diff(vp); starts = vp[:-1]
    pi = np.concatenate([pi[starts[a]:starts[a] + K[a]] for a in order]); cl = np.concatenate([cl[starts[a]:starts[a] + K[a]] for a in order])
    vp = np.concatenate([[0], np.cumsum(K[order])])
    assert np.diff(vp).max() > 128
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    poses = np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1)
    P = pkg.LidarProblem(vp, pi, cl, poses)
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(vp, pi, cl, poses, W)
    g, br, bc, bl = P.get_system()
    H = pkg.env_blocks_to_dense(br, bc, bl, W); H_ref = lo.assemble_dense(blocks, W)
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    assert np.abs(H - H_ref).max() <= 1e-7 * np.abs(H_ref).max()
    assert abs(P.residual(poses) - lo.only_residual(vp, pi, cl, poses)) <= 1e-8 * abs(r_ref)
    P.close()
    out, s = pkg.lidar_lm(vp, pi, cl, poses)
    ref_poses, info = lo.damping_iter(vp, pi, cl, poses)
    assert abs(s["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"] and np.abs(out - ref_poses).max() <= 1e-6
    """, timeout=900)
