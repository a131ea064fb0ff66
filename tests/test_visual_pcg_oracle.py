"""ITERATIVE_SCHUR for the visual LM (lvba_visual_opts::linear_solver) on the CPU oracle (tests/visual_pcg_oracle.py): the
conjugate gradients of Ceres' rule against the exact solve, its terminations, the residual reset and min_linear_iter, and the LM
with the inexact step against the exact LM of oracle/visual_oracle.py."""
import numpy as np

from oracle import synth
from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_pcg_oracle as vp


def _small(seed=5):
    return synth.make_problem(12, 0, 60, seed=seed, lidar=False)


def _spd(n, seed, cond=1e3):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((6 * n, 6 * n)))
    return (Q * np.geomspace(1.0, cond, 6 * n)) @ Q.T, rng.standard_normal(6 * n)


def test_tight_eta_gives_the_exact_step():
    pr = vo.VisualProblem(*vs.args(_small()))
    ref = vo.single_step(vo.VisualProblem(*vs.args(_small())), 1e4)
    # the quadratic-model test alone stops once Q stagnates in double, which leaves the step accurate to about sqrt(eps):
    # as many iterations as the system has unknowns are forced through min_linear_iter
    n = 6 * pr.nc
    got = vp.single_step(pr, 1e4, eta=1e-14, min_iter=n, max_iter=n)
    assert got["iters"] == n and got["term"] in (vp.SUCCESS, vp.NO_CONVERGENCE)
    for k in ("cam_step", "pt_step"):
        assert np.abs(got[k] - ref[k]).max() <= 1e-9 * np.abs(ref[k]).max(), k
    assert abs(got["model"] - ref["model"]) <= 1e-9 * abs(ref["model"])


def test_zero_rhs_takes_no_iteration():
    A, _ = _spd(3, 1)
    x, it, term = vp.cg(A, np.zeros(18))
    assert (it, term) == (0, vp.SUCCESS) and not x.any()


def test_indefinite_system_stops_at_nonpositive_curvature():
    # positive definite diagonal blocks (so the preconditioner is the identity), eigenvalues 1 +- 2 overall
    A = np.block([[np.eye(6), 2 * np.eye(6)], [2 * np.eye(6), np.eye(6)]])
    b = np.random.default_rng(2).standard_normal(12)
    x, it, term = vp.cg(A, b, eta=1e-14, max_iter=1000)
    assert term == vp.NO_CONVERGENCE and it >= 1
    # the current x comes back: the same run stopped one iteration earlier has it
    x_prev = vp.cg(A, b, eta=1e-30, max_iter=it - 1)[0] if it > 1 else np.zeros(12)
    assert np.array_equal(x, x_prev)


def test_nonpositive_preconditioner_pivot_is_failure():
    A, b = _spd(2, 3)
    A[0, 0] = -1.0
    assert vp.cg(A, b)[1:] == (0, vp.FAILURE)


def test_long_run_resets_the_residual():
    A, b = _spd(8, 4, cond=1e8)
    x, it, term = vp.cg(A, b, eta=1e-15, max_iter=10000)
    assert it > 2 * vp.RESET_PERIOD
    assert term == vp.SUCCESS and np.linalg.norm(A @ x - b) <= 1e-3 * np.linalg.norm(b)


def test_min_linear_iter_runs_past_a_met_test():
    A, b = _spd(4, 5)
    _, it0, t0 = vp.cg(A, b, eta=0.5)
    _, it1, t1 = vp.cg(A, b, eta=0.5, min_iter=it0 + 5)
    assert t0 == t1 == vp.SUCCESS and it1 == it0 + 5
    _, it2, t2 = vp.cg(A, b, eta=1e-30, max_iter=7)
    assert (it2, t2) == (7, vp.NO_CONVERGENCE)


def test_lm_matches_the_exact_lm():
    exact, ie = vo.ceres_lm(vo.VisualProblem(*vs.args(_small())))
    pcg, ip = vp.ceres_lm(vo.VisualProblem(*vs.args(_small())))
    assert abs(ip["cost"] - ie["cost"]) <= 1e-6 * ie["cost"], (ip["cost"], ie["cost"])
    assert ip["accepted"] >= 1 and max(ip["cg_iters"]) >= 1


def test_loop_closed_scene_lm():
    p = vs.make_scene(3, M=40, n_short=80, long_tracks=[(8, 36)])
    exact, ie = vo.ceres_lm(vo.VisualProblem(*vs.args(p)))
    _, ip = vp.ceres_lm(vo.VisualProblem(*vs.args(p)))
    assert abs(ip["cost"] - ie["cost"]) <= 1e-6 * ie["cost"], (ip["cost"], ie["cost"])
