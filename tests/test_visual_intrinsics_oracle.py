"""The intrinsics block of the visual LM (lvba_visual_opts::refine_intrinsics) on the CPU oracle (tests/visual_intr_oracle.py):
its Jacobian columns against central differences, the bordered Schur step (k + 1 camera solves and the k x k corner, the
device's algorithm) against the dense normal equations over every column, and the recovery of miscalibrated intrinsics."""
import numpy as np
import pytest

from oracle import synth
from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_fixed_oracle as vf
import visual_intr_oracle as vi
import visual_loss_oracle as vl

MASKS = [vi.FOCAL, vi.PRINCIPAL, vi.DISTORTION, vi.FOCAL | vi.PRINCIPAL, 0xFF, 0x10]


def _small(seed=5):
    return synth.make_problem(12, 0, 60, seed=seed, lidar=False)


def test_intr_jacobian_matches_central_differences():
    p = _small()
    pr = vo.VisualProblem(*vs.args(p))
    o = np.nonzero(pr.obs_ok)[0]
    q, t, X = pr.q[pr.obs_cam[o]], pr.t[pr.obs_cam[o]], pr.X[pr.obs_trk[o]]
    uv = pr.obs_uv[o]
    J = vi.intr_jacobian(q, t, X, pr.intr, pr.sp)
    for i in range(8):
        h = 1e-6 * max(1.0, abs(pr.intr[i]))
        ip, im = pr.intr.copy(), pr.intr.copy()
        ip[i] += h; im[i] -= h
        fd = (vo.reproj_eval(q, t, X, uv, ip, pr.sp, False)[0] - vo.reproj_eval(q, t, X, uv, im, pr.sp, False)[0]) / (2 * h)
        assert np.abs(J[:, :, i] - fd).max() <= 1e-7 * max(1.0, np.abs(fd).max()), i


def test_intr_jacobian_is_zero_behind_the_camera():
    p = _small()
    pr = vo.VisualProblem(*vs.args(p))
    X = np.array([[0.0, 0.0, -5.0]])
    J = vi.intr_jacobian(np.array([[1.0, 0, 0, 0]]), np.zeros((1, 3)), X, pr.intr, pr.sp)
    assert not J.any()


def _problem(p, mask, loss, cams):
    lr, lp = loss
    pr = vi.IntrProblem(*vs.args(p), mask=mask, loss_reproj=lr, loss_plane=lp)
    if cams == "some":
        vf.with_constant(pr, [0, 3, 4])
    elif cams == "all":
        vf.with_constant(pr, range(pr.M))
    return pr


@pytest.mark.parametrize("cams", ["fixed0", "some", "all"])
@pytest.mark.parametrize("loss", [(None, None), ((vl.HUBER, 1.0), (vl.HUBER, 0.1)), ((vl.CAUCHY, 1.0), None)],
                         ids=["plain", "huber", "cauchy"])
@pytest.mark.parametrize("mask", MASKS)
def test_bordered_step_matches_full_normal_equations(mask, loss, cams):
    p = vl.with_outliers(_small(7), 0.05, 20.0, 50.0, 7)[0] if loss[0] else _small(7)
    pr = _problem(p, mask, loss, cams)
    if cams == "all":
        assert pr.nc == 0
    for radius in (1e4, 1e1):
        a = vi.step_full(pr, radius)
        b = vi.step_bordered(pr, radius)
        assert np.abs(a["y"] - b["y"]).max() <= 1e-8 * np.abs(a["y"]).max()
        assert abs(a["model"] - b["model"]) <= 1e-9 * abs(a["model"])


def test_held_entries_and_mask_zero_are_the_plain_problem():
    p = _small(9)
    base = vo.single_step(vo.VisualProblem(*vs.args(p)))
    pr = vi.IntrProblem(*vs.args(p), mask=0)
    s = vi.step_full(pr)
    assert np.allclose(s["y"], base["y"], rtol=0, atol=1e-12 * np.abs(base["y"]).max())


def test_lm_recovers_miscalibrated_intrinsics():
    """Exact pixels (the scene's own projections, rounded to float32 as obs_uv is) and planes through the true landmarks: the
    true state is a minimum of zero reprojection error, so fx, fy (1 % off) and k1 (0.02 off) must come back to it, not merely
    closer.  The fixed intrinsics cannot get there."""
    p = synth.make_problem(30, 0, 400, seed=21, lidar=False)
    trk = np.repeat(np.arange(len(p["X_gt"])), np.diff(p["obs_ptr"]))
    R = vo.quat_to_rot(p["q_gt"])
    uv, _ = synth.project(R[p["obs_cam"]], p["t_gt"][p["obs_cam"]], p["X_gt"][trk])
    p["obs_uv"] = uv.astype(np.float32)
    p["q"][0], p["t"][0] = p["q_gt"][0], p["t_gt"][0]          # camera 0, held constant, at its true pose: the gauge
    truth = p["intr"].copy()
    bad = vi.miscalibrated(p, 0.01, 0.02)
    pr, info = vi.ceres_lm(vi.IntrProblem(*vs.args(bad), mask=vi.FOCAL | 0x10), max_iter=100, f_tol=1e-14, p_tol=1e-14, g_tol=1e-14)
    fixed, _ = vo.ceres_lm(vo.VisualProblem(*vs.args(bad)), max_iter=100, f_tol=1e-14, p_tol=1e-14, g_tol=1e-14)
    assert info["cost"] < 1e-3 * fixed.cost()
    # float32 pixels carry ~3e-5 px of rounding: the intrinsics come back to within 1e-5 relative (fx, fy) and 1e-5 (k1)
    assert np.abs(pr.intr[:2] / truth[:2] - 1).max() <= 1e-5, pr.intr[:2] / truth[:2] - 1
    assert abs(pr.intr[4] - truth[4]) <= 1e-5, pr.intr[4] - truth[4]
    assert np.array_equal(pr.intr[[2, 3, 5, 6, 7]], bad["intr"][[2, 3, 5, 6, 7]])
