"""The robust losses of path B on the CPU (tests/visual_loss_oracle.py): rho and rho' of Huber and Cauchy against differences of
rho, the corrected gradient J~^T r~ against differences of 1/2 sum rho, and the restated Ceres LM with a loss on a scene with
wrong matches: a stationary point, no lower cost nearby for an independent minimiser, cameras closer to ground truth than the
plain solve's.  Also the C ABI of the loss fields and its validation, which needs no device."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
from scipy import optimize

from oracle import synth
from oracle import visual_oracle as vo
import visual_loss_oracle as vl

ROOT = Path(__file__).resolve().parents[1]
KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
LOSSES = [(vl.HUBER, 1.0), (vl.HUBER, 0.1), (vl.HUBER, 3.0), (vl.CAUCHY, 1.0), (vl.CAUCHY, 0.1), (vl.CAUCHY, 4.0)]


def _args(p):
    return [p[k] for k in KEYS]


@pytest.mark.parametrize("kind,a", LOSSES)
def test_rho_and_derivative_against_differences(kind, a):
    b = a * a
    s = np.array([0.0, 1e-6 * b, 0.3 * b, b * (1 - 1e-3), b, b * (1 + 1e-3), 2.0 * b, 17.0 * b, 1e4 * b])
    rho, d1 = vl.loss_rho(kind, a, s)
    h = 1e-7 * np.maximum(s, b)
    fd = (vl.loss_rho(kind, a, s + h)[0] - vl.loss_rho(kind, a, s - h)[0]) / (2 * h)
    assert np.all(np.abs(d1 - fd) <= 1e-7 * np.abs(d1)), (d1, fd)
    # rho(0) = 0, rho'(0) = 1, rho <= s and rho' non-increasing (rho'' <= 0: the Corrector only scales)
    assert rho[0] == 0.0 and d1[0] == 1.0
    assert np.all(rho <= s + 1e-15 * s) and np.all(np.diff(d1) <= 0)
    if kind == vl.HUBER:
        assert np.array_equal(rho[s <= b], s[s <= b])


def _problem(seed=5, n_poses=8, n_tracks=40, outliers=False):
    p = synth.make_problem(n_poses, 0, n_tracks, seed=seed, lidar=False)
    if outliers:
        p, _ = vl.with_outliers(p, 0.05, 20.0, 50.0, seed)
    return p


@pytest.mark.parametrize("loss_reproj,loss_plane", [((vl.HUBER, 1.0), (vl.HUBER, 0.1)), ((vl.CAUCHY, 1.0), (vl.CAUCHY, 0.1)),
                                                    ((vl.HUBER, 0.7), None), (None, (vl.CAUCHY, 0.05))])
def test_corrected_gradient_is_the_gradient_of_the_robust_cost(loss_reproj, loss_plane):
    p = _problem(outliers=True)
    pr = vl.RobustProblem(*_args(p), fixed_cam=0, loss_reproj=loss_reproj, loss_plane=loss_plane)
    res, J = pr.residuals(jac=True)
    g = J.T @ res
    fd = vl.tangent_gradient_fd(pr)
    assert np.abs(g - fd).max() <= 1e-6 * np.abs(g).max()
    # and the cost is 1/2 sum rho, not 1/2 r~.r~
    assert pr.cost() < 0.5 * float(vo.VisualProblem(*_args(p)).residuals()[0] @ vo.VisualProblem(*_args(p)).residuals()[0])


def test_no_loss_is_the_plain_oracle_bit_for_bit():
    p = _problem()
    a = vo.VisualProblem(*_args(p))
    b = vl.RobustProblem(*_args(p))
    ra, Ja = a.residuals(jac=True)
    rb, Jb = b.residuals(jac=True)
    assert np.array_equal(ra, rb) and (Ja != Jb).nnz == 0 and a.cost() == b.cost()
    _, ia = vo.ceres_lm(a)
    _, ib = vl.ceres_lm(b)
    assert (ia["iters"], ia["accepted"], ia["term"], ia["cost0"], ia["cost"]) == (ib["iters"], ib["accepted"], ib["term"], ib["cost0"], ib["cost"])


def _cam_error(p, q, t):
    R = vo.quat_to_rot(q); Rg = vo.quat_to_rot(p["q_gt"])
    c = -np.einsum("nji,nj->ni", R, t); cg = -np.einsum("nji,nj->ni", Rg, p["t_gt"])
    return float(np.sqrt(((c - cg) ** 2).sum(1)).mean())


@pytest.mark.parametrize("kind", [vl.HUBER, vl.CAUCHY])
def test_robust_lm_on_wrong_matches(kind):
    p = _problem(seed=9, n_poses=10, n_tracks=60, outliers=True)
    pr = vl.RobustProblem(*_args(p), fixed_cam=0, loss_reproj=(kind, 1.0), loss_plane=(kind, 0.1))
    g0 = vl.tangent_gradient_fd(pr)
    pr, info = vl.ceres_lm(pr, max_iter=300, f_tol=-1.0, p_tol=-1.0)     # until the radius collapses at the rounding floor
    assert info["accepted"] > 0
    # at the optimum the plane residuals are near 0, where sqrt(e^2 + 1e-12) bends within |e| ~ 1e-6: a smaller step
    g1 = vl.tangent_gradient_fd(pr, h=1e-8)
    assert np.abs(g1).max() <= 1e-6 * np.abs(g0).max(), (np.abs(g1).max(), np.abs(g0).max(), info["term"])
    # an independent minimiser of the same cost, started at the result, finds nothing lower
    c1 = pr.cost()
    r = optimize.minimize(lambda d: pr.cost(*pr.plus(d)), np.zeros(pr.ncols), method="BFGS", options=dict(maxiter=200))
    assert r.fun >= c1 * (1 - 1e-10), (r.fun, c1)
    # the cameras end closer to ground truth than the plain solve's
    plain, _ = vo.ceres_lm(vo.VisualProblem(*_args(p), fixed_cam=0), max_iter=300)
    assert _cam_error(p, pr.q, pr.t) < _cam_error(p, plain.q, plain.t)


# ---- C ABI without a device ------------------------------------------------------------------------------------------------
def test_opts_layout_and_defaults(pkg, tmp_path):
    src = tmp_path / "opts.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "lvba_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %d %d %d\\n", sizeof(lvba_visual_opts), offsetof(lvba_visual_opts, reproj_loss),'
                   ' offsetof(lvba_visual_opts, reproj_loss_scale), offsetof(lvba_visual_opts, plane_loss), offsetof(lvba_visual_opts, plane_loss_scale),'
                   ' (int)LVBA_LOSS_NONE, (int)LVBA_LOSS_HUBER, (int)LVBA_LOSS_CAUCHY); return 0; }\n')
    exe = tmp_path / "opts"
    r = subprocess.run(["gcc", "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    V = pkg.VisualOpts
    assert got == [C.sizeof(V), V.reproj_loss.offset, V.reproj_loss_scale.offset, V.plane_loss.offset, V.plane_loss_scale.offset,
                   pkg.LOSS_NONE, pkg.LOSS_HUBER, pkg.LOSS_CAUCHY]
    o = pkg.visual_default_opts()
    assert (o.reproj_loss, o.reproj_loss_scale, o.plane_loss, o.plane_loss_scale) == (pkg.LOSS_NONE, 1.0, pkg.LOSS_NONE, 0.1)
    o = pkg.visual_default_opts(reproj_loss=pkg.LOSS_HUBER, plane_loss=(pkg.LOSS_CAUCHY, 0.25))
    assert (o.reproj_loss, o.reproj_loss_scale, o.plane_loss, o.plane_loss_scale) == (pkg.LOSS_HUBER, 1.0, pkg.LOSS_CAUCHY, 0.25)
    assert o.deterministic == 0 and o.max_iter == 50


BAD = [("reproj_loss", 3, None), ("plane_loss", -1, None), ("reproj_loss", 1, 0.0), ("reproj_loss", 2, -1.0), ("plane_loss", 1, float("nan")),
       ("plane_loss", 2, float("inf")), ("reproj_loss", 1, float("-inf"))]


@pytest.mark.parametrize("field,kind,scale", BAD)
def test_invalid_loss_is_refused_before_device_work(pkg, field, kind, scale):
    """An unknown kind or a non-finite / non-positive scale of a loss: LVBA_ERR_INVALID_ARG, whether or not a device exists, and
    the caller's buffers are untouched."""
    lib = pkg.load_library()
    p = _problem()
    o = pkg.visual_default_opts()
    setattr(o, field, kind)
    if scale is not None:
        setattr(o, field + "_scale", scale)
    q = np.ascontiguousarray(p["q"], np.float64); t = np.ascontiguousarray(p["t"], np.float64); X = np.ascontiguousarray(p["X"], np.float64)
    q0, t0, X0 = q.copy(), t.copy(), X.copy()
    pl = np.ascontiguousarray(p["plane_nd"], np.float64); op = np.ascontiguousarray(p["obs_ptr"], np.int64)
    oc = np.ascontiguousarray(p["obs_cam"], np.int32); uv = np.ascontiguousarray(p["obs_uv"], np.float32); it = np.ascontiguousarray(p["intr"], np.float64)
    s = pkg.Summary()
    s_bytes = bytes(s)
    P = lambda a, t_: a.ctypes.data_as(C.POINTER(t_))  # noqa: E731
    rc = lib.lvba_visual_lm(C.c_int32(len(q)), C.c_int64(len(X)), P(q, C.c_double), P(t, C.c_double), P(X, C.c_double), P(pl, C.c_double),
                            P(op, C.c_int64), P(oc, C.c_int32), P(uv, C.c_float), P(it, C.c_double), C.c_double(p["sigma_px"]),
                            C.c_double(p["sigma_plane"]), C.c_int32(0), C.byref(o), C.byref(s))
    assert rc == -1, rc
    assert field.encode() in lib.lvba_last_error()
    assert np.array_equal(q, q0) and np.array_equal(t, t0) and np.array_equal(X, X0) and bytes(s) == s_bytes


def test_none_kind_ignores_its_scale(pkg):
    """A scale of 0 or NaN beside LVBA_LOSS_NONE is not an error: without a device the call gets as far as the device."""
    if pkg.device_count() > 0:
        pytest.skip("checks the path of a machine without a device")
    p = _problem()
    o = pkg.visual_default_opts()
    o.reproj_loss_scale = 0.0; o.plane_loss_scale = float("nan")
    with pytest.raises(pkg.LvbaError) as e:
        pkg.visual_lm(*_args(p), opts=o)
    assert e.value.status == -2
