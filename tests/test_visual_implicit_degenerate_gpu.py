"""The matrix-free product of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_implicit.h, the visual_imp_* kernels) on the H100,
on ill-conditioned and edge-case landmarks, against the 50-digit reference (oracle/visual_mp.py).

The problems of tests/test_visual_implicit_mp_oracle.py (the degenerate landmark family with ballast tracks, isolated with the
repeat class; the rule moves every one of them to the matrix-free product, which is asserted), through reset_lm(linear_solver=1)
and one step, in the default and the deterministic mode: the damped operator A = S + diag(dadd), built column by column through
lvba_visual_apply_system, every block of it within C_S of the reference per class; rhs (lvba_visual_get_system(rhs, NULL)),
the point steps back-substituted by the reference from the device's own camera step, the cost and the model-cost change within
C_RHS, C_PT and C_COST (the constants of the explicit path, calibrated on the CPU); and every off-diagonal entry within the
symmetry bound of the double-double product, |A_ij - A_ji| <= ulp + 64 eps^2 T_ij (vm.symmetry_ratio), here and on the
400-camera scenes of tests/test_visual_implicit_gpu.py with the float64 term scale.  For contrast, the explicit product
(visual_pcg_product_kernel) on problems that many short tracks on three cameras hold under the rule: bitwise symmetric, the
stored blocks plus the LM diagonal bit for bit, and within the same bounds.  The worst ratio per class is printed.
"""
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import visual_mp as vm
from oracle import visual_oracle as vo

sys.path.insert(0, str(Path(__file__).resolve().parent))
import degenerate_landmarks as dl  # noqa: E402
import visual_big_scene as vs  # noqa: E402
import visual_fixed_oracle as vf  # noqa: E402
import visual_loss_oracle as vl  # noqa: E402
from test_visual_implicit_gpu import _loop, _mixed, _operator, _rhs  # noqa: E402
from test_visual_implicit_mp_oracle import C_PREC, PREC_CASES, bound_S, family_problems, prec_ratios  # noqa: E402
from test_visual_mp_oracle import groups_of, unbounded  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def problems():
    out = family_problems()
    sh, perm = vs.shuffled(out["shared"], 20261017)
    sh["cls"] = out["shared"]["cls"][perm]
    out["shared shuffled"] = sh
    out["isolated explicit"] = dl.ballast(dl.isolated(classes=dl.REPEAT), **dl.EXPLICIT)
    for p in out.values():
        p["lin"] = vm.linearize(p)
    return out


def _oracle(p, cam_fixed=None):
    pr = vl.RobustProblem(*vs.args(p), loss_reproj=p.get("loss_px"), loss_plane=p.get("loss_pl"))
    if cam_fixed is not None:
        vf.with_constant(pr, [0] + list(np.nonzero(cam_fixed)[0]))
    return pr


def _device(pkg, p, radius, scaling, det, cam_fixed=None, product=1):
    o = pkg.visual_default_opts(reproj_loss=p.get("loss_px"), plane_loss=p.get("loss_pl"))
    o.deterministic = int(det)
    P = pkg.VisualProblem(*vs.args(p))
    try:
        P.reset_lm(o, cam_fixed=cam_fixed, linear_solver=1)
        assert P.schur_product() == product
        cs, ps, model, cost = P.step(radius, jacobi_scaling=scaling)
        out = dict(A=_operator(P), rhs=_rhs(P), cam=P.structure()[0], cam_step=cs, pt_step=ps, model=model, cost=cost)
        if product == 0:
            out["S"] = P.get_system()
    finally:
        P.close()
    return out


def _check(p, dev, pr, radius, scaling, capsys, label, by_class=True, name=None):
    """every A block, rhs row and point step within the bounds, per class; cost and model for the whole problem; the symmetry
    bound on every off-diagonal entry"""
    assert np.array_equal(dev["cam"], np.nonzero(pr.cam_active)[0]), label
    sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
    n = sysm["n_rows"]
    A = dev["A"]
    assert A.shape == (6 * n, 6 * n)
    whole = vm.damped(sysm)
    touched = np.zeros((n, n), bool)
    for (i, j) in whole["S"]:
        touched[i, j] = True
    assert not (A.reshape(n, 6, n, 6).any(axis=(1, 3)) & ~touched).any(), (label, "a block no landmark touches")
    A_of = lambda i, j: A[6 * i:6 * i + 6, 6 * j:6 * j + 6]   # noqa: E731
    rhs = dev["rhs"].reshape(n, 6)
    dp, dph, model, modelh = vm.backsub(sysm, dev["cam_step"])
    tv = vo.valid_tracks(p["plane_nd"])
    groups = groups_of(p, "x") if by_class else {"all": np.arange(int(tv.sum()))}
    rows = []
    for g, idx in groups.items():
        lms = [sysm["lm"][a] for a in idx]
        rs, _, _ = vm.ratios(vm.damped(sysm, lms), A_of)
        _, rr, _ = vm.ratios(vm.assemble(sysm, lms), rhs=rhs)
        rp = max((vm.ratio(e, h) for e, h in zip(np.abs(dev["pt_step"][tv][idx] - dp[idx]).max(1), dph[idx])), default=0.0)
        rows.append((g, rs, rr, rp))
    base = vm.assemble(sysm)
    rc = vm.ratio(abs(dev["cost"] - base["cost"]), base["cost_hat"])
    rm = vm.ratio(abs(dev["model"] - model), modelh)
    sym = vm.symmetry_ratio(A, vm.dense(whole["T"], n))
    with capsys.disabled():
        print(f"\n{label}: cost {rc:.3g} model {rm:.3g} (bound {vm.C_COST:g})  symmetry {sym:.3g} (bound 1)")
        for g, rs, rr, rp in rows:
            print(f"  {g:14s} A {rs:9.3g} (bound {vm.C_S:g})  rhs {rr:9.3g} (bound {vm.C_RHS:g})  point {rp:9.3g} (bound {vm.C_PT:g})")
    for g, rs, rr, rp in rows:
        if unbounded(g, radius):
            assert np.isfinite([rs, rr, rp]).all(), (label, g)
            continue
        assert rs <= bound_S(name, g) and rr <= vm.C_RHS and rp <= vm.C_PT, (label, g, rs, rr, rp)
    assert rc <= vm.C_COST and rm <= vm.C_COST, (label, rc, rm)
    return sysm, sym


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
@pytest.mark.parametrize("radius,scaling", [(1e4, True), (1e12, False)])
def test_isolated_landmarks_meet_the_bounds(gpu_pkg, problems, det, radius, scaling, capsys):
    """every landmark on cameras of its own, the repeat class and two ballast tracks: each block of A is one class's"""
    p = problems["isolated"]
    _, sym = _check(p, _device(gpu_pkg, p, radius, scaling, det), _oracle(p), radius, scaling, capsys,
                    f"isolated, radius {radius:g}, scaling {scaling}, det={det}", name="isolated")
    assert sym <= 1.0


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
@pytest.mark.parametrize("name", ["tile_and_big", "distort", "huber_edge", "cauchy_far"])
def test_own_problems_meet_the_bounds(gpu_pkg, problems, name, det, capsys):
    """the 128 / 129 / 300 split (both track kernels, <8> and <128>), strong distortion, Huber at its threshold and Cauchy far
    beyond it"""
    p = problems[name]
    if name == "tile_and_big":
        P = gpu_pkg.VisualProblem(*vs.args(p))
        try:
            assert P.big_counts()["n_big"] == 4        # 129 and 300 take visual_imp_track_kernel<128>, the rest <8>
        finally:
            P.close()
    _, sym = _check(p, _device(gpu_pkg, p, 1e4, True, det), _oracle(p), 1e4, True, capsys, f"{name}, det={det}", name=name)
    assert sym <= 1.0


@pytest.mark.parametrize("name", ["shared", "shared shuffled"])
def test_shared_trajectory_meets_the_bounds(gpu_pkg, problems, name, capsys):
    """every class on one trajectory 1 km from the origin at its perturbed start, in caller order and shuffled"""
    p = problems[name]
    for det in (0, 1):
        _, sym = _check(p, _device(gpu_pkg, p, 1e4, True, det), _oracle(p), 1e4, True, capsys, f"{name}, det={det}", by_class=False)
        assert sym <= 1.0


def test_constant_cameras_meet_the_bounds(gpu_pkg, problems, capsys):
    """cam_fixed on every third camera that sees a degenerate landmark: their J_c records are zero"""
    p = problems["shared"]
    m = dl.fixed_mask(p)
    assert m.sum() >= 5
    _, sym = _check(p, _device(gpu_pkg, p, 1e4, True, 0, cam_fixed=m), _oracle(p, m), 1e4, True, capsys, "shared, cam_fixed",
                    by_class=False)
    assert sym <= 1.0


@pytest.mark.parametrize("make", [_mixed, _loop], ids=["mixed", "loop_closed"])
def test_long_track_scenes_meet_the_symmetry_bound(gpu_pkg, make, capsys):
    """400 cameras with tracks of up to 1000 observations, and a loop closure: T from the float64 oracle's Jacobian"""
    p = make()
    for det in (0, 1):
        o = gpu_pkg.visual_default_opts()
        o.deterministic = det
        P = gpu_pkg.VisualProblem(*vs.args(p))
        try:
            P.reset_lm(o, linear_solver=1)
            assert P.schur_product() == 1
            P.step(1e4)
            A = _operator(P)
        finally:
            P.close()
        sym = vm.symmetry_ratio(A, vm.term_scale_f64(vo.VisualProblem(*vs.args(p)), 1e4, True))
        with capsys.disabled():
            print(f"\n{make.__name__}, det={det}: symmetry {sym:.3g} (bound 1)")
        assert sym <= 1.0


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
def test_explicit_product_for_contrast(gpu_pkg, problems, det, capsys):
    """the isolated problem held on the explicit S by many short tracks on three cameras: ITERATIVE_SCHUR's explicit operator is
    bitwise symmetric, equals the stored blocks plus the LM diagonal bit for bit, and is within the same bounds"""
    p = problems["isolated explicit"]
    radius = 1e4
    dev = _device(gpu_pkg, p, radius, True, det, product=0)
    A = dev["A"]
    assert np.array_equal(A, A.T)
    cam, rhs, br, bc, bl = dev["S"]
    n = len(cam)
    S = np.zeros_like(A)
    for k, (i, j) in enumerate(zip(br, bc)):
        b = bl[k] if i != j else np.tril(bl[k]) + np.tril(bl[k], -1).T      # a diagonal block through its lower triangle
        S[6 * i:6 * i + 6, 6 * j:6 * j + 6] = b
        S[6 * j:6 * j + 6, 6 * i:6 * i + 6] = b.T
    lo = np.tril(np.ones((6 * n, 6 * n), bool))
    off = ~np.eye(6 * n, dtype=bool)
    assert np.array_equal(A[off & lo], S[off & lo])                       # every entry but the diagonal: the stored one
    sysm, _ = _check(p, dev, _oracle(p), radius, True, capsys, f"isolated explicit, det={det}", name="isolated")
    ref = vm.damped(sysm)                  # the diagonal: the stored one plus dadd, against the reference's dadd
    dadd = np.diag(A) - np.diag(S)
    err = np.abs(dadd - ref["dadd"].ravel())
    assert (err <= vm.C_S * vm.EPS * ref["dadd_hat"].ravel() + np.spacing(np.abs(np.diag(A)))).all()


@pytest.mark.parametrize("name,radius,scaling", PREC_CASES[:3])
def test_one_preconditioned_iteration(gpu_pkg, problems, name, radius, scaling):
    """min_linear_iter = max_linear_iter = 1: the camera step is s_c o alpha (D + diag dadd)^-1 rhs; after a fit of alpha every
    row within C_PREC eps kappa(M_r) of the 50-digit direction (C_PREC calibrated on the host solve): the device's D_r"""
    p = problems[name]
    pr = _oracle(p)
    P = gpu_pkg.VisualProblem(*vs.args(p))
    try:
        P.reset_lm(gpu_pkg.visual_default_opts(reproj_loss=p.get("loss_px"), plane_loss=p.get("loss_pl")), linear_solver=1,
                   min_linear_iter=1, max_linear_iter=1)
        assert P.schur_product() == 1
        cs, _, _, _ = P.step(radius, jacobi_scaling=scaling)
        st = P.linear_stats()
    finally:
        P.close()
    assert (st["cg_iters_last"], st["term_last"]) == (1, 1)
    sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
    s_cam = np.array([[float(c) for c in row] for row in sysm["s_cam"]])
    y = cs[pr.cam_active] / s_cam
    # near_z rows are left out: their M_r (kappa ~1e20) is the difference of terms ~1e4x larger, so eps kappa(M_r) does not
    # bound how far the device's and the host's rounding of D_r move the direction (device 7.9e14, host 4.9e4 on one row)
    per, _ = prec_ratios(sysm, y.ravel(), groups_of(p, name), skip=("near_z",))
    assert max(per.values()) <= C_PREC, per
