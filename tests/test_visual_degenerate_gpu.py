"""The visual LM on the GPU (boundary B2) on ill-conditioned and edge-case landmarks, against the 50-digit reference
(oracle/visual_mp.py).

The landmark family of tests/degenerate_landmarks.py: far facades at grazing angles (kappa of the damped landmark block up to
~1e10), two-view pairs of tiny parallax, views from one centre (a block singular but for the LM diagonal), views with z just
above and just below the 1e-8 cut-off, landmarks on their plane to 1e-9 (the kink of sqrt(e^2 + 1e-12)), scenes 1e3 - 1e5 m
from the origin, cameras whose U - W C^-1 W^T nearly cancels, tracks of 128 / 129 / 300 observations (tile path and
visual_big.h), strong distortion at the image corners, Huber at s = a^2 to a few ulps and Cauchy at s >> a^2.  Through
VisualProblem.reset_lm + step + get_system, in the default and the deterministic mode, every S block, rhs row, point step
(back-substituted by the reference from the device's own camera step), the cost and the model-cost change are held to the
bounds of tests/test_visual_mp_oracle.py (constants C_S, C_RHS, C_PT, C_COST of visual_mp.py, calibrated there on the CPU
from two float64 implementations).  The worst ratio per class is printed.
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

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def problems():
    out = {"isolated": dl.isolated(), "tile_and_big": dl.tile_and_big(), "shared": dl.shared(), "distort": dl.distort(),
           "huber_edge": dl.huber_edge(), "cauchy_far": dl.cauchy_far()}
    sh, perm = vs.shuffled(out["shared"], 20261017)
    sh["cls"] = out["shared"]["cls"][perm]
    out["shared shuffled"] = sh
    for p in out.values():
        p["lin"] = vm.linearize(p)
    return out


def _oracle(p, cam_fixed=None):
    pr = vl.RobustProblem(*vs.args(p), loss_reproj=p.get("loss_px"), loss_plane=p.get("loss_pl"))
    if cam_fixed is not None:
        vf.with_constant(pr, [0] + list(np.nonzero(cam_fixed)[0]))
    return pr


def _device(pkg, p, radius, scaling, det, cam_fixed=None):
    o = pkg.visual_default_opts(reproj_loss=p.get("loss_px"), plane_loss=p.get("loss_pl"))
    o.deterministic = int(det)
    P = pkg.VisualProblem(*vs.args(p))
    try:
        P.reset_lm(o, cam_fixed=cam_fixed)
        cs, ps, model, cost = P.step(radius, jacobi_scaling=scaling)
        cam, rhs, br, bc, bl = P.get_system()
    finally:
        P.close()
    blocks = {(int(a), int(b)): bl[k] for k, (a, b) in enumerate(zip(br, bc))}
    return dict(cam=cam, rhs=rhs, blocks=blocks, cam_step=cs, pt_step=ps, model=model, cost=cost)


def _check(p, dev, pr, radius, scaling, capsys, label, by_class=True):
    """every S block, rhs row and point step within the bounds, per class; cost and model for the whole problem"""
    assert np.array_equal(dev["cam"], np.nonzero(pr.cam_active)[0]), label
    sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
    whole = vm.assemble(sysm)
    for k, b in dev["blocks"].items():
        if k not in whole["S"]:
            assert not b.any(), (label, "a block no landmark touches", k)
    zero = np.zeros((6, 6))
    S_of = lambda i, j: dev["blocks"].get((i, j), zero)   # noqa: E731
    dp, dph, model, modelh = vm.backsub(sysm, dev["cam_step"])
    tv = vo.valid_tracks(p["plane_nd"])
    cls = p["cls"][tv]
    groups = {str(c): np.nonzero(cls == c)[0] for c in sorted(set(cls))} if by_class else {"all": np.arange(len(cls))}
    rows = []
    for g, idx in groups.items():
        ref = vm.assemble(sysm, [sysm["lm"][a] for a in idx])
        rs, rr, _ = vm.ratios(ref, S_of, dev["rhs"])
        rp = max((vm.ratio(e, h) for e, h in zip(np.abs(dev["pt_step"][tv][idx] - dp[idx]).max(1), dph[idx])), default=0.0)
        rows.append((g, rs, rr, rp))
    rc = vm.ratio(abs(dev["cost"] - whole["cost"]), whole["cost_hat"])
    rm = vm.ratio(abs(dev["model"] - model), modelh)
    with capsys.disabled():
        print(f"\n{label}: cost {rc:.3g} model {rm:.3g} (bound {vm.C_COST:g})")
        for g, rs, rr, rp in rows:
            print(f"  {g:14s} S {rs:9.3g} (bound {vm.C_S:g})  rhs {rr:9.3g} (bound {vm.C_RHS:g})  point {rp:9.3g} (bound {vm.C_PT:g})")
    for g, rs, rr, rp in rows:
        if radius > 1e8 and g == "rotation":      # no bound applies (tests/test_visual_mp_oracle.py): finite results only
            assert np.isfinite([rs, rr, rp]).all(), (label, g)
            continue
        assert rs <= vm.C_S and rr <= vm.C_RHS and rp <= vm.C_PT, (label, g, rs, rr, rp)
    assert rc <= vm.C_COST and rm <= vm.C_COST, (label, rc, rm)


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
@pytest.mark.parametrize("radius,scaling", [(1e4, True), (1e12, False)])
def test_isolated_landmarks_meet_the_bounds(gpu_pkg, problems, det, radius, scaling, capsys):
    """every landmark on cameras of its own: each S block and rhs row is one class's"""
    p = problems["isolated"]
    _check(p, _device(gpu_pkg, p, radius, scaling, det), _oracle(p), radius, scaling, capsys,
           f"isolated, radius {radius:g}, scaling {scaling}, det={det}")


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
@pytest.mark.parametrize("name", ["tile_and_big", "distort", "huber_edge", "cauchy_far"])
def test_own_problems_meet_the_bounds(gpu_pkg, problems, name, det, capsys):
    """the 128 / 129 / 300 tile / big split, strong distortion, Huber at its threshold and Cauchy far beyond it"""
    p = problems[name]
    if name == "tile_and_big":
        P = gpu_pkg.VisualProblem(*vs.args(p))
        try:
            assert P.big_counts()["n_big"] == 4        # 129 and 300; the two of 128 take the tiles
        finally:
            P.close()
    _check(p, _device(gpu_pkg, p, 1e4, True, det), _oracle(p), 1e4, True, capsys, f"{name}, det={det}")


@pytest.mark.parametrize("name", ["shared", "shared shuffled"])
def test_shared_trajectory_meets_the_bounds(gpu_pkg, problems, name, capsys):
    """every class on one trajectory 1 km from the origin, at its perturbed start, in caller order and with the landmarks
    (and every landmark's observations) shuffled"""
    p = problems[name]
    for det in (0, 1):
        _check(p, _device(gpu_pkg, p, 1e4, True, det), _oracle(p), 1e4, True, capsys, f"{name}, det={det}", by_class=False)


def test_constant_cameras_meet_the_bounds(gpu_pkg, problems, capsys):
    """cam_fixed on every third camera that sees a degenerate landmark: those observations have no camera columns"""
    p = problems["shared"]
    m = dl.fixed_mask(p)
    assert m.sum() >= 5
    _check(p, _device(gpu_pkg, p, 1e4, True, 0, cam_fixed=m), _oracle(p, m), 1e4, True, capsys, "shared, cam_fixed", by_class=False)


def test_lm_from_the_perturbed_start_matches_oracle(gpu_pkg, problems):
    """23 iterations of visual_lm from the shared problem's perturbed start: the same accept / reject sequence and first cost
    as the float64 oracle, and the end state within 1e-6 or within 16x the oracle's own spread under a 1e-15 perturbation of
    its inputs.  Past those iterations the cameras that only degenerate landmarks constrain (views from one centre, cut-off
    views, cameras of one or two landmarks) drift along their near-null directions, and the oracle's own accept / reject
    sequence changes under that perturbation."""
    p = problems["shared"]
    n_it = 23
    pr, info = vo.ceres_lm(vo.VisualProblem(*vs.args(p)), max_iter=n_it)
    seq_ref = [t["rho"] > 1e-3 for t in info["trace"]]
    o = gpu_pkg.visual_default_opts()
    o.max_iter = n_it
    P = gpu_pkg.VisualProblem(*vs.args(p))
    try:
        P.reset_lm(o)
        seq = []
        for _ in range(n_it):
            st = P.iterate(1)
            seq.append(st["accepted"] > 0)
            if st["termination"] != 0:
                break
    finally:
        P.close()
    assert seq == seq_ref
    q, t, X, s = gpu_pkg.visual_lm(*vs.args(p), opts=o)
    assert s["iterations"] == info["iters"] and s["accepted"] == info["accepted"]
    sysm = vm.system(p["lin"], pr.cam_col, 1e4, True)
    whole = vm.assemble(sysm)
    assert vm.ratio(abs(s["cost_first"] - whole["cost"]), whole["cost_hat"]) <= vm.C_COST
    rng = np.random.default_rng(5)
    p2 = dict(p)
    p2["X"] = p["X"] * (1 + 1e-15 * rng.standard_normal(p["X"].shape))
    p2["t"] = p["t"] * (1 + 1e-15 * rng.standard_normal(p["t"].shape))
    pr2, info2 = vo.ceres_lm(vo.VisualProblem(*vs.args(p2)), max_iter=n_it)
    sc = abs(info2["cost"] - info["cost"])
    sx = max(np.abs(pr2.q - pr.q).max(), np.abs(pr2.t - pr.t).max(), np.abs(pr2.X - pr.X).max())
    assert abs(s["cost_last"] - info["cost"]) <= max(1e-6 * info["cost"], 16 * sc)
    assert max(np.abs(q - pr.q).max(), np.abs(t - pr.t).max(), np.abs(X - pr.X).max()) <= max(1e-6, 16 * sx)
