"""The matrix-free product of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_implicit.h) on the degenerate landmark family against
the 50-digit reference (oracle/visual_mp.py), without a GPU: the host-compiled matrix-free passes (tests/emu/visual_implicit_emu.cpp,
emu_imp_operator: one linearisation, then ProdTrackF / ProdRowF on every unit vector) give the damped operator
A = S + diag(dadd) column by column, rhs, the cost, and the point steps and model-cost change of vbig::BacksubStridePass over
the matrix-free records.

Calibration: on the whole family (tests/degenerate_landmarks.py, every problem but tile_and_big with two ballast tracks whose
cameras each take several views, so that RowPartF sums runs on long tracks; isolated with the repeat class), at radius 1e4 and
1e12, with Jacobi scaling on and off, every A block, rhs row and point step is held to the bounds C_S, C_RHS and C_PT of the
explicit path, and the cost and model to C_COST (rotation at radius 1e12 exempt, as there).  The worst ratio per class is
printed, beside the float64 oracle's and the explicit host passes' on the same problem and camera step.  Three (problem, class)
pairs exceed C_S in the float64 arithmetic the explicit and the matrix-free passes share (WIDE_S below); there the float64
oracle meets C_S, so the reference's error scale is not what is too tight.

Preconditioner: with one CG iteration the camera step is alpha M^-1 rhs, M = blockdiag(D_r + diag dadd_r); per row it is held to
C_PREC eps kappa(M_r) of the 50-digit direction after a fit of alpha (calibrated here on the host-compiled solve).

Symmetry: the double-double product is the exact operator of the rounded records rounded once, so every off-diagonal entry meets
|A_ij - A_ji| <= ulp(max(|A_ij|, |A_ji|)) + 64 eps^2 T_ij (vm.symmetry_ratio, T_ij the sum of the absolute values of the entry's
terms).  The same product restated in plain double from the exported records misses that bound by at least 100x on the far,
cancel and repeat classes and on a long-track scene: the bound has teeth.
"""
import ctypes
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import visual_mp as vm
from oracle import visual_oracle as vo

sys.path.insert(0, str(Path(__file__).resolve().parent))
import degenerate_landmarks as dl  # noqa: E402
import visual_big_scene as vs  # noqa: E402
import visual_loss_oracle as vl  # noqa: E402
from test_visual_big_emu import Local  # noqa: E402
import test_visual_implicit_emu as tie  # noqa: E402
import test_visual_mp_oracle as tvm  # noqa: E402
from test_visual_mp_oracle import groups_of, unbounded  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
SETTINGS = [(1e4, True), (1e4, False), (1e12, True), (1e12, False)]
TEETH = ("far", "cancel", "repeat")


def family_problems():
    """the problems of the matrix-free calibration: the family with ballast tracks (long tracks on cameras of their own, each
    camera seen several times: RowPartF's runs), isolated with the repeat class"""
    out = {"isolated": dl.ballast(dl.isolated(classes=dl.REPEAT)), "tile_and_big": dl.tile_and_big()}
    for name, make in (("shared", dl.shared), ("distort", dl.distort), ("huber_edge", dl.huber_edge), ("cauchy_far", dl.cauchy_far)):
        out[name] = dl.ballast(make())
    return out


@pytest.fixture(scope="module")
def family():
    out = family_problems()
    for p in out.values():
        p["lin"] = vm.linearize(p)
    return out


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("imp_mp") / "libvisual_implicit_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_implicit_emu.cpp"),
                        "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(P(t))


def oracle_problem(p):
    return vl.RobustProblem(*vs.args(p), loss_reproj=p.get("loss_px"), loss_plane=p.get("loss_pl"))


def operator(emu, p, radius, scaling, y_cam=None):
    """emu_imp_operator on the whole problem (camera 0 constant, as the library's gauge): the dense operator A [6n, 6n] from the
    n*6 unit vectors, and the linearisation's outputs; y_cam: the scaled camera step to back-substitute (default zero)"""
    L = Local(p, 0)
    n, n6, Tv, T = L.n, 6 * L.n, L.Tv, len(p["X"])
    nnz = int(L.trk_ptr[-1])
    q, t, X = (np.ascontiguousarray(a, np.float64) for a in (L.pr.q, L.pr.t, L.pr.X))
    lp, ll = p.get("loss_px") or (0, 1.0), p.get("loss_pl") or (0, 1.0)
    o = dict(ys=np.zeros((n6, n6)), pt_step=np.zeros((T, 3)), model=np.zeros(1), rec=np.zeros((max(nnz, 1), 24)),
             params=np.zeros((max(Tv, 1), 16)), row_ptr=np.zeros(n + 1, np.int64), row_obs=np.zeros(max(nnz, 1), np.int64),
             row_trk=np.zeros(max(nnz, 1), np.int32), rhs=np.zeros(max(n6, 1)), colsq=np.zeros(max(n6, 1)), dadd=np.zeros(max(n6, 1)),
             s_cam=np.zeros(max(n6, 1)), D=np.zeros(max(n, 1) * 36), s_pt=np.zeros(max(Tv, 1) * 3), out=np.zeros(2))
    xs = np.ascontiguousarray(np.eye(n6))
    yc = np.ascontiguousarray(np.zeros(n6) if y_cam is None else y_cam, np.float64)
    emu.emu_imp_operator(ctypes.c_int(n), ctypes.c_int64(Tv), *L.common(), ctypes.c_int(lp[0]), ctypes.c_double(lp[1]),
                         ctypes.c_int(ll[0]), ctypes.c_double(ll[1]), ctypes.c_int(T), _p(q), _p(t), _p(X), ctypes.c_int(int(scaling)),
                         ctypes.c_double(radius), ctypes.c_int(n6), _p(xs), _p(o["ys"]), _p(yc), _p(o["pt_step"]), _p(o["model"]),
                         _p(o["rec"]), _p(o["params"]), _p(o["row_ptr"], ctypes.c_int64), _p(o["row_obs"], ctypes.c_int64),
                         _p(o["row_trk"], ctypes.c_int), *[_p(o[k]) for k in ("rhs", "colsq", "dadd", "s_cam", "D", "s_pt", "out")])
    o["A"] = o.pop("ys").T                            # column k is the product of unit vector k
    o["L"] = L
    return o


def plain_double(o):
    """ProdTrackF / ProdRowF restated in plain double (numpy) on the exported records of `o`, applied to every unit vector:
    u_l = C_l^-1 sum J_X^T (J_c x_row), y_r = sum J_c^T (J_c x_r - J_X u_l) + dadd o x_r, every sum in observation order"""
    L = o["L"]
    n6 = 6 * L.n
    rec = o["rec"]
    Jc = rec[:, 2:14].reshape(-1, 2, 6); JX = rec[:, 14:20].reshape(-1, 2, 3)
    p = o["params"]
    Ci = p[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
    x = np.eye(n6).reshape(L.n, 6, n6)
    y = np.zeros((L.n, 6, n6))
    for k in range(L.Tv):
        obs = [s for s in range(L.trk_ptr[k], L.trk_ptr[k + 1]) if L.row[s] >= 0]
        a = np.zeros((3, n6))
        for s in obs:
            a += JX[s].T @ (Jc[s] @ x[L.row[s]])
        u = Ci[k] @ a
        for s in obs:
            y[L.row[s]] += Jc[s].T @ (Jc[s] @ x[L.row[s]] - JX[s] @ u)
    return y.reshape(n6, n6) + np.diag(o["dadd"][:n6])


def class_rows(sysm, idx):
    """the system rows the landmarks idx touch"""
    return sorted({i for a in idx for i in sysm["lm"][a]["urows"]})


# (problem, class) -> the bound on the A blocks where the float64 arithmetic of the passes (landmark_step's sym3_inverse and the
# per-observation records, shared by visual_big.h and visual_implicit.h) exceeds C_S on the family; worst ratios measured:
# matrix-free host 231 / explicit host 231 / H100 147 (repeat), 115 / 115 / 157 (far beside the repeat class), 1.4e3 / - / 189
# (the Cauchy problem's ballast).  On the two isolated pairs the float64 oracle (LU per landmark) meets C_S: the shared
# arithmetic is what exceeds it.  On the Cauchy ballast all three float64 implementations agree at 1.4e3: there the reference's
# first-order scale of the loss-corrected terms is what is too tight.
WIDE_S = {("isolated", "repeat"): 1024.0, ("isolated", "far"): 1024.0, ("cauchy_far", "ballast"): 8192.0}


def bound_S(name, g):
    return WIDE_S.get((name, g), vm.C_S)


def damped_ratios(sysm, A, groups):
    """{group: the worst |A block - reference| / (eps scale)} of the dense operator A"""
    A_of = lambda i, j: A[6 * i:6 * i + 6, 6 * j:6 * j + 6]    # noqa: E731
    return {g: vm.ratios(vm.damped(sysm, [sysm["lm"][a] for a in idx]), A_of)[0] for g, idx in groups.items()}


@pytest.fixture(scope="module")
def measured(family, emu, tmp_path_factory):
    """(problem, group, radius, scaling) -> dict of ratios: "imp" (A, rhs, point step, cost, model, symmetry) of the host
    matrix-free passes, "oracle" and "expl" (S, rhs, point step) of the float64 oracle and of the explicit host passes
    (visual_big.h) on the same problem and camera step (the oracle's)"""
    lib = tvm._emu_lib(tmp_path_factory.mktemp("vloss_emu"))
    out = {}
    for name, p in family.items():
        pr = oracle_problem(p)
        groups = groups_of(p, name)
        for radius, scaling in SETTINGS:
            sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
            orc = tvm.run_oracle(pr, radius, scaling)
            o = operator(emu, p, radius, scaling, orc["y_cam"])
            n = sysm["n_rows"]
            cam_step = np.zeros((pr.M, 6)); cam_step[pr.cam_active] = (o["s_cam"][:6 * n] * orc["y_cam"]).reshape(-1, 6)
            imp = dict(S=None, rhs=o["rhs"][:6 * n].reshape(n, 6), cost=o["out"][0], model=o["model"][0],
                       pt_step=o["pt_step"][pr.tv], cam_step=cam_step)
            per, (rc, rm) = tvm.measure(p, sysm, imp, groups)
            ra = damped_ratios(sysm, o["A"], groups)
            po, _ = tvm.measure(p, sysm, orc, groups)
            px, _ = tvm.measure(p, sysm, tvm.run_emu(lib, p, pr, radius, scaling, orc["y_cam"]), groups)
            sym = vm.symmetry_ratio(o["A"], vm.dense(vm.damped(sysm)["T"], n))
            for g, v in per.items():
                out[(name, g, radius, scaling)] = dict(imp=(ra[g],) + v[1:] + (rc, rm, sym), oracle=po[g], expl=px[g])
    return out


def test_every_problem_takes_the_matrix_free_product(emu, family):
    """every problem of the family is over the rule (with ballast, and also without: a camera row of a few short tracks weighs
    8 envelope blocks against 16 observations); with many short tracks on three cameras of their own it is under it"""
    def rule(p):
        c = tie._counts(p)
        return emu.emu_imp_choose(*[ctypes.c_int64(x) for x in c[:3]], ctypes.c_int(c[3]))
    for name, p in family.items():
        assert rule(p) == 1, name
    for make in (dl.isolated, dl.shared, dl.distort, dl.huber_edge, dl.cauchy_far):
        assert rule(make()) == 1, make.__name__
        assert rule(dl.ballast(make(), **dl.EXPLICIT)) == 0, make.__name__
    iso = family["isolated"]
    op = iso["obs_ptr"]
    for a in np.nonzero(np.isin(iso["cls"], ["repeat", "ballast"]))[0]:
        cams = iso["obs_cam"][op[a]:op[a + 1]]
        assert len(np.unique(cams)) < len(cams)           # a camera seen more than once: a run in its row


def test_host_matrix_free_passes_meet_the_bounds(measured, capsys):
    """every ratio within its constant, the A blocks of WIDE_S's pairs within theirs; on the isolated pairs the float64 oracle
    meets C_S (shared arithmetic of the passes), on the Cauchy ballast it does not (the reference's scale)"""
    worst = {}
    for (name, g, radius, scaling), v in measured.items():
        if unbounded(g, radius):
            assert np.isfinite(v["imp"]).all(), (name, g, radius, scaling)
            continue
        w = worst.setdefault((name, g), np.zeros(12))
        np.maximum(w, tuple(v["imp"]) + tuple(v["oracle"]) + tuple(v["expl"]), out=w)
    with capsys.disabled():
        print("\nhost matrix-free passes: |float64 - mp| / (eps E), worst over radius 1e4 / 1e12 and Jacobi scaling on / off;"
              " symmetry: |A_ij - A_ji| over its bound; the float64 oracle's and the explicit host passes' S / rhs / point:")
        print(f"  {'problem':12s} {'group':14s} {'A':>9s} {'rhs':>9s} {'point':>9s} {'cost':>9s} {'model':>9s} {'symmetry':>9s}"
              f" {'orc S':>9s} {'orc rhs':>9s} {'orc pt':>9s} {'expl S':>9s} {'expl rhs':>9s} {'expl pt':>9s}")
        for (name, g), w in sorted(worst.items()):
            print(f"  {name:12s} {g:14s} " + " ".join(f"{x:9.3g}" for x in w))
        print("  bounds: C_S {:g} C_RHS {:g} C_PT {:g} C_COST {:g}, symmetry 1; A of {}".format(
            vm.C_S, vm.C_RHS, vm.C_PT, vm.C_COST, ", ".join(f"{n} {g} {b:g}" for (n, g), b in WIDE_S.items())))
    for (name, g, radius, scaling), v in measured.items():
        if unbounded(g, radius):
            continue
        const = (bound_S(name, g), vm.C_RHS, vm.C_PT, vm.C_COST, vm.C_COST, 1.0)
        assert all(x <= c for x, c in zip(v["imp"], const)), (name, g, radius, scaling, v)
    for (name, g) in (("isolated", "repeat"), ("isolated", "far")):
        assert worst[(name, g)][6] <= vm.C_S, (name, g, "the float64 oracle")
    assert worst[("cauchy_far", "ballast")][6] > vm.C_S                     # every float64 implementation alike
    for (name, g) in (("isolated", "repeat"), ("cauchy_far", "ballast")):    # far exceeds C_S on the H100 only (157)
        assert worst[(name, g)][0] > vm.C_S, (name, g, "no longer exceeds C_S: drop it from WIDE_S")


def _long_track_scene():
    """60 cameras, a 200-observation track over all of them (each seen three or four times) and a repeated-camera track"""
    return vs.make_scene(5, M=60, n_short=60, long_tracks=((200, 0),), extra_tracks=([3, 3, 4, 3, 5],))


def test_plain_double_misses_the_symmetry_bound(emu, family, capsys):
    """the double-double product meets the symmetry bound; the same product in plain double misses it by at least 100x on the
    far, cancel and repeat classes and on a long-track scene"""
    p = family["isolated"]
    pr = oracle_problem(p)
    rows = []
    for radius, scaling in ((1e4, True), (1e12, False)):
        sysm = vm.system(p["lin"], pr.cam_col, radius, scaling)
        o = operator(emu, p, radius, scaling)
        Apd = plain_double(o)
        for g, idx in groups_of(p, "isolated").items():
            r = np.array([6 * i + a for i in class_rows(sysm, idx) for a in range(6)])
            T = vm.dense(vm.damped(sysm, [sysm["lm"][a] for a in idx])["T"], sysm["n_rows"])[np.ix_(r, r)]
            d = np.abs(Apd[np.ix_(r, r)] - o["A"][np.ix_(r, r)])
            assert (d <= 1e3 * vm.EPS * T + np.spacing(np.abs(o["A"][np.ix_(r, r)]))).all(), g   # the same operator, to rounding
            rows.append((f"isolated {g}, radius {radius:g}", vm.symmetry_ratio(o["A"][np.ix_(r, r)], T),
                         vm.symmetry_ratio(Apd[np.ix_(r, r)], T), g in TEETH))
    q = _long_track_scene()
    pq = vo.VisualProblem(*vs.args(q))
    for radius, scaling in ((1e4, True), (1e12, False)):
        o = operator(emu, q, radius, scaling)
        T = vm.term_scale_f64(pq, radius, scaling)
        rows.append((f"long track, radius {radius:g}", vm.symmetry_ratio(o["A"], T), vm.symmetry_ratio(plain_double(o), T), True))
    with capsys.disabled():
        print("\nsymmetry |A_ij - A_ji| / (ulp + 64 eps^2 T_ij), worst entry: double-double product, plain-double restatement")
        for lab, dd, pd, _ in rows:
            print(f"  {lab:34s} {dd:9.3g} {pd:11.3g}")
    for lab, dd, pd, teeth in rows:
        assert dd <= 1.0, lab
        if teeth:
            assert pd >= 100.0, lab


def test_preconditioner_blocks_match_the_reference(emu, family):
    """D_r + diag(dadd_r), the blocks the preconditioner inverts (RowPartF / RowSumF with their runs), are A's diagonal blocks
    of the reference within the A bound of their class"""
    for name in ("isolated", "tile_and_big"):
        p = family[name]
        pr = oracle_problem(p)
        for radius, scaling in ((1e4, True), (1e12, False)):
            sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
            o = operator(emu, p, radius, scaling)
            n = sysm["n_rows"]
            D = o["D"][:36 * n].reshape(n, 6, 6) + np.einsum("ra,ab->rab", o["dadd"][:6 * n].reshape(n, 6), np.eye(6))
            for g, idx in groups_of(p, name).items():
                if unbounded(g, radius):
                    continue
                ref = vm.damped(sysm, [sysm["lm"][a] for a in idx])
                for i in class_rows(sysm, idx):
                    assert vm.ratio(np.abs(D[i] - ref["S"][(i, i)]).max(), ref["S_hat"][(i, i)]) <= bound_S(name, g), (name, g, i)
                    assert np.array_equal(D[i], D[i].T)


# ------------------------------------------------------------------ one preconditioned CG iteration
# With min_linear_iter = max_linear_iter = 1 the camera step is alpha M^-1 rhs (x_0 = 0, p_0 = M^-1 r_0), M = blockdiag(D_r +
# diag dadd_r).  Per row r, after fitting the scalar alpha to the 50-digit direction M_ref^-1 rhs_ref (computed at 50 digits
# from the reference's blocks rounded to float64), |y_r - alpha ref_r|_max <= C_PREC eps kappa_inf(M_r) |alpha ref_r|_max.
# Calibrated below on the host-compiled solve (vpcg::solve_with with PrecDF, tests/emu/visual_implicit_emu.cpp): the smallest
# power of two at least 4x the worst ratio.  Radius 1e12 is left out: there the near_z, rotation, far and repeat blocks are
# indefinite in float64 and the preconditioner ends the solve in FAILURE (the LM's invalid step), as Ceres' does.
C_PREC = 2.0 ** 18


def prec_ratios(sysm, y, groups, skip=()):
    """{group: worst row ratio} of the scaled camera step y [n_rows * 6] against alpha M_ref^-1 rhs_ref, alpha fitted over every
    row with a reference direction; and alpha"""
    from mpmath import mp
    n = sysm["n_rows"]
    ref = vm.damped(sysm)
    rhs = vm.assemble(sysm)["rhs"]
    d = np.zeros((n, 6)); kap = np.zeros(n)
    for i in range(n):
        if (i, i) not in ref["S"]:
            continue
        M = ref["S"][(i, i)]
        x = mp.lu_solve(mp.matrix(M.tolist()), mp.matrix(rhs[i].tolist()))
        d[i] = [float(v) for v in x]
        kap[i] = np.abs(M).sum(1).max() * np.abs(np.linalg.inv(M)).sum(1).max()
    y = y.reshape(n, 6)
    alpha = float((d * y).sum() / (d * d).sum())
    out = {}
    for g, idx in groups.items():
        if g in skip:
            continue
        rows = {i for a in idx for i in sysm["lm"][a]["urows"]}
        out[g] = max((np.abs(y[i] - alpha * d[i]).max() / (vm.EPS * kap[i] * abs(alpha) * np.abs(d[i]).max())
                      for i in rows if np.abs(d[i]).max() > 0), default=0.0)
    return out, alpha


PREC_CASES = [("isolated", 1e4, True), ("isolated", 1e4, False), ("tile_and_big", 1e4, True), ("distort", 1e4, True),
              ("huber_edge", 1e4, True), ("cauchy_far", 1e4, True)]


def one_iteration(emu, p, radius, scaling):
    """the host CG's step after one iteration (PrecDF) on the matrix-free operator, and (iterations, termination)"""
    o = operator(emu, p, radius, scaling)
    L = o["L"]
    n6 = 6 * L.n
    lp, ll = p.get("loss_px") or (0, 1.0), p.get("loss_pl") or (0, 1.0)
    r = tie.run(emu, L, radius, scaling, losses=(lp[0], lp[1], ll[0], ll[1]), dadd=o["dadd"][:n6], eta=0.1, min_iter=1, max_iter=1)
    return r["x_sol"][:n6], (int(r["info"][0]), int(r["info"][1]))


def test_one_preconditioned_iteration_calibration(emu, family, capsys):
    """the host-compiled CG (PrecDF, one iteration) on the matrix-free operator: every row within C_PREC; the constant is the
    smallest power of two at least 4x the worst row"""
    worst = {}
    for name, radius, scaling in PREC_CASES:
        p = family[name]
        pr = oracle_problem(p)
        sysm = vm.system(p["lin"], pr.cam_col, radius, scaling, p.get("loss_px"), p.get("loss_pl"))
        y, info = one_iteration(emu, p, radius, scaling)
        assert info == (1, 1), (name, info)                   # one iteration, NO_CONVERGENCE at the iteration limit
        per, _ = prec_ratios(sysm, y, groups_of(p, name))
        for g, v in per.items():
            worst[(name, g, radius)] = v
    w = max(worst.values())
    with capsys.disabled():
        print("\none preconditioned CG iteration, host: |y_r - alpha ref_r| / (eps kappa(M_r) |alpha ref_r|), worst row per class:")
        for k, v in sorted(worst.items()):
            print(f"  {k[0]:12s} {k[1]:14s} radius {k[2]:7.0e} {v:9.3g}")
        print(f"  worst {w:.3g}; smallest power of two >= 4x: {2.0 ** np.ceil(np.log2(4 * w)):g}; in use C_PREC = {C_PREC:g}")
    assert 4 * w <= C_PREC


def test_explicit_operator_is_bitwise_symmetric(emu, family, tmp_path_factory):
    """the explicit product (vpcg::ProdF, as visual_pcg_product_kernel: one stored block for both triangles), applied to every
    unit vector on the S of the explicit host passes, is symmetric bit for bit"""
    so = tmp_path_factory.mktemp("pcg_emu") / "libvisual_pcg_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_pcg_emu.cpp"), "-o", str(so)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    pcg = ctypes.CDLL(str(so))
    p = family["isolated"]
    L = Local(p, 0)
    n, n6 = L.n, 6 * L.n
    o = tie.run(emu, L, 1e4, True)
    S = np.ascontiguousarray(o["S"])
    dadd = np.ascontiguousarray(np.clip(o["colsq"][:n6], 1e-6, 1e32) / 1e4)
    first = np.ascontiguousarray(L.first, np.int32)
    last = np.ascontiguousarray(np.searchsorted(L.first, np.arange(n), side="right") - 1, np.int32)
    A = np.zeros((n6, n6))
    y = np.zeros(n6)
    for k in range(n6):
        x = np.zeros(n6); x[k] = 1.0
        pcg.emu_pcg_product(ctypes.c_int(n), _p(first, ctypes.c_int), _p(last, ctypes.c_int), _p(L.row_start, ctypes.c_longlong),
                            _p(S), _p(dadd), _p(x), _p(y))
        A[:, k] = y
    assert np.array_equal(A, A.T)
