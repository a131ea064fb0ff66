"""The 50-digit visual reference (oracle/visual_mp.py), the degenerate landmark family (tests/degenerate_landmarks.py) and the
error bounds that the GPU test tests/test_visual_degenerate_gpu.py holds the device to — all without a GPU.

Bounds (oracle/visual_mp.py): every S block, rhs row and point step within C eps E of the 50-digit value, E its first-order
float64 error scale; the cost and the model-cost change of a whole problem likewise.  The constants are calibrated here from
two float64 implementations measured against the 50-digit reference over the whole family (isolated, the 128 / 129 / 300 tile
and big split, the shared trajectory at its perturbed start, distort, huber_edge, cauchy_far), at radius 1e4 and 1e12, with
Jacobi scaling on and off: oracle/visual_oracle.py with tests/visual_loss_oracle.py (a sparse LU of the whole system,
np.linalg.inv per landmark) and the big-landmark passes of global-lvba_b200/csrc/visual_big.h compiled for the host
(tests/emu/visual_loss_emu.cpp: the device's sym3_inverse and per-observation arithmetic).  The point steps are compared
with the 50-digit back-substitution of each implementation's own camera step.  Each constant is the smallest power of two at
least 4x the worst ratio observed (rotation landmarks at radius 1e12 excluded, see below):

    worst ratio      S                 rhs               point step        cost              model
    float64 oracle   12.5 (far)        0.109 (ordinary)  0.151 (big 129)   0.067             8.6e-9
    host big passes  23.2 (far)        0.109 (ordinary)  0.102 (big 129)   0.039             8.4e-9
    constant         C_S = 128         C_RHS = 0.5       C_PT = 1          C_COST = 0.5 (cost and model)

The model-cost scale is loose (|J_c dc| and |J_X dp| nearly cancel in J dx, and their hats do not): its bound catches only
gross errors.

No constant was chosen by looking at GPU output.  At radius 1e12 the rotation class has kappa ~1e13 or more: no bound means
anything there, and only finite S, rhs and steps are required.

Reached by the family (test_family_is_not_vacuous): kappa_l 4e4 (far, near_z, rotation) at radius 1e4 and 3e12 (far) at
1e12; z down to 1e-7 and views at z = 5e-9, below the 1e-8 cut-off; |e| down to 5e-15; Huber s / a^2 - 1 from -6 to +5 ulps
and up to 2e5 a^2; Cauchy s up to 2e9 a^2; coordinates 1e5 m from the origin; the radial factor down to 1e-3.

The bounds discriminate (test_bounds_reject_float64_mistakes): C^-1 formed in float32 for one landmark, the plane term dropped
from one landmark, the Jacobi scale of one point column off by 1e6 ulp, and Huber's rho' taken as a / s instead of a / sqrt(s)
each put at least one ratio at least 4x above its constant.  The device's sym3_inverse in float32, the cut-off at z > 0,
another constant than 1e-12 in plane_eval or Huber's test against a instead of a^2 each make the host big passes of
visual_math.h fail test_float64_implementations_meet_the_bounds.
"""
import ctypes
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import synth
from oracle import visual_mp as vm
from oracle import visual_oracle as vo

sys.path.insert(0, str(Path(__file__).resolve().parent))
import degenerate_landmarks as dl  # noqa: E402
import visual_big_scene as vs  # noqa: E402
import visual_loss_oracle as vl  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
SETTINGS = [(1e4, True), (1e4, False), (1e12, True), (1e12, False)]


def oracle_problem(p, fixed_cam=0):
    return vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam, loss_reproj=p.get("loss_px"), loss_plane=p.get("loss_pl"))


def system(p, lin, cam_row, radius, scaling):
    return vm.system(lin, cam_row, radius, scaling, p.get("loss_px"), p.get("loss_pl"))


@pytest.fixture(scope="module")
def family():
    out = {"isolated": dl.isolated(), "tile_and_big": dl.tile_and_big(), "shared": dl.shared(), "distort": dl.distort(),
           "huber_edge": dl.huber_edge(), "cauchy_far": dl.cauchy_far()}
    for p in out.values():
        p["lin"] = vm.linearize(p)
    return out


def test_matches_float64_oracle_on_well_conditioned_landmarks():
    """synth.make_problem: ordinary landmarks 3-20 m from their cameras, where float64 is accurate to ~1e-12"""
    p = synth.make_problem(12, 0, 60, seed=3, lidar=False)
    pr = vo.VisualProblem(*vs.args(p))
    lin = vm.linearize(p)
    for radius, scaling in ((1e4, True), (3.0, False)):
        ref = vo.single_step(pr, radius, scaling)
        sysm = vm.system(lin, pr.cam_col, radius, scaling)
        A = vm.assemble(sysm)
        n = sysm["n_rows"]
        S = np.zeros((6 * n, 6 * n))
        for (i, j), b in A["S"].items():
            S[6 * i:6 * i + 6, 6 * j:6 * j + 6] = b; S[6 * j:6 * j + 6, 6 * i:6 * i + 6] = b.T
        assert np.abs(S - ref["S_nodamp"]).max() <= 1e-9 * np.abs(S).max()
        assert np.abs(A["rhs"].ravel() - ref["rhs"]).max() <= 1e-9 * np.abs(ref["rhs"]).max()
        assert abs(A["cost"] - ref["cost"]) <= 1e-12 * ref["cost"]
        dp, _, model, _ = vm.backsub(sysm, ref["cam_step"])
        assert np.abs(dp - ref["pt_step"][pr.tv]).max() <= 1e-9 * np.abs(dp).max()
        assert abs(model - ref["model"]) <= 1e-9 * abs(model)
    # the forward-mode Jacobian through the manifold plus is the analytic one of reproj_eval (Q9 tangent basis)
    op = p["obs_ptr"]
    for a in range(0, 60, 7):
        for k, s in enumerate(range(op[a], op[a + 1])):
            c = p["obs_cam"][s]
            r, Jq, Jt, JX = vo.reproj_eval(p["q"][[c]], p["t"][[c]], p["X"][[a]], p["obs_uv"][[s]].astype(np.float64), p["intr"], p["sigma_px"])
            o = lin[a]["obs"][k]
            Jm = np.array([[float(x) for x in row] for row in o["J"]])
            Ja = np.concatenate([Jq[0], Jt[0], JX[0]], 1)
            assert np.abs(Jm - Ja).max() <= 1e-11 * np.abs(Ja).max()
            assert np.abs(np.array([float(x) for x in o["r"]]) - r[0]).max() <= 1e-9


# ------------------------------------------------------------------ float64 implementations
def _emu_lib(tmp):
    so = tmp / "libvisual_loss_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_loss_emu.cpp"), "-o", str(so)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def _ptr(a, t):
    return a.ctypes.data_as(P(t))


def run_emu(lib, p, pr, radius, scaling, y_cam):
    """visual_big.h's passes over every landmark (tests/emu/visual_loss_emu.cpp) with the camera step y_cam (scaled);
    returns S(i, j), rhs [n, 6], cost, model, pt_step [Tv, 3], cam_step [M, 6] (= s_cam y_cam)"""
    op = np.asarray(p["obs_ptr"], np.int64)
    tv = np.nonzero(pr.tv)[0]
    K = np.diff(op)[tv]
    Tv, n = len(tv), pr.nc
    trk_ptr = np.zeros(Tv + 1, np.int32); trk_ptr[1:] = np.cumsum(K)
    trk_id = tv.astype(np.int32)
    sel = np.concatenate([np.arange(op[a], op[a + 1]) for a in tv]).astype(np.int64)
    cam = np.ascontiguousarray(np.asarray(p["obs_cam"])[sel], np.int32)
    row = np.ascontiguousarray(pr.cam_col[cam], np.int32)
    uv = np.ascontiguousarray(np.asarray(p["obs_uv"], np.float32)[sel])
    plane = np.ascontiguousarray(np.asarray(p["plane_nd"], np.float64)[tv])
    first = np.arange(n)
    for a in range(Tv):
        r = row[trk_ptr[a]:trk_ptr[a + 1]]; r = r[r >= 0]
        if len(r):
            first[r] = np.minimum(first[r], r.min())
    first = np.minimum.accumulate(first[::-1])[::-1].astype(np.int32)
    row_start = np.zeros(n + 1, np.int64); row_start[1:] = np.cumsum(np.arange(n) - first + 1)
    intr = np.ascontiguousarray(p["intr"], np.float64)
    lp, ll = p.get("loss_px") or (0, 1.0), p.get("loss_pl") or (0, 1.0)
    kind = np.array([lp[0], ll[0]], np.int32); la = np.array([lp[1], ll[1]], np.float64)
    q, t, X = (np.ascontiguousarray(a, np.float64) for a in (pr.q, pr.t, pr.X))
    o = dict(cam_colsq0=np.zeros(6 * n), pt_colsq0=np.zeros(3 * Tv), S=np.zeros(max(int(row_start[-1]), 1) * 36), rhs=np.zeros(6 * n),
             cam_colsq=np.zeros(6 * n), cam_grad=np.zeros(6 * n), X_cand=X.copy(), pt_step=np.zeros_like(X), out=np.zeros(5))
    yc = np.ascontiguousarray(y_cam, np.float64)
    lib.emu_vloss_step(ctypes.c_int(n), ctypes.c_int64(Tv), _ptr(trk_ptr, ctypes.c_int), _ptr(trk_id, ctypes.c_int), _ptr(cam, ctypes.c_int),
                       _ptr(row, ctypes.c_int), _ptr(uv, ctypes.c_float), _ptr(plane, ctypes.c_double), _ptr(intr, ctypes.c_double),
                       ctypes.c_double(float(p["sigma_px"])), ctypes.c_double(float(p["sigma_plane"])), _ptr(kind, ctypes.c_int),
                       _ptr(la, ctypes.c_double), _ptr(first, ctypes.c_int), _ptr(row_start, ctypes.c_longlong), _ptr(q, ctypes.c_double),
                       _ptr(t, ctypes.c_double), _ptr(X, ctypes.c_double), ctypes.c_int(int(scaling)), ctypes.c_double(radius),
                       ctypes.c_double(1e-6), ctypes.c_double(1e32), _ptr(yc, ctypes.c_double),
                       *[_ptr(o[k], ctypes.c_double) for k in ("cam_colsq0", "pt_colsq0", "S", "rhs", "cam_colsq", "cam_grad", "X_cand",
                                                                "pt_step", "out")])
    blocks = o["S"].reshape(-1, 36)
    s_cam = 1.0 / (1.0 + np.sqrt(o["cam_colsq0"])) if scaling else np.ones(6 * n)
    cam_step = np.zeros((pr.M, 6)); cam_step[pr.cam_active] = (s_cam * yc).reshape(n, 6)
    return dict(S=lambda i, j: blocks[row_start[i] + j - first[i]].reshape(6, 6), rhs=o["rhs"].reshape(n, 6), cost=o["out"][0],
                model=o["out"][2], pt_step=o["pt_step"][tv], cam_step=cam_step)


def run_oracle(pr, radius, scaling):
    ref = vo.single_step(pr, radius, scaling)
    S = ref["S_nodamp"]
    nc6 = 6 * pr.nc
    return dict(S=lambda i, j: S[6 * i:6 * i + 6, 6 * j:6 * j + 6], rhs=ref["rhs"].reshape(-1, 6), cost=ref["cost"], model=ref["model"],
                pt_step=ref["pt_step"][pr.tv], cam_step=ref["cam_step"], y_cam=ref["y"][:nc6])


def measure(p, sysm, dev, groups):
    """{group: (S, rhs, point step) ratios} over the landmark groups {name: indices into sysm['lm']}, and the whole problem's
    (cost, model) ratios, for the results `dev` of one implementation"""
    dp, dph, model, modelh = vm.backsub(sysm, dev["cam_step"])
    out = {}
    for g, idx in groups.items():
        ref = vm.assemble(sysm, [sysm["lm"][a] for a in idx])
        rs, rr, _ = vm.ratios(ref, dev["S"], dev["rhs"])
        rp = max((vm.ratio(e, h) for e, h in zip(np.abs(dev["pt_step"][idx] - dp[idx]).max(1), dph[idx])), default=0.0)
        out[g] = (rs, rr, rp)
    whole = vm.assemble(sysm)
    rc = vm.ratio(abs(dev["cost"] - whole["cost"]), whole["cost_hat"])
    rm = vm.ratio(abs(dev["model"] - model), modelh)
    return out, (float(rc), float(rm))


def groups_of(p, name):
    cls = p["cls"][vo.valid_tracks(p["plane_nd"])]
    if name == "shared":
        return {"shared": np.arange(len(cls))}
    return {str(c): np.nonzero(cls == c)[0] for c in sorted(set(cls))}


def unbounded(group, radius):
    return radius > 1e8 and group == "rotation"


@pytest.fixture(scope="module")
def measured(family, tmp_path_factory):
    """(implementation, problem, group, radius, scaling) -> (S, rhs, point step, cost, model) ratios"""
    lib = _emu_lib(tmp_path_factory.mktemp("vloss_emu"))
    out = {}
    for name, p in family.items():
        pr = oracle_problem(p)
        for radius, scaling in SETTINGS:
            sysm = system(p, p["lin"], pr.cam_col, radius, scaling)
            orc = run_oracle(pr, radius, scaling)
            emu = run_emu(lib, p, pr, radius, scaling, orc["y_cam"])
            for impl, dev in (("float64 oracle", orc), ("host big passes", emu)):
                per, (rc, rm) = measure(p, sysm, dev, groups_of(p, name))
                for g, (rs, rr, rp) in per.items():
                    out[(impl, name, g, radius, scaling)] = (rs, rr, rp, rc, rm)
    return out


def _worst(measured, impl=None):
    vals = [v for (i, _, g, r, _), v in measured.items() if (impl is None or i == impl) and not unbounded(g, r)]
    return np.max(np.array(vals), axis=0)


CONST = (vm.C_S, vm.C_RHS, vm.C_PT, vm.C_COST, vm.C_COST)


@pytest.mark.parametrize("impl", ["float64 oracle", "host big passes"])
def test_float64_implementations_meet_the_bounds(measured, impl):
    for (i, name, g, radius, scaling), v in measured.items():
        if i == impl and not unbounded(g, radius):
            assert all(x <= c for x, c in zip(v, CONST)), (name, g, radius, scaling, v)


def test_bounds_calibration(measured, capsys):
    """each constant is the smallest power of two at least 4x the worst ratio of the float64 implementations; the table is
    printed so that a change in the float64 arithmetic shows"""
    worst = _worst(measured)
    with capsys.disabled():
        print("\nobserved |float64 - mp| / (eps E), worst over radius 1e4 / 1e12 and Jacobi scaling on / off:")
        print(f"  {'implementation':16s} {'problem':12s} {'group':14s} {'S':>9s} {'rhs':>9s} {'point':>9s} {'cost':>9s} {'model':>9s}")
        keys = sorted({(i, n, g) for i, n, g, _, _ in measured})
        for i, n, g in keys:
            v = np.max([val for (i2, n2, g2, r, _), val in measured.items() if (i2, n2, g2) == (i, n, g) and not unbounded(g, r)], axis=0)
            print(f"  {i:16s} {n:12s} {g:14s} " + " ".join(f"{x:9.3g}" for x in v))
        for impl in ("float64 oracle", "host big passes"):
            print(f"  worst {impl}: " + " ".join(f"{x:.3g}" for x in _worst(measured, impl)))
        calib = [2.0 ** math.ceil(math.log2(4 * w)) if w > 0 else 1.0 for w in worst]
        print("  smallest powers of two >= 4x worst: C_S {:g} C_RHS {:g} C_PT {:g} C_COST {:g} / {:g}; in use: {:g} {:g} {:g} {:g}".format(
            *calib, vm.C_S, vm.C_RHS, vm.C_PT, vm.C_COST))
    assert all(4 * w <= c for w, c in zip(worst, CONST))


def test_rotation_at_radius_1e12_is_finite(family, measured):
    """the float64 oracle and the host passes give finite S, rhs and steps where no bound applies"""
    p = family["isolated"]
    pr = oracle_problem(p)
    for scaling in (True, False):
        ref = vo.single_step(pr, 1e12, scaling)
        assert np.isfinite(ref["S_nodamp"]).all() and np.isfinite(ref["rhs"]).all()
        assert np.isfinite(ref["cam_step"]).all() and np.isfinite(ref["pt_step"]).all()
    assert all(np.isfinite(v).all() for v in measured.values())


def test_family_is_not_vacuous(family, capsys):
    """the ranges the family reaches, from the 50-digit reference"""
    iso = family["isolated"]
    pr = oracle_problem(iso)
    kap = {}
    for radius in (1e4, 1e12):
        sysm = system(iso, iso["lin"], pr.cam_col, radius, True)
        cls = iso["cls"][pr.tv]
        for L, c in zip(sysm["lm"], cls):
            kap[(c, radius)] = max(kap.get((c, radius), 0.0), L["kappa"])
    obs = [o for L in iso["lin"] for o in L["obs"]]
    z_valid = min(float(o["z"]) for o in obs if o["valid"])
    cut = [float(o["z"]) for o in obs if not o["valid"]]
    e = [abs(float(L["plane"]["e"])) for L in iso["lin"]]
    he = family["huber_edge"]
    a2 = vm.mpf(he["loss_px"][1]) ** 2
    rel = [float((L["obs"][0]["r"][0] ** 2 + L["obs"][0]["r"][1] ** 2) / a2 - 1) / vm.EPS for L in he["lin"][:12]]
    far = [float((L["obs"][0]["r"][0] ** 2 + L["obs"][0]["r"][1] ** 2) / a2) for L in he["lin"][12:]]
    cf = family["cauchy_far"]
    cfar = max(float((o["r"][0] ** 2 + o["r"][1] ** 2) / vm.mpf(cf["loss_px"][1]) ** 2) for L in cf["lin"] for o in L["obs"])
    off = max(np.abs(iso["t"]).max(), np.abs(iso["X"]).max())
    d = family["distort"]
    k1, k2 = d["intr"][4], d["intr"][5]
    Xc = []
    for a, L in enumerate(d["lin"]):
        c = d["obs_cam"][d["obs_ptr"][a]]
        R = vo.quat_to_rot(d["q"][[c]])[0]
        x = R @ d["X"][a] + d["t"][c]
        Xc.append((x[0] / x[2]) ** 2 + (x[1] / x[2]) ** 2)
    rad = min(abs(1 + k1 * r2 + k2 * r2 * r2) for r2 in Xc)
    with capsys.disabled():
        print("\nreached by the degenerate landmark family:")
        for (c, radius), k in sorted(kap.items()):
            print(f"  kappa_l {c:9s} radius {radius:7.0e}: {k:9.3g}")
        print(f"  smallest z of a view {z_valid:.3g}, views cut off at z {sorted(cut)[:3]}...; smallest |e| {min(e):.3g}")
        print(f"  Huber s / a^2 - 1 in ulps {sorted(rel)}; far {min(far):.3g} .. {max(far):.3g} a^2; Cauchy s up to {cfar:.3g} a^2")
        print(f"  largest coordinate {off:.3g} m; smallest radial factor {rad:.3g}")
    assert max(kap.values()) >= 1e8 and max(k for (c, r), k in kap.items() if c != "rotation") >= 1e8
    assert z_valid < 1e-6 and len(cut) >= 6 and all(0 < z < 1e-8 for z in cut)
    assert min(e) < 1e-8
    assert min(rel) < 0 < max(rel) and max(abs(x) for x in rel) <= 16
    assert max(far) > 1e5 and cfar > 1e8
    assert off >= 1e4
    assert rad < 0.1


def test_bounds_reject_float64_mistakes(family):
    """deliberate float64 mistakes in the float64 oracle's results put a ratio at least 4x above its constant: C^-1 of one
    landmark in float32 (its point step), the plane term of one landmark dropped, one point column's Jacobi scale off by 1e6
    ulp in the step's conversion, Huber's rho' = a / s instead of a / sqrt(s)"""
    iso = family["isolated"]
    pr = oracle_problem(iso)
    sysm = system(iso, iso["lin"], pr.cam_col, 1e4, True)
    orc = run_oracle(pr, 1e4, True)
    groups = {"all": np.arange(int(pr.tv.sum()))}
    per, costs = measure(iso, sysm, orc, groups)
    base = per["all"] + costs
    assert all(x <= c for x, c in zip(base, CONST))
    l = int(np.argmin([L["kappa"] for L in sysm["lm"]]))          # the best-conditioned landmark: the hardest to catch
    L = sysm["lm"][l]
    sp = np.array([float(c) for c in L["s_pt"]])

    def ratios_with(dev):
        per, costs = measure(iso, sysm, dev, groups)
        return np.array(per["all"] + costs) / np.array(CONST)

    # C^-1 in float32 for landmark l: its point step y = -C^-1 b
    dev = dict(orc); dev["pt_step"] = orc["pt_step"].copy()
    y = orc["pt_step"][l] / sp
    b = -L["C"] @ y
    dev["pt_step"][l] = sp * -(np.linalg.inv(L["C"].astype(np.float32)).astype(np.float64) @ b)
    assert ratios_with(dev).max() >= 4
    # one point column's Jacobi scale off by 1e6 ulp where the step is scaled back
    dev = dict(orc); dev["pt_step"] = orc["pt_step"].copy()
    dev["pt_step"][l, 0] *= 1 + 1e6 * vm.EPS
    assert ratios_with(dev).max() >= 4
    # the plane term dropped from landmark l (the float64 oracle without its plane residual)
    keep = vo.plane_eval
    a_trk = L["track"]

    def no_plane(X, plane_nd, sigma):
        r, J = keep(X, plane_nd, sigma)
        k = int(np.nonzero(np.nonzero(pr.tv)[0] == a_trk)[0][0])
        r = r.copy(); J = J.copy(); r[k] = 0.0; J[k] = 0.0
        return r, J
    vo.plane_eval = no_plane
    try:
        dev = run_oracle(oracle_problem(iso), 1e4, True)
    finally:
        vo.plane_eval = keep
    assert ratios_with(dev).max() >= 4
    # Huber's rho' = a / s on the huber_edge problem
    he = family["huber_edge"]
    prh = oracle_problem(he)
    sysh = system(he, he["lin"], prh.cam_col, 1e4, True)
    gh = {"all": np.arange(int(prh.tv.sum()))}
    keep_rho = vl.loss_rho

    def wrong_rho(kind, a, s):
        rho, d = keep_rho(kind, a, s)
        if kind == vl.HUBER:
            s = np.asarray(s, np.float64)
            d = np.where(s > a * a, np.maximum(vl._TINY, a / np.where(s > a * a, s, 1.0)), d)
        return rho, d
    vl.loss_rho = wrong_rho
    try:
        dev = run_oracle(oracle_problem(he), 1e4, True)
    finally:
        vl.loss_rho = keep_rho
    per, costs = measure(he, sysh, dev, gh)
    assert (np.array(per["all"] + costs) / np.array(CONST)).max() >= 4
