"""The passes of the DOGLEG trust-region strategy (global-lvba_b200/csrc/visual_dogleg.h) without a GPU, through the host policy
(tests/emu/visual_dogleg_emu.cpp): D, g, the Gauss-Newton step, alpha (through |J~ v|^2), the chosen step of each case, its
model cost change and the candidate landmarks against tests/visual_dogleg_oracle.py to 1e-10, on scenes with 129- and
300-observation tracks, a camera that sees a landmark twice, constant cameras, landmarks without a plane and a loss.  Then the
same with the items of every pass in a shuffled order, which must give the same bits."""
import ctypes
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import synth
import visual_big_scene as vs
import visual_dogleg_oracle as dl
import visual_fixed_oracle as vf
import visual_loss_oracle as vl

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
sys.path.insert(0, str(ROOT / "tests"))
from test_visual_big_emu import Local  # noqa: E402

KJV = 9                                              # vdog::kJv; the scalars: gg nn gn alpha case beta cg cn |s|, then the J~ v sums
NSCAL = KJV + 4


def _lib(tmp):
    so = Path(tmp) / "libvisual_dogleg_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_dogleg_emu.cpp"),
                        "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _lib(tmp_path_factory.mktemp("emu"))


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(P(t))


def _scene(name):
    if name == "small":
        return synth.make_problem(30, 600, 300, seed=11), None, None
    if name == "long":
        p = vs.make_scene(5, M=120, n_short=150, long_tracks=((129, 10), (300, 0)), extra_tracks=([3, 3, 4, 5],))
        p["plane_nd"][[2, 7]] = 0.0                       # two landmarks without a plane: not in the problem
        return p, (vl.HUBER, 1.0), None
    if name == "constant":
        return synth.make_problem(30, 600, 300, seed=11), (vl.CAUCHY, 1.0), (0, 3, 4)
    raise KeyError(name)


def setup(name):
    """The scene, its local layout, the oracle problem and the inputs of the passes at the start state"""
    p, loss, cams = _scene(name)
    L = Local(p, 0)
    pr = vl.RobustProblem(*vs.args(p), loss_reproj=loss)
    if cams is not None:
        vf.with_constant(pr, cams)
        L.pr = pr
        L.n = pr.nc
        L.row = np.ascontiguousarray(pr.cam_col[L.cam], np.int32)
    res, J = pr.residuals(jac=True)
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel()))
    Js = (J @ sp.diags(scale)).tocsr()
    D, g, alpha = dl.linearise(Js, res)
    y = dl.gauss_newton(Js, res, D, dl.MIN_MU)
    nc6 = 6 * pr.nc
    inp = dict(s_cam=scale[:nc6], s_pt=scale[nc6:], colsq=np.asarray(Js.multiply(Js).sum(0)).ravel()[:nc6],
               grad=(Js.T @ res)[:nc6], y=y[:nc6], pt_step=np.zeros((pr.T, 3)))
    inp["pt_step"][pr.tv] = (scale[nc6:] * y[nc6:]).reshape(-1, 3)
    ref = dict(D=D, g=g, GN=D * y, alpha=alpha, Js=Js, res=res, scale=scale)
    return p, loss, L, pr, inp, ref


def run(emu, p, loss, L, inp, radii):
    n = 6 * L.n + 3 * L.Tv
    T = len(p["X"])
    lp, ap = loss if loss else (0, 1.0)
    c = {k: np.ascontiguousarray(v, np.float64) for k, v in inp.items()}
    q, t, X = (np.ascontiguousarray(p[k], np.float64) for k in ("q", "t", "X"))
    radii = np.ascontiguousarray(radii, np.float64)
    o = dict(D=np.zeros(n), g=np.zeros(n), gn=np.zeros(n), sc=np.zeros((len(radii), NSCAL)), v=np.zeros((len(radii), n)),
             Xc=np.zeros((len(radii), T, 3)), scal=np.zeros((len(radii), 3)))
    emu.emu_dogleg_run(ctypes.c_int(L.n), ctypes.c_int64(L.Tv), *L.common(), ctypes.c_int(lp), ctypes.c_double(ap), ctypes.c_int(0),
                       ctypes.c_double(0.1), _p(q), _p(t), _p(X), ctypes.c_int64(T), _p(c["s_cam"]), _p(c["s_pt"]), _p(c["colsq"]),
                       _p(c["grad"]), _p(c["y"]), _p(c["pt_step"]), ctypes.c_int(len(radii)), _p(radii),
                       *[_p(o[k]) for k in ("D", "g", "gn", "sc", "v", "Xc", "scal")])
    return o


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


def _radii(ref):
    gnorm, gn_norm = np.linalg.norm(ref["g"]), np.linalg.norm(ref["GN"])
    a = ref["alpha"] * gnorm
    assert a < gn_norm
    return [2.0 * gn_norm, 0.5 * a, 0.5 * (a + gn_norm)]      # cases 1, 2, 3 (the first fresh, the others reusing)


@pytest.mark.parametrize("name", ["small", "long", "constant"])
def test_passes_match_the_oracle(emu, name):
    p, loss, L, pr, inp, ref = setup(name)
    radii = _radii(ref)
    o = run(emu, p, loss, L, inp, radii)
    for k, r in (("D", "D"), ("g", "g"), ("gn", "GN")):
        assert _rel(o[k], ref[r]) <= 1e-10, k
    Js, res = ref["Js"], ref["res"]
    for j, (radius, case) in enumerate(zip(radii, (dl.GAUSS_NEWTON, dl.CAUCHY, dl.INTERPOLATED))):
        sc = o["sc"][j]
        assert abs(sc[3] - ref["alpha"]) <= 1e-10 * ref["alpha"]
        c, s, snorm, beta = dl.dogleg_step(ref["g"], ref["GN"], ref["alpha"], radius)
        assert int(sc[4]) == c == case
        assert abs(sc[8] - snorm) <= 1e-10 * snorm and abs(sc[5] - beta) <= 1e-10
        v = s / ref["D"]
        assert _rel(o["v"][j], v) <= 1e-10
        Jv = Js @ v
        model = -float(Jv @ (res + 0.5 * Jv))
        assert abs(o["scal"][j][0] - model) <= 1e-10 * abs(model)
        assert abs(sc[KJV + 3] - float(Jv @ Jv)) <= 1e-10 * float(Jv @ Jv)
        Xn = pr.plus(v * ref["scale"])[2]
        assert _rel(o["Xc"][j][pr.tv], Xn[pr.tv]) <= 1e-12
    if name == "long":
        assert sorted(np.diff(L.trk_ptr))[-2:] == [129, 300]


def _dump(name, out):
    p, loss, L, pr, inp, ref = setup(name)
    import tempfile
    o = run(_lib(tempfile.mkdtemp()), p, loss, L, inp, _radii(ref))
    np.savez(out, **o)


def test_shuffled_items_give_the_same_bits(tmp_path):
    outs = []
    for seed in (None, "7"):
        env = dict(os.environ)
        env.pop("LVBA_EMU_SHUFFLE", None)
        if seed:
            env["LVBA_EMU_SHUFFLE"] = seed
        f = tmp_path / f"o{seed}.npz"
        code = (f"import sys; sys.path[:0] = {json.dumps([str(ROOT), str(ROOT / 'tests')])}; "
                f"import test_visual_dogleg_emu as t; t._dump('long', {json.dumps(str(f))})")
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=str(ROOT))
        assert r.returncode == 0, r.stderr
        outs.append(np.load(f))
    a, b = outs
    for k in a.files:
        assert np.array_equal(a[k], b[k]), k
