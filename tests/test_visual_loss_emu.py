"""The robust-loss passes of path B (the kLoss instantiations of global-lvba_b200/csrc/visual_big.h) checked without a GPU: run
through the host policy over EVERY landmark of a problem, each treated as big (tests/emu/visual_loss_emu.cpp), against
tests/visual_loss_oracle.py — cost 1/2 sum rho, column norms of the corrected Jacobian, the point-block gradient, the reduced camera
system and its rhs, and, given the oracle's camera step, the landmark step and the model-cost change.  Tolerances of
tests/test_visual_big_gpu.py.  Re-run with shuffled items and under ASan/UBSan."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import visual_big_scene as vs
import visual_loss_oracle as vl
from test_visual_big_emu import Local

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
LOSSES = [((vl.HUBER, 1.0), (vl.HUBER, 0.1)), ((vl.CAUCHY, 1.0), (vl.CAUCHY, 0.1)), ((vl.HUBER, 0.5), None), (None, (vl.CAUCHY, 0.02))]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libvisual_loss_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []),
           "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_loss_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(so))
    lib.emu_vloss_cost.restype = ctypes.c_double
    return lib


def _ptr(a, t):
    return a.ctypes.data_as(P(t))


def _loss_args(lr, lp):
    kind = np.array([(lr or (vl.NONE, 1.0))[0], (lp or (vl.NONE, 1.0))[0]], np.int32)
    a = np.array([(lr or (vl.NONE, 1.0))[1], (lp or (vl.NONE, 1.0))[1]], np.float64)
    return kind, a


def _step(emu, L, kind, a, radius, scaling, y_cam):
    pr = L.pr
    q, t, X = (np.ascontiguousarray(v, np.float64) for v in (pr.q, pr.t, pr.X))
    n6, nb = max(L.n, 1) * 6, max(int(L.row_start[-1]), 1)
    o = dict(cam_colsq0=np.zeros(n6), pt_colsq0=np.zeros(max(L.Tv, 1) * 3), S=np.zeros(nb * 36), rhs=np.zeros(n6),
             cam_colsq=np.zeros(n6), cam_grad=np.zeros(n6), X_cand=X.copy(), pt_step=np.zeros_like(X), out=np.zeros(5))
    yc = np.ascontiguousarray(y_cam, np.float64)
    emu.emu_vloss_step(ctypes.c_int(L.n), ctypes.c_int64(L.Tv), *L.common(), _ptr(kind, ctypes.c_int), _ptr(a, ctypes.c_double),
                       _ptr(L.first, ctypes.c_int), _ptr(L.row_start, ctypes.c_longlong), _ptr(q, ctypes.c_double), _ptr(t, ctypes.c_double),
                       _ptr(X, ctypes.c_double), ctypes.c_int(int(scaling)), ctypes.c_double(radius), ctypes.c_double(1e-6), ctypes.c_double(1e32),
                       _ptr(yc, ctypes.c_double), *[_ptr(o[k], ctypes.c_double) for k in
                       ("cam_colsq0", "pt_colsq0", "S", "rhs", "cam_colsq", "cam_grad", "X_cand", "pt_step", "out")])
    S = np.zeros((6 * L.n, 6 * L.n))
    blocks = o["S"].reshape(-1, 6, 6)
    for r in range(L.n):
        for c in range(L.first[r], r + 1):
            b = blocks[L.row_start[r] + c - L.first[r]]
            S[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
            S[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
    o["S_dense"] = S
    return o


def _cost(emu, L, kind, a, q, t, X):
    q, t, X = (np.ascontiguousarray(v, np.float64) for v in (q, t, X))
    return emu.emu_vloss_cost(ctypes.c_int64(L.Tv), *L.common(), _ptr(kind, ctypes.c_int), _ptr(a, ctypes.c_double),
                              _ptr(q, ctypes.c_double), _ptr(t, ctypes.c_double), _ptr(X, ctypes.c_double))


def check(emu, p, lr, lp, fixed_cam=0, radius=1e4, scaling=True):
    L = Local(p, fixed_cam)
    L.pr = pr = vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam, loss_reproj=lr, loss_plane=lp)
    kind, a = _loss_args(lr, lp)
    ref = vl.single_step(pr, radius, scaling)
    nc6 = 6 * pr.nc
    o = _step(emu, L, kind, a, radius, scaling, ref["y"][:nc6] if nc6 else np.zeros(6))
    assert abs(o["out"][0] - ref["cost"]) <= 1e-10 * ref["cost"]
    res, J = pr.residuals(jac=True)
    colsq = np.asarray(J.multiply(J).sum(0)).ravel()
    got = np.concatenate([o["cam_colsq0"][:nc6], o["pt_colsq0"][:3 * L.Tv]])
    assert np.abs(got - colsq).max() <= 1e-10 * np.abs(colsq).max()
    g_pt = (J.T @ res)[nc6:]
    assert abs(o["out"][1] - np.abs(g_pt).max()) <= 1e-8 * np.abs(g_pt).max()
    if nc6:
        assert np.abs(o["S_dense"] - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
        assert np.abs(o["rhs"][:nc6] - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    assert np.abs(o["pt_step"] - ref["pt_step"]).max() <= 1e-6 * max(np.abs(ref["pt_step"]).max(), 1e-300)
    assert abs(o["out"][2] - ref["model"]) <= 1e-7 * abs(ref["model"])
    qn, tn, Xn = pr.plus(np.concatenate([ref["cam_step"][pr.cam_active].ravel(), ref["pt_step"][pr.tv].ravel()]))
    c_cand = pr.cost(qn, tn, Xn)
    assert abs(_cost(emu, L, kind, a, qn, tn, Xn) - c_cand) <= 1e-10 * c_cand
    assert abs(_cost(emu, L, kind, a, pr.q, pr.t, pr.X) - ref["cost"]) <= 1e-10 * ref["cost"]
    # the loss is in effect: the robust cost is below the plain one
    assert ref["cost"] < vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam).cost()


def _scene():
    p = vs.make_scene(41, M=80, n_short=150, long_tracks=((129, 10), (200, 30)), extra_tracks=([3, 3, 4, 3, 5],))
    p, _ = vl.with_outliers(p, 0.05, 20.0, 50.0, 41)
    return p


@pytest.mark.parametrize("fixed_cam", [0, -1])
@pytest.mark.parametrize("lr,lp", LOSSES)
def test_loss_passes_match_oracle(emu, lr, lp, fixed_cam):
    check(emu, _scene(), lr, lp, fixed_cam)


def test_loss_passes_unscaled_small_radius(emu):
    check(emu, _scene(), (vl.HUBER, 1.0), (vl.HUBER, 0.1), 0, radius=3.0, scaling=False)


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261016")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__, "-k", "not rerun"],
                       capture_output=True, text=True, cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
