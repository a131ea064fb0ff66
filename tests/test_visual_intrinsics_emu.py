"""The passes of the intrinsics block of the visual LM (global-lvba_b200/csrc/visual_intr.h) without a GPU: run through the host
policy (tests/emu/visual_intrinsics_emu.cpp) over tile-sized and long landmarks (129 to 700 observations), their border, corner,
rhs_k, column norms, corner solve and back-substitution against tests/visual_intr_oracle.py; then once more with the items of
every pass in a shuffled order, and under the address and UB sanitizers."""
import ctypes
import os
import subprocess
import sys
from ctypes import POINTER as P
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

from oracle import synth  # noqa: E402
import visual_big_scene as vs  # noqa: E402
import visual_intr_oracle as vi  # noqa: E402
import visual_loss_oracle as vl  # noqa: E402
from test_visual_big_emu import Local, _asan  # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libvisual_intrinsics_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []),
           "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_intrinsics_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def _d(a):
    return np.ascontiguousarray(a, np.float64).ctypes.data_as(P(ctypes.c_double))


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


KSYS = 60                                  # vintr::kSys: C (upper triangle) | rhs_k | column norms | gradient


def _ut(i, j):                             # vintr::ut
    return i * 8 - i * (i - 1) // 2 + (j - i)


def _loss(l):
    return (0, 1.0) if l is None else l


def check(emu, p, mask, losses=(None, None), fixed_cam=0, radius=1e4):
    L = Local(p, fixed_cam)
    pr = vi.IntrProblem(*vs.args(p), fixed_cam=fixed_cam, mask=mask, loss_reproj=losses[0], loss_plane=losses[1])
    ref = vi.step_bordered(pr, radius)
    s = ref["system"]
    scale, nc6, nb, fr = s["scale"], 6 * pr.nc, pr.nb, pr.free
    sk = np.zeros(8); sk[fr] = scale[nb:]
    yk = np.zeros(8); yk[fr] = ref["y"][nb:]
    s_cam, s_pt = np.ascontiguousarray(scale[:nc6]), np.ascontiguousarray(scale[nc6:nb])
    y_cam = np.ascontiguousarray(ref["y"][:nc6])
    keep = [s_cam, s_pt, sk, yk, y_cam]
    q, t, X = (np.ascontiguousarray(a, np.float64) for a in (pr.q, pr.t, pr.X))
    n6 = 6 * L.n
    colsq0, sys_, B = np.zeros(8), np.zeros(KSYS), np.zeros(8 * max(n6, 1))
    Xc, ps, out = X.copy(), np.zeros_like(X), np.zeros(3)
    (lp, ap), (ll, al) = _loss(losses[0]), _loss(losses[1])
    emu.emu_vintr_step(ctypes.c_int(L.n), ctypes.c_int64(L.Tv), *L.common(), ctypes.c_int(lp), ctypes.c_double(ap), ctypes.c_int(ll),
                       ctypes.c_double(al), _d(q), _d(t), _d(X), _d(s_cam), _d(s_pt), _d(sk), ctypes.c_double(radius),
                       ctypes.c_double(1e-6), ctypes.c_double(1e32), _d(y_cam), _d(yk),
                       *[a.ctypes.data_as(P(ctypes.c_double)) for a in (colsq0, sys_, B, Xc, ps, out)])
    del keep
    # unscaled column norms: the Jacobi scale of the free entries
    assert _rel(1.0 / (1.0 + np.sqrt(colsq0[fr])), scale[nb:]) <= 1e-12
    Bm = B[:8 * n6].reshape(8, n6)[fr].T if n6 else np.zeros((0, pr.k))
    if n6:
        assert _rel(Bm, s["B"]) <= 1e-11
    C = np.array([[sys_[_ut(min(i, j), max(i, j))] for j in fr] for i in fr])
    assert _rel(C, s["C"]) <= 1e-11
    assert _rel(sys_[36 + fr], s["rhs_k"]) <= 1e-11
    assert _rel(sys_[44 + fr], s["Dk"] * radius) <= 1e-11 or np.all(s["Dk"] * radius <= 1e-6)
    # the corner solve and the camera step of visual_intr_corner_kernel
    A = s["S"] + np.diag(s["Dc"])
    Y = np.linalg.solve(A, s["B"]) if nc6 else np.zeros((0, pr.k))
    yv = np.linalg.solve(A, s["rhs_c"]) if nc6 else np.zeros(0)
    Sig = np.ascontiguousarray(s["C"] + np.diag(s["Dk"]) - s["B"].T @ Y)
    r = np.ascontiguousarray(s["rhs_k"] - s["B"].T @ yv)
    assert emu.emu_vintr_corner_solve(ctypes.c_int(pr.k), Sig.ctypes.data_as(P(ctypes.c_double)), r.ctypes.data_as(P(ctypes.c_double))) == 1
    assert _rel(r, ref["y"][nb:]) <= 1e-9
    # back-substitution: the landmark step and the model cost change
    assert _rel(ps[pr.tv], ref["delta"][nc6:nb].reshape(-1, 3)) <= 1e-9
    assert abs(out[0] - ref["model"]) <= 1e-9 * abs(ref["model"])
    return L


def test_corner_solve_refuses_a_nonpositive_pivot(emu):
    S = np.array([[1.0, 2.0], [2.0, 1.0]]); r = np.ones(2)
    assert emu.emu_vintr_corner_solve(ctypes.c_int(2), S.ctypes.data_as(P(ctypes.c_double)), r.ctypes.data_as(P(ctypes.c_double))) == 0


@pytest.mark.parametrize("mask", [vi.FOCAL, vi.PRINCIPAL, vi.DISTORTION, 0xFF])
@pytest.mark.parametrize("fixed_cam", [0, -1])
def test_tile_scene(emu, mask, fixed_cam):
    p = vi.miscalibrated(synth.make_problem(14, 0, 80, seed=5, lidar=False))
    check(emu, p, mask, fixed_cam=fixed_cam)
    check(emu, p, mask, fixed_cam=fixed_cam, radius=3.0)


@pytest.mark.parametrize("losses", [((vl.HUBER, 1.0), (vl.HUBER, 0.1)), ((vl.CAUCHY, 1.0), None)], ids=["huber", "cauchy"])
def test_losses(emu, losses):
    p = vl.with_outliers(vi.miscalibrated(synth.make_problem(14, 0, 80, seed=6, lidar=False)), 0.05, 20.0, 50.0, 6)[0]
    check(emu, p, vi.FOCAL | vi.DISTORTION, losses)


def test_long_landmarks(emu):
    p = vi.miscalibrated(vs.make_scene(23, M=120, n_short=60, long_tracks=((129, 0), (300, 0), (700, 10))))
    p["plane_nd"][::13, :3] = 0.0
    L = check(emu, p, 0xFF)
    assert np.diff(L.trk_ptr).max() >= 700
    check(emu, p, vi.FOCAL, fixed_cam=-1)


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    """The passes do not depend on the order in which the items of a pass run, and the host policy finds no memory or UB error."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261018")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="7")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
