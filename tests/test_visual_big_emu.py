"""Path B for landmarks with more observations than one batch CTA holds (global-lvba_b200/csrc/visual_big.h) checked without a
GPU: the passes run through the host policy over EVERY landmark of a problem, each treated as big (tests/emu/visual_big_emu.cpp),
against oracle/visual_oracle.py — cost, column norms, the point-block gradient, the reduced camera system before the camera LM
diagonal and its rhs, and, given the oracle's camera step, the landmark step and the model-cost change.  Tolerances of
tests/test_visual_gpu.py.  Re-run with shuffled items and under ASan/UBSan."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import visual_oracle as vo
import visual_big_scene as vs

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libvisual_big_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []),
           "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_big_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(so))
    lib.emu_vbig_cost.restype = ctypes.c_double
    return lib


def _ptr(a, t):
    return a.ctypes.data_as(P(t))


class Local:
    """The library's local layout of a problem: landmarks with a valid plane (caller order), system rows = the active cameras
    in index order, the envelope of the reduced camera system."""

    def __init__(self, p, fixed_cam):
        self.pr = vo.VisualProblem(*vs.args(p), fixed_cam=fixed_cam)
        op = np.asarray(p["obs_ptr"], np.int64)
        tv = np.nonzero(self.pr.tv)[0]
        K = np.diff(op)[tv]
        self.Tv, self.n = len(tv), self.pr.nc
        self.trk_ptr = np.zeros(self.Tv + 1, np.int32); self.trk_ptr[1:] = np.cumsum(K)
        self.trk_id = tv.astype(np.int32)
        sel = np.concatenate([np.arange(op[a], op[a + 1]) for a in tv]).astype(np.int64) if self.Tv else np.zeros(0, np.int64)
        self.cam = np.ascontiguousarray(np.asarray(p["obs_cam"])[sel], np.int32)
        self.row = np.ascontiguousarray(self.pr.cam_col[self.cam], np.int32)
        self.uv = np.ascontiguousarray(np.asarray(p["obs_uv"], np.float32)[sel])
        self.plane = np.ascontiguousarray(np.asarray(p["plane_nd"], np.float64)[tv])
        first = np.arange(self.n)
        for a in range(self.Tv):
            r = self.row[self.trk_ptr[a]:self.trk_ptr[a + 1]]
            r = r[r >= 0]
            if len(r):
                first[r] = np.minimum(first[r], r.min())
        for r in range(self.n - 2, -1, -1):
            first[r] = min(first[r], first[r + 1])
        self.first = first.astype(np.int32)
        self.row_start = np.zeros(self.n + 1, np.int64); self.row_start[1:] = np.cumsum(np.arange(self.n) - first + 1)
        self.intr = np.ascontiguousarray(p["intr"], np.float64)
        self.sp, self.spl = float(p["sigma_px"]), float(p["sigma_plane"])

    def common(self):
        return [_ptr(self.trk_ptr, ctypes.c_int), _ptr(self.trk_id, ctypes.c_int), _ptr(self.cam, ctypes.c_int), _ptr(self.row, ctypes.c_int),
                _ptr(self.uv, ctypes.c_float), _ptr(self.plane, ctypes.c_double), _ptr(self.intr, ctypes.c_double),
                ctypes.c_double(self.sp), ctypes.c_double(self.spl)]

    def cost(self, emu, q, t, X):
        q, t, X = (np.ascontiguousarray(a, np.float64) for a in (q, t, X))
        return emu.emu_vbig_cost(ctypes.c_int64(self.Tv), *self.common(), _ptr(q, ctypes.c_double), _ptr(t, ctypes.c_double), _ptr(X, ctypes.c_double))

    def step(self, emu, radius, scaling, y_cam):
        pr = self.pr
        q, t, X = (np.ascontiguousarray(a, np.float64) for a in (pr.q, pr.t, pr.X))
        n6, nb = max(self.n, 1) * 6, max(int(self.row_start[-1]), 1)
        o = dict(cam_colsq0=np.zeros(n6), pt_colsq0=np.zeros(max(self.Tv, 1) * 3), S=np.zeros(nb * 36), rhs=np.zeros(n6),
                 cam_colsq=np.zeros(n6), cam_grad=np.zeros(n6), X_cand=X.copy(), pt_step=np.zeros_like(X), out=np.zeros(5))
        yc = None if y_cam is None else np.ascontiguousarray(y_cam, np.float64)
        emu.emu_vbig_step(ctypes.c_int(self.n), ctypes.c_int64(self.Tv), *self.common(), _ptr(self.first, ctypes.c_int),
                          _ptr(self.row_start, ctypes.c_longlong), _ptr(q, ctypes.c_double), _ptr(t, ctypes.c_double), _ptr(X, ctypes.c_double),
                          ctypes.c_int(int(scaling)), ctypes.c_double(radius), ctypes.c_double(1e-6), ctypes.c_double(1e32),
                          None if yc is None else _ptr(yc, ctypes.c_double), *[_ptr(o[k], ctypes.c_double) for k in
                          ("cam_colsq0", "pt_colsq0", "S", "rhs", "cam_colsq", "cam_grad", "X_cand", "pt_step", "out")])
        S = np.zeros((6 * self.n, 6 * self.n))
        blocks = o["S"].reshape(-1, 6, 6)
        for r in range(self.n):
            for c in range(self.first[r], r + 1):
                b = blocks[self.row_start[r] + c - self.first[r]]
                S[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
                S[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
        o["S_dense"] = S
        return o


def check(emu, p, fixed_cam=0, radius=1e4, scaling=True):
    L = Local(p, fixed_cam)
    pr = L.pr
    ref = vo.single_step(pr, radius, scaling)
    nc6 = 6 * pr.nc
    o = L.step(emu, radius, scaling, ref["y"][:nc6])
    # cost and column norms (unscaled): the Jacobi scale of the oracle
    assert abs(o["out"][0] - ref["cost"]) <= 1e-10 * ref["cost"]
    res, J = pr.residuals(jac=True)
    colsq = np.asarray(J.multiply(J).sum(0)).ravel()
    got = np.concatenate([o["cam_colsq0"][:nc6], o["pt_colsq0"][:3 * L.Tv]])
    assert np.abs(got - colsq).max() <= 1e-10 * np.abs(colsq).max()
    if scaling:
        assert np.abs(1.0 / (1.0 + np.sqrt(got)) - ref["scale"]).max() <= 1e-12
    # point-block gradient max (unscaled)
    g_pt = (J.T @ res)[nc6:]
    if len(g_pt):
        assert abs(o["out"][1] - np.abs(g_pt).max()) <= 1e-8 * np.abs(g_pt).max()
    # reduced camera system before the camera LM diagonal, and its rhs
    if nc6:
        assert np.abs(o["S_dense"] - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
        assert np.abs(o["rhs"][:nc6] - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    # given the oracle's camera step: the landmark step, the model-cost change, the candidate cost
    assert np.abs(o["pt_step"] - ref["pt_step"]).max() <= 1e-6 * max(np.abs(ref["pt_step"]).max(), 1e-300)
    assert abs(o["out"][2] - ref["model"]) <= 1e-7 * abs(ref["model"])
    qn, tn, Xn = pr.plus(np.concatenate([ref["cam_step"][pr.cam_active].ravel(), ref["pt_step"][pr.tv].ravel()]))
    Xn_emu = o["X_cand"].copy()
    assert np.abs(Xn_emu[pr.tv] - Xn[pr.tv]).max() <= 1e-6 * max(np.abs(ref["pt_step"]).max(), 1e-300)
    c_cand = pr.cost(qn, tn, Xn)
    assert abs(L.cost(emu, qn, tn, Xn) - c_cand) <= 1e-10 * c_cand
    assert abs(L.cost(emu, pr.q, pr.t, pr.X) - ref["cost"]) <= 1e-10 * ref["cost"]
    return L


@pytest.mark.parametrize("fixed_cam", [0, -1])
def test_problem_small(emu, problem_small, fixed_cam):
    check(emu, problem_small, fixed_cam)
    check(emu, problem_small, fixed_cam, radius=3.0, scaling=False)


def test_long_tracks_over_consecutive_cameras(emu):
    """Landmarks of 129, 300 and 1000 observations; 1000 > the 420 cameras, so that track sees most cameras two or three times."""
    M = 420 if not os.environ.get("LVBA_EMU_RERUN") else 320
    p = vs.make_scene(5, M=M, n_short=150, long_tracks=((129, 10), (300, 50), (1000, 0)))
    L = check(emu, p, 0)
    assert sorted(np.diff(L.trk_ptr))[-3:] == [129, 300, 1000]
    check(emu, p, -1)


def test_duplicate_fixed_and_behind_camera_landmarks(emu):
    """A landmark that sees one camera several times, one whose only cameras are the fixed camera, one behind its first camera
    (zero residual there, utils.hpp:78), and landmarks without a valid plane (skipped)."""
    p = vs.make_scene(8, M=40, n_short=60, extra_tracks=([3, 3, 4, 3, 5], [0], [0, 0], [7, 8, 9, 10]))
    T = len(p["obs_ptr"]) - 1
    vs.put_behind(p, T - 1)
    p["plane_nd"][::9, :3] = 0.0
    for fixed_cam in (0, -1):
        check(emu, p, fixed_cam)


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    """The passes do not depend on the order in which the items of a pass run (the device runs them concurrently), and the host
    policy finds no memory or UB error."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261015")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="7")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
