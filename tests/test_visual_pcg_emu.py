"""The passes of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_pcg.h) without a GPU, through the host policy
(tests/emu/visual_pcg_emu.cpp): the envelope product against a dense product on banded, tall and loop-closed envelopes, and the
whole conjugate-gradients solve against tests/visual_pcg_oracle.py (the same iteration count and termination, the step to
1e-12); then once more with the items of every pass in a shuffled order."""
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

import visual_pcg_oracle as vp  # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libvisual_pcg_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_pcg_emu.cpp"), "-o", str(so)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def envelope(first):
    """first made monotone (as Envelope::build makes it), last and row_start."""
    first = np.minimum.accumulate(np.asarray(first, np.int64)[::-1])[::-1]
    n = len(first)
    last = np.array([max([i for i in range(n) if first[i] <= k], default=k) for k in range(n)], np.int32)
    row_start = np.concatenate([[0], np.cumsum(np.arange(n) - first + 1)]).astype(np.int64)
    return first.astype(np.int32), last, row_start


def system(first, seed, couple=0.3):
    """A symmetric positive definite system on the envelope (random blocks, diagonally dominant) in envelope storage, the
    diagonal blocks' upper triangles filled with garbage (the device reads their lower triangles), and the damping."""
    rng = np.random.default_rng(seed)
    f, last, rs = envelope(first)
    n = len(f)
    A = np.zeros((6 * n, 6 * n))
    blocks = np.zeros((rs[-1], 6, 6))
    for r in range(n):
        for c in range(f[r], r):
            if rng.random() < couple or c == r - 1:
                B = rng.standard_normal((6, 6))
                blocks[rs[r] + c - f[r]] = B
                A[6 * r:6 * r + 6, 6 * c:6 * c + 6] = B; A[6 * c:6 * c + 6, 6 * r:6 * r + 6] = B.T
    rowsum = np.abs(A).sum(1)
    for r in range(n):
        G = rng.standard_normal((6, 6))
        D = G @ G.T + np.diag(rowsum[6 * r:6 * r + 6] + 1.0)
        A[6 * r:6 * r + 6, 6 * r:6 * r + 6] = D
        stored = np.tril(D) + np.triu(rng.standard_normal((6, 6)), 1)
        blocks[rs[r] + r - f[r]] = stored
    dadd = rng.uniform(0.0, 2.0, 6 * n)
    return (f, last, rs), np.ascontiguousarray(blocks.reshape(-1)), dadd, A + np.diag(dadd)


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(P(t))


def _env(e):
    f, last, rs = e
    return ctypes.c_int(len(f)), _p(f, ctypes.c_int), _p(last, ctypes.c_int), _p(rs, ctypes.c_longlong)


N = 48
SHAPES = {
    "banded": [max(0, r - 3) for r in range(N)],
    "tall": [max(0, r - 30) for r in range(N)],               # shared-window columns of up to 30 rows below a pivot
    "loop_closed": [0 if r >= N - 4 else max(0, r - 2) for r in range(N)],   # the last rows reach back to the first
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_envelope_product(emu, shape):
    e, blocks, dadd, A = system(SHAPES[shape], 1)
    x = np.random.default_rng(2).standard_normal(6 * N)
    y = np.zeros(6 * N)
    emu.emu_pcg_product(*_env(e), _p(blocks), _p(dadd), _p(x), _p(y))
    assert np.abs(y - A @ x).max() <= 1e-12 * np.abs(A @ x).max()


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("eta,min_iter,max_iter", [(0.1, 0, 500), (1e-6, 0, 500), (0.1, 15, 500), (1e-14, 0, 7), (1e-12, 25, 500)])
def test_solve_matches_the_oracle(emu, shape, eta, min_iter, max_iter):
    e, blocks, dadd, A = system(SHAPES[shape], 3)
    b = np.random.default_rng(4).standard_normal(6 * N)
    x = np.zeros(6 * N); info = np.zeros(2, np.int32)
    emu.emu_pcg_solve(*_env(e), _p(blocks), _p(dadd), _p(b), ctypes.c_double(eta), ctypes.c_int(min_iter), ctypes.c_int(max_iter),
                      _p(x), _p(info, ctypes.c_int))
    xr, it, term = vp.cg(A, b, eta, min_iter, max_iter)
    assert (int(info[0]), int(info[1])) == (it, term)
    assert np.abs(x - xr).max() <= 1e-12 * np.abs(xr).max()
    if min_iter > 2 * vp.RESET_PERIOD:
        assert it >= min_iter                                 # the run passes two residual resets


def test_zero_rhs_and_bad_preconditioner(emu):
    e, blocks, dadd, A = system(SHAPES["banded"], 5)
    x = np.ones(6 * N); info = np.full(2, -1, np.int32)
    emu.emu_pcg_solve(*_env(e), _p(blocks), _p(dadd), _p(np.zeros(6 * N)), ctypes.c_double(0.1), ctypes.c_int(0), ctypes.c_int(500),
                      _p(x), _p(info, ctypes.c_int))
    assert tuple(info) == (0, vp.SUCCESS) and not x.any()
    d = dadd.copy(); d[6 * 7 + 2] = -1e6                          # a damped diagonal block that is not positive definite
    emu.emu_pcg_solve(*_env(e), _p(blocks), _p(d), _p(np.ones(6 * N)), ctypes.c_double(0.1), ctypes.c_int(0), ctypes.c_int(500),
                      _p(x), _p(info, ctypes.c_int))
    assert tuple(info) == (0, vp.FAILURE)


def test_indefinite_system_stops_without_convergence(emu):
    e, blocks, dadd, A = system(SHAPES["banded"], 6)
    d = dadd.copy()
    bl = blocks.reshape(-1, 6, 6)
    f, last, rs = e
    for r in range(N - 1):                                         # strong coupling of neighbours: positive blocks, indefinite A
        bl[rs[r + 1] + r - f[r + 1]] *= 50.0
    A2 = np.zeros_like(A)
    for r in range(N):
        for c in range(f[r], r + 1):
            B = bl[rs[r] + c - f[r]]
            if c == r:
                B = np.tril(B) + np.tril(B, -1).T
            A2[6 * r:6 * r + 6, 6 * c:6 * c + 6] = B; A2[6 * c:6 * c + 6, 6 * r:6 * r + 6] = B.T
    A2 += np.diag(d)
    assert np.linalg.eigvalsh(A2).min() < 0
    b = np.random.default_rng(7).standard_normal(6 * N)
    x = np.zeros(6 * N); info = np.zeros(2, np.int32)
    emu.emu_pcg_solve(*_env(e), _p(np.ascontiguousarray(bl.reshape(-1))), _p(d), _p(b), ctypes.c_double(1e-14), ctypes.c_int(0),
                      ctypes.c_int(500), _p(x), _p(info, ctypes.c_int))
    xr, it, term = vp.cg(A2, b, 1e-14, 0, 500)
    assert (int(info[0]), int(info[1])) == (it, term) and term == vp.NO_CONVERGENCE
    assert np.abs(x - xr).max() <= 1e-10 * max(np.abs(xr).max(), 1e-300)


def test_rerun_with_shuffled_items():
    """The passes do not depend on the order in which the items of a pass run."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261018")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
