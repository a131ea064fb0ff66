"""The matrix-free reduced camera system of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_implicit.h) without a GPU, through the
host policy (tests/emu/visual_implicit_emu.cpp), over every landmark of a problem: its build against the explicit passes of
visual_big.h on the same problem (rhs, column norms, gradient, cost and gradient max to rounding), its diagonal blocks and its
product against S + diag(dadd) of tests/visual_pcg_oracle.py, and the whole conjugate-gradients solve on it against the oracle's
cg.  Then the same with the items of every pass in a shuffled order, which must give the same bits.  Also the rule that
chooses between the two products, on the counts of the benchmark and test scenes."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import synth
from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_pcg_oracle as vp

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
sys.path.insert(0, str(ROOT / "tests"))
from test_visual_big_emu import Local  # noqa: E402

HUBER, CAUCHY = 1, 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libvisual_implicit_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_implicit_emu.cpp"),
                        "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(so))


def _p(a, t=ctypes.c_double):
    return a.ctypes.data_as(P(t))


def run(emu, L, radius=1e4, scaling=True, losses=(0, 1.0, 0, 0.1), dadd=None, x=None, eta=0.1, min_iter=0, max_iter=500):
    n, n6 = L.n, 6 * L.n
    pr = L.pr
    q, t, X = (np.ascontiguousarray(a, np.float64) for a in (pr.q, pr.t, pr.X))
    o = {k: np.zeros(max(n6, 1)) for k in ("rhs_x", "colsq_x", "grad_x", "rhs", "colsq", "grad", "y", "x_sol")}
    o.update(S=np.zeros(max(int(L.row_start[-1]), 1) * 36), D=np.zeros(max(n, 1) * 36), out_x=np.zeros(2), out=np.zeros(2),
             info=np.zeros(2, np.int32))
    dadd = np.ascontiguousarray(np.zeros(n6) if dadd is None else dadd, np.float64)
    x = np.ascontiguousarray(np.zeros(n6) if x is None else x, np.float64)
    lp, ap, ll, al = losses
    emu.emu_imp_run(ctypes.c_int(n), ctypes.c_int64(L.Tv), *L.common(), ctypes.c_int(lp), ctypes.c_double(ap), ctypes.c_int(ll),
                    ctypes.c_double(al), _p(L.first, ctypes.c_int), _p(L.row_start, ctypes.c_longlong), _p(q), _p(t), _p(X),
                    ctypes.c_int(int(scaling)), ctypes.c_double(radius),
                    *[_p(o[k]) for k in ("S", "rhs_x", "colsq_x", "grad_x", "out_x", "rhs", "colsq", "grad", "D", "out")],
                    _p(dadd), _p(x), _p(o["y"]), ctypes.c_double(eta), ctypes.c_int(min_iter), ctypes.c_int(max_iter), _p(o["x_sol"]),
                    _p(o["info"], ctypes.c_int))
    S = np.zeros((n6, n6))
    blocks = o["S"][:int(L.row_start[-1]) * 36].reshape(-1, 6, 6)
    for r in range(n):
        for c in range(L.first[r], r + 1):
            b = blocks[L.row_start[r] + c - L.first[r]]
            S[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
            S[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
    o["S_dense"] = S
    return o


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def check(emu, p, fixed_cam=0, radius=1e4, scaling=True, losses=(0, 1.0, 0, 0.1), oracle=True):
    L = Local(p, fixed_cam)
    n6 = 6 * L.n
    o = run(emu, L, radius, scaling, losses)
    # the build: the explicit passes' values to rounding
    for k in ("rhs", "colsq", "grad"):
        assert _rel(o[k][:n6], o[k + "_x"][:n6]) <= 1e-12, k
    assert abs(o["out"][0] - o["out_x"][0]) <= 1e-13 * o["out_x"][0]
    assert abs(o["out"][1] - o["out_x"][1]) <= 1e-12 * o["out_x"][1]
    # the damping of the camera columns, as visual_cam_diag_kernel makes it
    dadd = np.clip(o["colsq"][:n6], 1e-6, 1e32) / radius
    A = vp.sym_lower(o["S_dense"]) + np.diag(dadd)
    if oracle:
        ref = vp.single_step(L.pr, radius, scaling=scaling)
        A_ref = ref["S"]                                  # the damped system: S + diag(dadd)
        assert _rel(A, A_ref) <= 1e-8
    else:
        A_ref = A
    # the diagonal blocks: those of S + diag(dadd)
    D = o["D"][:L.n * 36].reshape(-1, 6, 6)
    for r in range(L.n):
        blk = A_ref[6 * r:6 * r + 6, 6 * r:6 * r + 6]
        assert np.abs(D[r] + np.diag(dadd[6 * r:6 * r + 6]) - blk).max() <= 1e-10 * np.abs(blk).max(), r
    # the product, for a random x
    x = np.random.default_rng(3).standard_normal(n6)
    o = run(emu, L, radius, scaling, losses, dadd=dadd, x=x)
    assert _rel(o["y"][:n6], A_ref @ x) <= 1e-11
    # the whole solve: the oracle's cg on the same A
    for eta, mn, mx in ((0.1, 0, 500), (1e-3, 0, 500), (1e-14, 0, 7)):
        o = run(emu, L, radius, scaling, losses, dadd=dadd, x=x, eta=eta, min_iter=mn, max_iter=mx)
        xr, it, term = vp.cg(A, o["rhs"][:n6], eta, mn, mx)
        assert (int(o["info"][0]), int(o["info"][1])) == (it, term), (eta, mx)
        assert _rel(o["x_sol"][:n6], xr) <= 1e-10, (eta, mx)
    return L


@pytest.mark.parametrize("fixed_cam", [0, -1])
def test_small_scene(emu, problem_small, fixed_cam):
    check(emu, problem_small, fixed_cam)
    check(emu, problem_small, fixed_cam, radius=3.0, scaling=False)


def test_long_tracks(emu):
    """Landmarks of 129 and 300 observations beside short ones."""
    p = vs.make_scene(5, M=120, n_short=150, long_tracks=((129, 10), (300, 0)))
    L = check(emu, p, 0)
    assert sorted(np.diff(L.trk_ptr))[-2:] == [129, 300]


def test_repeated_camera_constant_cameras_and_no_plane(emu):
    """A landmark that sees one camera several times, one seen only by the constant camera, landmarks without a valid plane."""
    p = vs.make_scene(8, M=40, n_short=60, extra_tracks=([3, 3, 4, 3, 5], [0], [0, 0], [7, 8, 8, 8, 9, 10]))
    p["plane_nd"][::9, :3] = 0.0
    for fixed_cam in (0, -1):
        check(emu, p, fixed_cam)


@pytest.mark.parametrize("losses", [(HUBER, 1.0, HUBER, 0.1), (CAUCHY, 0.5, CAUCHY, 0.05)], ids=["huber", "cauchy"])
def test_robust_losses(emu, losses):
    p = vs.make_scene(8, M=40, n_short=60, extra_tracks=([3, 3, 4, 3, 5],))
    check(emu, p, 0, losses=losses, oracle=False)


def _counts(p, fixed_cam=0):
    """The plan's counts of lvba_visual_counts (free observations, pair contributions to S, envelope blocks, rows), from the
    library's rules: rows = the non-constant cameras with observations in index order; per landmark C(n, 2) + sum C(n_row, 2)
    pair contributions over its n free observations; the envelope from the lowest row of every landmark's clique."""
    L = Local(p, fixed_cam)
    free = pairs = 0
    for a in range(L.Tv):
        r = L.row[L.trk_ptr[a]:L.trk_ptr[a + 1]]
        r = r[r >= 0]
        free += len(r)
        _, c = np.unique(r, return_counts=True)
        pairs += len(r) * (len(r) - 1) // 2 + int((c * (c - 1) // 2).sum())
    return free, pairs, int(L.row_start[-1]), L.n


def test_selection_rule(emu):
    choose = lambda free, pairs, nb, n: emu.emu_imp_choose(ctypes.c_int64(free), ctypes.c_int64(pairs), ctypes.c_int64(nb), ctypes.c_int(n))
    # config C (what bench.py builds) and the same with 200 tracks of 200-1000 observations (tools/bench_visual_pcg.py): counts
    # of the library's plan
    assert choose(549213, 1379750, 40754, 1999) == 0
    assert choose(669267, 42152656, 1994896, 1999) == 1
    small = synth.make_problem(14, 0, 80, seed=5, lidar=False)
    mixed = vs.make_scene(17, M=400, n_short=300, long_tracks=((128, 5), (129, 20), (300, 60), (1000, 0)), extra_tracks=([3, 3, 4, 3, 5],))
    loop = vs.make_scene(11, M=400, long_tracks=[(20, 390)])
    assert choose(*_counts(small)) == 0
    assert choose(*_counts(mixed)) == 1
    assert choose(*_counts(loop)) == 1
    assert choose(0, 0, 0, 0) == 0 and choose(10, 10 ** 9, 10 ** 9, 0) == 0


def test_rerun_with_shuffled_items():
    """The passes do not depend on the order in which the items of a pass run, and give the same bits in any order."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261018")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout


def test_shuffled_items_give_the_same_bits(emu, problem_small, tmp_path):
    """One run in index order and one with shuffled items (in a child process, which reads LVBA_EMU_SHUFFLE once) agree bit for
    bit on everything the matrix-free passes write."""
    out = {}
    for tag, shuffle in (("plain", None), ("shuffled", "7")):
        env = dict(os.environ)
        env.pop("LVBA_EMU_SHUFFLE", None)
        if shuffle:
            env["LVBA_EMU_SHUFFLE"] = shuffle
        f = tmp_path / f"{tag}.npz"
        code = ("import sys, numpy as np; sys.path[:0] = [%r, %r]; import test_visual_implicit_emu as t;"
                "import ctypes; from oracle import synth;"
                "emu = ctypes.CDLL(%r); L = t.Local(synth.make_problem(14, 0, 80, seed=5, lidar=False), 0);"
                "o = t.run(emu, L, x=np.random.default_rng(1).standard_normal(6 * L.n), dadd=np.full(6 * L.n, 0.5));"
                "np.savez(%r, **{k: v for k, v in o.items() if k not in ('S', 'S_dense', 'rhs_x', 'colsq_x', 'grad_x', 'out_x')})"
                % (str(ROOT), str(ROOT / "tests"), str(emu._name), str(f)))
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=str(ROOT), env=env, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
        out[tag] = dict(np.load(f))
    for k, v in out["plain"].items():
        assert v.tobytes() == out["shuffled"][k].tobytes(), k
