"""The damping rule of the LiDAR LM (global-lvba_b200/csrc/balm_rule.h: one accept / reject decision, the update of u and v and
the stop test, shared by lvba_lidar_iterate and every window of lvba_lidar_lm_batch) checked without a GPU: run on the host
(tests/emu/balm_rule_emu.cpp) and held against oracle.lidar_oracle.balm_update, the rule of the oracle's damping_iter, over the
same sequences of pass results.  Accepts, rejects, non-finite candidates and the stop test give the same u, v, decisions and
termination, bit for bit."""
import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import lidar_oracle as lo

ROOT = Path(__file__).resolve().parents[1]
TERM_MAX_ITER, TERM_FUNCTION_TOL = 0, 1
V = 37.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libbalm_rule_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "balm_rule_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(str(so))
    lib.balm_rule_run.restype = C.c_int
    return lib


def run_emu(lib, u0, v0, rel_tol, batched, sc, verbose=0):
    n = len(sc)
    sc = np.ascontiguousarray(sc, np.float64).ravel()
    u, v = np.zeros(n), np.zeros(n)
    acc, term = np.zeros(n, np.int32), np.zeros(n, np.int32)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
    k = lib.balm_rule_run(C.c_double(u0), C.c_double(v0), C.c_double(rel_tol), C.c_int(batched), C.c_int(verbose), C.c_int(n),
                          P(sc, C.c_double), C.c_double(V), P(u, C.c_double), P(v, C.c_double), P(acc, C.c_int), P(term, C.c_int))
    return [(float(u[i]), float(v[i]), bool(acc[i]), int(term[i])) for i in range(k)]


def run_oracle(u0, v0, rel_tol, batched, sc):
    """damping_iter's use of the rule: residual1 from the pass that rebuilt H (every pass of a window of the batch)."""
    u, v, rebuilt, out = u0, v0, True, []
    for r1_sum, q1_sum, bad, r2_sum in sc:
        if rebuilt:
            r1 = r1_sum / V
        u, v, acc, stop = lo.balm_update(u, v, r1, r2_sum / V, q1_sum / V, rel_tol, bad=bad != 0.0)
        out.append((u, v, acc, TERM_FUNCTION_TOL if stop else TERM_MAX_ITER))
        rebuilt = batched or acc
        if stop:
            break
    return out


def random_passes(rng, n):
    """Pass results [r1 sum, q1, non-finite flag, r2 sum]: decreases of every size (the 1/3 floor of the update included),
    increases, a non-finite trial residual, model or step, and changes below the stop threshold."""
    sc, r1 = [], 5.0 + rng.random()
    for _ in range(n):
        kind = rng.integers(0, 7)
        q1 = r1 * 10.0 ** rng.uniform(-4, -1)
        bad = 0.0
        if kind == 0:
            r2 = r1 - q1 * rng.uniform(0.01, 2.0)          # accepted, rho anywhere in (0, 2)
        elif kind == 1:
            r2 = r1 * (1 + 10.0 ** rng.uniform(-5, -1))    # rejected
        elif kind == 2:
            r2 = [math.nan, math.inf][rng.integers(0, 2)]
        elif kind == 3:
            r2, q1 = r1 - 0.5 * q1, [math.nan, math.inf][rng.integers(0, 2)]
        elif kind == 4:
            r2, bad = r1 - 0.5 * q1, 1.0
        elif kind == 5:
            r2 = r1 * (1 + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-9, -7))    # a change below the stop threshold of 1e-6
        else:
            r2 = r1 - q1 * rng.uniform(2.0, 5.0)           # a decrease far beyond the model: rho > 2
        sc.append([r1 * V, q1 * V, bad, r2 * V])
        if math.isfinite(r2) and r2 < r1 and bad == 0.0 and math.isfinite(q1):
            r1 = r2
    return sc


@pytest.mark.parametrize("batched", [0, 1])
@pytest.mark.parametrize("rel_tol", [1e-6, -1.0])
def test_rule_equals_the_oracle(emu, rel_tol, batched):
    seen = set()
    for seed in range(16):
        rng = np.random.default_rng(seed)
        sc = random_passes(rng, 40)
        u0, v0 = [(0.01, 2.0), (1e-4, 3.0), (10.0, 2.0)][seed % 3]
        got = run_emu(emu, u0, v0, rel_tol, batched, sc)
        assert got == run_oracle(u0, v0, rel_tol, batched, sc), seed
        seen |= {(a, t) for _, _, a, t in got}
    # accepts and rejects, and with the test on, stops after both
    assert seen == ({(True, 0), (False, 0), (True, 1), (False, 1)} if rel_tol > 0 else {(True, 0), (False, 0)})


def test_handwritten_sequence(emu, capfd):
    """An accept with rho = 1/2, one at the 1/3 floor, five rejects (an increase, residual1 kept from the last build while
    sc[0] changes, a NaN and an infinite trial, the device's non-finite flag), an accept that resets v, then a decrease below
    rel_tol: stop.  The verbose line carries the caller's label."""
    sc = [[4.0 * V, 2.0 * V, 0, 3.0 * V],                    # rho = 1/2: u *= 1
          [3.0 * V, 0.1 * V, 0, 2.9 * V],                    # rho ~ 1: u *= 1/3
          [2.9 * V, 0.1 * V, 0, 3.5 * V],
          [9.9 * V, 0.1 * V, 0, 3.0 * V],                    # not rebuilt: residual1 stays 2.9
          [2.9 * V, 0.1 * V, 0, math.nan],
          [2.9 * V, 0.1 * V, 0, math.inf],
          [2.9 * V, 0.1 * V, 1, 2.0 * V],                    # flagged: rejected though r2 < r1
          [2.9 * V, 0.9 * V, 0, 2.0 * V],
          [2.0 * V, 0.5 * V, 0, 2.0 * V * (1 - 1e-8)]]
    got = run_emu(emu, 0.01, 2.0, 1e-6, 0, sc, verbose=1)
    assert got == run_oracle(0.01, 2.0, 1e-6, 0, sc)
    assert [a for _, _, a, _ in got] == [True, True, False, False, False, False, False, True, True]
    assert [v for _, v, _, _ in got] == [2.0, 2.0, 4.0, 8.0, 16.0, 32.0, 64.0, 2.0, 2.0]
    assert [t for *_, t in got] == [TERM_MAX_ITER] * 8 + [TERM_FUNCTION_TOL]
    assert got[0][0] == 0.01 and got[1][0] == 0.01 * (1.0 / 3.0)
    err = capfd.readouterr().err.splitlines()
    assert len(err) == 9
    assert err[0] == "[emu] iter 0: (4 3) u: 0.01 v: 2 q: 1 q1: 2"
    assert err[3].startswith("[emu] iter 3: (2.9 3) ") and err[4].startswith("[emu] iter 4: (2.9 nan) ")
