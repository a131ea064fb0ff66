"""The 50-digit plane-factor oracle (oracle/balm_mp.py), the degenerate voxel family (tests/degenerate_voxels.py) and the
error bounds that the GPU test tests/test_lidar_degenerate_gpu.py holds the device to — all without a GPU.

Bounds, per voxel v with delta_v = 8 eps (|C_v| + |vBar_v|^2) and kappa_v = (|C_v| + |vBar_v|^2) / (lambda_1 - lambda_0):
    residual      |res - res_mp|        <= C_R sum_v delta_v
    gradient row  |g_i - g_i,mp|_max    <= C_G eps sum_{v at i} kappa_v max|Auk_v|
    Hessian block |H_ij - H_ij,mp|_max  <= C_H eps sum_{v at i, j} kappa_v tmax_v
(tmax_v: the largest term summed into the voxel's blocks, balm_mp.voxel).  The constants are calibrated here, on the CPU,
from two float64 implementations measured against the 50-digit oracle over the whole family (isolated, K = 128 / 129, and the shared arrangement
at its perturbed LM start): oracle/lidar_oracle.py (LAPACK eigh) and the big-voxel passes of global-lvba_b200/csrc/lidar_big.h compiled for the host (tests/emu/big_emu.cpp,
cyclic Jacobi).  Each constant is the smallest power of two at least 4x the worst ratio observed:

    worst ratio      residual            g                   H
    float64 oracle   0.053 (strip129)    1.8 (plane)         2.0 (strip, shared arrangement)
    host big passes  0.23  (line128)     1.6 (disc)          3.2 (strip129)
    constant         C_R = 1             C_G = 8             C_H = 16

No constant was chosen by looking at GPU output.
"""
import ctypes
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
from mpmath import mpf

from oracle import balm_mp as bm
from oracle import lidar_oracle as lo
from oracle import synth

sys.path.insert(0, str(Path(__file__).resolve().parent))
import degenerate_voxels as dv  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def family():
    """the isolated family, the K = 128 / 129 strip and line voxels, and the shared arrangement at its perturbed LM start
    (poses up to 1 km from the far voxels), with their 50-digit results"""
    out = {}
    sh = dv.shared()
    sh["poses"] = sh["poses0"]
    for name, p in (("isolated", dv.isolated()), ("tile_and_big", dv.tile_and_big()), ("shared", sh)):
        p["refs"] = bm.evaluate(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
        out[name] = p
    return out


def test_matches_float64_oracle_on_well_conditioned_voxels():
    """synth.make_problem: ordinary 0.5 m patches, where float64 is accurate to ~1e-11"""
    p = synth.make_problem(30, 600, 0, seed=0, visual=False)
    W = 30
    refs = bm.evaluate(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    ref = bm.assemble(p["vox_ptr"], p["pose_idx"], refs, W)
    r, g, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    H = lo.assemble_dense(blocks, W)
    Href = np.zeros_like(H)
    for (i, j), b in ref["H"].items():
        Href[6 * i:6 * i + 6, 6 * j:6 * j + 6] = b
        Href[6 * j:6 * j + 6, 6 * i:6 * i + 6] = b.T
    assert abs(r - ref["res"]) <= 1e-9 * r
    assert np.abs(g - ref["g"]).max() <= 1e-9 * np.abs(g).max()
    assert np.abs(H - Href).max() <= 1e-9 * np.abs(H).max()


def test_eigenvector_signs_do_not_matter(family):
    p = family["isolated"]
    for a in range(0, len(p["vox_ptr"]) - 1, 7):
        s = slice(int(p["vox_ptr"][a]), int(p["vox_ptr"][a + 1]))
        x = bm.voxel(p["clusters"][s], p["poses"][p["pose_idx"][s]])
        y = bm.voxel(p["clusters"][s], p["poses"][p["pose_idx"][s]], flip=True)
        for k in ("res", "g", "Hd", "Hp"):
            assert np.array_equal(x[k], y[k]), (p["cls"][a], k)


def _fd_voxels(p):
    """one voxel of every class seen from 2..8 poses, with an integral N (the Hessian divides by int(N))"""
    seen = {}
    for a in range(len(p["vox_ptr"]) - 1):
        K = p["vox_ptr"][a + 1] - p["vox_ptr"][a]
        s = slice(int(p["vox_ptr"][a]), int(p["vox_ptr"][a + 1]))
        N = p["clusters"][s, 9].sum()
        if 2 <= K <= 8 and N == math.floor(N) and p["cls"][a] not in seen:
            seen[p["cls"][a]] = a
    return sorted(seen.items())


def test_derivatives_equal_finite_differences_at_50_digits(family):
    """g and H are the first and second derivatives of lambda_0 along the reference's retraction R Exp(dphi), p + dp
    (bavoxel.hpp:722-727), by fourth-order central differences at h = 1e-10 in 50 digits (truncation ~h^4, rounding
    ~1e-50 / h^2): agreement to 1e-13 of the sum of |terms| is limited only by the float64 rounding of g and H.
    Bulk voxels of non-integral N are left out: their Hessian divides by int(N), their residual by N."""
    p = family["isolated"]
    rng = np.random.Generator(np.random.Philox(key=9))
    h = mpf("1e-10")
    for cls, a in _fd_voxels(p):
        s = slice(int(p["vox_ptr"][a]), int(p["vox_ptr"][a + 1]))
        cl, ps = p["clusters"][s], p["poses"][p["pose_idx"][s]]
        r = bm.voxel(cl, ps)
        K = len(cl)
        d = rng.normal(size=(K, 6))
        f = {m: bm.lambda0(cl, [bm.retract(ps[k], [m * h * mpf(float(x)) for x in d[k]]) for k in range(K)])
             for m in (-2, -1, 0, 1, 2)}
        fd1 = (f[-2] - 8 * f[-1] + 8 * f[1] - f[2]) / (12 * h)
        fd2 = (-f[2] + 16 * f[1] - 30 * f[0] + 16 * f[-1] - f[-2]) / (12 * h * h)
        H = np.zeros((6 * K, 6 * K))
        for k in range(K):
            H[6 * k:6 * k + 6, 6 * k:6 * k + 6] = r["Hd"][k]
        for q, (i, j) in enumerate(zip(*np.triu_indices(K, 1))):
            H[6 * i:6 * i + 6, 6 * j:6 * j + 6] = r["Hp"][q]
            H[6 * j:6 * j + 6, 6 * i:6 * i + 6] = r["Hp"][q].T
        dv_ = d.ravel()
        gd = math.fsum(r["g"].ravel() * dv_)
        dHd = math.fsum((dv_[:, None] * H * dv_[None, :]).ravel())
        hterms = np.abs(dv_[:, None] * H * dv_[None, :]).sum()
        # at an exact minimum (flat, axis: lambda_0 = 0) g = 0 and fd1 is the truncation error alone, ~h^4
        assert abs(float(fd1) - gd) <= 1e-13 * np.abs(r["g"].ravel() * dv_).sum() + 1e-25 * hterms, cls
        assert abs(float(fd2) - dHd) <= 1e-13 * hterms, cls


def test_family_reaches_every_branch(family, capsys):
    """the device's own solver choice (common.cuh), evaluated in float64 on each voxel's covariance"""
    p = family["isolated"]
    tb = family["tile_and_big"]
    count = {k: 0 for k in ("fast path", "fallback (build and residual)", "det(C) <= 0", "2x2 step, b12 = 0 or < 1e-6",
                            "v1 axis tie", "|vBar|^2 > 1e6 |C|", "non-integral N", "N > 1e6", "slot of N = 1",
                            "K > 128 (big path)")}
    per_class = {}
    for a in range(len(p["vox_ptr"]) - 1):
        s = slice(int(p["vox_ptr"][a]), int(p["vox_ptr"][a + 1]))
        b = bm.device_branch(bm.covariance64(p["clusters"][s], p["poses"][p["pose_idx"][s]]))
        r = p["refs"][a]
        hits = [("fast path", b["fast"]), ("fallback (build and residual)", not b["fast"]), ("det(C) <= 0", b["det"] <= 0),
                ("2x2 step, b12 = 0 or < 1e-6", b["b12"] is not None and b["b12"] < 1e-6), ("v1 axis tie", b["tie"]),
                ("|vBar|^2 > 1e6 |C|", r["vbar"] ** 2 > 1e6 * r["cmax"]), ("non-integral N", r["N"] != math.floor(r["N"])),
                ("N > 1e6", r["N"] > 1e6), ("slot of N = 1", bool((p["clusters"][s, 9] == 1).any())),
                ("K > 128 (big path)", s.stop - s.start > 128)]
        for k, hit in hits:
            if hit:
                count[k] += 1
                per_class.setdefault(k, set()).add(str(p["cls"][a]))
    count["K > 128 (big path)"] += int((np.diff(tb["vox_ptr"]) > 128).sum())
    with capsys.disabled():
        print("\nbranches reached by the degenerate voxel family (isolated arrangement):")
        for k, n in count.items():
            print(f"  {k:32s} {n:4d}  {sorted(per_class.get(k, {'big'}))}")
    for k, n in count.items():
        assert n >= (1 if k == "det(C) <= 0" else 10), (k, n)
    assert {"strip", "line"} <= per_class["fallback (build and residual)"]
    assert "plane" in per_class["fast path"]


# ------------------------------------------------------------------ float64 implementations against the bounds
def _emu_lib(tmp):
    so = tmp / "libbig_emu.so"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "big_emu.cpp"), "-o", str(so)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(so))
    lib.emu_big_accumulate.restype = ctypes.c_double
    return lib


def _run_big_emu(lib, p):
    """lidar_big.h's params / slots / pairs passes over every voxel; returns (res, g, upper(i, j))"""
    W = len(p["poses"])
    vp = np.ascontiguousarray(p["vox_ptr"], np.int64); pi = np.ascontiguousarray(p["pose_idx"], np.int32)
    cl = np.ascontiguousarray(p["clusters"], np.float64); ps = np.ascontiguousarray(p["poses"], np.float64)
    first = np.arange(W)
    for a in range(len(vp) - 1):
        sl = pi[vp[a]:vp[a + 1]]
        first[sl] = np.minimum(first[sl], sl.min())
    first = np.minimum.accumulate(first[::-1])[::-1].astype(np.int32)
    row_start = np.concatenate([[0], np.cumsum(np.arange(W) - first + 1)]).astype(np.int64)
    H = np.zeros((row_start[-1], 36)); g = np.zeros((W, 6))
    P = ctypes.POINTER
    r = lib.emu_big_accumulate(ctypes.c_int64(len(vp) - 1), vp.ctypes.data_as(P(ctypes.c_int64)), pi.ctypes.data_as(P(ctypes.c_int32)),
                               cl.ctypes.data_as(P(ctypes.c_double)), ps.ctypes.data_as(P(ctypes.c_double)), first.ctypes.data_as(P(ctypes.c_int)),
                               row_start.ctypes.data_as(P(ctypes.c_longlong)), H.ctypes.data_as(P(ctypes.c_double)), g.ctypes.data_as(P(ctypes.c_double)),
                               ctypes.c_int(0))
    return r, g, lambda i, j: H[row_start[j] + i - first[j]].reshape(6, 6).T if i != j else H[row_start[i] + i - first[i]].reshape(6, 6)


def _run_oracle(p):
    W = len(p["poses"])
    r, g, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    Hs = lo.assemble_sparse(blocks, W)
    return r, g, lambda i, j: Hs[6 * i:6 * i + 6, 6 * j:6 * j + 6].toarray()


@pytest.fixture(scope="module")
def measured(family, tmp_path_factory):
    """(implementation, class) -> worst (residual, g, H) ratio against the 50-digit oracle"""
    lib = _emu_lib(tmp_path_factory.mktemp("big_emu"))
    out = {}
    for name, p in family.items():
        for c in sorted(set(p["cls"])):
            idx = np.nonzero(p["cls"] == c)[0]
            q = dv.reorder(p, idx)
            ref = bm.assemble(q["vox_ptr"], q["pose_idx"], [p["refs"][a] for a in idx], len(q["poses"]))
            c = c if name != "shared" else f"shared {c}"
            out[("float64 oracle", str(c))] = bm.ratios(ref, *_run_oracle(q))
            out[("host big passes", str(c))] = bm.ratios(ref, *_run_big_emu(lib, q))
    return out


@pytest.mark.parametrize("impl", ["float64 oracle", "host big passes"])
def test_float64_implementations_meet_the_bounds(measured, impl):
    for (name, c), (rr, rg, rh) in measured.items():
        if name == impl:
            assert rr <= bm.C_R and rg <= bm.C_G and rh <= bm.C_H, (c, rr, rg, rh)


def test_bounds_calibration(measured, capsys):
    """each constant is a power of two at least 4x the worst ratio of the float64 implementations (section of the module
    docstring); the table is printed so that a change in the float64 arithmetic shows"""
    worst = np.max(np.array(list(measured.values())), axis=0)
    with capsys.disabled():
        print("\nobserved |float64 - mp| / bound scale, per class:          residual        g        H")
        for (impl, c), (rr, rg, rh) in sorted(measured.items()):
            print(f"  {impl:16s} {c:10s}                           {rr:9.3g} {rg:9.3g} {rh:9.3g}")
        calib = [2.0 ** math.ceil(math.log2(4 * w)) for w in worst]
        print(f"  worst {worst}; smallest powers of two >= 4x worst: C_R {calib[0]:g} C_G {calib[1]:g} C_H {calib[2]:g}; "
              f"in use: {bm.C_R:g} {bm.C_G:g} {bm.C_H:g}")
    assert 4 * worst[0] <= bm.C_R and 4 * worst[1] <= bm.C_G and 4 * worst[2] <= bm.C_H
