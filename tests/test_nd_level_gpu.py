"""The tree levels of the substructured block LDL^T on the GPU (global-lvba_b200/csrc/nd_kernels.cuh): the SYRK of every level
runs beside the spike it reads from (programmatic dependent launch + per-CTA row counters), which runs beside the factorisation.
Whatever the order the three kernels happen to interleave in, every solve — through the CUDA graph and eagerly — must give the
sparse-LU solution to 1e-10 and agree with every other solve of the same system to 1e-11 (only the order of the SYRK's RED.ADDs
differs from run to run).  Solves alternate between two systems of the same structure and different values, so that a consumer
that read a row before its producer wrote it would find the other system's numbers there, not the same ones again."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import solver_systems as ss  # noqa: E402

pytestmark = pytest.mark.gpu
TOL, AGREE, REPS = 1e-10, 1e-11, 5


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as graft
    p = graft.load_package()
    p.load_library()
    if p.device_count() < 1:
        pytest.fail("no CUDA device: the LVBA hot path has no CPU fallback")
    return p


def band(n, b):
    return [max(0, r - b) for r in range(n)]


def ragged(n=1040):
    """four stretches of different band widths: right-hand-side counts 6 (wa + wc) that are not multiples of the 64-wide SYRK tile"""
    width = np.concatenate([np.full(n // 4, 30), np.full(n // 4, 3), np.full(n // 4, 17), np.full(n - 3 * (n // 4), 9)])
    return [max(0, r - int(width[r])) for r in range(n)]


def separators(n, b, p):
    """separator rows of a plain band of half-width b cut into p chunks (nd_plan.h build_plan: equal interiors, separators as wide
    as the band)"""
    out, cursor = [], 0
    for c in range(p - 1):
        m = max(4, (n - cursor - (p - c - 1) * b) // (p - c))
        out.append((cursor + m, cursor + m + b))
        cursor = cursor + m + b
    return out


def two_systems(first_raw, seed, **kw):
    """two systems of one envelope with different values, and their sparse-LU solutions"""
    out = []
    for q in range(2):
        first, blocks, dadd, rhs, A = ss.make(first_raw, seed=seed + 7919 * q, **kw)
        out.append((first, blocks, dadd, rhs, ss.reference_solve(A, rhs)))
    return out


def check_alternating(pkg, monkeypatch, systems, chunks):
    first_x = [None, None]
    for graph in ("1", "0"):
        monkeypatch.setenv("LVBA_ND_GRAPH", graph)
        for rep in range(2 * REPS):
            q = rep % 2
            first, blocks, dadd, rhs, xr = systems[q]
            x, _, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=chunks)
            assert info["path"] == pkg.SOLVE_CHUNKED and info["chunks"] == chunks, info
            scale = np.abs(xr).max()
            assert np.abs(x - xr).max() <= TOL * scale, (graph, rep, np.abs(x - xr).max(), scale)
            if first_x[q] is None:
                first_x[q] = x
            assert np.abs(x - first_x[q]).max() <= AGREE * scale, (graph, rep, np.abs(x - first_x[q]).max(), scale)


@pytest.mark.parametrize("n,b,chunks", [(2000, 30, 16), (2000, 30, 32), (1999, 20, 32), (5000, 30, 64)])
def test_every_solve_matches_sparse_lu_and_the_others(pkg, monkeypatch, n, b, chunks):
    check_alternating(pkg, monkeypatch, two_systems(band(n, b), seed=3 * n + b + chunks), chunks)


@pytest.mark.parametrize("chunks", [8, 21])
def test_ragged_envelope(pkg, monkeypatch, chunks):
    check_alternating(pkg, monkeypatch, two_systems(ragged(), seed=91 + chunks, fill=0.6), chunks)


@pytest.mark.parametrize("which", [2, 3])
def test_singular_pivot_in_a_separator_is_reported(pkg, monkeypatch, which):
    """A block row decoupled from everything, with a zero diagonal block and no damping, inside a separator (not a chunk
    interior): its pivot block in the dense separator factorisation is exactly zero.  which = 2: a separator of the first tree
    level; 3: the root of eight chunks."""
    n, b, chunks = 900, 12, 8
    s0, s1 = separators(n, b, chunks)[which]
    r = s0 + 5
    assert s0 <= r < s1
    first, blocks, dadd, rhs, A = ss.make(band(n, b), seed=5)
    f, rs = ss.layout(band(n, b))
    blocks = blocks.copy(); dadd = dadd.copy()
    blocks[rs[r]:rs[r + 1]] = 0.0                # row r: its couplings to the left and its diagonal block
    for q in range(r + 1, n):                    # column r: the couplings of the rows below
        if f[q] <= r:
            blocks[rs[q] + r - f[q]] = 0.0
    dadd[6 * r:6 * r + 6] = 0.0
    for graph in ("1", "0"):
        monkeypatch.setenv("LVBA_ND_GRAPH", graph)
        with pytest.raises(pkg.LvbaError):
            pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=chunks)
