"""The substructured block LDL^T on the GPU (global-lvba_b200/csrc/nd_solver.cuh): for symmetric INDEFINITE block-banded
systems (SURVEY.md Q5) every path of the library — one CTA, the twisted pair, p chunks + separator tree — must give the same
solution as a sparse LU of the same matrix, to 1e-10 of its largest entry.  Replaces Eigen::SimplicialLDLT
(reference include/BALM/bavoxel.hpp:695-710) / Ceres DENSE_SCHUR (src/lvba_system.cpp:1573-1575).
The plan and the layout passes are checked without a GPU in tests/test_nd_solver_emu.py."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import solver_systems as ss  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-10


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


@pytest.mark.parametrize("n,b,chunks", [(600, 30, 2), (601, 30, 4), (2000, 30, 16), (1999, 20, 32), (2000, 30, 32), (1203, 9, 16),
                                          (5000, 30, 64), (777, 5, 11)])
def test_chunked_matches_sparse_lu_and_the_other_paths(pkg, n, b, chunks):
    first, blocks, dadd, rhs, A = ss.make(band(n, b), seed=n + chunks)
    xr = ss.reference_solve(A, rhs)
    scale = np.abs(xr).max()
    xc, ms, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=chunks)
    assert info["path"] == pkg.SOLVE_CHUNKED and info["chunks"] == chunks, info
    assert np.abs(xc - xr).max() <= TOL * scale, (np.abs(xc - xr).max(), scale)
    xt, _, it = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_TWISTED)
    assert it["path"] == pkg.SOLVE_TWISTED
    assert np.abs(xt - xr).max() <= TOL * scale
    assert np.abs(xc - xt).max() <= TOL * scale
    if n <= 2000:
        x1, _, _ = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_ONE_CTA)
        assert np.abs(x1 - xc).max() <= TOL * scale
        xg, _, _ = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_SHARED_WINDOW)
        assert np.abs(xg - xc).max() <= TOL * scale


def test_ragged_envelope_and_chunks_shorter_than_the_band(pkg):
    n = 1040
    width = np.concatenate([np.full(260, 30), np.full(260, 3), np.full(260, 17), np.full(260, 9)])
    first, blocks, dadd, rhs, A = ss.make([max(0, r - int(width[r])) for r in range(n)], seed=9, fill=0.6)
    xr = ss.reference_solve(A, rhs)
    scale = np.abs(xr).max()
    for chunks in (2, 3, 8, 16, 21):
        xc, _, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=chunks)
        assert info["chunks"] == chunks
        assert np.abs(xc - xr).max() <= TOL * scale, (chunks, np.abs(xc - xr).max())
    # interiors (~11 rows) shorter than the band (30): consecutive separators couple directly
    first, blocks, dadd, rhs, A = ss.make(band(300, 30), seed=10)
    xr = ss.reference_solve(A, rhs)
    xc, _, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=8)
    assert info["chunks"] >= 6
    assert np.abs(xc - xr).max() <= TOL * np.abs(xr).max()


def test_automatic_choice_and_repeated_solves(pkg):
    """AUTO picks the chunked path for long chains; the captured graph must give the same answer at every replay."""
    first, blocks, dadd, rhs, A = ss.make(band(2000, 30), seed=3)
    xr = ss.reference_solve(A, rhs)
    x, ms, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_AUTO, reps=5)
    assert info["path"] == pkg.SOLVE_CHUNKED and info["chunks"] >= 4, info
    assert np.abs(x - xr).max() <= TOL * np.abs(xr).max()
    # a short chain keeps the twisted pair / one CTA
    first, blocks, dadd, rhs, A = ss.make(band(200, 12), seed=4)
    x, ms, info = pkg.env_solve(first, blocks, dadd, rhs)
    assert info["path"] in (pkg.SOLVE_ONE_CTA, pkg.SOLVE_TWISTED)
    assert np.abs(x - ss.reference_solve(A, rhs)).max() <= TOL * np.abs(x).max()


def test_singular_pivot_is_reported(pkg):
    first, blocks, dadd, rhs, A = ss.make(band(900, 12), seed=5)
    rs = ss.layout(band(900, 12))[1]
    blocks = blocks.copy()
    blocks[rs[451] - 1] = 0.0                    # diagonal block of row 450 := 0 and no damping there
    dadd = dadd.copy(); dadd[6 * 450:6 * 451] = 0.0
    # row 450's pivot block is then -sum(L D L^T) of its column couplings: generically non-singular; force exact singularity by
    # decoupling the row completely
    f = ss.layout(band(900, 12))[0]
    blocks[rs[450]:rs[451]] = 0.0
    for r in range(451, 900):
        if f[r] <= 450:
            blocks[rs[r] + 450 - f[r]] = 0.0
    with pytest.raises(pkg.LvbaError):
        pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=8)


def test_spike_beside_the_factorisation_gives_the_same_solution(pkg, monkeypatch):
    """The spike kernels start beside the factorisation they read from (programmatic dependent launch + progress counters);
    the arithmetic is fixed up to the order of the SYRK's RED.ADDs, so repeated solves agree to rounding — also without the
    CUDA graph (a consumer that ran ahead of its producer would read stale columns only now and then, and be wrong by far
    more than rounding)."""
    first, blocks, dadd, rhs, A = ss.make(band(2000, 30), seed=77)
    x0, _, info = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=16)
    assert info["chunks"] == 16
    xr = ss.reference_solve(A, rhs)
    assert np.abs(x0 - xr).max() <= TOL * np.abs(xr).max()
    for graph in ("1", "0"):
        monkeypatch.setenv("LVBA_ND_GRAPH", graph)
        for rep in range(5):
            x_pipe, _, _ = pkg.env_solve(first, blocks, dadd, rhs, path=pkg.SOLVE_CHUNKED, chunks=16, reps=3)
            assert np.abs(x_pipe - xr).max() <= TOL * np.abs(xr).max(), (graph, rep, np.abs(x_pipe - xr).max())
            assert np.abs(x_pipe - x0).max() <= 1e-11 * np.abs(xr).max(), (graph, rep, np.abs(x_pipe - x0).max())
