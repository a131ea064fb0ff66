"""Random symmetric (indefinite) block-envelope systems for the solver tests: envelope storage as the library keeps it + a
scipy sparse copy for the reference solve."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def layout(first_raw):
    n = len(first_raw)
    first = np.minimum(np.asarray(first_raw, np.int64), np.arange(n))
    first = np.minimum.accumulate(first[::-1])[::-1]
    row_start = np.zeros(n + 1, np.int64)
    row_start[1:] = np.cumsum(np.arange(n) - first + 1)
    return first.astype(np.int32), row_start


def make(first_raw, seed, indefinite=True, fill=0.85):
    """returns first, blocks [nblocks, 36], dadd, rhs, sparse matrix (A + diag(dadd)) in CSC"""
    rng = np.random.default_rng(seed)
    first, rs = layout(first_raw)
    n = len(first)
    nb = int(rs[-1])
    blocks = rng.normal(0, 1, (nb, 6, 6))
    keep = rng.random(nb) < fill
    blocks[~keep] = 0.0
    rows = np.repeat(np.arange(n), np.arange(n) - first + 1)
    cols = np.concatenate([np.arange(first[r], r + 1) for r in range(n)])
    diag = rows == cols
    height = (np.arange(n) - first + 2)[rows[diag]]
    D = rng.normal(0, 1, (n, 6, 6))
    D = D @ D.transpose(0, 2, 1) + (14.0 * height)[:, None, None] * np.eye(6)
    if indefinite:
        D[1::3] *= -1.0
    full = blocks.copy()
    full[diag] = D
    stored = full.copy()
    garbage = np.triu(rng.normal(0, 99, (n, 6, 6)), 1)                  # the upper triangle of a diagonal block is never read
    stored[diag] = np.tril(D) + garbage
    dadd = rng.uniform(0.05, 0.2, 6 * n)
    rhs = rng.normal(0, 1, 6 * n)
    # sparse copy: lower blocks + mirrored strictly-lower blocks
    r_idx = (6 * rows[:, None, None] + np.arange(6)[None, :, None]) + np.zeros((1, 1, 6), np.int64)
    c_idx = (6 * cols[:, None, None] + np.arange(6)[None, None, :]) + np.zeros((1, 6, 1), np.int64)
    lower = sp.coo_matrix((full.ravel(), (r_idx.ravel(), c_idx.ravel())), shape=(6 * n, 6 * n))
    off = ~diag
    upper = sp.coo_matrix((full[off].ravel(), (c_idx[off].ravel(), r_idx[off].ravel())), shape=(6 * n, 6 * n))
    A = (lower + upper + sp.diags(dadd)).tocsc()
    return first, stored.reshape(nb, 36), dadd, rhs, A


def reference_solve(A, rhs):
    return spla.spsolve(A, rhs)


def damped(br, bc, blocks, n, u):
    """first[] and dadd = u diag(A) of a system as get_system() returns it (envelope blocks row by row, the diagonal block
    last in each row): the damped system the LM step solves"""
    first = np.full(n, n, np.int32)
    np.minimum.at(first, br, bc)
    return first, u * np.concatenate([np.diag(b) for b in blocks[br == bc]])
