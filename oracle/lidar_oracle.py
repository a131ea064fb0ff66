"""CPU ORACLE for hot path A — BALM2 LiDAR bundle adjustment (numpy, float64).

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, bench.py's cpu_baseline
leg and __graft_entry__.smoke() may import this.  The shipped solver is the
CUDA library (global-lvba_b200/csrc) and never calls into this file.

PARITY: PINNED AGAINST THE REFERENCE'S OWN SOURCE for this path — tests/test_ref_pin.py holds every function below
against tests/golden/ref_balm.npz, written by include/BALM/tools.hpp + include/BALM/bavoxel.hpp compiled where they lie
(oracle/ref_driver.cpp -> oracle/_ref/libbalm_ref.so) on stand-ins for Eigen / PCL (oracle/ref_shim/: own Jacobi
eigen-solver and envelope LDL^T under the reference's lines — NOT Eigen; see ref_shim/mini_eigen.h for what that leaves
open).  Observed: H / g / sum(lambda_0) 1e-11 relative, damping_iter end poses 2e-11.  The reference ships no tests,
fixtures or golden vectors of its own (SURVEY.md §4, §8c).  Also pinned by finite-difference identities
(tests/test_oracle_lidar.py): the analytic gradient/Hessian below must equal the derivatives of the residual-only
function along the reference's own retraction R <- R*Exp(dphi), p <- p + dp.

Each function restates, line for line, the cited reference code:

  transform_clusters   PointCluster::transform         include/BALM/tools.hpp:450-456
  voxel_eig            sig accumulation + eigen solve  include/BALM/bavoxel.hpp:87-110
  acc_evaluate2        VOX_HESS::acc_evaluate2         include/BALM/bavoxel.hpp:68-174
  only_residual        evaluate_only_residual          include/BALM/bavoxel.hpp:176-203
  so3_exp              Exp                             include/BALM/tools.hpp:62-77
  damping_iter         BALM2::damping_iter             include/BALM/bavoxel.hpp:662-767
  balm_update          its accept / reject and stop    include/BALM/bavoxel.hpp:733-762

Storage differs from the reference on purpose (SURVEY.md §0.3): the reference
keeps a dense vector<PointCluster>(win_size) per voxel and a dense 6W x 6W
Hessian; here a voxel stores only its non-empty (N != 0) slots as CSR
(vox_ptr, pose_idx, clusters[nnz,10] = Pxx Pxy Pxz Pyy Pyz Pzz vx vy vz N) and
H is returned as block-COO / scipy sparse.  Empty slots contribute exact zeros
in the reference (transform of a zero cluster is zero), so results agree.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def hat(v):
    """tools.hpp:105-112, batched (...,3)->(...,3,3)."""
    v = np.asarray(v)
    out = np.zeros(v.shape[:-1] + (3, 3))
    out[..., 0, 1], out[..., 0, 2] = -v[..., 2], v[..., 1]
    out[..., 1, 0], out[..., 1, 2] = v[..., 2], -v[..., 0]
    out[..., 2, 0], out[..., 2, 1] = -v[..., 1], v[..., 0]
    return out


def so3_exp(w):
    """tools.hpp:62-77 (identity below 1e-11), batched (n,3)->(n,3,3)."""
    w = np.atleast_2d(np.asarray(w, np.float64))
    th = np.linalg.norm(w, axis=1)
    big = th >= 1e-11
    axis = w / np.where(big, th, 1.0)[:, None]
    K = hat(axis)
    R = np.eye(3)[None] + np.sin(th)[:, None, None] * K + (1.0 - np.cos(th))[:, None, None] * (K @ K)
    R[~big] = np.eye(3)
    return R


def unpack_clusters(clusters):
    c = np.asarray(clusters, np.float64)
    P = np.empty((c.shape[0], 3, 3))
    P[:, 0, 0], P[:, 0, 1], P[:, 0, 2] = c[:, 0], c[:, 1], c[:, 2]
    P[:, 1, 0], P[:, 1, 1], P[:, 1, 2] = c[:, 1], c[:, 3], c[:, 4]
    P[:, 2, 0], P[:, 2, 1], P[:, 2, 2] = c[:, 2], c[:, 4], c[:, 5]
    return P, c[:, 6:9].copy(), c[:, 9].copy()


def transform_clusters(P, v, n, R, t):
    """tools.hpp:450-456: v' = R v + N p ; P' = R P R^T + rp + rp^T + N p p^T."""
    Rv = np.einsum("nij,nj->ni", R, v)
    vt = Rv + n[:, None] * t
    rp = np.einsum("ni,nj->nij", Rv, t)
    Pt = R @ P @ np.transpose(R, (0, 2, 1)) + rp + np.transpose(rp, (0, 2, 1)) \
        + n[:, None, None] * np.einsum("ni,nj->nij", t, t)
    return Pt, vt


def _voxel_sums(vox_ptr, Pt, vt, n):
    starts = vox_ptr[:-1]
    sP = np.add.reduceat(Pt.reshape(-1, 9), starts, axis=0).reshape(-1, 3, 3)
    sv = np.add.reduceat(vt, starts, axis=0)
    sN = np.add.reduceat(n, starts)
    return sP, sv, sN


def voxel_eig(vox_ptr, pose_idx, clusters, poses):
    """bavoxel.hpp:87-100: merged covariance and its ascending eigen system."""
    P, v, n = unpack_clusters(clusters)
    R = poses[pose_idx, :9].reshape(-1, 3, 3)
    t = poses[pose_idx, 9:12]
    Pt, vt = transform_clusters(P, v, n, R, t)
    sP, sv, sN = _voxel_sums(vox_ptr, Pt, vt, n)
    vbar = sv / sN[:, None]
    C = sP / sN[:, None, None] - np.einsum("ni,nj->nij", vbar, vbar)
    lam, U = np.linalg.eigh(C)            # ascending, like SelfAdjointEigenSolver
    return lam, U, vbar, sN, (P, v, n, R, t)


def only_residual(vox_ptr, pose_idx, clusters, poses):
    """bavoxel.hpp:176-203 — returns sum_v lambda_0 (NOT divided by V)."""
    lam, *_ = voxel_eig(vox_ptr, pose_idx, clusters, poses)
    return float(lam[:, 0].sum())


def acc_evaluate2(vox_ptr, pose_idx, clusters, poses, n_poses, want_blocks=True):
    """bavoxel.hpp:68-174.  Returns (residual_sum, g[W,6], (bi, bj, blocks)).

    Block COO holds every (i, j) block contribution for i <= j (upper
    triangle incl. diagonal) exactly as lines 148 and 165 accumulate them; the
    mirror of lines 171-173 is applied by assemble_dense / assemble_sparse.
    """
    lam, U, vbar, sN, (P, v, n, R, t) = voxel_eig(vox_ptr, pose_idx, clusters, poses)
    V = len(vox_ptr) - 1
    K = np.diff(vox_ptr)
    row = np.repeat(np.arange(V), K)
    NN = np.trunc(sN)                                  # int NN = sig.N (line 101)
    uk = U[:, :, 0]
    umumT = np.zeros((V, 3, 3))
    for m in (1, 2):                                   # lines 107-110
        um = U[:, :, m]
        umumT += (2.0 / (lam[:, 0] - lam[:, m]))[:, None, None] * np.einsum("ni,nj->nij", um, um)
    ukukT = np.einsum("ni,nj->nij", uk, uk)

    # ---- per active slot (lines 112-149), all slots of all voxels batched
    uk_s, NN_s, vbar_s = uk[row], NN[row], vbar[row]
    vihat = hat(v)
    RiTuk = np.einsum("nji,nj->ni", R, uk_s)
    RiTukhat = hat(RiTuk)
    PiRiTuk = np.einsum("nij,nj->ni", P, RiTuk)
    viRiTuk = np.einsum("nij,nj->ni", vihat, RiTuk)
    viRiTukukT = np.einsum("ni,nj->nij", viRiTuk, uk_s)
    ti_v = t - vbar_s
    ukTti_v = np.einsum("ni,ni->n", uk_s, ti_v)
    combo1 = hat(PiRiTuk) + vihat * ukTti_v[:, None, None]
    combo2 = np.einsum("nij,nj->ni", R, v) + n[:, None] * ti_v
    Auk = np.empty((len(n), 3, 6))
    Auk[:, :, :3] = (R @ P + np.einsum("ni,nj->nij", ti_v, v)) @ RiTukhat - R @ combo1
    Auk[:, :, 3:] = np.einsum("ni,nj->nij", combo2, uk_s) \
        + np.einsum("ni,ni->n", combo2, uk_s)[:, None, None] * np.eye(3)[None]
    Auk /= NN_s[:, None, None]
    jjt = np.einsum("nij,ni->nj", Auk, uk_s)           # Auk^T uk
    g = np.zeros((n_poses, 6))
    np.add.at(g, pose_idx, jjt)
    residual = float(lam[:, 0].sum())
    if not want_blocks:
        return residual, g, None

    um_s = umumT[row]
    Hd = np.einsum("nai,nab,nbj->nij", Auk, um_s, Auk)
    Hd[:, :3, :3] += (2.0 / NN_s)[:, None, None] * ((combo1 - RiTukhat @ P) @ RiTukhat) \
        - (2.0 / NN_s / NN_s)[:, None, None] * np.einsum("ni,nj->nij", viRiTuk, viRiTuk) \
        - 0.5 * hat(jjt[:, :3])
    HRt = (2.0 / NN_s * (1.0 - n / NN_s))[:, None, None] * viRiTukukT
    Hd[:, :3, 3:] += HRt
    Hd[:, 3:, :3] += np.transpose(HRt, (0, 2, 1))
    Hd[:, 3:, 3:] += (2.0 / NN_s * (n - n * n / NN_s))[:, None, None] * ukukT[row]
    bi = [pose_idx.astype(np.int64)]; bj = [pose_idx.astype(np.int64)]; bl = [Hd]

    # ---- pairs i<j inside each voxel (lines 151-167), grouped by K
    for k in np.unique(K):
        if k < 2:
            continue
        vs = np.nonzero(K == k)[0]
        base = vox_ptr[vs]
        ii, jj = np.triu_indices(int(k), 1)
        si = (base[:, None] + ii[None, :]).ravel()
        sj = (base[:, None] + jj[None, :]).ravel()
        um_p = np.repeat(umumT[vs], len(ii), axis=0)
        NNp = np.repeat(NN[vs], len(ii))
        Hb = np.einsum("nai,nab,nbj->nij", Auk[si], um_p, Auk[sj])
        Hb[:, :3, :3] += (-2.0 / NNp / NNp)[:, None, None] * np.einsum("ni,nj->nij", viRiTuk[si], viRiTuk[sj])
        Hb[:, :3, 3:] += (-2.0 * n[sj] / NNp / NNp)[:, None, None] * viRiTukukT[si]
        Hb[:, 3:, :3] += (-2.0 * n[si] / NNp / NNp)[:, None, None] * np.transpose(viRiTukukT[sj], (0, 2, 1))
        Hb[:, 3:, 3:] += (-2.0 * n[si] * n[sj] / NNp / NNp)[:, None, None] * np.repeat(ukukT[vs], len(ii), axis=0)
        bi.append(pose_idx[si].astype(np.int64)); bj.append(pose_idx[sj].astype(np.int64)); bl.append(Hb)
    return residual, g, (np.concatenate(bi), np.concatenate(bj), np.concatenate(bl))


def assemble_sparse(blocks, n_poses):
    """Sum block-COO into a full symmetric CSR matrix (mirror of lines 171-173)."""
    bi, bj, bl = blocks
    r = (6 * bi[:, None, None] + np.arange(6)[None, :, None]) + np.zeros((1, 1, 6), np.int64)
    c = (6 * bj[:, None, None] + np.arange(6)[None, None, :]) + np.zeros((1, 6, 1), np.int64)
    up = sp.coo_matrix((bl.ravel(), (r.ravel(), c.ravel())), shape=(6 * n_poses, 6 * n_poses)).tocsr()
    off = bi != bj
    lo = sp.coo_matrix((np.transpose(bl[off], (0, 2, 1)).ravel(),
                        (c[off].transpose(0, 2, 1).ravel(), r[off].transpose(0, 2, 1).ravel())),
                       shape=up.shape).tocsr()
    return (up + lo).tocsr()


def assemble_dense(blocks, n_poses):
    return assemble_sparse(blocks, n_poses).toarray()


def retract(poses, dx):
    """bavoxel.hpp:722-727: R_j <- R_j Exp(dx[6j:6j+3]), p_j <- p_j + dx[6j+3:6j+6]."""
    W = poses.shape[0]
    dx = dx.reshape(W, 6)
    R = poses[:, :9].reshape(W, 3, 3) @ so3_exp(dx[:, :3])
    out = poses.copy()
    out[:, :9] = R.reshape(W, 9)
    out[:, 9:12] = poses[:, 9:12] + dx[:, 3:]
    return out


def lm_step(H, g, u):
    """bavoxel.hpp:692-710: D = diag(H); (H + u D) dx = -g."""
    d = H.diagonal()
    A = (H + sp.diags(u * d)).tocsc()
    dx = spla.spsolve(A, -g.ravel())
    return dx, d


def balm_update(u, v, residual1, residual2, q1, rel_tol, bad=False):
    """The decision of one damping_iter pass (bavoxel.hpp:733-762): accept the trial poses when the residual drops, and the new
    damping u, v; then the stop test (:760, off for rel_tol < 0).  A non-finite trial residual or model, or `bad` (a non-finite
    step or singular pivot on the device), counts as no decrease.  Returns (u, v, accepted, stop)."""
    if bad or not (np.isfinite(residual2) and np.isfinite(q1)):
        residual2 = np.nan
    q = residual1 - residual2
    accepted = q > 0
    if accepted:
        rho = q / q1
        v = 2.0
        qq = 1 - (2 * rho - 1) ** 3
        u *= (1.0 / 3.0) if qq < 1.0 / 3.0 else qq
    else:
        u *= v
        v *= 2
    stop = rel_tol >= 0 and abs(residual1 - residual2) / residual1 < rel_tol
    return u, v, bool(accepted), bool(stop)


def damping_iter(vox_ptr, pose_idx, clusters, poses, u0=0.01, v0=2.0, max_iter=10, rel_tol=1e-6,
                 log=None):
    """bavoxel.hpp:662-767 incl. quirks Q1-Q3 of SURVEY.md §8a.  Returns (poses, info)."""
    W = poses.shape[0]
    V = len(vox_ptr) - 1
    u, v = u0, v0
    poses = poses.copy()
    is_calc_hess = True
    info = {"iters": 0, "r_first": None, "r_last": None, "accepted": 0, "trace": []}
    residual1 = None
    H = g = None
    for it in range(max_iter):
        if is_calc_hess:
            rs, g, blocks = acc_evaluate2(vox_ptr, pose_idx, clusters, poses, W)
            H = assemble_sparse(blocks, W)
            residual1 = rs / V                          # AVG_THR, line 635
            if info["r_first"] is None:
                info["r_first"] = residual1
        dx, d = lm_step(H, g, u)
        trial = retract(poses, dx)
        q1 = 0.5 * dx.dot(u * d * dx - g.ravel())       # line 729
        residual2 = only_residual(vox_ptr, pose_idx, clusters, trial) / V
        q1 /= V                                         # line 732
        info["trace"].append(dict(it=it, r1=residual1, r2=residual2, u=u, v=v, q=residual1 - residual2, q1=q1,
                                  dx_inf=float(np.abs(dx).max())))
        if log:
            log(info["trace"][-1])
        info["iters"] = it + 1
        u, v, is_calc_hess, stop = balm_update(u, v, residual1, residual2, q1, rel_tol)
        if is_calc_hess:
            poses = trial
            info["accepted"] += 1
            info["r_last"] = residual2
        elif info["r_last"] is None:
            info["r_last"] = residual1
        if stop:
            break
    info["u_last"], info["v_last"] = u, v
    return poses, info


def window_ba(win_ptr, vox_ptr, pose_idx, clusters, poses, min_voxels_per_pose=3, **lm_kw):
    """The window loop of LvbaSystem::runWindowBA (reference src/lvba_system.cpp:232-302) restated on the flat
    layout of lvba_lidar_lm_batch: window w owns poses win_ptr[w]..win_ptr[w+1]-1; every voxel lies in one window;
    pose_idx indexes the concatenated pose array.  Each window with at least `min_voxels_per_pose` voxels per pose
    (`plvec_voxels.size() < 3 * x_win.size()` -> continue, :262-266) runs its own damping_iter (:264); the others keep
    their poses.  Returns (poses, [info or None per window])."""
    win_ptr = np.asarray(win_ptr)
    poses = np.array(poses, dtype=np.float64, copy=True)
    first_pose = pose_idx[np.asarray(vox_ptr[:-1])] if len(vox_ptr) > 1 else np.zeros(0, np.int64)
    win_of_vox = np.searchsorted(win_ptr, first_pose, side="right") - 1
    infos = []
    for w in range(len(win_ptr) - 1):
        lo_, hi_ = int(win_ptr[w]), int(win_ptr[w + 1])
        vs = np.nonzero(win_of_vox == w)[0]
        if hi_ - lo_ <= 0 or len(vs) == 0 or len(vs) < min_voxels_per_pose * (hi_ - lo_):
            infos.append(None)
            continue
        vp = np.zeros(len(vs) + 1, np.int64)
        sl = [np.arange(vox_ptr[a], vox_ptr[a + 1]) for a in vs]
        vp[1:] = np.cumsum([len(x) for x in sl])
        idx = np.concatenate(sl)
        new, info = damping_iter(vp, (pose_idx[idx] - lo_).astype(np.int32), clusters[idx], poses[lo_:hi_], **lm_kw)
        poses[lo_:hi_] = new
        infos.append(info)
    return poses, infos
