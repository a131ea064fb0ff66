"""Constant pose sets on the oracle of the LiDAR LM (oracle/lidar_oracle.py): BALM2's damping_iter with Ceres'
SetParameterBlockConstant on every pose of a set — the rows and columns of the free poses only, every voxel kept in the cost.
D = diag(H_ff); q1 = 1/2 dx_f^T (u D dx_f - g_f) / V; the damping rule is lidar_oracle.balm_update unchanged; constant poses are
never touched.  With no free pose the residual is evaluated once (iterations 0, Ceres' function tolerance)."""
import numpy as np
import scipy.sparse as sp

from oracle import lidar_oracle as lo


def mask_of(W, poses):
    m = np.zeros(W, bool)
    m[list(poses)] = True
    return m


def free_index(fixed, W):
    """the free poses in ascending order (the rows of the pose system) and their 6 W columns"""
    free = np.arange(W) if fixed is None else np.flatnonzero(~np.asarray(fixed, bool))
    cols = (6 * free[:, None] + np.arange(6)[None, :]).ravel()
    return free, cols


def restricted(H, g, fixed):
    """H_ff (sparse or dense) and g_f of the full system H [6W, 6W], g [W, 6]"""
    W = np.asarray(g).reshape(-1, 6).shape[0]
    if fixed is None or not np.any(fixed):             # no constant pose: the system as it is
        return H, np.asarray(g).ravel()
    _, cols = free_index(fixed, W)
    Hf = H[cols][:, cols] if sp.issparse(H) else np.asarray(H)[np.ix_(cols, cols)]
    return Hf, np.asarray(g).ravel()[cols]


def first_step(H, g, u, fixed):
    """dx [W, 6] of (H_ff + u diag(H_ff)) dx_f = -g_f, zeros for constant poses (dense solve)"""
    W = np.asarray(g).reshape(-1, 6).shape[0]
    Hf, gf = restricted(np.asarray(H.toarray() if sp.issparse(H) else H), g, fixed)
    dx = np.zeros(6 * W)
    _, cols = free_index(fixed, W)
    if len(cols):
        dx[cols] = np.linalg.solve(Hf + np.diag(u * np.diag(Hf)), -gf)
    return dx.reshape(W, 6)


def damping_iter_fixed(vox_ptr, pose_idx, clusters, poses, fixed=None, u0=0.01, v0=2.0, max_iter=10, rel_tol=1e-6):
    """lidar_oracle.damping_iter with the poses of the boolean mask `fixed` (None: none) held constant.  Returns (poses, info)."""
    W = poses.shape[0]
    V = len(vox_ptr) - 1
    fixed = np.zeros(W, bool) if fixed is None else np.asarray(fixed, bool)
    free, cols = free_index(fixed, W)
    u, v = u0, v0
    poses = poses.copy()
    info = {"iters": 0, "r_first": None, "r_last": None, "accepted": 0, "trace": []}
    if len(free) == 0:                                  # nothing to solve: the residual once
        r = lo.only_residual(vox_ptr, pose_idx, clusters, poses) / V
        info.update(r_first=r, r_last=r, u_last=u, v_last=v, term="function_tol")
        return poses, info
    is_calc_hess = True
    residual1 = None
    H = g = None
    for it in range(max_iter):
        if is_calc_hess:
            rs, g_all, blocks = lo.acc_evaluate2(vox_ptr, pose_idx, clusters, poses, W)
            H, g = restricted(lo.assemble_sparse(blocks, W), g_all, fixed)
            residual1 = rs / V
            if info["r_first"] is None:
                info["r_first"] = residual1
        dx_f, d = lo.lm_step(H, g, u)
        dx = np.zeros(6 * W)
        dx[cols] = dx_f
        trial = lo.retract(poses, dx)
        trial[fixed] = poses[fixed]                     # constant poses are never touched
        q1 = 0.5 * dx_f.dot(u * d * dx_f - g.ravel())
        residual2 = lo.only_residual(vox_ptr, pose_idx, clusters, trial) / V
        q1 /= V
        info["trace"].append(dict(it=it, r1=residual1, r2=residual2, u=u, v=v, q1=q1))
        info["iters"] = it + 1
        u, v, is_calc_hess, stop = lo.balm_update(u, v, residual1, residual2, q1, rel_tol)
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


def window_ba_fixed(win_ptr, vox_ptr, pose_idx, clusters, poses, fixed=None, min_voxels_per_pose=3, **lm_kw):
    """lidar_oracle.window_ba with constant poses (a mask over the concatenated poses): every window runs its own
    damping_iter_fixed; the skip rule counts all poses of a window.  Returns (poses, [info or None per window])."""
    win_ptr = np.asarray(win_ptr)
    W = len(poses)
    fixed = np.zeros(W, bool) if fixed is None else np.asarray(fixed, bool)
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
        new, info = damping_iter_fixed(vp, (pose_idx[idx] - lo_).astype(np.int32), clusters[idx], poses[lo_:hi_], fixed[lo_:hi_], **lm_kw)
        poses[lo_:hi_] = new
        infos.append(info)
    return poses, infos
