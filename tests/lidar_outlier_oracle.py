"""Oracle of BALM2's voxel outlier removal, which the reference carries commented out in include/BALM/bavoxel.hpp:
VOX_HESS::evaluate_residual (:205-234), VOX_HESS::remove_residual (:236-268) and BALM2::remove_outlier (:650-660).

remove_outlier_loop restates the reference literally: a sequential walk that erases from a list.  remove_outlier_mask is the
same rule written the way the library computes it on the device (lidar_outliers.h): removed_i = (lambda_i >= thr) and i < k*,
where k* is the first i with lambda_i < thr and #{j < i : lambda_j >= thr} = reject_num (V when there is none).
damping_iter_with_removal chains damping_iter, remove_outlier and damping_iter as a caller of the reference would."""
import math

import numpy as np

from oracle import lidar_oracle as lo


def evaluate_residual(vox_ptr, pose_idx, clusters, poses):
    """lambda_0 of every voxel (evaluate_residual, :205-234)."""
    lam, *_ = lo.voxel_eig(np.asarray(vox_ptr), np.asarray(pose_idx), np.asarray(clusters), np.asarray(poses))
    return lam[:, 0].copy()


def rule_params(ratio, V):
    """(index of thr in the sorted lambdas, reject_num) of remove_outlier :655-656, or None where the library refuses."""
    if not (math.isfinite(ratio) and 0.0 <= ratio < 1.0):
        return None
    k = math.floor((1.0 - ratio) * float(V))
    if k < 1:
        return None
    return k - 1, math.floor(ratio * float(V))


def remove_outlier_loop(lam, ratio):
    """remove_outlier + remove_residual as the reference writes them: returns the removed mask [V]."""
    lam = [float(x) for x in lam]
    V = len(lam)
    residuals = sorted(lam)                                          # std::sort, ascending
    threshold = residuals[math.floor((1 - ratio) * V) - 1]
    reject_num = float(math.floor(ratio * V))                        # int, then passed on as a double
    voxels = list(range(V))                                          # plvec_voxels, by original index
    rej_cnt = 0
    i = 0
    while i < len(voxels):
        if lam[voxels[i]] >= threshold:
            del voxels[i]                                            # plvec_voxels.erase(begin() + i)
            rej_cnt += 1
            continue
        i += 1
        if rej_cnt == reject_num:
            break
    removed = np.ones(V, bool)
    removed[voxels] = False
    return removed


def remove_outlier_mask(lam, ratio):
    """The same rule in the vectorised k* form of the device passes."""
    lam = np.asarray(lam, np.float64)
    V = len(lam)
    k_thr, reject_num = rule_params(ratio, V)
    thr = np.sort(lam, kind="stable")[k_thr]
    flag = lam >= thr
    before = np.concatenate(([0], np.cumsum(flag)[:-1]))
    stop = np.nonzero((~flag) & (before == reject_num))[0]
    k_star = int(stop[0]) if len(stop) else V
    return flag & (np.arange(V) < k_star)


def kept_problem(vox_ptr, pose_idx, clusters, removed):
    """The CSR and records of the voxels not in `removed`, in their order."""
    vox_ptr = np.asarray(vox_ptr, np.int64)
    keep = np.nonzero(~np.asarray(removed, bool))[0]
    counts = np.diff(vox_ptr)[keep]
    slots = np.concatenate([np.arange(vox_ptr[a], vox_ptr[a + 1]) for a in keep]) if len(keep) else np.zeros(0, np.int64)
    vp = np.concatenate(([0], np.cumsum(counts))).astype(np.int64)
    return vp, np.asarray(pose_idx)[slots].copy(), np.asarray(clusters)[slots].copy()


def damping_iter_with_removal(vox_ptr, pose_idx, clusters, poses, ratio, **lm_kw):
    """damping_iter, remove_outlier(ratio) at its end poses, damping_iter on the kept voxels.  Returns (poses, removed)."""
    p1, _ = lo.damping_iter(vox_ptr, pose_idx, clusters, poses, **lm_kw)
    removed = remove_outlier_loop(evaluate_residual(vox_ptr, pose_idx, clusters, p1), ratio)
    vp, pi, cl = kept_problem(vox_ptr, pose_idx, clusters, removed)
    p2, _ = lo.damping_iter(vp, pi, cl, p1, **lm_kw)
    return p2, removed
