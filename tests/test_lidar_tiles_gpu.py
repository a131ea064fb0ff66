"""The LiDAR Hessian build does not depend on the order in which the caller lists the voxels: the library orders them by
lowest pose and sums every H block of a tile on chip (global-lvba_b200/csrc/lidar_tiles.h).  The same problem with its voxels
shuffled, already in lowest-pose order (the direct upload path) and in the caller's order gives H, g and the residual of the
numpy oracle, at the tolerances of tests/test_lidar_gpu.py."""
import numpy as np
import pytest

from oracle import lidar_oracle as lo

pytestmark = pytest.mark.gpu


def reorder(p, perm):
    vp, pi, cl = p["vox_ptr"], p["pose_idx"], p["clusters"]
    K = np.diff(vp)[perm]
    nvp = np.zeros(len(perm) + 1, np.int64)
    nvp[1:] = np.cumsum(K)
    idx = np.concatenate([np.arange(vp[a], vp[a + 1]) for a in perm])
    return dict(p, vox_ptr=nvp, pose_idx=np.ascontiguousarray(pi[idx]), clusters=np.ascontiguousarray(cl[idx]))


@pytest.mark.parametrize("order", ["caller", "shuffled", "lowest_pose"])
def test_build_matches_oracle_in_any_voxel_order(gpu_pkg, problem_A, order):
    p, W = problem_A, 50
    V = len(p["vox_ptr"]) - 1
    if order == "shuffled":
        p = reorder(p, np.random.default_rng(20261015).permutation(V))
    elif order == "lowest_pose":
        p = reorder(p, np.argsort(p["pose_idx"][p["vox_ptr"][:-1]], kind="stable"))
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    r = P.build()
    g, br, bc, bl = P.get_system()
    res = P.residual()
    P.close()
    r_ref, g_ref, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    H = gpu_pkg.env_blocks_to_dense(br, bc, bl, W)
    H_ref = lo.assemble_dense(blocks, W)
    assert abs(r - r_ref) <= 1e-8 * abs(r_ref)
    assert abs(res - r_ref) <= 1e-8 * abs(r_ref)
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    assert np.abs(H - H_ref).max() <= 1e-7 * np.abs(H_ref).max()
