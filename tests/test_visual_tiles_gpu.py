"""The reduced camera system build does not depend on the order in which the caller lists the landmarks: the library orders
them by the lowest system row of their clique and sums every S block and camera row of a tile on chip
(global-lvba_b200/csrc/visual_tiles.h).  The same problem with its landmarks in the caller's order, shuffled and already in
lowest-row order, with and without a fixed camera, gives S, rhs, the cost and one LM step of the numpy oracle, at the
tolerances of tests/test_visual_gpu.py."""
import numpy as np
import pytest

from oracle import visual_oracle as vo

pytestmark = pytest.mark.gpu

KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


def reorder(p, perm):
    op, cam, uv = p["obs_ptr"], p["obs_cam"], p["obs_uv"]
    K = np.diff(op)[perm]
    nop = np.zeros(len(perm) + 1, np.int64)
    nop[1:] = np.cumsum(K)
    idx = np.concatenate([np.arange(op[a], op[a + 1]) for a in perm])
    return dict(p, X=np.ascontiguousarray(p["X"][perm]), plane_nd=np.ascontiguousarray(p["plane_nd"][perm]), obs_ptr=nop,
                obs_cam=np.ascontiguousarray(cam[idx]), obs_uv=np.ascontiguousarray(uv[idx]))


def lowest_row_order(p, fixed_cam):
    """Landmarks by the lowest active camera they see (rows follow the camera index), cameras unsorted inside a landmark."""
    op, cam = p["obs_ptr"], p["obs_cam"]
    low = np.array([min([c for c in cam[op[a]:op[a + 1]] if c != fixed_cam], default=0) for a in range(len(op) - 1)])
    return np.argsort(low, kind="stable")


@pytest.mark.parametrize("fixed_cam", [0, -1])
@pytest.mark.parametrize("order", ["caller", "shuffled", "lowest_row"])
def test_system_and_step_match_oracle_in_any_landmark_order(gpu_pkg, problem_small, order, fixed_cam):
    p = problem_small
    T = len(p["obs_ptr"]) - 1
    if order == "shuffled":
        p = reorder(p, np.random.default_rng(20261015).permutation(T))
    elif order == "lowest_row":
        p = reorder(p, lowest_row_order(p, fixed_cam))
    args = [p[k] for k in KEYS]
    P = gpu_pkg.VisualProblem(*args, fixed_cam=fixed_cam)
    pr = vo.VisualProblem(*args, fixed_cam=fixed_cam)
    assert abs(P.cost() - pr.cost()) <= 1e-10 * pr.cost()
    cs, ps, model, cost = P.step(1e4)
    ref = vo.single_step(vo.VisualProblem(*args, fixed_cam=fixed_cam), 1e4, True)
    assert abs(cost - ref["cost"]) <= 1e-10 * ref["cost"]
    assert abs(model - ref["model"]) <= 1e-7 * abs(ref["model"])
    assert np.abs(cs - ref["cam_step"]).max() <= 1e-6 * np.abs(ref["cam_step"]).max()
    assert np.abs(ps - ref["pt_step"]).max() <= 1e-6 * np.abs(ref["pt_step"]).max()
    cam, rhs, br, bc, bl = P.get_system()
    S = gpu_pkg.env_blocks_to_dense(br, bc, bl, len(cam))
    assert np.array_equal(cam, np.nonzero(pr.cam_active)[0])
    assert np.abs(S - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
    assert np.abs(rhs.ravel() - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    P.close()
