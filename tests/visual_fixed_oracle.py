"""Constant camera sets on the oracle of the visual LM (oracle/visual_oracle.py, tests/visual_loss_oracle.py): the Ceres problem with
SetParameterBlockConstant on every camera of a set — the columns of the free cameras only, every residual block kept."""
import numpy as np


def mask_of(M, cams):
    m = np.zeros(M, bool)
    m[list(cams)] = True
    return m


def with_constant(pr, cams):
    """pr (a VisualProblem or RobustProblem) with exactly the cameras `cams` constant."""
    used = np.zeros(pr.M, bool)
    used[pr.obs_cam[pr.obs_ok]] = True
    used[list(cams)] = False
    pr.fixed = -1
    pr.cam_active = used
    pr.cam_col = np.full(pr.M, -1, np.int64)
    pr.cam_col[used] = np.arange(used.sum())
    pr.nc = int(used.sum())
    pr.ncols = 6 * pr.nc + 3 * pr.npt
    return pr
