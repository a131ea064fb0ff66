"""CPU oracle of path B with robust losses (numpy, float64): oracle/visual_oracle.py's problem with a ceres::LossFunction on the
reprojection and on the plane residual blocks.  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restated from ceres-solver 2.1.0 (not vendored; nothing to hold it against here):
  HuberLoss(a), CauchyLoss(a)   loss_function.cc, b = a^2
  Corrector                     corrector.cc: rho'' <= 0 for both losses, so the residual and the Jacobian of a block are
                                multiplied by sqrt(rho'(s)), s = |r|^2 of the block, and nothing else changes
  cost                          1/2 sum rho(s) over the blocks, also for the candidate of the trust-region test
Everything downstream (Jacobi scaling, LM diagonal, Schur system, gradient, model cost change) uses the corrected residuals and
Jacobian, so oracle/visual_oracle.py's single_step and trust-region loop apply to them unchanged: they take every cost from
RobustProblem.cost().  With both losses None everything equals oracle/visual_oracle.py bit for bit.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import visual_oracle as vo

NONE, HUBER, CAUCHY = 0, 1, 2
_TINY = np.finfo(np.float64).tiny          # DBL_MIN


def loss_rho(kind, a, s):
    """rho(s), rho'(s) of lvba_loss_kind `kind` with scale a (ceres HuberLoss / CauchyLoss), elementwise."""
    s = np.asarray(s, np.float64)
    b = a * a
    if kind == HUBER:
        big = s > b
        r = np.sqrt(np.where(big, s, 1.0))
        return np.where(big, 2.0 * a * r - b, s), np.where(big, np.maximum(_TINY, a / r), 1.0)
    if kind == CAUCHY:
        c = 1.0 / b
        u = 1.0 + s * c
        return b * np.log(u), np.maximum(_TINY, 1.0 / u)
    if kind == NONE:
        return s.copy(), np.ones_like(s)
    raise ValueError(f"unknown loss kind {kind}")


class RobustProblem(vo.VisualProblem):
    """vo.VisualProblem with loss_reproj / loss_plane = None or (kind, a)."""

    def __init__(self, *args, loss_reproj=None, loss_plane=None, **kw):
        super().__init__(*args, **kw)
        self.loss_reproj, self.loss_plane = loss_reproj, loss_plane

    def _blocks(self, res):
        """squared norm of every residual block: the reprojection 2-vectors, then the planes; and the rows of each block"""
        nr = int(self.obs_ok.sum())
        s_obs = res[0:2 * nr:2] ** 2 + res[1:2 * nr:2] ** 2
        return nr, s_obs, res[2 * nr:] ** 2

    def _rho(self, res):
        nr, s_obs, s_pl = self._blocks(res)
        lr = self.loss_reproj or (NONE, 1.0)
        lp = self.loss_plane or (NONE, 1.0)
        rho_o, d_o = loss_rho(lr[0], lr[1], s_obs)
        rho_p, d_p = loss_rho(lp[0], lp[1], s_pl)
        return nr, rho_o, d_o, rho_p, d_p

    def residuals(self, q=None, t=None, X=None, jac=False):
        """The corrected residuals r~ = sqrt(rho') r and Jacobian J~ = sqrt(rho') J, per block."""
        res, J = super().residuals(q, t, X, jac)
        if self.loss_reproj is None and self.loss_plane is None:
            return res, J
        nr, _, d_o, _, d_p = self._rho(res)
        w = np.concatenate([np.repeat(np.sqrt(d_o), 2), np.sqrt(d_p)])
        res = res * w
        if J is not None:
            J = (sp.diags(w) @ J).tocsr()
        return res, J

    def cost(self, q=None, t=None, X=None):
        """1/2 sum rho over the residual blocks."""
        if self.loss_reproj is None and self.loss_plane is None:
            return super().cost(q, t, X)
        res, _ = vo.VisualProblem.residuals(self, q, t, X, jac=False)
        _, rho_o, _, rho_p, _ = self._rho(res)
        return 0.5 * float(rho_o.sum() + rho_p.sum())


TERM = {"max_iter": 0, "function": 1, "parameter": 2, "gradient": 3, "radius": 4, "invalid_steps": 5}


def tangent_gradient_fd(prob: RobustProblem, h=1e-7):
    """Central differences of cost() along every tangent column (cameras via the Q9 manifold, t and X additive).  The step is
    small because Huber's rho is only C^1 at s = a^2: a difference across that point is off by O(h)."""
    g = np.zeros(prob.ncols)
    for j in range(prob.ncols):
        d = np.zeros(prob.ncols); d[j] = h
        g[j] = (prob.cost(*prob.plus(d)) - prob.cost(*prob.plus(-d))) / (2 * h)
    return g


def with_outliers(p, frac=0.05, lo=20.0, hi=50.0, seed=0):
    """A copy of the scene dict p whose observations, a fraction `frac` of them, are moved by lo..hi px in a random direction."""
    rng = np.random.default_rng(seed)
    q = dict(p)
    uv = np.array(p["obs_uv"], np.float32).copy()
    n = len(uv)
    k = rng.choice(n, max(1, int(round(frac * n))), replace=False)
    ang = rng.uniform(0, 2 * np.pi, len(k)); mag = rng.uniform(lo, hi, len(k))
    uv[k, 0] += (mag * np.cos(ang)).astype(np.float32); uv[k, 1] += (mag * np.sin(ang)).astype(np.float32)
    q["obs_uv"] = uv
    return q, k
