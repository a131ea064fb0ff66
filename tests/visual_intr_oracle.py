"""CPU oracle of path B with the intrinsics as a parameter block (numpy, float64): tests/visual_loss_oracle.py's problem with
(fx fy cx cy k1 k2 p1 p2) one more ceres parameter block of size 8 in every ReprojErrorWhitenedDistorted, a SubsetManifold
holding the entries whose bit of `mask` is clear (lvba_visual_opts::refine_intrinsics).  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Columns: [cameras (6 per active camera) | landmarks (3 per valid landmark) | free intrinsics (k)].  Everything else is the
trust-region loop of oracle/visual_oracle.py (ceres_lm), restated here over these columns: Jacobi scaling of every column,
the LM diagonal, the tolerances, ||x|| over all 8 intrinsics and the step over the free ones.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import visual_oracle as vo
import visual_loss_oracle as vl

FOCAL, PRINCIPAL, DISTORTION = 0x03, 0x0C, 0xF0


def intr_jacobian(q, t, X, intr, sigma):
    """d r / d intr (n, 2, 8) of the whitened reprojection residual of vo.reproj_eval; zero where z <= 1e-8."""
    fx, fy, cx, cy, k1, k2, p1, p2 = intr
    Xc = vo.quat_rotate(q, X) + t
    z = Xc[:, 2]
    valid = z > 1e-8
    zs = np.where(valid, z, 1.0)
    xn, yn = Xc[:, 0] / zs, Xc[:, 1] / zs
    r2 = xn * xn + yn * yn
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    J = np.zeros((len(z), 2, 8))
    J[:, 0, 0] = xd; J[:, 0, 2] = 1.0
    J[:, 0, 4] = fx * xn * r2; J[:, 0, 5] = fx * xn * r2 * r2; J[:, 0, 6] = fx * 2 * xn * yn; J[:, 0, 7] = fx * (r2 + 2 * xn * xn)
    J[:, 1, 1] = yd; J[:, 1, 3] = 1.0
    J[:, 1, 4] = fy * yn * r2; J[:, 1, 5] = fy * yn * r2 * r2; J[:, 1, 6] = fy * (r2 + 2 * yn * yn); J[:, 1, 7] = fy * 2 * xn * yn
    J /= sigma
    J[~valid] = 0.0
    return J


class IntrProblem(vl.RobustProblem):
    """vl.RobustProblem with the free intrinsics (bits of mask) as the last k columns."""

    def __init__(self, *args, mask=0, **kw):
        super().__init__(*args, **kw)
        self.mask = int(mask)
        self.free = np.array([i for i in range(8) if (self.mask >> i) & 1], np.int64)
        self.k = len(self.free)

    @property
    def nb(self):                             # columns of the cameras and landmarks (tests/visual_fixed_oracle.py may change them)
        return self.ncols

    @property
    def nall(self):
        return self.ncols + self.k

    def _with_intr(self, intr, fn):
        saved = self.intr
        if intr is not None:
            self.intr = np.asarray(intr, np.float64)
        try:
            return fn()
        finally:
            self.intr = saved

    def residuals_k(self, q=None, t=None, X=None, intr=None, jac=False):
        """Corrected residuals and, with jac, the corrected Jacobian over all nall columns (csr)."""
        def run():
            res, J = vo.VisualProblem.residuals(self, q, t, X, jac)
            Jk = None
            if jac:
                o = np.nonzero(self.obs_ok)[0]
                qq = self.q if q is None else q; tt = self.t if t is None else t; XX = self.X if X is None else X
                Jo = intr_jacobian(qq[self.obs_cam[o]], tt[self.obs_cam[o]], XX[self.obs_trk[o]], self.intr, self.sp)
                Jk = np.zeros((len(res), self.k))
                Jk[:2 * len(o)] = Jo[:, :, self.free].reshape(2 * len(o), self.k)
            if self.loss_reproj is not None or self.loss_plane is not None:
                _, _, d_o, _, d_p = self._rho(res)
                w = np.concatenate([np.repeat(np.sqrt(d_o), 2), np.sqrt(d_p)])
                res = res * w
                if jac:
                    J = (sp.diags(w) @ J).tocsr(); Jk = Jk * w[:, None]
            if jac:
                J = sp.hstack([J, sp.csr_matrix(Jk)]).tocsr()
            return res, J
        return self._with_intr(intr, run)

    def cost_k(self, q=None, t=None, X=None, intr=None):
        return self._with_intr(intr, lambda: vl.RobustProblem.cost(self, q, t, X))

    def plus_k(self, delta):
        q, t, X = vo.VisualProblem.plus(self, delta[:self.nb])
        intr = self.intr.copy()
        intr[self.free] += delta[self.nb:]
        return q, t, X, intr

    def x_norm_k(self):
        return float(np.sqrt(vo.VisualProblem.x_norm(self) ** 2 + (self.intr ** 2).sum()))


def _scaled(prob, radius, scaling=True, min_diag=1e-6, max_diag=1e32):
    res, J = prob.residuals_k(jac=True)
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.nall)
    Js = (J @ sp.diags(scale)).tocsr()
    diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
    return res, J, Js, scale, np.sqrt(diag / radius)


def step_full(prob: IntrProblem, radius=1e4, scaling=True):
    """One LM step from the dense normal equations over every column: dict(y (scaled), delta, model, scale)."""
    res, _, Js, scale, lm = _scaled(prob, radius, scaling)
    A = (Js.T @ Js).toarray() + np.diag(lm * lm)
    y = np.linalg.solve(A, -(Js.T @ res))
    Jy = Js @ y
    return dict(y=y, delta=y * scale, model=-float(Jy @ (res + 0.5 * Jy)), scale=scale)


def bordered_system(prob: IntrProblem, radius=1e4, scaling=True):
    """The landmarks eliminated: S (camera system without its LM diagonal), B (border), C (corner without its LM diagonal),
    rhs_c, rhs_k, and the LM diagonals Dc, Dk (squared), all Jacobi-scaled as the device builds them."""
    res, _, Js, scale, lm = _scaled(prob, radius, scaling)
    A = (Js.T @ Js).toarray()
    g = Js.T @ res
    nc6, nb = 6 * prob.nc, prob.nb
    d2 = lm * lm
    pts = np.arange(nc6, nb)
    oth = np.concatenate([np.arange(nc6), np.arange(nb, prob.nall)])
    V = A[np.ix_(pts, pts)] + np.diag(d2[pts])
    W = A[np.ix_(oth, pts)]
    Vi = np.linalg.inv(V)
    R = A[np.ix_(oth, oth)] - W @ Vi @ W.T
    r = -(g[oth] - W @ Vi @ g[pts])
    return dict(S=R[:nc6, :nc6], B=R[:nc6, nc6:], C=R[nc6:, nc6:], rhs_c=r[:nc6], rhs_k=r[nc6:],
                Dc=d2[:nc6], Dk=d2[nb:], V=V, W=W, g_p=g[pts], scale=scale, res=res, Js=Js)


def step_bordered(prob: IntrProblem, radius=1e4, scaling=True):
    """The device's algorithm: Y = A^-1 B and y = A^-1 r_c with A the damped camera system (k + 1 solves), the k x k Schur
    complement Sigma = C + D_k - B^T Y, dk = Sigma^-1 (rhs_k - B^T y), dc = y - Y dk, then the landmark back-substitution."""
    s = bordered_system(prob, radius, scaling)
    nc6 = 6 * prob.nc
    A = s["S"] + np.diag(s["Dc"])
    if nc6:
        Y = np.linalg.solve(A, s["B"]); y = np.linalg.solve(A, s["rhs_c"])
    else:
        Y = np.zeros((0, prob.k)); y = np.zeros(0)
    Sig = s["C"] + np.diag(s["Dk"]) - s["B"].T @ Y
    L = np.linalg.cholesky(Sig)
    yk = np.linalg.solve(L.T, np.linalg.solve(L, s["rhs_k"] - s["B"].T @ y))
    yc = y - Y @ yk
    Wc, Wk = s["W"][:nc6], s["W"][nc6:]
    yp = np.linalg.solve(s["V"], -(s["g_p"] + Wc.T @ yc + Wk.T @ yk))
    yall = np.concatenate([yc, yp, yk])
    Jy = s["Js"] @ yall
    return dict(y=yall, delta=yall * s["scale"], model=-float(Jy @ (s["res"] + 0.5 * Jy)), system=s)


def ceres_lm(prob: IntrProblem, max_iter=50, radius0=1e4, scaling=True, f_tol=1e-6, g_tol=1e-10, p_tol=1e-8):
    """oracle/visual_oracle.py's ceres_lm over the columns of IntrProblem (the intrinsics refined in place: prob.intr)."""
    min_diag, max_diag = 1e-6, 1e32
    radius, nu = radius0, 2.0
    info = {"iters": 0, "accepted": 0, "term": "max_iter"}
    res, J = prob.residuals_k(jac=True)
    cost = prob.cost_k()
    info["cost0"] = cost
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.nall)
    Js = (J @ sp.diags(scale)).tocsr()
    if np.abs(J.T @ res).max() <= g_tol:
        info["term"] = "gradient"; info["cost"] = cost
        return prob, info
    reuse_diag, diag, invalid = False, None, 0
    for it in range(1, max_iter + 1):
        info["iters"] = it
        if not reuse_diag:
            diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
        lm = np.sqrt(diag / radius)
        A = (Js.T @ Js + sp.diags(lm * lm)).tocsc()
        y = spla.spsolve(A, -(Js.T @ res))
        reuse_diag = True
        Jy = Js @ y
        model = -float(Jy @ (res + 0.5 * Jy))
        if not np.all(np.isfinite(y)) or model <= 0:
            invalid += 1
            radius *= 0.5
            if invalid >= 5:
                info["term"] = "invalid_steps"; break
            continue
        invalid = 0
        delta = y * scale
        qn, tn, Xn, In = prob.plus_k(delta)
        cand = prob.cost_k(qn, tn, Xn, In)
        ca, tv = prob.cam_active, prob.tv
        step_norm = float(np.sqrt(((qn[ca] - prob.q[ca]) ** 2).sum() + ((tn[ca] - prob.t[ca]) ** 2).sum()
                                  + ((Xn[tv] - prob.X[tv]) ** 2).sum() + ((In - prob.intr) ** 2).sum()))
        rho = (cost - cand) / model
        if step_norm <= p_tol * (prob.x_norm_k() + p_tol):
            info["term"] = "parameter"; break
        if abs(cost - cand) <= f_tol * cost:
            info["term"] = "function"; break
        if rho > 1e-3:
            prob.q, prob.t, prob.X, prob.intr = qn, tn, Xn, In
            cost = cand
            info["accepted"] += 1
            res, J = prob.residuals_k(jac=True)
            Js = (J @ sp.diags(scale)).tocsr()
            radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3))
            nu = 2.0
            reuse_diag = False
            if np.abs(J.T @ res).max() <= g_tol:
                info["term"] = "gradient"; break
        else:
            radius /= nu
            nu *= 2
            if radius < 1e-32:
                info["term"] = "radius"; break
    info["cost"] = cost
    return prob, info


def miscalibrated(p, dfocal=0.01, dk1=0.02):
    """A copy of the scene dict p whose intrinsics have fx and fy off by the factor 1 + dfocal and k1 off by dk1 (the true ones
    stay in p["intr"] of the original)."""
    q = dict(p)
    intr = np.array(p["intr"], np.float64).copy()
    intr[0] *= 1 + dfocal; intr[1] *= 1 + dfocal; intr[4] += dk1
    q["intr"] = intr
    return q
