"""CPU ORACLE for hot path B — visual BA with LiDAR plane priors (numpy, float64).

TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/lidar_oracle.py header).

PARITY: the two cost functors ARE pinned against the reference's own source (include/utils.hpp:51-147 compiled where it
lies, evaluated with T = double and with T = Jet as ceres::AutoDiffCostFunction does: oracle/ref_driver.cpp,
tests/golden/ref_balm.npz, tests/test_ref_pin.py — residuals 1e-10, Jacobians 1e-12, the z_c <= 1e-8 branch and a
non-unit quaternion included).  THE SOLVER IS UNPINNED: it is ceres-solver 2.1.0 (README.md:21, CMakeLists.txt:33), a
third-party dependency that is neither vendored under /root/reference nor installed here; its trust-region algorithm
is restated below from the published algorithm and no Ceres binary exists here to hold it against.  What is restated:

  reproj_residual / jac   ReprojErrorWhitenedDistorted   include/utils.hpp:61-111
  plane_residual / jac    PointPlaneErrorWhitened        include/utils.hpp:133-139
  problem structure       optimizeCameraPoses            src/lvba_system.cpp:1571-1643
                          (camera 0 constant :1582-1583; only landmarks with a valid
                          plane :1598-1603; loss = nullptr :1630,:1639; 50 iterations,
                          DENSE_SCHUR :1573-1574)
  trust-region LM         ceres-solver 2.1.0 published algorithm (SURVEY.md Q9-Q11, A.3):
                          Jacobi column scaling 1/(1+||J0[:,j]||) fixed at iteration 0,
                          LM diagonal sqrt(clamp(diag(J~^T J~),1e-6,1e32)/radius), radius0 1e4,
                          step acceptance rho > 1e-3, radius /= max(1/3, 1-(2rho-1)^3) on
                          accept, radius /= nu (nu*=2) on reject, function / parameter /
                          gradient tolerances 1e-6 / 1e-8 / 1e-10, cost = 1/2 sum r^2.
  quaternion manifold     ceres::EigenQuaternionManifold applied to {w,x,y,z} memory
                          (src/lvba_system.cpp:1579) — the "Q9" mislabelled-order Plus.

The analytic Jacobians here replace Ceres' Jet auto-diff; they are pinned by
finite differences and by scipy.optimize.least_squares on small problems
(tests/test_oracle_visual.py).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from .lidar_oracle import hat


def quat_rotate(q, X):
    """ceres::QuaternionRotatePoint (normalises q), batched.  q = (w,x,y,z)."""
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, v = q[..., :1], q[..., 1:]
    uv = 2.0 * np.cross(v, X)
    return X + w * uv + np.cross(v, uv)


def quat_to_rot(q):
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - w * z); R[..., 0, 2] = 2 * (x * z + w * y)
    R[..., 1, 0] = 2 * (x * y + w * z); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - w * x)
    R[..., 2, 0] = 2 * (x * z - w * y); R[..., 2, 1] = 2 * (y * z + w * x); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def plus_jacobian(q):
    """EigenQuaternionManifold::PlusJacobian on memory m = (w,x,y,z) read as Eigen (x,y,z,w).
    Rows = memory slots m0..m3, columns = tangent delta (SURVEY.md Q9).  (n,4,3)."""
    m0, m1, m2, m3 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    J = np.empty(q.shape[:-1] + (4, 3))
    J[..., 0, 0], J[..., 0, 1], J[..., 0, 2] = m3, m2, -m1
    J[..., 1, 0], J[..., 1, 1], J[..., 1, 2] = -m2, m3, m0
    J[..., 2, 0], J[..., 2, 1], J[..., 2, 2] = m1, -m0, m3
    J[..., 3, 0], J[..., 3, 1], J[..., 3, 2] = -m0, -m1, -m2
    return J


def manifold_plus(q, delta):
    """EigenQuaternionManifold::Plus on (w,x,y,z) memory (Q9): treat (m3; m0,m1,m2) as a
    Hamilton quaternion (w; v) and left-multiply by (cos|d|; sin|d|/|d| d)."""
    nd = np.linalg.norm(delta, axis=-1)
    out = q.copy()
    nz = nd > 0
    if not np.any(nz):
        return out
    d = delta[nz]; n = nd[nz]
    s = (np.sin(n) / n)[:, None] * d
    c = np.cos(n)
    bw = q[nz, 3]; bv = q[nz, 0:3]
    rw = c * bw - np.einsum("ni,ni->n", s, bv)
    rv = c[:, None] * bv + bw[:, None] * s + np.cross(s, bv)
    out[nz, 0:3] = rv
    out[nz, 3] = rw
    return out


def reproj_eval(q, t, X, uv, intr, sigma, want_jac=True):
    """utils.hpp:61-111 for a batch of observations.  q,t,X,uv are per observation.
    Returns r (n,2) and, if asked, Jq (n,2,3 tangent, Q9 basis), Jt (n,2,3), JX (n,2,3)."""
    fx, fy, cx, cy, k1, k2, p1, p2 = intr
    qn = q / np.linalg.norm(q, axis=-1, keepdims=True)
    RX = quat_rotate(q, X)
    Xc = RX + t
    z = Xc[:, 2]
    valid = z > 1e-8                                     # line 78
    zs = np.where(valid, z, 1.0)
    xn, yn = Xc[:, 0] / zs, Xc[:, 1] / zs
    r2 = xn * xn + yn * yn
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    r = np.stack([(fx * xd + cx - uv[:, 0]) / sigma, (fy * yd + cy - uv[:, 1]) / sigma], 1)
    r[~valid] = 0.0
    if not want_jac:
        return r, None, None, None
    g = 2 * (k1 + 2 * k2 * r2)
    Dd = np.empty((len(z), 2, 2))
    Dd[:, 0, 0] = rad + xn * xn * g + 2 * p1 * yn + 6 * p2 * xn
    Dd[:, 0, 1] = xn * yn * g + 2 * p1 * xn + 2 * p2 * yn
    Dd[:, 1, 0] = Dd[:, 0, 1]
    Dd[:, 1, 1] = rad + yn * yn * g + 6 * p1 * yn + 2 * p2 * xn
    Dn = np.zeros((len(z), 2, 3))
    Dn[:, 0, 0] = 1 / zs; Dn[:, 0, 2] = -xn / zs
    Dn[:, 1, 1] = 1 / zs; Dn[:, 1, 2] = -yn / zs
    F = np.array([[fx / sigma, 0.0], [0.0, fy / sigma]])
    Jpix = F[None] @ Dd @ Dn                             # d r / d Xc   (n,2,3)
    Rm = quat_to_rot(q)
    JX = Jpix @ Rm
    Jt = Jpix.copy()
    # d(R(q)X)/dq ambient (unit form X + 2w v x X + 2 v x (v x X)), then Q9 tangent basis
    w = qn[:, 0]; v = qn[:, 1:]
    vxX = np.cross(v, X)
    dW = 2.0 * vxX                                       # (n,3)
    dV = -2.0 * w[:, None, None] * hat(X) - 2.0 * hat(vxX) - 2.0 * hat(v) @ hat(X)   # (n,3,3)
    Jamb = np.concatenate([dW[:, :, None], dV], 2)       # (n,3,4)
    Jq = Jpix @ Jamb @ plus_jacobian(qn)
    for J in (Jq, Jt, JX):
        J[~valid] = 0.0
    return r, Jq, Jt, JX


def plane_eval(X, plane_nd, sigma):
    """utils.hpp:133-139: r = sqrt(e^2 + 1e-12)/max(1e-9, sigma), e = -(n.X + d)."""
    s = max(1e-9, sigma)
    e = -(np.einsum("ni,ni->n", plane_nd[:, :3], X) + plane_nd[:, 3])
    root = np.sqrt(e * e + 1e-12)
    r = root / s
    J = (e / root)[:, None] * (-plane_nd[:, :3]) / s
    return r, J


def valid_tracks(plane_nd):
    """has_valid_plane, src/lvba_system.cpp:1598: finite and !n.isZero(1e-6)."""
    n, d = plane_nd[:, :3], plane_nd[:, 3]
    return np.isfinite(n).all(1) & np.isfinite(d) & (np.abs(n) > 1e-6).any(1)


class VisualProblem:
    """Index bookkeeping for the Ceres problem of src/lvba_system.cpp:1571-1643."""

    def __init__(self, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane,
                 fixed_cam=0):
        self.q = np.array(q, np.float64); self.t = np.array(t, np.float64); self.X = np.array(X, np.float64)
        self.plane_nd = np.asarray(plane_nd, np.float64)
        self.obs_ptr = np.asarray(obs_ptr, np.int64); self.obs_cam = np.asarray(obs_cam, np.int64)
        self.obs_uv = np.asarray(obs_uv, np.float32).astype(np.float64)
        self.intr = np.asarray(intr, np.float64); self.sp = sigma_px; self.spl = sigma_plane
        self.M, self.T = self.q.shape[0], self.X.shape[0]
        self.fixed = fixed_cam
        self.tv = valid_tracks(self.plane_nd)
        L = np.diff(self.obs_ptr)
        self.obs_trk = np.repeat(np.arange(self.T), L)
        self.obs_ok = self.tv[self.obs_trk]
        # cameras that carry at least one residual and are not constant are "active"
        used = np.zeros(self.M, bool); used[self.obs_cam[self.obs_ok]] = True
        if 0 <= self.fixed < self.M:
            used[self.fixed] = False
        self.cam_active = used
        self.cam_col = np.full(self.M, -1, np.int64)
        self.cam_col[used] = np.arange(used.sum())
        self.nc = int(used.sum())
        self.pt_col = np.full(self.T, -1, np.int64)
        self.pt_col[self.tv] = np.arange(self.tv.sum())
        self.npt = int(self.tv.sum())
        self.ncols = 6 * self.nc + 3 * self.npt

    # ---- evaluation --------------------------------------------------
    def residuals(self, q=None, t=None, X=None, jac=False):
        q = self.q if q is None else q; t = self.t if t is None else t; X = self.X if X is None else X
        o = np.nonzero(self.obs_ok)[0]
        cam = self.obs_cam[o]; trk = self.obs_trk[o]
        r, Jq, Jt, JX = reproj_eval(q[cam], t[cam], X[trk], self.obs_uv[o], self.intr, self.sp, jac)
        tr = np.nonzero(self.tv)[0]
        rp, Jp = plane_eval(X[tr], self.plane_nd[tr], self.spl)
        res = np.concatenate([r.ravel(), rp])
        if not jac:
            return res, None
        nr = len(o)
        rows, cols, vals = [], [], []
        rr = (2 * np.arange(nr))[:, None, None] + np.arange(2)[None, :, None] + np.zeros((1, 1, 3), np.int64)
        act = self.cam_col[cam] >= 0
        for blk, off in ((Jq, 0), (Jt, 3)):
            cc = (6 * self.cam_col[cam] + off)[:, None, None] + np.arange(3)[None, None, :] + np.zeros((1, 2, 1), np.int64)
            rows.append(rr[act].ravel()); cols.append(cc[act].ravel()); vals.append(blk[act].ravel())
        cc = (6 * self.nc + 3 * self.pt_col[trk])[:, None, None] + np.arange(3)[None, None, :] + np.zeros((1, 2, 1), np.int64)
        rows.append(rr.ravel()); cols.append(cc.ravel()); vals.append(JX.ravel())
        rows.append(np.repeat(2 * nr + np.arange(len(tr)), 3))
        cols.append(((6 * self.nc + 3 * self.pt_col[tr])[:, None] + np.arange(3)[None, :]).ravel())
        vals.append(Jp.ravel())
        J = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                          shape=(len(res), self.ncols)).tocsr()
        return res, J

    def cost(self, q=None, t=None, X=None):
        r, _ = self.residuals(q, t, X, jac=False)
        return 0.5 * float(r @ r)

    def plus(self, delta):
        """x (+) delta in the tangent space: cameras via the Q9 manifold, t and X additive."""
        q, t, X = self.q.copy(), self.t.copy(), self.X.copy()
        ca = np.nonzero(self.cam_active)[0]
        dc = delta[:6 * self.nc].reshape(self.nc, 6)
        q[ca] = manifold_plus(self.q[ca], dc[:, :3])
        t[ca] = self.t[ca] + dc[:, 3:]
        tr = np.nonzero(self.tv)[0]
        X[tr] = self.X[tr] + delta[6 * self.nc:].reshape(self.npt, 3)
        return q, t, X

    def x_norm(self):
        ca = self.cam_active; tv = self.tv
        return float(np.sqrt((self.q[ca] ** 2).sum() + (self.t[ca] ** 2).sum() + (self.X[tv] ** 2).sum()))


def schur_system(J, r, D, nc):
    """Explicit reduced camera system of SURVEY.md A.3 (small problems only):
    S = B - E C^-1 E^T, rhs = -(g_c - E C^-1 g_p), with B,C including D^2."""
    A = (J.T @ J + sp.diags(D * D)).tocsc()
    g = J.T @ r
    nct = 6 * nc
    B = A[:nct, :nct].toarray(); E = A[:nct, nct:].toarray(); C = A[nct:, nct:].toarray()
    Cinv = np.linalg.inv(C)
    S = B - E @ Cinv @ E.T
    rhs = -(g[:nct] - E @ Cinv @ g[nct:])
    return S, rhs


def ceres_lm(prob: VisualProblem, max_iter=50, radius0=1e4, log=None, scaling=True, f_tol=1e-6, g_tol=1e-10, p_tol=1e-8):
    """Ceres 2.1 TrustRegionMinimizer + LevenbergMarquardtStrategy, restated.  Every cost is prob.cost() (with a loss,
    tests/visual_loss_oracle.py, 1/2 sum rho rather than 1/2 r.r of the corrected residuals).  The tolerances default to the
    library's (lvba_visual_default_opts)."""
    min_diag, max_diag = 1e-6, 1e32
    radius, nu = radius0, 2.0
    info = {"iters": 0, "accepted": 0, "trace": [], "term": "max_iter"}
    res, J = prob.residuals(jac=True)
    cost = prob.cost()
    info["cost0"] = cost
    if scaling:
        scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel()))
    else:
        scale = np.ones(prob.ncols)
    info["scale"] = scale
    Js = (J @ sp.diags(scale)).tocsr()
    grad = J.T @ res
    if np.abs(grad).max() <= g_tol:
        info["term"] = "gradient"; info["cost"] = cost
        return prob, info
    reuse_diag = False
    diag = None
    invalid = 0
    for it in range(1, max_iter + 1):
        info["iters"] = it
        if not reuse_diag:
            diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
        lm = np.sqrt(diag / radius)
        A = (Js.T @ Js + sp.diags(lm * lm)).tocsc()
        b = -(Js.T @ res)
        y = spla.spsolve(A, b)
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
        qn, tn, Xn = prob.plus(delta)
        cand = prob.cost(qn, tn, Xn)
        # Ceres: step_norm = ||x - candidate_x|| in the ambient space
        ca, tv = prob.cam_active, prob.tv
        step_norm = float(np.sqrt(((qn[ca] - prob.q[ca]) ** 2).sum() + ((tn[ca] - prob.t[ca]) ** 2).sum()
                                  + ((Xn[tv] - prob.X[tv]) ** 2).sum()))
        rho = (cost - cand) / model
        info["trace"].append(dict(it=it, cost=cost, cand=cand, rho=rho, radius=radius, step=step_norm, model=model))
        if log:
            log(info["trace"][-1])
        if step_norm <= p_tol * (prob.x_norm() + p_tol):
            info["term"] = "parameter"; break
        if abs(cost - cand) <= f_tol * cost:
            # Ceres 2.x tests FunctionToleranceReached() before IsStepSuccessful():
            # the minimiser returns with x (not the candidate) as the solution.
            info["term"] = "function"; break
        if rho > 1e-3:
            prob.q, prob.t, prob.X = qn, tn, Xn
            cost = cand
            info["accepted"] += 1
            res, J = prob.residuals(jac=True)
            Js = (J @ sp.diags(scale)).tocsr()
            grad = J.T @ res
            radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3))
            nu = 2.0
            reuse_diag = False
            if np.abs(grad).max() <= g_tol:
                info["term"] = "gradient"; break
        else:
            radius /= nu
            nu *= 2
            if radius < 1e-32:
                info["term"] = "radius"; break
    info["cost"] = cost
    info["radius"] = radius
    return prob, info


def single_step(prob: VisualProblem, radius=1e4, scaling=True, min_diag=1e-6, max_diag=1e32):
    """One linearisation + LM solve at the current state (what lvba_visual_step computes).
    Returns dict(cost, model, cam_step[M,6], pt_step[T,3], scale, S, rhs) — S/rhs only for small problems."""
    res, J = prob.residuals(jac=True)
    cost = prob.cost()
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.ncols)
    Js = (J @ sp.diags(scale)).tocsr()
    diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
    lm = np.sqrt(diag / radius)
    A = (Js.T @ Js + sp.diags(lm * lm)).tocsc()
    y = spla.spsolve(A, -(Js.T @ res))
    Jy = Js @ y
    model = -float(Jy @ (res + 0.5 * Jy))
    delta = y * scale
    cam_step = np.zeros((prob.M, 6)); pt_step = np.zeros((prob.T, 3))
    cam_step[prob.cam_active] = delta[:6 * prob.nc].reshape(prob.nc, 6)
    pt_step[prob.tv] = delta[6 * prob.nc:].reshape(prob.npt, 3)
    out = dict(cost=cost, model=model, cam_step=cam_step, pt_step=pt_step, scale=scale, y=y)
    if prob.ncols <= 6000:
        out["S"], out["rhs"] = schur_system(Js, res, lm, prob.nc)
        out["S_nodamp"] = out["S"] - np.diag((lm * lm)[:6 * prob.nc])
    return out
