"""numpy restatement of ITERATIVE_SCHUR for the visual LM (lvba_visual_opts::linear_solver, global-lvba_b200/csrc/visual_pcg.h):
Ceres' ConjugateGradientsSolver::Solve with the SCHUR_JACOBI preconditioner on the explicit reduced camera system, restated from
the ceres-solver 2.1.0 sources, and the LM of oracle/visual_oracle.py with that solve in place of the exact one.  Small problems
only (dense matrices).  oracle/visual_oracle.py is reused as it is."""
import sys
from pathlib import Path

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import visual_oracle as vo  # noqa: E402

SUCCESS, NO_CONVERGENCE, FAILURE = 0, 1, 2
RESET_PERIOD = 10


def _bad(v):
    return v == 0.0 or not np.isfinite(v)


def sym_lower(A):
    """A with every diagonal 6x6 block replaced by its lower triangle mirrored (how the device reads the diagonal blocks)."""
    A = np.array(A, np.float64)
    for r in range(A.shape[0] // 6):
        b = A[6 * r:6 * r + 6, 6 * r:6 * r + 6]
        A[6 * r:6 * r + 6, 6 * r:6 * r + 6] = np.tril(b) + np.tril(b, -1).T
    return A


def block_jacobi(A):
    """The inverses of the 6x6 diagonal blocks of A through their Cholesky factors, or None on a pivot that is not finite and > 0."""
    n = A.shape[0] // 6
    out = np.zeros((n, 6, 6))
    for r in range(n):
        b = A[6 * r:6 * r + 6, 6 * r:6 * r + 6]
        L = np.zeros((6, 6))
        for j in range(6):
            v = b[j, j] - L[j, :j] @ L[j, :j]
            if not (v > 0.0 and np.isfinite(v)):
                return None
            L[j, j] = np.sqrt(v)
            for i in range(j + 1, 6):
                L[i, j] = (b[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
        Li = np.linalg.solve(L, np.eye(6))
        out[r] = Li.T @ Li
    return out


def cg(A, b, eta=0.1, min_iter=0, max_iter=500):
    """ConjugateGradientsSolver::Solve with r_tolerance = -1 (LevenbergMarquardtStrategy), x0 = 0, and a FAILURE at once on any
    non-finite rho, beta, pq or alpha.  A: the damped symmetric system.  Returns (x, iterations, termination)."""
    A = np.asarray(A, np.float64); b = np.asarray(b, np.float64)
    n = b.size // 6
    x = np.zeros_like(b)
    if float(b @ b) == 0.0:
        return x, 0, SUCCESS
    Minv = block_jacobi(A)
    if Minv is None:
        return x, 0, FAILURE
    r = b.copy()
    p = np.zeros_like(b)
    rho, Q0 = 0.0, 0.0
    i = 0
    while True:
        i += 1
        z = np.einsum("rab,rb->ra", Minv, r.reshape(n, 6)).ravel()
        last_rho, rho = rho, float(r @ z)
        if _bad(rho):
            return x, i, FAILURE
        if i == 1:
            p = z
        else:
            beta = rho / last_rho
            if _bad(beta):
                return x, i, FAILURE
            p = z + beta * p
        q = A @ p
        pq = float(p @ q)
        if np.isnan(pq):
            return x, i, FAILURE
        if pq <= 0 or np.isinf(pq):
            return x, i, NO_CONVERGENCE
        alpha = rho / pq
        if not np.isfinite(alpha):
            return x, i, FAILURE
        x = x + alpha * p
        r = b - A @ x if i % RESET_PERIOD == 0 else r - alpha * q
        Q1 = -float(x @ (b + r))
        zeta = i * (Q1 - Q0) / Q1
        if zeta < eta and i >= min_iter:
            return x, i, SUCCESS
        Q0 = Q1
        if i >= max_iter:
            return x, i, NO_CONVERGENCE


def _solve(Js, res, lm, nc, eta, min_iter, max_iter):
    """y of the damped system through the Schur complement: cameras by cg, then the landmarks' back-substitution."""
    A = (Js.T @ Js + sp.diags(lm * lm)).toarray()
    g = Js.T @ res
    k = 6 * nc
    B, E, Cp = A[:k, :k], A[:k, k:], A[k:, k:]
    Ci = np.linalg.inv(Cp)
    S = B - E @ Ci @ E.T
    rhs = -(g[:k] - E @ Ci @ g[k:])
    yc, it, term = cg(sym_lower(S), rhs, eta, min_iter, max_iter) if k else (np.zeros(0), 0, SUCCESS)
    yp = Ci @ (-g[k:] - E.T @ yc)
    return np.concatenate([yc, yp]), it, term, S, rhs


def single_step(prob, radius=1e4, eta=0.1, min_iter=0, max_iter=500, scaling=True, min_diag=1e-6, max_diag=1e32):
    """visual_oracle.single_step with the camera system solved by cg: dict(cost, model, cam_step, pt_step, scale, y, S, rhs,
    dadd (the camera LM diagonal), iters, term)."""
    res, J = prob.residuals(jac=True)
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.ncols)
    Js = (J @ sp.diags(scale)).tocsr()
    diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
    lm = np.sqrt(diag / radius)
    y, it, term, S, rhs = _solve(Js, res, lm, prob.nc, eta, min_iter, max_iter)
    Jy = Js @ y
    delta = y * scale
    cam_step = np.zeros((prob.M, 6)); pt_step = np.zeros((prob.T, 3))
    cam_step[prob.cam_active] = delta[:6 * prob.nc].reshape(prob.nc, 6)
    pt_step[prob.tv] = delta[6 * prob.nc:].reshape(prob.npt, 3)
    return dict(cost=prob.cost(), model=-float(Jy @ (res + 0.5 * Jy)), cam_step=cam_step, pt_step=pt_step, scale=scale, y=y,
                S=S, rhs=rhs, dadd=(lm * lm)[:6 * prob.nc], iters=it, term=term)


def ceres_lm(prob, max_iter=50, radius0=1e4, eta=0.1, min_iter=0, max_linear_iter=500, scaling=True, f_tol=1e-6, g_tol=1e-10,
             p_tol=1e-8):
    """visual_oracle.ceres_lm with the camera system solved by cg.  A FAILURE is an invalid step, as a non-finite step or a
    model cost change <= 0 is.  info gains cg_iters (per solve) and cg_terms."""
    min_diag, max_diag = 1e-6, 1e32
    radius, nu = radius0, 2.0
    info = {"iters": 0, "accepted": 0, "term": "max_iter", "cg_iters": [], "cg_terms": []}
    res, J = prob.residuals(jac=True)
    cost = prob.cost()
    info["cost0"] = cost
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.ncols)
    Js = (J @ sp.diags(scale)).tocsr()
    if np.abs(J.T @ res).max() <= g_tol:
        info["term"] = "gradient"; info["cost"] = cost
        return prob, info
    invalid = 0
    for it in range(1, max_iter + 1):
        info["iters"] = it
        diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag)
        lm = np.sqrt(diag / radius)
        y, cgi, term, _, _ = _solve(Js, res, lm, prob.nc, eta, min_iter, max_linear_iter)
        info["cg_iters"].append(cgi); info["cg_terms"].append(term)
        Jy = Js @ y
        model = -float(Jy @ (res + 0.5 * Jy))
        if term == FAILURE or not np.all(np.isfinite(y)) or model <= 0:
            invalid += 1
            radius *= 0.5
            if invalid >= 5:
                info["term"] = "invalid_steps"; break
            continue
        invalid = 0
        qn, tn, Xn = prob.plus(y * scale)
        cand = prob.cost(qn, tn, Xn)
        ca, tv = prob.cam_active, prob.tv
        step_norm = float(np.sqrt(((qn[ca] - prob.q[ca]) ** 2).sum() + ((tn[ca] - prob.t[ca]) ** 2).sum()
                                  + ((Xn[tv] - prob.X[tv]) ** 2).sum()))
        rho = (cost - cand) / model
        if step_norm <= p_tol * (prob.x_norm() + p_tol):
            info["term"] = "parameter"; break
        if abs(cost - cand) <= f_tol * cost:
            info["term"] = "function"; break
        if rho > 1e-3:
            prob.q, prob.t, prob.X = qn, tn, Xn
            cost = cand
            info["accepted"] += 1
            res, J = prob.residuals(jac=True)
            Js = (J @ sp.diags(scale)).tocsr()
            radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3))
            nu = 2.0
            if np.abs(J.T @ res).max() <= g_tol:
                info["term"] = "gradient"; break
        else:
            radius /= nu
            nu *= 2
            if radius < 1e-32:
                info["term"] = "radius"; break
    info["cost"] = cost
    info["radius"] = radius
    return prob, info


__all__ = ["cg", "block_jacobi", "sym_lower", "single_step", "ceres_lm", "vo", "SUCCESS", "NO_CONVERGENCE", "FAILURE"]
