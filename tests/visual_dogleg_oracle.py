"""CPU oracle of the DOGLEG trust-region strategy of the visual LM (numpy, float64) on the problems of oracle/visual_oracle.py and
tests/visual_loss_oracle.py.  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restated from ceres-solver 2.1.0 (DoglegStrategy with TRADITIONAL_DOGLEG, TrustRegionMinimizer; not vendored, nothing to hold
it against here), the same rule global-lvba_b200/csrc/visual_dogleg.h states with its constants.  Everything is in the
Jacobi-scaled space of oracle/visual_oracle.ceres_lm: Js = J diag(scale), the scale fixed at iteration 0.  dogleg() records
per pass the case, alpha, mu, the radius, rho and whether the pass reused the linearisation.
"""
from __future__ import annotations

import warnings

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

MIN_MU, MAX_MU, MU_INCREASE = 1e-8, 1.0, 10.0
DECREASE, INCREASE = 0.25, 0.75
GAUSS_NEWTON, CAUCHY, INTERPOLATED = 1, 2, 3


def linearise(Js, res, min_diag=1e-6, max_diag=1e32):
    """D, g = Js^T res / D and alpha = |g|^2 / |Js (g / D)|^2 (ComputeGradient, ComputeCauchyPoint)."""
    D = np.sqrt(np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag))
    g = (Js.T @ res) / D
    Jg = Js @ (g / D)
    return D, g, float(g @ g) / float(Jg @ Jg)


def gauss_newton(Js, res, D, mu):
    """y of the damped solve (Js^T Js + mu D^2) y = -Js^T res (the LM step at radius 1 / mu), or None when it is not finite."""
    A = (Js.T @ Js + sp.diags(mu * D * D)).tocsc()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        y = spla.spsolve(A, -(Js.T @ res))
    return y if np.all(np.isfinite(y)) else None


def dogleg_step(g, GN, alpha, radius):
    """ComputeTraditionalDoglegStep: (case, s in the D-scaled space, |s|, beta)."""
    gnorm, gn_norm = float(np.linalg.norm(g)), float(np.linalg.norm(GN))
    if gn_norm <= radius:
        return GAUSS_NEWTON, GN.copy(), gn_norm, 0.0
    if gnorm * alpha >= radius:
        return CAUCHY, -(radius / gnorm) * g, radius, 0.0
    b_dot_a = -alpha * float(g @ GN)
    a2 = (alpha * gnorm) ** 2
    bma2 = a2 - 2.0 * b_dot_a + gn_norm ** 2
    c = b_dot_a - a2
    d = np.sqrt(c * c + bma2 * (radius * radius - a2))
    beta = (d - c) / bma2 if c <= 0 else (radius * radius - a2) / (d + c)
    s = (-alpha * (1.0 - beta)) * g + beta * GN
    return INTERPOLATED, s, float(np.linalg.norm(s)), float(beta)


def dogleg(prob, max_iter=50, radius0=1e4, scaling=True, f_tol=1e-6, g_tol=1e-10, p_tol=1e-8, min_radius=1e-32,
           min_rel_decrease=1e-3, min_diag=1e-6, max_diag=1e32):
    """The trust-region loop with the dogleg strategy; every cost is prob.cost().  Returns (prob, info): info has iters,
    accepted, builds (linearisations), reused, term, cost0, cost, radius and trace (one dict per pass)."""
    info = {"iters": 0, "accepted": 0, "builds": 0, "reused": 0, "trace": [], "term": "max_iter"}
    res, J = prob.residuals(jac=True)
    cost = prob.cost()
    info["cost0"] = cost
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.ncols)
    radius, mu, reuse, invalid = radius0, MIN_MU, False, 0
    D = g = GN = None
    alpha = 0.0
    for _ in range(max_iter):
        fresh = not reuse
        solved = not fresh
        if fresh:
            Js = (J @ sp.diags(scale)).tocsr()
            if mu < MAX_MU:
                info["builds"] += 1
                if np.abs(J.T @ res).max() <= g_tol:
                    info["term"] = "gradient"
                    break
            D, g, alpha = linearise(Js, res, min_diag, max_diag)
            while mu < MAX_MU:
                y = gauss_newton(Js, res, D, mu)
                if y is not None:
                    GN = D * y
                    solved = True
                    break
                mu *= MU_INCREASE
                if mu < MAX_MU:
                    info["builds"] += 1
        info["iters"] += 1
        if not fresh:
            info["reused"] += 1
        reuse = True
        rec = dict(it=info["iters"], reused=not fresh, mu=mu, radius=radius, cost=cost, case=0, alpha=alpha, rho=None,
                   accepted=False, valid=False)
        model = step_norm = cand = np.nan
        if solved:
            case, s, snorm, _ = dogleg_step(g, GN, alpha, radius)
            v = s / D
            Jv = Js @ v
            model = -float(Jv @ (res + 0.5 * Jv))
            qn, tn, Xn = prob.plus(v * scale)
            cand = prob.cost(qn, tn, Xn)
            ca, tv = prob.cam_active, prob.tv
            step_norm = float(np.sqrt(((qn[ca] - prob.q[ca]) ** 2).sum() + ((tn[ca] - prob.t[ca]) ** 2).sum()
                                      + ((Xn[tv] - prob.X[tv]) ** 2).sum()))
            rec.update(case=case, cand=cand, model=model, step=v, snorm=snorm, gnorm=float(np.linalg.norm(g)),
                       gn_norm=float(np.linalg.norm(GN)))
        info["trace"].append(rec)
        if not (solved and np.isfinite(model) and np.isfinite(step_norm) and model > 0):
            invalid += 1
            mu *= MU_INCREASE
            reuse = False
            if invalid >= 5:
                info["term"] = "invalid_steps"
                break
            continue
        rec["valid"] = True
        invalid = 0
        rho = (cost - cand) / model
        rec["rho"] = rho
        if step_norm <= p_tol * (prob.x_norm() + p_tol):
            info["term"] = "parameter"
            break
        if abs(cost - cand) <= f_tol * cost:
            info["term"] = "function"
            break
        if np.isfinite(cand) and rho > min_rel_decrease:
            rec["accepted"] = True
            prob.q, prob.t, prob.X = qn, tn, Xn
            cost = cand
            info["accepted"] += 1
            if rho < DECREASE:
                radius *= 0.5
            if rho > INCREASE:
                radius = max(radius, 3.0 * snorm)
            mu = max(MIN_MU, 2.0 * mu / MU_INCREASE)
            reuse = False
            res, J = prob.residuals(jac=True)
        else:
            radius *= 0.5
        if radius < min_radius:
            info["term"] = "radius"
            break
    info["cost"] = cost
    info["radius"] = radius
    info["mu"] = mu
    return prob, info
