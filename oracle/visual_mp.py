"""EXTENDED-PRECISION ORACLE of the visual reduced camera system (mpmath, 50 digits), one landmark at a time.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  The float64 oracle (visual_oracle.py) and the CUDA library round in float64; on
landmarks whose damped, Jacobi-scaled block C is ill-conditioned (far facades at grazing angles, short baselines, views from
one centre), on coordinates far from the origin and on the edges of the forward model, neither can tell which of them is the
more accurate.  This file restates the same lines in 50-digit arithmetic, independently of visual_oracle.py and of the
analytic Jacobians of global-lvba_b200/csrc/visual_math.h, on exactly the float64 inputs the library receives (obs_uv is
float32 and converts exactly; every float64 constant of the reference, 1e-8 and 1e-12, is taken as the double it is):

  observation    ReprojErrorWhitenedDistorted              include/utils.hpp:61-111 (QuaternionRotatePoint normalises q,
                                                           the z <= 1e-8 cut-off, Brown-Conrady distortion)
  its Jacobian   forward-mode derivatives (the Dual type below) through EigenQuaternionManifold::Plus on {w,x,y,z} memory
                 read as Eigen (x,y,z,w) (SURVEY.md Q9), at delta = 0: exp(delta) = (1; delta) to first order
  plane          PointPlaneErrorWhitened                   include/utils.hpp:133-139
  losses         ceres HuberLoss / CauchyLoss and the Corrector (rho'' <= 0: r, J times sqrt(rho')), as loss_eval /
                 obs_loss / plane_loss define them
  LM system      Jacobi scale 1/(1 + ||J[:, j]||), LM diagonal clamp(||J~[:, j]||^2, min, max) / radius, C and C^-1 (mp LU),
                 g_p, every camera pair's -W_i C^-1 W_j^T, U, rhs, cost; given a camera step, the back-substituted point
                 step and the model-cost change

Each landmark's results are rounded once to float64 at the end; the camera pairs of a long track are summed in exact integer
arithmetic from 200-bit fixed-point copies of the 50-digit W_i C^-1 and W_j (as balm_mp._pairs), and blocks that several
landmarks touch add their float64 contributions (an error of eps times the block's scale, far inside every bound).

Every result comes with an error scale ("hat"): its float64 rounding error over eps, to first order.  Each quantity is carried
as (V, E) = (|value|, error / eps) through the same sums and products (a product's E = E_a V_b + V_a E_b), so that a float64
evaluation is expected within C eps E.  The E of the inputs:
  J_c, J_X    amp_o |J|,  amp_o = max(1, (|RX|_1 + |t|_1) / z): cancellation in X_c = RX + t, relative to the depth
  r           |r| + pix_o + |dr/dX_c|_1 (|RX|_1 + |t|_1),  pix_o = (|f| |x_d|_terms + |c| + |u|) / sigma: the cancellation of
              u_pred - u, and the rounding of X_c carried through the projection
  J_plane     |J_p| + |n| 1e-12 (|n.X|_terms + |d|) / (root^3 sigma_p) (dJ_p/de = 1e-12 n / (root^3 sigma_p));
  r_plane     |r_p| + |e| (|n.X|_terms + |d|) / (root sigma_p)
  C^-1        |C^-1| C^ |C^-1| (first-order perturbation of an inverse)
and, with a loss, everything times sqrt(rho').  Bounds (constants calibrated in tests/test_visual_mp_oracle.py):
  |S_ij - S_ij,mp|_max <= C_S eps max S^_ij      |rhs_i - rhs_i,mp|_max <= C_RHS eps max rhs^_i
  |dp_l - dp_l,mp|_max <= C_PT eps max dp^_l     |cost - cost_mp| <= C_COST eps cost^,  |model - model_mp| <= C_COST eps model^
Also returned per landmark: kappa_l = ||C_l||_inf ||C_l^-1||_inf and max_o amp_o.
"""
from __future__ import annotations

import math

import numpy as np
from mpmath import mp, mpf
from mpmath.libmp import to_fixed

mp.dps = 50
EPS = float(np.finfo(np.float64).eps)
_FIX = 200
_DBL_MIN = mpf(float(np.finfo(np.float64).tiny))
_ZCUT = mpf(1e-8)           # utils.hpp:78, the double nearest 1e-8
_PLANE_EPS = mpf(1e-12)     # utils.hpp:138, the double nearest 1e-12
NONE, HUBER, CAUCHY = 0, 1, 2

# Bound constants, calibrated in tests/test_visual_mp_oracle.py (see its docstring)
C_S, C_RHS, C_PT, C_COST = 128.0, 0.5, 1.0, 0.5


class Dual:
    """v + sum_k d[k] e_k: forward-mode first derivatives over mpf, 9 seeds (rotation tangent, t, X)"""
    __slots__ = ("v", "d")

    def __init__(self, v, d=None):
        self.v = v
        self.d = d if d is not None else [mpf(0)] * 9

    def __add__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v + o.v, [a + b for a, b in zip(self.d, o.d)])
        return Dual(self.v + o, self.d)
    __radd__ = __add__

    def __sub__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v - o.v, [a - b for a, b in zip(self.d, o.d)])
        return Dual(self.v - o, self.d)

    def __rsub__(self, o):
        return Dual(o - self.v, [-a for a in self.d])

    def __neg__(self):
        return Dual(-self.v, [-a for a in self.d])

    def __mul__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v * o.v, [self.v * b + o.v * a for a, b in zip(self.d, o.d)])
        return Dual(self.v * o, [a * o for a in self.d])
    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, Dual):
            iv = 1 / o.v
            q = self.v * iv
            return Dual(q, [(a - q * b) * iv for a, b in zip(self.d, o.d)])
        return Dual(self.v / o, [a / o for a in self.d])

    def __rtruediv__(self, o):
        q = o / self.v
        return Dual(q, [-q * a / self.v for a in self.d])

    def sqrt(self):
        s = mp.sqrt(self.v)
        h = 1 / (2 * s)
        return Dual(s, [a * h for a in self.d])


def _seed(v, k):
    d = [mpf(0)] * 9
    d[k] = mpf(1)
    return Dual(mpf(v), d)


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def observation(q, t, X, uv, intr, sigma_px):
    """utils.hpp:61-111 for one observation at 50 digits: r [2] and J [2][9] (d/d(rotation tangent, t, X)) as mpf, and the
    hats' ingredients z, amp, pix"""
    m = [mpf(float(x)) for x in q]
    dth = [_seed(0, k) for k in range(3)]
    # EigenQuaternionManifold::Plus(x, delta) = Quaternion(exp delta) * Quaternion(x); Eigen reads memory m as (x,y,z,w)
    ew, ev = m[3], m[0:3]
    w_new = ew - (dth[0] * ev[0] + dth[1] * ev[1] + dth[2] * ev[2])
    cr = _cross(dth, ev)
    v_new = [dth[i] * ew + cr[i] + ev[i] for i in range(3)]
    mem = [v_new[0], v_new[1], v_new[2], w_new]
    # ceres::QuaternionRotatePoint reads memory as (w,x,y,z) and normalises
    inv = 1 / (mem[0] * mem[0] + mem[1] * mem[1] + mem[2] * mem[2] + mem[3] * mem[3]).sqrt()
    w, x, y, z = (c * inv for c in mem)
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
         [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
         [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    Xd = [_seed(X[i], 6 + i) for i in range(3)]
    td = [_seed(t[i], 3 + i) for i in range(3)]
    RX = [R[i][0] * Xd[0] + R[i][1] * Xd[1] + R[i][2] * Xd[2] for i in range(3)]
    Xc = [RX[i] + td[i] for i in range(3)]
    zc = Xc[2]
    amp_num = sum(abs(c.v) for c in RX) + sum(abs(mpf(float(c))) for c in t)
    zero = [[mpf(0)] * 9, [mpf(0)] * 9]
    if not (zc.v > _ZCUT):
        return dict(r=[mpf(0), mpf(0)], J=zero, z=zc.v, amp=mpf(1), pix=[mpf(0), mpf(0)], xc_err=mpf(0), valid=False)
    fx, fy, cx, cy, k1, k2, p1, p2 = (mpf(float(c)) for c in intr)
    xn, yn = Xc[0] / zc, Xc[1] / zc
    r2 = xn * xn + yn * yn
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    u, v = mpf(float(uv[0])), mpf(float(uv[1]))
    sg = mpf(float(sigma_px))
    res = [(fx * xd + cx - u) / sg, (fy * yd + cy - v) / sg]
    ax, ay, ar2 = abs(xn.v), abs(yn.v), r2.v
    arad = 1 + abs(k1) * ar2 + abs(k2) * ar2 * ar2
    xterm = ax * arad + 2 * abs(p1) * ax * ay + abs(p2) * (ar2 + 2 * ax * ax)
    yterm = ay * arad + abs(p1) * (ar2 + 2 * ay * ay) + 2 * abs(p2) * ax * ay
    pix = [(abs(fx) * xterm + abs(cx) + abs(u)) / sg, (abs(fy) * yterm + abs(cy) + abs(v)) / sg]
    return dict(r=[c.v for c in res], J=[res[0].d, res[1].d], z=zc.v, amp=max(mpf(1), amp_num / zc.v), pix=pix, xc_err=amp_num,
                valid=True)


def plane(pl, X, sigma_pl):
    """utils.hpp:133-139: r = sqrt(e^2 + 1e-12) / max(1e-9, sigma), e = -(n.X + d); J = dr/dX"""
    n = [mpf(float(c)) for c in pl[:3]]
    d = mpf(float(pl[3]))
    Xm = [mpf(float(c)) for c in X]
    s = mpf(max(1e-9, float(sigma_pl)))
    e = -(n[0] * Xm[0] + n[1] * Xm[1] + n[2] * Xm[2] + d)
    root = mp.sqrt(e * e + _PLANE_EPS)
    k = e / root / s
    terms = sum(abs(n[i] * Xm[i]) for i in range(3)) + abs(d)
    return dict(r=root / s, J=[-k * c for c in n], e=e, root=root, s=s, n=n, terms=terms)


def loss(kind, a, s):
    """rho(s), rho'(s) of ceres HuberLoss / CauchyLoss with scale a, b = a^2, at 50 digits (loss_eval)"""
    a = mpf(float(a))
    b = a * a
    if kind == HUBER and s > b:
        r = mp.sqrt(s)
        return 2 * a * r - b, max(_DBL_MIN, a / r)
    if kind == CAUCHY:
        u = 1 + s / b
        return b * mp.log(u), max(_DBL_MIN, 1 / u)
    return s, mpf(1)


# ------------------------------------------------------------------ pass 1: the forward model of every observation
def linearize(p):
    """observation() of every observation and plane() of every landmark with a valid plane, at the problem's state.
    Returns a list over the valid landmarks (caller order) of dict(track, cams, obs [...], plane)."""
    from oracle.visual_oracle import valid_tracks
    tv = np.nonzero(valid_tracks(np.asarray(p["plane_nd"], np.float64)))[0]
    op = np.asarray(p["obs_ptr"], np.int64)
    out = []
    for a in tv:
        X = p["X"][a]
        obs = []
        for s in range(op[a], op[a + 1]):
            c = int(p["obs_cam"][s])
            obs.append(observation(p["q"][c], p["t"][c], X, p["obs_uv"][s], p["intr"], p["sigma_px"]))
        out.append(dict(track=int(a), cams=np.asarray(p["obs_cam"][op[a]:op[a + 1]], np.int64), obs=obs,
                        plane=plane(p["plane_nd"][a], X, p["sigma_plane"])))
    return out


def _abs(A):
    return np.array([[float(abs(x)) for x in row] for row in A])


def _to_fix(x, scale):
    return to_fixed(mpf(x)._mpf_, scale)


def _pair_blocks(Y, W):
    """-Y_i W_j^T for every i > j: Y, W [R][6][3] of mpf -> {(i, j): 6x6 float64}, exact integer sums rounded once"""
    R = len(Y)
    if R < 2:
        return {}
    ymax = max(abs(x) for Yi in Y for row in Yi for x in row)
    wmax = max(abs(x) for Wi in W for row in Wi for x in row)
    if ymax == 0 or wmax == 0:
        return {(i, j): np.zeros((6, 6)) for i in range(R) for j in range(i)}
    sy = _FIX - int(mp.floor(mp.log(ymax, 2))); sw = _FIX - int(mp.floor(mp.log(wmax, 2)))
    Yi = np.array([[[_to_fix(x, sy) for x in row] for row in Yk] for Yk in Y], dtype=object).reshape(6 * R, 3)
    Wi = np.array([[[_to_fix(x, sw) for x in row] for row in Wk] for Wk in W], dtype=object).reshape(6 * R, 3)
    P = Yi @ Wi.T
    den = 1 << (sy + sw)
    out = {}
    for i in range(R):
        for j in range(i):
            blk = P[6 * i:6 * i + 6, 6 * j:6 * j + 6]
            out[(i, j)] = np.array([[-int(blk[a, b]) / den for b in range(6)] for a in range(6)])
    return out


# ------------------------------------------------------------------ pass 2: the LM system at one radius / scaling
def system(lin, cam_row, radius=1e4, scaling=True, loss_px=None, loss_pl=None, min_diag=1e-6, max_diag=1e32):
    """The reduced camera system's contributions of every landmark of `lin` (linearize()), for system rows cam_row [M]
    (-1: a constant camera).  loss_px / loss_pl: None or (kind, a).  Returns dict(n_rows, s_cam [n_rows, 6] (mp), lm [...])."""
    lpx = loss_px or (NONE, 1.0)
    lpl = loss_pl or (NONE, 1.0)
    n_rows = int(cam_row.max()) + 1 if len(cam_row) and cam_row.max() >= 0 else 0
    # corrector weights and the unscaled column norms of every camera (Jacobi scale, fixed at this state)
    colsq = [[mpf(0)] * 6 for _ in range(n_rows)]
    for L in lin:
        for k, o in enumerate(L["obs"]):
            rho, rho1 = loss(lpx[0], lpx[1], o["r"][0] ** 2 + o["r"][1] ** 2)
            o["w"], o["rho"] = mp.sqrt(rho1), rho
            row = cam_row[L["cams"][k]]
            if row >= 0:
                for c in range(6):
                    colsq[row][c] += rho1 * (o["J"][0][c] ** 2 + o["J"][1][c] ** 2)
        P = L["plane"]
        rho, rho1 = loss(lpl[0], lpl[1], P["r"] ** 2)
        P["w"], P["rho"] = mp.sqrt(rho1), rho
    one = mpf(1)
    s_cam = [[one / (1 + mp.sqrt(c)) if scaling else one for c in row] for row in colsq]
    lms = [_landmark(L, cam_row, s_cam, radius, scaling, min_diag, max_diag) for L in lin]
    return dict(n_rows=n_rows, s_cam=s_cam, lm=lms, cam_row=cam_row, radius=radius, min_diag=min_diag, max_diag=max_diag)


def _landmark(L, cam_row, s_cam, radius, scaling, min_diag, max_diag):
    obs, P = L["obs"], L["plane"]
    K = len(obs)
    one = mpf(1)
    # point columns: unscaled norms of the corrected Jacobian, the Jacobi scale, the scaled blocks
    Jp = [P["w"] * c for c in P["J"]]
    colsq = [Jp[m] ** 2 + sum(o["w"] ** 2 * (o["J"][0][6 + m] ** 2 + o["J"][1][6 + m] ** 2) for o in obs) for m in range(3)]
    s_pt = [one / (1 + mp.sqrt(c)) if scaling else one for c in colsq]
    rows = [int(cam_row[c]) for c in L["cams"]]
    JX, Jc, r = [], [], []
    for k, o in enumerate(obs):
        w = o["w"]
        JX.append([[w * o["J"][a][6 + m] * s_pt[m] for m in range(3)] for a in range(2)])
        Jc.append([[w * o["J"][a][c] * s_cam[rows[k]][c] for c in range(6)] if rows[k] >= 0 else [mpf(0)] * 6 for a in range(2)])
        r.append([w * o["r"][0], w * o["r"][1]])
    Jps = [Jp[m] * s_pt[m] for m in range(3)]
    rp = P["w"] * P["r"]
    C = [[sum(JX[k][a][i] * JX[k][a][j] for k in range(K) for a in range(2)) + Jps[i] * Jps[j] for j in range(3)] for i in range(3)]
    rad = mpf(float(radius))
    D = [min(max(C[i][i], mpf(float(min_diag))), mpf(float(max_diag))) / rad for i in range(3)]
    for i in range(3):
        C[i][i] += D[i]
    Ci = mp.inverse(mp.matrix(C))
    Ci = [[Ci[i, j] for j in range(3)] for i in range(3)]
    gp = [sum(JX[k][a][m] * r[k][a] for k in range(K) for a in range(2)) + Jps[m] * rp for m in range(3)]
    # per camera row of this landmark: U, W, g_c (several observations of one camera add up)
    urows = sorted(set(x for x in rows if x >= 0))
    ix = {x: i for i, x in enumerate(urows)}
    R = len(urows)
    U = [[[mpf(0)] * 6 for _ in range(6)] for _ in range(R)]
    csq = [[mpf(0)] * 6 for _ in range(R)]
    W = [[[mpf(0)] * 3 for _ in range(6)] for _ in range(R)]
    gc = [[mpf(0)] * 6 for _ in range(R)]
    for k in range(K):
        if rows[k] < 0:
            continue
        i = ix[rows[k]]
        for a in range(2):
            jc, jx = Jc[k][a], JX[k][a]
            for c in range(6):
                gc[i][c] += jc[c] * r[k][a]
                csq[i][c] += jc[c] * jc[c]
                for d in range(6):
                    U[i][c][d] += jc[c] * jc[d]
                for m in range(3):
                    W[i][c][m] += jc[c] * jx[m]
    Y = [[[sum(W[i][c][n] * Ci[n][m] for n in range(3)) for m in range(3)] for c in range(6)] for i in range(R)]
    wp = [sum(Ci[m][n] * gp[n] for n in range(3)) for m in range(3)]
    diag = [np.array([[float(U[i][c][d] - sum(Y[i][c][m] * W[i][d][m] for m in range(3))) for d in range(6)] for c in range(6)])
            for i in range(R)]
    rhs = [np.array([float(-(gc[i][c] - sum(W[i][c][m] * wp[m] for m in range(3)))) for c in range(6)]) for i in range(R)]
    off = _pair_blocks(Y, W)
    # error scales, first order: every quantity as (V, E) = (|value|, its float64 rounding error / eps), in float64
    w = [float(o["w"]) for o in obs]
    sp = np.array([float(c) for c in s_pt])
    VX = [_abs(JX[k]) for k in range(K)]
    EX = [float(obs[k]["amp"]) * VX[k] for k in range(K)]
    Vc = [_abs(Jc[k]) for k in range(K)]
    Ec = [float(obs[k]["amp"]) * Vc[k] for k in range(K)]
    Vr = [np.array([float(abs(x)) for x in r[k]]) for k in range(K)]
    Er = [w[k] * np.array([float(abs(obs[k]["r"][a]) + obs[k]["pix"][a] + obs[k]["xc_err"] * sum(abs(x) for x in obs[k]["J"][a][3:6]))
                           for a in range(2)]) for k in range(K)]
    n_abs = np.array([float(abs(c)) for c in P["n"]])
    Vp = np.array([float(abs(c)) for c in Jps])
    Ep = Vp + float(P["w"]) * sp * n_abs * float(P["terms"] * _PLANE_EPS / (P["root"] ** 3 * P["s"]))
    Vrp = float(abs(rp))
    Erp = float(P["w"]) * float(abs(P["r"]) + P["terms"] * abs(P["e"]) / (P["root"] * P["s"]))
    VC = _abs(C)
    EC = sum((EX[k].T @ VX[k] + VX[k].T @ EX[k] for k in range(K)), np.zeros((3, 3))) + 2 * np.outer(Ep, Vp) + VC
    VCi = _abs(Ci)
    ECi = VCi @ EC @ VCi
    Vgp = sum((VX[k].T @ Vr[k] for k in range(K)), np.zeros(3)) + Vp * Vrp
    Egp = sum((EX[k].T @ Vr[k] + VX[k].T @ Er[k] for k in range(K)), np.zeros(3)) + Ep * Vrp + Vp * Erp
    EU = np.zeros((R, 6, 6)); VU = np.zeros((R, 6, 6)); VW = np.zeros((R, 6, 3)); EW = np.zeros((R, 6, 3)); Egc = np.zeros((R, 6))
    for k in range(K):
        if rows[k] >= 0:
            i = ix[rows[k]]
            EU[i] += Ec[k].T @ Vc[k] + Vc[k].T @ Ec[k]
            VU[i] += Vc[k].T @ Vc[k]
            VW[i] += Vc[k].T @ VX[k]; EW[i] += Ec[k].T @ VX[k] + Vc[k].T @ EX[k]
            Egc[i] += Ec[k].T @ Vr[k] + Vc[k].T @ Er[k]
    VY = VW @ VCi
    EY = EW @ VCi + VW @ ECi
    pair_e = (np.einsum("icm,jdm->ijcd", EY, VW) + np.einsum("icm,jdm->ijcd", VY, EW)).max(axis=(2, 3)) if R else np.zeros((0, 0))
    Sh = {(urows[i], urows[j]): pair_e[i, j] + (EU[i].max() if i == j else 0.0) for i in range(R) for j in range(i + 1)}
    rhsh = [(Egc[i] + EY[i] @ Vgp + VY[i] @ Egp).max() for i in range(R)]
    # the term scale of every entry: sum |J_c|^T |J_c| (diagonal blocks) + sum_o |E_o| |C^-1| sum_o |E_o|^T
    Tp = np.einsum("icm,jdm->ijcd", VY, VW) if R else np.zeros((0, 0, 6, 6))
    Tl = {(urows[i], urows[j]): Tp[i, j] + (VU[i] if i == j else 0.0) for i in range(R) for j in range(i + 1)}
    S = {(urows[i], urows[i]): diag[i] for i in range(R)}
    for (i, j), blk in off.items():
        S[(urows[i], urows[j])] = blk
    cost = sum(o["rho"] for o in obs) + P["rho"]
    costh = sum(w[k] * float(abs(obs[k]["r"][a])) * Er[k][a] for k in range(K) for a in range(2)) \
        + float(P["w"] * abs(P["r"])) * Erp + float(abs(cost))
    kappa = float(VC.sum(1).max() * VCi.sum(1).max())
    return dict(track=L["track"], rows=rows, urows=urows, S=S, S_hat=Sh, T=Tl, csq=dict(zip(urows, csq)),
                csq_hat=dict(zip(urows, (np.diag(EU[i]) for i in range(R)))), rhs=dict(zip(urows, rhs)), rhs_hat=dict(zip(urows, rhsh)),
                cost=float(cost / 2), cost_hat=costh, kappa=kappa, amp=max([float(o["amp"]) for o in obs] + [1.0]),
                z_min=min([float(o["z"]) for o in obs]), e=float(P["e"]), C=np.array([[float(x) for x in row] for row in C]), s_pt=s_pt, Ci=Ci, gp=gp, JX=JX, r=r, Jps=Jps, rp=rp,
                V=dict(X=VX, r=Vr, p=Vp, rp=Vrp, Ci=VCi, gp=Vgp), E=dict(X=EX, r=Er, p=Ep, rp=Erp, Ci=ECi, gp=Egp),
                obs=obs, cams=L["cams"], wo=[o["w"] for o in obs])


# ------------------------------------------------------------------ pass 3: back-substitution of a camera step
def backsub(sysm, cam_step):
    """Given the camera step cam_step [M, 6] (unscaled, delta = s_c y_c; constant cameras ignored): every landmark's point step
    dp = s_p o y_p, y_p = -C^-1 (g_p + sum_o J~_X^T J_c delta_c), and its model-cost change -sum J~y (r~ + J~y / 2), with
    error scales.  Returns (dp [Tv, 3], dp_hat [Tv], model, model_hat)."""
    dps, dph, model, modelh = [], [], mpf(0), 0.0
    for L in sysm["lm"]:
        K = len(L["obs"])
        V, E = L["V"], L["E"]
        jc, Vjc, Ejc = [], [], []
        for k in range(K):
            o = L["obs"][k]
            row, cam, w = L["rows"][k], L["cams"][k], L["wo"][k]
            if row < 0:
                jc.append([mpf(0), mpf(0)]); Vjc.append(np.zeros(2)); Ejc.append(np.zeros(2))
                continue
            dc = [mpf(float(x)) for x in cam_step[cam]]
            jc.append([w * sum(o["J"][a][c] * dc[c] for c in range(6)) for a in range(2)])
            Vjc.append(float(w) * _abs(o["J"])[:, :6] @ np.abs(cam_step[cam]))
            Ejc.append(float(o["amp"]) * Vjc[-1])
        b = [L["gp"][m] + sum(L["JX"][k][a][m] * jc[k][a] for k in range(K) for a in range(2)) for m in range(3)]
        y = [-sum(L["Ci"][m][n] * b[n] for n in range(3)) for m in range(3)]
        dp = [L["s_pt"][m] * y[m] for m in range(3)]
        Vb = V["gp"] + sum((V["X"][k].T @ Vjc[k] for k in range(K)), np.zeros(3))
        Eb = E["gp"] + sum((E["X"][k].T @ Vjc[k] + V["X"][k].T @ Ejc[k] for k in range(K)), np.zeros(3))
        Vy = V["Ci"] @ Vb
        Ey = E["Ci"] @ Vb + V["Ci"] @ Eb + Vy
        sp = np.array([float(c) for c in L["s_pt"]])
        m_l = mpf(0); mh = 0.0
        for k in range(K):
            for a in range(2):
                jy = jc[k][a] + sum(L["JX"][k][a][m] * y[m] for m in range(3))
                m_l -= jy * (L["r"][k][a] + jy / 2)
                Vjy = Vjc[k][a] + V["X"][k][a] @ Vy
                Ejy = Ejc[k][a] + E["X"][k][a] @ Vy + V["X"][k][a] @ Ey
                mh += Ejy * (V["r"][k][a] + Vjy) + Vjy * E["r"][k][a]
        jy = sum(L["Jps"][m] * y[m] for m in range(3))
        m_l -= jy * (L["rp"] + jy / 2)
        Vjy = V["p"] @ Vy
        Ejy = E["p"] @ Vy + V["p"] @ Ey
        mh += Ejy * (V["rp"] + Vjy) + Vjy * E["rp"]
        model += m_l; modelh += mh
        dps.append([float(x) for x in dp]); dph.append(float((sp * Ey).max()))
    return np.array(dps).reshape(-1, 3), np.array(dph), float(model), modelh


# ------------------------------------------------------------------ a whole problem
def assemble(sysm, lms=None):
    """S {(i, j): 6x6} for i >= j (the lower envelope, scaled, before the camera LM diagonal, as lvba_visual_get_system
    returns it), rhs [n_rows, 6], the cost, and their scales, summed over the landmarks `lms` (default: all)"""
    lms = sysm["lm"] if lms is None else lms
    n = sysm["n_rows"]
    S, Sh = {}, {}
    rhs = np.zeros((n, 6)); rhsh = np.zeros(n); touched = np.zeros(n, bool)
    for L in lms:
        for k, b in L["S"].items():
            S[k] = S.get(k, 0.0) + b
            Sh[k] = Sh.get(k, 0.0) + L["S_hat"][k]
        for i, v in L["rhs"].items():
            rhs[i] += v; rhsh[i] += L["rhs_hat"][i]; touched[i] = True
    return dict(S=S, S_hat=Sh, rhs=rhs, rhs_hat=rhsh, rows=touched, cost=math.fsum(L["cost"] for L in lms),
                cost_hat=math.fsum(L["cost_hat"] for L in lms))


def damped(sysm, lms=None):
    """The damped operator A = S + diag(dadd) that ITERATIVE_SCHUR applies, summed over the landmarks `lms` (default: all), as
    full 6x6 blocks in both triangles (A_ji = A_ij^T): dadd = clamp(sum J~_c^2, min_diag, max_diag) / radius per camera column
    (visual_cam_diag_kernel), each block with its error scale, and T, the sum of the absolute values of the terms of every
    entry (sum |J_c|^T |J_c| on the diagonal blocks, plus dadd, plus sum_l |W_il| |C_l^-1| |W_jl|^T, |W_il| = sum_o |E_o|).
    Returns dict(S, S_hat, T) keyed (i, j) over both triangles, so that ratios(damped(...), A_block) applies, and dadd,
    dadd_hat [n_rows, 6]."""
    lms = sysm["lm"] if lms is None else lms
    ref = assemble(sysm, lms)
    n = sysm["n_rows"]
    csq = {}; csqh = np.zeros((n, 6))
    T = {}
    for L in lms:
        for i, v in L["csq"].items():
            c = csq.setdefault(i, [mpf(0)] * 6)
            for a in range(6):
                c[a] += v[a]
            csqh[i] += L["csq_hat"][i]
        for k, b in L["T"].items():
            T[k] = T.get(k, 0.0) + b
    rad, lo, hi = mpf(float(sysm["radius"])), mpf(float(sysm["min_diag"])), mpf(float(sysm["max_diag"]))
    dadd = np.zeros((n, 6)); daddh = np.zeros((n, 6))
    for i, c in csq.items():
        for a in range(6):
            dadd[i, a] = float(min(max(c[a], lo), hi) / rad)
            daddh[i, a] = (csqh[i, a] / float(rad) if lo < c[a] < hi else 0.0) + dadd[i, a]
    A, Ah, At = {}, {}, {}
    for (i, j), b in ref["S"].items():
        if i == j:
            A[(i, i)] = b + np.diag(dadd[i])
            Ah[(i, i)] = ref["S_hat"][(i, i)] + daddh[i].max()
            At[(i, i)] = T[(i, i)] + np.diag(dadd[i])
        else:
            A[(i, j)], A[(j, i)] = b, b.T
            Ah[(i, j)] = Ah[(j, i)] = ref["S_hat"][(i, j)]
            At[(i, j)], At[(j, i)] = T[(i, j)], T[(i, j)].T
    return dict(S=A, S_hat=Ah, T=At, dadd=dadd, dadd_hat=daddh)


def dense(blocks, n):
    """{(i, j): 6x6} -> the [6n, 6n] matrix"""
    M = np.zeros((6 * n, 6 * n))
    for (i, j), b in blocks.items():
        M[6 * i:6 * i + 6, 6 * j:6 * j + 6] = b
    return M


# The symmetry bound of an operator applied through the Jacobian blocks in double-double (visual_implicit.h, vimp::DD): each
# entry is the exact operator of the rounded records, which is symmetric, rounded once, so that
#   |A_ij - A_ji| <= ulp(max(|A_ij|, |A_ji|)) + C_SYM eps^2 T_ij
# with T_ij the sum of the absolute values of the entry's terms (damped(), term_scale_f64()).  A product rounded in plain
# double misses it by the cancellation in its terms, ~eps T_ij.
C_SYM = 64.0


def symmetry_ratio(A, T):
    """max over the off-diagonal entries of |A_ij - A_ji| / (ulp(max(|A_ij|, |A_ji|)) + C_SYM eps^2 T_ij), for the dense
    operator A and its term scale T (a ratio <= 1 meets the bound); NaN anywhere gives NaN"""
    d = np.abs(A - A.T)
    bound = np.spacing(np.maximum(np.abs(A), np.abs(A.T))) + C_SYM * EPS * EPS * np.maximum(T, T.T)
    np.fill_diagonal(d, 0.0)
    return float(np.max(d / bound)) if d.size else 0.0


def term_scale_f64(prob, radius=1e4, scaling=True, min_diag=1e-6, max_diag=1e32):
    """T of damped() in float64, from the absolute values of the float64 oracle's Jacobian (visual_oracle.VisualProblem or
    visual_loss_oracle.RobustProblem: corrected with a loss): |J_c|^T |J_c| + diag(dadd) + |E| |C^-1| |E|^T, with E per
    observation as |J_c|^T |J_X| and C the damped point blocks.  For scenes too large for the 50-digit linearisation; T is
    needed to its order of magnitude only.  Returns the dense [6 nc, 6 nc] matrix."""
    import scipy.sparse as sp
    res, J = prob.residuals(jac=True)
    scale = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(0)).ravel())) if scaling else np.ones(prob.ncols)
    Js = (J @ sp.diags(scale)).tocsc()
    nc6 = 6 * prob.nc
    diag = np.clip(np.asarray(Js.multiply(Js).sum(0)).ravel(), min_diag, max_diag) / radius
    Jc, Jp = abs(Js[:, :nc6]), Js[:, nc6:]
    CC = (Jp.T @ Jp).tocoo()                                  # block diagonal: a residual row touches one landmark
    Cb = np.zeros((prob.npt, 3, 3))
    np.add.at(Cb, (CC.row // 3, CC.row % 3, CC.col % 3), CC.data)
    Cb += np.einsum("la,ab->lab", diag[nc6:].reshape(-1, 3), np.eye(3))
    Ci = np.abs(np.linalg.inv(Cb)) if prob.npt else Cb
    E = (Jc.T @ abs(Jp)).tocsc()
    Cib = sp.block_diag(list(Ci), format="csc")
    T = (Jc.T @ Jc).toarray() + np.diag(diag[:nc6]) + (E @ Cib @ E.T).toarray()
    return T


def ratios(ref, S_block=None, rhs=None, cost=None):
    """|dev - mp| / (eps scale) of the worst S block, the worst rhs row and the cost, for device results S_block(i, j) -> the
    6x6 block (i >= j), rhs [n_rows, 6] and cost (each None to skip: ratio 0)"""
    rs = 0.0
    if S_block is not None:
        rs = max((ratio(np.abs(S_block(i, j) - b).max(), ref["S_hat"][(i, j)]) for (i, j), b in ref["S"].items()), default=0.0)
    rr = 0.0
    if rhs is not None and ref["rows"].any():
        on = ref["rows"]
        rr = max(ratio(e, h) for e, h in zip(np.abs(rhs[on] - ref["rhs"][on]).max(1), ref["rhs_hat"][on]))
    rc = 0.0 if cost is None else ratio(abs(cost - ref["cost"]), ref["cost_hat"])
    return float(rs), float(rr), float(rc)


def ratio(err, scale):
    """err / (eps scale); a result with no terms (scale 0, e.g. a camera seen only beyond the z cut-off) must be exact.  NaN
    in err gives NaN."""
    if scale > 0:
        return err / (EPS * scale)
    return 0.0 if err == 0 else (math.inf if err == err else math.nan)
