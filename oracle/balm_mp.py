"""EXTENDED-PRECISION ORACLE of the BALM2 plane factor (mpmath, 50 digits), one voxel at a time.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  The float64 oracle (lidar_oracle.py) and the CUDA library round in float64; on
voxels whose two smallest eigenvalues are close, or whose covariance is a small difference of large terms, neither can
tell which of them is the more accurate.  This file restates the same lines in 50-digit arithmetic, independently of
lidar_oracle.py, on exactly the float64 inputs the library receives (clusters, poses, pose_idx are converted exactly):

  transform        PointCluster::transform + operator+=   include/BALM/tools.hpp:441-456
  voxel            VOX_HESS::acc_evaluate2, one voxel       include/BALM/bavoxel.hpp:68-174
  lambda0          evaluate_only_residual, one voxel        include/BALM/bavoxel.hpp:176-203
  so3_exp/retract  Exp and the LM retraction                include/BALM/tools.hpp:62-77, bavoxel.hpp:722-727

The eigen system is mpmath.eigsy, eigenvalues ascending, every eigenvector's largest component made positive (every use
is even in u, SURVEY.md Q6; `flip` negates them all to show that).  Clusters may carry a non-integral N (weighted points):
the covariance divides by the sum of N, the Hessian by its integer part (`int NN = sig.N`, bavoxel.hpp:101), as the
library and lidar_oracle.py do.

Each voxel's results are rounded once to float64 at the end.  The slot-pair blocks H_ij = F_i D F_j^T are summed in exact
integer arithmetic from 200-bit fixed-point copies of the 50-digit per-slot factors F_i (see _pairs), which keeps voxels
seen from 160 poses to about a second.

device_branch restates, in float64, the tests by which global-lvba_b200/csrc/common.cuh picks a solver for a covariance
(eig3_sym_plane / sym3_smallest_eigenvalue: Newton fast path or Jacobi fallback), so that a test can show which branches a
family of voxels reaches.
"""
from __future__ import annotations

import math

import numpy as np
from mpmath import mp, mpf
from mpmath.libmp import to_fixed

mp.dps = 50
EPS = float(np.finfo(np.float64).eps)
_FIX = 200                     # bits of the fixed-point pair products

# Bound constants (see tests/test_balm_mp_oracle.py for their calibration against the float64 oracle and the host-compiled
# big-voxel passes): |res - res_mp| <= C_R sum_v delta_v, |g_i - g_i,mp| <= C_G g_scale_i, |H_ij - H_ij,mp| <= C_H H_scale_ij
C_R, C_G, C_H = 1.0, 8.0, 16.0


# ------------------------------------------------------------------ 3-vector / 3x3 helpers on lists of mpf
def _mv(A, x):
    return [A[i][0] * x[0] + A[i][1] * x[1] + A[i][2] * x[2] for i in range(3)]


def _mtv(A, x):
    return [A[0][i] * x[0] + A[1][i] * x[1] + A[2][i] * x[2] for i in range(3)]


def _mm(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def _hat(v):
    """tools.hpp:105-112"""
    z = mpf(0)
    return [[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]]


def _dot(a, b):
    return sum((x * y for x, y in zip(a, b)), mpf(0))


def _unpack(rec, pose):
    c = [mpf(float(x)) for x in rec]
    P = [[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]]
    R = [[mpf(pose[3 * i + j]) for j in range(3)] for i in range(3)]
    t = [mpf(pose[9 + i]) for i in range(3)]
    return P, c[6:9], c[9], R, t


def transform(P, v, n, R, t):
    """tools.hpp:450-456: v' = R v + N p;  P' = R P R^T + R v p^T + p (R v)^T + N p p^T"""
    Rv = _mv(R, v)
    RP = _mm(R, P)
    Pt = [[RP[i][0] * R[j][0] + RP[i][1] * R[j][1] + RP[i][2] * R[j][2] + Rv[i] * t[j] + t[i] * Rv[j] + n * t[i] * t[j]
           for j in range(3)] for i in range(3)]
    return Pt, [Rv[i] + n * t[i] for i in range(3)]


def _merged(slots):
    """tools.hpp:441-447 (operator+=) over the transformed slots; bavoxel.hpp:97-98: vBar, P/N - vBar vBar^T"""
    Ps = [[mpf(0)] * 3 for _ in range(3)]; vs = [mpf(0)] * 3; Ns = mpf(0)
    for P, v, n, R, t in slots:
        Pt, vt = transform(P, v, n, R, t)
        for i in range(3):
            vs[i] += vt[i]
            for j in range(3):
                Ps[i][j] += Pt[i][j]
        Ns += n
    vbar = [x / Ns for x in vs]
    C = [[Ps[i][j] / Ns - vbar[i] * vbar[j] for j in range(3)] for i in range(3)]
    return C, vbar, Ns


def eig(C, flip=False):
    """SelfAdjointEigenSolver (bavoxel.hpp:98): ascending eigenvalues, eigenvectors u[m] with a fixed sign"""
    E, Q = mp.eigsy(mp.matrix(C))
    order = sorted(range(3), key=lambda k: E[k])
    lam = [E[k] for k in order]
    u = []
    for k in order:
        col = [Q[i, k] for i in range(3)]
        big = max(range(3), key=lambda i: abs(col[i]))
        s = -1 if (col[big] < 0) != flip else 1
        u.append([s * x for x in col])
    return lam, u


def so3_exp(w):
    """tools.hpp:62-77 in 50 digits (identity below 1e-11)"""
    th = mp.sqrt(_dot(w, w))
    if th < mpf("1e-11"):
        return [[mpf(int(i == j)) for j in range(3)] for i in range(3)]
    K = _hat([x / th for x in w])
    KK = _mm(K, K)
    s, c = mp.sin(th), mp.cos(th)
    return [[int(i == j) + s * K[i][j] + (1 - c) * KK[i][j] for j in range(3)] for i in range(3)]


def retract(pose, dx):
    """bavoxel.hpp:722-727 for one pose: R <- R Exp(dx[:3]), p <- p + dx[3:], returned as 12 mpf"""
    R = [[mpf(pose[3 * i + j]) for j in range(3)] for i in range(3)]
    Rn = _mm(R, so3_exp(dx[:3]))
    return [Rn[i][j] for i in range(3) for j in range(3)] + [mpf(pose[9 + i]) + dx[3 + i] for i in range(3)]


def lambda0(clusters, poses):
    """evaluate_only_residual for one voxel (bavoxel.hpp:176-203): clusters [K,10], poses [K,12] (float64 or mpf)"""
    C, _, _ = _merged([_unpack(clusters[k], poses[k]) for k in range(len(clusters))])
    E = mp.eigsy(mp.matrix(C), eigvals_only=True)
    return min(E[k] for k in range(3))


def _to_fix(x, scale):
    return to_fixed(mpf(x)._mpf_, scale)


def _pairs(F, D):
    """every H_ij = F_i D F_j^T, i < j, of one voxel: F [K][6][3] and D [3] in 50 digits -> float64 [K(K-1)/2, 6, 6]"""
    K = len(F)
    fmax = max(abs(x) for Fi in F for row in Fi for x in row)
    dmax = max(abs(d) for d in D)
    if K < 2 or fmax == 0:
        return np.zeros((K * (K - 1) // 2, 6, 6))
    sf = _FIX - int(mp.floor(mp.log(fmax, 2))); sd = _FIX - int(mp.floor(mp.log(dmax, 2)))
    Fi = np.array([[[_to_fix(x, sf) for x in row] for row in Fk] for Fk in F], dtype=object).reshape(6 * K, 3)
    Di = np.array([_to_fix(d, sd) for d in D], dtype=object)
    Hall = Fi @ (Fi * Di[None, :]).T                     # exact, scale 2^(2 sf + sd)
    den = 1 << (2 * sf + sd)
    ii, jj = np.triu_indices(K, 1)
    out = np.empty((len(ii), 6, 6))
    for p, (i, j) in enumerate(zip(ii, jj)):
        blk = Hall[6 * i:6 * i + 6, 6 * j:6 * j + 6]
        out[p] = [[int(blk[a, b]) / den for b in range(6)] for a in range(6)]   # int / int: correctly rounded
    return out


def voxel(clusters, poses, flip=False):
    """acc_evaluate2 (bavoxel.hpp:68-174) for ONE voxel: clusters [K,10] body-frame records of its slots in ascending pose
    order, poses [K,12] the poses of those slots.  Returns a dict of float64 results:
      res        lambda_0                          (:174)
      g [K,6]    Auk_i^T u_k per slot              (:141-142)
      Hd [K,6,6] diagonal blocks H_ii              (:143-149)
      Hp [K(K-1)/2,6,6] H_ij for i < j in np.triu_indices order (:151-167)
    and what the error bounds need: lam [3], gap = lambda_1 - lambda_0, cmax = max|C|, vbar = |vBar|, N, amax = max|Auk|,
    hmax = the largest entry of the voxel's blocks and tmax = the largest entry of the terms summed into them.  A float64
    evaluation rounds those terms, not the sum: a voxel seen from one pose has g = H = 0 exactly (the pose moves the whole
    voxel rigidly) while every term is of order |Auk|^2 / gap, so the Hessian bound scales with tmax.  The bound is first
    order in the covariance rounding and assumes points within sensor range of their poses: a voxel 1 km from the poses
    that see it has body-frame moments ~1e6 m^2, whose rounding the float64 oracle itself carries ~100x past it."""
    K = len(clusters)
    slots = [_unpack(clusters[k], poses[k]) for k in range(K)]
    C, vbar, Ns = _merged(slots)
    lam, u = eig(C, flip)
    NN = mpf(int(mp.floor(Ns)))                          # int NN = sig.N (:101)
    uk = u[0]
    w1, w2 = 2 / (lam[0] - lam[1]), 2 / (lam[0] - lam[2])   # umumT weights (:107-110)
    g = np.empty((K, 6)); Hd = np.empty((K, 6, 6)); F = []
    amax = tmax = mpf(0)
    for i, (P, v, n, R, t) in enumerate(slots):          # :112-149
        vihat = _hat(v)
        RiTuk = _mtv(R, uk)
        RiTukhat = _hat(RiTuk)
        PiRiTuk = _mv(P, RiTuk)
        viRiTuk = _mv(vihat, RiTuk)
        ti_v = [t[a] - vbar[a] for a in range(3)]
        ukTti_v = _dot(uk, ti_v)
        hP = _hat(PiRiTuk)
        combo1 = [[hP[a][b] + vihat[a][b] * ukTti_v for b in range(3)] for a in range(3)]
        Rv = _mv(R, v)
        combo2 = [Rv[a] + n * ti_v[a] for a in range(3)]
        RP = _mm(R, P)
        L = _mm([[RP[a][b] + ti_v[a] * v[b] for b in range(3)] for a in range(3)], RiTukhat)
        Rc1 = _mm(R, combo1)
        c2uk = _dot(combo2, uk)
        A = [[(L[a][b] - Rc1[a][b]) / NN for b in range(3)]
             + [(combo2[a] * uk[b] + (c2uk if a == b else 0)) / NN for b in range(3)] for a in range(3)]   # Auk, 3 x 6
        amax = max([amax] + [abs(x) for row in A for x in row])
        jjt = [A[0][c] * uk[0] + A[1][c] * uk[1] + A[2][c] * uk[2] for c in range(6)]
        a1 = [A[0][c] * u[1][0] + A[1][c] * u[1][1] + A[2][c] * u[1][2] for c in range(6)]
        a2 = [A[0][c] * u[2][0] + A[1][c] * u[2][1] + A[2][c] * u[2][2] for c in range(6)]
        H = [[w1 * a1[r] * a1[c] + w2 * a2[r] * a2[c] for c in range(6)] for r in range(6)]   # Auk^T umumT Auk
        M = _mm([[combo1[a][b] - x for b, x in enumerate(row)] for a, row in enumerate(_mm(RiTukhat, P))], RiTukhat)
        hj = _hat(jjt[:3])
        for a in range(3):
            for b in range(3):
                H[a][b] += 2 / NN * M[a][b] - 2 / NN / NN * viRiTuk[a] * viRiTuk[b] - hj[a][b] / 2
                HRt = 2 / NN * (1 - n / NN) * viRiTuk[a] * uk[b]
                H[a][3 + b] += HRt
                H[3 + b][a] += HRt
                H[3 + a][3 + b] += 2 / NN * (n - n * n / NN) * uk[a] * uk[b]
        b = viRiTuk + [n * x for x in uk]
        tmax = max([tmax, abs(w1) * max(abs(x) for x in a1) ** 2, abs(w2) * max(abs(x) for x in a2) ** 2,
                    2 / NN / NN * max(abs(x) for x in b) ** 2, 2 / NN * max(abs(x) for row in M for x in row),
                    max(abs(x) for x in jjt[:3]) / 2, 2 / NN * abs(1 - n / NN) * max(abs(x) for x in viRiTuk),
                    2 / NN * abs(n - n * n / NN)])
        g[i] = [float(x) for x in jjt]
        Hd[i] = [[float(x) for x in row] for row in H]
        # H_ij (i < j, :151-167) = w1 a1_i a1_j^T + w2 a2_i a2_j^T - 2/NN^2 b_i b_j^T with b = (viRiTuk, n u_k)
        F.append([[a1[r], a2[r], b[r]] for r in range(6)])
    Hp = _pairs(F, [w1, w2, -2 / NN / NN])
    hmax = max(np.abs(Hd).max(), np.abs(Hp).max() if len(Hp) else 0.0)
    return dict(res=float(lam[0]), g=g, Hd=Hd, Hp=Hp, lam=np.array([float(x) for x in lam]),
                gap=float(lam[1] - lam[0]), cmax=float(max(abs(x) for row in C for x in row)),
                vbar=float(mp.sqrt(_dot(vbar, vbar))), N=float(Ns), amax=float(amax), hmax=float(hmax), tmax=float(tmax))


# ------------------------------------------------------------------ a whole problem
def evaluate(vox_ptr, pose_idx, clusters, poses, flip=False):
    """voxel() for every voxel of a CSR problem; returns the list of per-voxel dicts"""
    out = []
    for a in range(len(vox_ptr) - 1):
        s = slice(int(vox_ptr[a]), int(vox_ptr[a + 1]))
        out.append(voxel(clusters[s], poses[pose_idx[s]], flip))
    return out


def kappa(r):
    """first-order conditioning of one voxel: (|C| + |vBar|^2) / (lambda_1 - lambda_0)"""
    return (r["cmax"] + r["vbar"] ** 2) / r["gap"]


def delta(r):
    """absolute rounding of the float64 covariance: 8 eps (|C| + |vBar|^2)"""
    return 8.0 * EPS * (r["cmax"] + r["vbar"] ** 2)


def assemble(vox_ptr, pose_idx, refs, n_poses):
    """The problem's residual, g and upper blocks summed over the voxels, and the per-entry bound scales:
      res, res_scale = sum_v delta_v
      g [W,6],  g_scale [W]  = eps sum_{v at pose i} kappa_v max|Auk_v|
      H {(i,j): 6x6} for i <= j,  H_scale {(i,j)} = eps sum_{v at i and j} kappa_v tmax_v
    where kappa_v = (|C| + |vBar|^2) / (lambda_1 - lambda_0): the covariance is rounded by ~eps (|C| + |vBar|^2), which moves
    the eigenvectors by that over the gap, and umumT scales with 1 / gap."""
    g = np.zeros((n_poses, 6)); gs = np.zeros(n_poses)
    H, Hs = {}, {}
    res = math.fsum(r["res"] for r in refs)
    res_scale = math.fsum(delta(r) for r in refs)
    for a, r in enumerate(refs):
        pi = pose_idx[int(vox_ptr[a]):int(vox_ptr[a + 1])]
        kap = kappa(r)
        g[pi] += r["g"]; gs[pi] += EPS * kap * r["amax"]
        for k, p in enumerate(pi):
            H[(p, p)] = H.get((p, p), 0.0) + r["Hd"][k]
            Hs[(p, p)] = Hs.get((p, p), 0.0) + EPS * kap * r["tmax"]
        for q, (i, j) in enumerate(zip(*np.triu_indices(len(pi), 1))):
            key = (pi[i], pi[j])
            H[key] = H.get(key, 0.0) + r["Hp"][q]
            Hs[key] = Hs.get(key, 0.0) + EPS * kap * r["tmax"]
    return dict(res=res, res_scale=res_scale, g=g, g_scale=gs, H=H, H_scale=Hs)


def ratios(ref, res, g, upper):
    """|dev - mp| / bound scale of a problem's residual, its worst g row and its worst H block, for device results res,
    g [W,6] and upper(i, j) -> the 6 x 6 block (i, j), i <= j"""
    rr = abs(res - ref["res"]) / ref["res_scale"]
    on = ref["g_scale"] > 0
    rg = (np.abs(g - ref["g"]).max(1)[on] / ref["g_scale"][on]).max(initial=0.0)
    rh = max((np.abs(upper(i, j) - blk).max() / ref["H_scale"][(i, j)] for (i, j), blk in ref["H"].items()), default=0.0)
    return float(rr), float(rg), float(rh)


# ------------------------------------------------------------------ the device's solver choice, restated in float64
def covariance64(clusters, poses):
    """the merged covariance in float64, in the order the device forms it (lidar.cuh transform_cluster, voxel_cov)"""
    acc = np.zeros(10)
    for rec, ps in zip(clusters, poses):
        R = ps[:9].reshape(3, 3); t = ps[9:12]
        P = np.array([[rec[0], rec[1], rec[2]], [rec[1], rec[3], rec[4]], [rec[2], rec[4], rec[5]]])
        Rv = R @ rec[6:9]
        Pt = R @ P @ R.T + np.outer(Rv, t) + np.outer(t, Rv) + rec[9] * np.outer(t, t)
        acc += [Pt[0, 0], Pt[0, 1], Pt[0, 2], Pt[1, 1], Pt[1, 2], Pt[2, 2], *(Rv + rec[9] * t), rec[9]]
    inv = 1.0 / acc[9]
    m = acc[6:9] * inv
    return np.array([acc[0] * inv - m[0] * m[0], acc[1] * inv - m[0] * m[1], acc[2] * inv - m[0] * m[2],
                     acc[3] * inv - m[1] * m[1], acc[4] * inv - m[1] * m[2], acc[5] * inv - m[2] * m[2]])


def device_branch(cov):
    """common.cuh eig3_sym_plane / sym3_smallest_eigenvalue on cov = (a00 a01 a02 a11 a12 a22) in float64:
      fast    the Newton root is taken (settled and |p'(lambda_0)| >= 1e-2 tr^2); otherwise the Jacobi solver decides
      det     the characteristic polynomial's c0 = det(C)
      b12     on the fast path, the off-diagonal of the 2 x 2 problem relative to its diagonal (0 when exactly 0)
      tie     on the fast path, the smallest |u_0| components tie in the v1 axis choice"""
    a00, a01, a02, a11, a12, a22 = (float(x) for x in cov)
    m00, m01, m02 = a11 * a22 - a12 * a12, a01 * a22 - a12 * a02, a01 * a12 - a11 * a02
    c2 = a00 + a11 + a22
    c1 = m00 + (a00 * a22 - a02 * a02) + (a00 * a11 - a01 * a01)
    c0 = a00 * m00 - a01 * m01 + a02 * m02
    lam, fp, settled = 0.0, -c1, False
    for _ in range(10):
        f = ((c2 - lam) * lam - c1) * lam + c0
        fp = (-3.0 * lam + 2.0 * c2) * lam - c1
        d = f / fp
        lam -= d
        if abs(d) <= 1e-16 * abs(c2):
            settled = True
            break
    out = dict(fast=bool(settled and abs(fp) >= 1e-2 * c2 * c2), det=c0, lam0=lam, b12=None, tie=False)
    if not out["fast"]:
        return out
    A = np.array([[a00, a01, a02], [a01, a11, a12], [a02, a12, a22]])
    r = A - lam * np.eye(3)
    xs = [np.cross(r[0], r[1]), np.cross(r[0], r[2]), np.cross(r[1], r[2])]
    e0 = xs[0]
    for x in xs[1:]:
        if x @ x > e0 @ e0:
            e0 = x
    e0 = e0 / math.sqrt(e0 @ e0)
    ax, ay, az = np.abs(e0)
    if ax <= ay and ax <= az:
        v1 = np.array([0.0, e0[2], -e0[1]]); out["tie"] = ax == ay or ax == az
    elif ay <= az:
        v1 = np.array([-e0[2], 0.0, e0[0]]); out["tie"] = ay == az
    else:
        v1 = np.array([e0[1], -e0[0], 0.0])
    v1 = v1 / math.sqrt(v1 @ v1)
    v2 = np.cross(e0, v1)
    b11, b12, b22 = v1 @ A @ v1, v1 @ A @ v2, v2 @ A @ v2
    out["b12"] = abs(b12) / (abs(b11) + abs(b22))
    return out
