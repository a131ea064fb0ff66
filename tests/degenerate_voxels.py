"""LiDAR voxels on the numerically hard side of the plane factor (bavoxel.hpp:68-203) — a deterministic generator.

Real maps accept a voxel as a plane when lambda_0 / lambda_2 is small (voxel_math.h judge_eigen); lambda_1 is not
constrained, so strips, kerbs, poles and exactly planar ground enter the LM beside ordinary patches.  Each class below
draws world points, sees them from K poses and stores body-frame PointClusters the way oracle/synth.make_lidar does
(float32-rounded points accumulated into P, v, N in float64):

  plane  0.5 m x 0.5 m patch, 1 cm normal noise                  the Newton fast path of both device solvers (control)
  strip  0.5 m x 2 cm, 1 cm noise: lambda_0 <= lambda_1 << lambda_2  the Jacobi fallbacks of the build and residual passes
  line   1 m x 3 mm x 3 mm rod: lambda_0 ~ lambda_1, large 2/(l0 - l1)  both fallbacks, large umumT
  flat   exactly planar (no noise), poses within 0.3 m of the patch  lambda_0 at the rounding level, det(C) <= 0
  disc   symmetric 6 x 6 grid: lambda_1 = lambda_2 to the last bits  the 2 x 2 step with b12 = 0 or tiny
  axis   exactly planar, normal along x, y or z at a power-of-two offset, poses at 90-degree rotations and t = 0, N = 64:
         the covariance has exact zeros, so u_0 has exact zeros and the v1 axis choice ties
  far    plane or strip 1e3 m or 1e4 m from the origin                cancellation in P/N - vbar vbar^T
  bulk   plane with slots of N ~ 1e6 (weighted points, some of non-integral N) beside slots of N = 1: NN = (int)N, large P
  big    strip or line seen from 129-160 poses                        the big-voxel passes (lidar_big.h)

Exactly rank-1 or rank-0 covariances are not generated: there 2 / (lambda_0 - lambda_1) = 2 / 0 and the plane factor is
undefined.

Two arrangements of the same world-frame voxels:
  isolated  every voxel has poses of its own, so every block of H and every row of g comes from one voxel;
  shared    one trajectory, every voxel seen from K distinct poses within +-4 of its centre pose: blocks mix classes.
            Every voxel lies within 10 m of its centre pose (a far voxel here is a plane or strip like any other).
"""
import numpy as np

from oracle import synth

CLASSES = ("plane", "strip", "line", "flat", "disc", "axis", "far", "bulk")
BIG_K = (129, 160)


def _rot(rng):
    return synth.so3_exp(rng.normal(0.0, 2.0, (1, 3)))[0]


def _signed_perm(rng):
    """one of the 24 rotations that map the axes onto the axes (90-degree multiples)"""
    while True:
        R = np.zeros((3, 3))
        R[np.arange(3), rng.permutation(3)] = rng.choice([-1.0, 1.0], 3)
        if np.linalg.det(R) > 0:
            return R


def _frame(rng, cls, centre=None):
    """(centre, n, e1, e2): plane normal n and two in-plane directions"""
    if cls == "axis":
        k = int(rng.integers(3))
        n = np.eye(3)[k]; e1 = np.eye(3)[(k + 1) % 3]; e2 = np.eye(3)[(k + 2) % 3]
        c = rng.uniform(-20.0, 20.0, 3)
        c[k] = float(rng.choice([-8.0, -4.0, -2.0, 2.0, 4.0, 8.0]))     # the normal coordinate, exact in float32
        return c, n, e1, e2
    n = rng.normal(size=3); n /= np.linalg.norm(n)
    h = np.array([1.0, 0, 0]) if abs(n[0]) < 0.9 else np.array([0, 1.0, 0])
    e1 = np.cross(n, h); e1 /= np.linalg.norm(e1)
    e2 = np.cross(n, e1)
    if centre is None:
        centre = rng.uniform(-30.0, 30.0, 3)
    return centre, n, e1, e2


def _points(rng, shape, frame, m, noisy=True):
    """m world points of one slot"""
    c, n, e1, e2 = frame
    if shape == "plane":
        a, b, e = rng.uniform(-0.25, 0.25, m), rng.uniform(-0.25, 0.25, m), rng.normal(0, 0.01, m) * noisy
    elif shape == "strip":
        a, b, e = rng.uniform(-0.25, 0.25, m), rng.uniform(-0.01, 0.01, m), rng.normal(0, 0.01, m)
    elif shape == "line":
        a, b, e = rng.uniform(-0.5, 0.5, m), rng.uniform(-1.5e-3, 1.5e-3, m), rng.uniform(-1.5e-3, 1.5e-3, m)
    elif shape == "disc":
        g = (np.arange(6) - 2.5) * 0.1
        a, b = np.repeat(g, 6), np.tile(g, 6)
        e = rng.normal(0, 0.01, 36) * noisy
    else:
        raise ValueError(shape)
    return c[None] + a[:, None] * e1[None] + b[:, None] * e2[None] + e[:, None] * n[None]


def _cluster(pw, R, t, w=None):
    """body-frame PointCluster record (Pxx Pxy Pxz Pyy Pyz Pzz vx vy vz N) of world points pw seen from pose (R, t)"""
    pb = ((pw - t[None]) @ R).astype(np.float32).astype(np.float64)          # R^T (pw - t), float32 like a scan
    w = np.ones(len(pb)) if w is None else w
    P = np.einsum("k,ki,kj->ij", w, pb, pb)
    return np.array([P[0, 0], P[0, 1], P[0, 2], P[1, 1], P[1, 2], P[2, 2], *(w @ pb), w.sum()])


def _voxel_spec(rng, cls):
    """(point shape, frame) of one voxel of class cls"""
    if cls == "far":
        shape = ("plane", "strip")[int(rng.integers(2))]
        d = rng.normal(size=3); d *= float(rng.choice([1e3, 1e4])) / np.linalg.norm(d)
        frame = _frame(rng, "far", centre=d)
    elif cls in ("flat", "axis", "bulk"):
        shape, frame = "plane", _frame(rng, cls)
    else:
        shape, frame = cls, _frame(rng, cls)
    return shape, frame


def _voxel_slots(rng, cls, shape, frame, poses):
    """cluster records of one voxel seen from the given poses [(R, t), ...]"""
    K = len(poses)
    if cls == "axis":                                     # N = 64 in total: 1/N and every mean are exact
        cut = np.sort(rng.choice(np.arange(1, 64 // 4), K - 1, replace=False)) * 4 if K > 1 else np.zeros(0, np.int64)
        counts = np.diff(np.concatenate([[0], cut, [64]]))
    else:
        counts = rng.integers(8, 41, K)
    out = []
    heavy = int(rng.integers(K)) if cls == "bulk" else -1
    for k, (R, t) in enumerate(poses):
        if cls == "bulk" and k != heavy and rng.random() < 0.5:
            out.append(_cluster(_points(rng, shape, frame, 1), R, t))                 # a single point, N = 1
        elif cls == "bulk":                                # 40 points of weight ~25000: N ~ 1e6, integral or not
            w = np.full(40, 25000.0 + (0.0123 if rng.random() < 0.5 else 0.0))
            out.append(_cluster(_points(rng, shape, frame, 40), R, t, w))
        else:
            noisy = cls not in ("flat", "axis") and not (cls == "disc" and rng.random() < 0.5)
            out.append(_cluster(_points(rng, shape, frame, int(counts[k]), noisy), R, t))
    return out


def _own_poses(rng, cls, frame, K):
    c = frame[0]
    if cls == "axis":
        return [(_signed_perm(rng), np.zeros(3)) for _ in range(K)]
    spread = 0.3 if cls == "flat" else 8.0
    return [(_rot(rng), c + rng.uniform(-spread, spread, 3)) for _ in range(K)]


def _pack(classes, slot_lists, pose_lists, poses):
    K = np.array([len(s) for s in slot_lists], np.int64)
    vox_ptr = np.concatenate([[0], np.cumsum(K)]).astype(np.int64)
    return dict(vox_ptr=vox_ptr, pose_idx=np.concatenate(pose_lists).astype(np.int32),
                clusters=np.array([r for s in slot_lists for r in s]), poses=poses, cls=np.array(classes))


def _poses_array(Rt):
    return np.array([np.concatenate([R.reshape(9), t]) for R, t in Rt])


def isolated(seed=0, per_class=24, k_max=8, big=6, big_k=BIG_K):
    """per_class voxels of every class with K in 1..k_max, and `big` strip / line voxels with K in big_k, each voxel with
    poses of its own (so every H block and g row belongs to one voxel)."""
    rng = np.random.Generator(np.random.Philox(key=1000 + seed))
    classes, slots, pidx, Rt = [], [], [], []
    todo = [(c, int(rng.integers(1, k_max + 1))) for c in CLASSES for _ in range(per_class)]
    todo += [(("strip", "line")[b % 2], int(rng.integers(big_k[0], big_k[1] + 1))) for b in range(big)]
    for cls, K in todo:
        shape, frame = _voxel_spec(rng, cls)
        own = _own_poses(rng, cls, frame, K)
        slots.append(_voxel_slots(rng, cls, shape, frame, own))
        pidx.append(np.arange(len(Rt), len(Rt) + K))
        Rt += own
        classes.append(cls if K <= 128 else "big")
    return _pack(classes, slots, pidx, _poses_array(Rt))


def tile_and_big(seed=0):
    """strip and line voxels seen from 128 poses (the most a tile holds) and the same voxels seen from one pose more
    (129: the big-voxel passes), each with poses of its own."""
    rng = np.random.Generator(np.random.Philox(key=2000 + seed))
    classes, slots, pidx, Rt = [], [], [], []
    for shape in ("strip", "line", "strip", "line"):
        frame = _frame(rng, shape)
        own = _own_poses(rng, shape, frame, 129)
        recs = _voxel_slots(rng, shape, shape, frame, own)
        for K in (128, 129):
            slots.append(recs[:K])
            pidx.append(np.arange(len(Rt), len(Rt) + K))
            Rt += own[:K]
            classes.append(f"{shape}{K}")
    return _pack(classes, slots, pidx, _poses_array(Rt))


def shared(seed=0, per_class=24, k_max=8, half=4, n_poses=60):
    """The classes on one trajectory: a voxel is seen from K distinct poses within +-half of its centre pose, so blocks
    and tiles mix classes and fast-path with fallback voxels.  Returns the problem at the generating poses, plus
    `poses0`, a perturbed start for the LM."""
    rng = np.random.Generator(np.random.Philox(key=3000 + seed))
    R_gt, p_gt = synth.make_trajectory(n_poses, rng)
    classes, slots, pidx = [], [], []
    for cls in CLASSES:
        for _ in range(per_class):
            c = int(rng.integers(n_poses))
            cand = np.arange(max(0, c - half), min(n_poses, c + half + 1))
            K = min(int(rng.integers(1, k_max + 1)), len(cand))
            sel = np.sort(rng.choice(cand, K, replace=False))
            shape, frame = _voxel_spec(rng, cls)
            frame = (p_gt[c] + rng.uniform(-10, 10, 3),) + frame[1:]   # within sensor range, like make_lidar
            slots.append(_voxel_slots(rng, cls, shape, frame, [(R_gt[j], p_gt[j]) for j in sel]))
            pidx.append(sel)
            classes.append(cls)
    poses = np.concatenate([R_gt.reshape(n_poses, 9), p_gt], 1)
    p = _pack(classes, slots, pidx, poses)
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (n_poses, 3)))
    p["poses0"] = np.concatenate([R0.reshape(n_poses, 9), p_gt + rng.normal(0, 0.02, (n_poses, 3))], 1)
    return p


def reorder(p, order):
    """the same problem with its voxels in another order"""
    K = np.diff(p["vox_ptr"]); starts = p["vox_ptr"][:-1]
    idx = np.concatenate([np.arange(starts[a], starts[a] + K[a]) for a in order])
    out = dict(p)
    out.update(vox_ptr=np.concatenate([[0], np.cumsum(K[order])]).astype(np.int64), pose_idx=p["pose_idx"][idx],
               clusters=p["clusters"][idx], cls=p["cls"][order])
    return out
