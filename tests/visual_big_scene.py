"""Visual BA scenes with long tracks, for the tests of the landmarks that have more than 128 observations
(global-lvba_b200/csrc/visual_big.h).

Cameras ride along a straight street (0.5 m apart, looking sideways at a facade 40-60 m away), so that one facade point is in
front of hundreds of consecutive cameras.  A track longer than the number of cameras wraps around: the sequence passes the
place again and the track holds several keypoints of one image, as a revisit joined by the matcher gives.  Short tracks of
3-8 observations fill the scene as in oracle/synth.make_visual.  Same layout as oracle/synth.make_problem's visual part."""
import numpy as np

from oracle import synth
from oracle import visual_oracle as vo

KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


def args(p):
    return [p[k] for k in KEYS]


def _cameras(M, rng):
    base = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])        # camera z = world +y, x = world +x
    R_gt = base[None] @ synth.so3_exp(rng.normal(0, 0.02, (M, 3)))
    p = np.stack([0.5 * np.arange(M), rng.normal(0, 0.1, M), 1.5 + rng.normal(0, 0.05, M)], 1)
    t_gt = -np.einsum("nij,nj->ni", R_gt, p)
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.005, (M, 3)))
    t0 = t_gt + rng.normal(0, 0.03, (M, 3))
    return R_gt, t_gt, R0, t0, p


def make_scene(seed, M=60, n_short=120, long_tracks=(), extra_tracks=()):
    """long_tracks: (K, first camera) pairs, cameras first, first + 1, ... modulo M.  extra_tracks: camera lists of further tracks
    (duplicates allowed) whose landmark lies 20 m in front of their first camera."""
    rng = np.random.Generator(np.random.Philox(key=seed))
    R_gt, t_gt, R0, t0, p = _cameras(M, rng)
    cams, Xs = [], []
    for _ in range(n_short):
        c = int(rng.integers(0, M))
        lo, hi = max(0, c - 10), min(M, c + 11)
        L = int(min(rng.integers(3, 9), hi - lo))
        cams.append(np.sort(rng.choice(np.arange(lo, hi), L, replace=False)))
        Xs.append(p[c] + np.array([rng.uniform(-5, 5), rng.uniform(5, 20), rng.uniform(-3, 3)]))
    for K, c0 in long_tracks:
        cc = (c0 + np.arange(K)) % M
        mid = p[cc].mean(0)
        cams.append(cc)
        Xs.append(np.array([mid[0] + rng.uniform(-3, 3), rng.uniform(40, 60), rng.uniform(-5, 5)]))
    for cl in extra_tracks:
        cams.append(np.asarray(cl, np.int64))
        Xs.append(p[cl[0]] + np.array([rng.uniform(-2, 2), 20.0, rng.uniform(-2, 2)]))
    X_gt = np.array(Xs)
    obs_ptr = np.zeros(len(cams) + 1, np.int64)
    obs_ptr[1:] = np.cumsum([len(c) for c in cams])
    obs_cam = np.concatenate(cams).astype(np.int32)
    trk = np.repeat(np.arange(len(cams)), np.diff(obs_ptr))
    uv, _ = synth.project(R_gt[obs_cam], t_gt[obs_cam], X_gt[trk])
    obs_uv = (uv + rng.normal(0, 0.5, uv.shape)).astype(np.float32)
    n = rng.normal(size=(len(cams), 3)); n /= np.linalg.norm(n, axis=1, keepdims=True)
    plane_nd = np.concatenate([n, -np.einsum("ni,ni->n", n, X_gt)[:, None]], 1)
    X0 = X_gt + rng.normal(0, 0.05, X_gt.shape)
    return dict(q=synth.rot_to_quat_wxyz(R0), t=t0, X=X0, plane_nd=plane_nd, obs_ptr=obs_ptr, obs_cam=obs_cam, obs_uv=obs_uv,
                intr=synth.INTR.copy(), sigma_px=synth.SIGMA_PX, sigma_plane=synth.SIGMA_PLANE)


def put_behind(p, a):
    """Move landmark a behind its first camera (z_c < 0): zero residual there (utils.hpp:78)."""
    c = p["obs_cam"][p["obs_ptr"][a]]
    R = vo.quat_to_rot(p["q"][c][None])[0]
    p["X"][a] = R.T @ (np.array([0.1, 0.1, -2.0]) - p["t"][c])


def shuffled(p, seed):
    """The same problem with the landmarks in another order (and every landmark's observations permuted)."""
    rng = np.random.default_rng(seed)
    op = p["obs_ptr"]
    T = len(op) - 1
    perm = rng.permutation(T)
    idx = np.concatenate([op[a] + rng.permutation(op[a + 1] - op[a]) for a in perm]).astype(np.int64)
    q = dict(p)
    q["obs_ptr"] = np.zeros(T + 1, np.int64); q["obs_ptr"][1:] = np.cumsum(np.diff(op)[perm])
    q["obs_cam"] = p["obs_cam"][idx]; q["obs_uv"] = p["obs_uv"][idx]
    q["X"] = p["X"][perm]; q["plane_nd"] = p["plane_nd"][perm]
    return q, perm
