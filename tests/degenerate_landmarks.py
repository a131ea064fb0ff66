"""Ill-conditioned and edge-case landmarks for the visual LM, for the 50-digit reference oracle/visual_mp.py.

The layout is the street of tests/visual_big_scene.py: cameras 0.5 m apart along world x, looking sideways (+y).  Every landmark
is labelled with its class:

  far       depth 1e2 - 1e5 m, plane normal perpendicular to the mean ray (a facade at a grazing angle)
  pair      2 views with 1e-3 - 1e-1 m of parallax
  rotation  3 views from one camera centre, plane normal perpendicular to the ray: C is singular but for the LM diagonal
  near_z    ordinary views, one view with z in 1e-7 - 1e-4 and one with z = 5e-9 (below the 1e-8 cut-off, utils.hpp:78)
  plane0    the landmark on its plane up to |e| in 1e-9 - 1e-5 (the kink of sqrt(e^2 + 1e-12))
  offset    the landmark and its cameras translated 1e3 - 1e5 m from the origin
  cancel    cameras that see only one or two landmarks, so that U - W C^-1 W^T nearly cancels
  big       far / pair geometry with 128 observations (the tile path) and with 129 and 300 (visual_big.h)
  ordinary  3 - 5 views at 5 - 20 m (a reference point for the others)

and problems of their own for what is global to a problem: `distort` (large k1 k2 p1 p2, landmarks near the corners, where the
radial factor approaches 0), `huber_edge` (reprojection s within a few ulps of a^2 on both sides, a = 1.7, and far beyond) and
`cauchy_far` (s up to 1e9 a^2).  Problems are the dicts of tests/visual_big_scene.py with `cls` [T] and, for the loss problems,
`loss_px` / `loss_pl` = (kind, a)."""
import numpy as np
from mpmath import mpf

from oracle import synth
from oracle import visual_mp as vm

BASE = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])      # camera z = world +y, camera x = world +x
CLASSES = ("ordinary", "far", "pair", "rotation", "near_z", "plane0", "offset", "cancel")


class _Scene:
    def __init__(self, seed, intr=None):
        self.rng = np.random.Generator(np.random.Philox(key=seed))
        self.R, self.c = [], []                  # camera rotations (world -> camera) and centres
        self.tracks = []                         # (cams, X_gt, plane normal or None, cls, e, perturb)
        self.intr = synth.INTR.copy() if intr is None else np.asarray(intr, np.float64)

    def camera(self, centre, tilt=0.02, R=None):
        self.R.append(BASE @ synth.so3_exp(self.rng.normal(0, tilt, (1, 3)))[0] if R is None else R)
        self.c.append(np.asarray(centre, np.float64))
        return len(self.R) - 1

    def street(self, x0, n, spacing=0.5, offset=(0.0, 0.0, 0.0)):
        return [self.camera(np.array([x0 + spacing * i, 0.0, 1.5]) + offset) for i in range(n)]

    def track(self, cams, X, cls, normal=None, e=None, perturb=True):
        self.tracks.append((list(cams), np.asarray(X, np.float64), normal, cls, e, perturb))

    def at(self, cam, xn, yn, depth):
        """the world point that camera `cam` sees at normalised (xn, yn) and depth"""
        return self.c[cam] + self.R[cam].T @ (depth * np.array([xn, yn, 1.0]))

    def near_camera(self, X, z):
        """a new camera that sees X at X_c = (1e-3 z, 2e-3 z, z)"""
        R = BASE @ synth.so3_exp(self.rng.normal(0, 0.02, (1, 3)))[0]
        return self.camera(X - R.T @ np.array([1e-3 * z, 2e-3 * z, z]), R=R)

    def build(self, perturb=False, noise_px=0.5):
        rng = self.rng
        M = len(self.R)
        R = np.array(self.R); c = np.array(self.c)
        t = -np.einsum("nij,nj->ni", R, c)
        cams = [np.asarray(tc[0], np.int32) for tc in self.tracks]
        X_gt = np.array([tc[1] for tc in self.tracks])
        obs_ptr = np.zeros(len(cams) + 1, np.int64); obs_ptr[1:] = np.cumsum([len(x) for x in cams])
        obs_cam = np.concatenate(cams).astype(np.int32)
        trk = np.repeat(np.arange(len(cams)), np.diff(obs_ptr))
        uv, _ = synth.project(R[obs_cam], t[obs_cam], X_gt[trk], self.intr)
        keep = np.array([self.tracks[a][5] for a in trk])
        obs_uv = np.where(keep[:, None], uv + rng.normal(0, noise_px, uv.shape), uv).astype(np.float32)
        plane_nd = np.zeros((len(cams), 4))
        X0 = X_gt.copy()
        for a, (cl, X, n, cls, e, pert) in enumerate(self.tracks):
            if n is None:
                n = rng.normal(size=3)
            n = n / np.linalg.norm(n)
            plane_nd[a, :3] = n
            plane_nd[a, 3] = -n @ X + (e if e is not None else 0.0)
            if pert and e is None:
                X0[a] = X + rng.normal(0, 0.05, 3)
        q = synth.rot_to_quat_wxyz(R)
        if perturb:
            hold = np.zeros(M, bool)
            for cl, _, _, cls, _, pert in self.tracks:
                if not pert:
                    hold[cl] = True
            Rp = R @ synth.so3_exp(rng.normal(0, 0.002, (M, 3)))
            tp = t + rng.normal(0, 0.01, (M, 3))
            q = np.where(hold[:, None], q, synth.rot_to_quat_wxyz(Rp)); t = np.where(hold[:, None], t, tp)
        return dict(q=q, t=t, X=X0, X_gt=X_gt, plane_nd=plane_nd, obs_ptr=obs_ptr, obs_cam=obs_cam, obs_uv=obs_uv,
                    intr=self.intr.copy(), sigma_px=synth.SIGMA_PX, sigma_plane=synth.SIGMA_PLANE,
                    cls=np.array([tc[3] for tc in self.tracks]))


def _perp(ray, rng):
    n = np.cross(ray, rng.normal(size=3))
    return n / np.linalg.norm(n)


def _add_class(S, cls, i, cams=None, x0=0.0):
    """one landmark of class `cls`, variant i; cams: street cameras to use (else new ones at x0)"""
    rng = S.rng
    def street(n, spacing=0.5, offset=(0.0, 0.0, 0.0)):
        return cams[:n] if cams is not None else S.street(x0, n, spacing, offset)
    if cls == "ordinary":
        cl = street(3 + i % 3)
        X = S.at(cl[0], rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(5, 20))
        S.track(cl, X, cls)
    elif cls == "far":
        D = 10.0 ** (2 + 3 * (i % 7) / 6)                   # 1e2 .. 1e5 m
        cl = street(5)
        X = S.at(cl[2], rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), D)
        ray = X - np.mean([S.c[k] for k in cl], 0)
        S.track(cl, X, cls, normal=_perp(ray / np.linalg.norm(ray), rng))
    elif cls == "pair":
        b = 10.0 ** (-3 + 2 * (i % 5) / 4)                  # 1e-3 .. 1e-1 m
        cl = street(2, spacing=b) if cams is None else [cams[0], S.camera(S.c[cams[0]] + [b, 0, 0])]
        X = S.at(cl[0], rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 20.0)
        S.track(cl, X, cls)
    elif cls == "rotation":
        c0 = np.array([x0, 0.0, 1.5]) if cams is None else S.c[cams[0]] + [0.0, 0.0, 0.3]
        cl = [S.camera(c0 + rng.normal(0, 1e-9, 3), tilt=0.05) for _ in range(3)]
        X = S.at(cl[0], 0.05, -0.05, 20.0)
        ray = X - c0
        S.track(cl, X, cls, normal=_perp(ray / np.linalg.norm(ray), rng))
    elif cls == "near_z":
        cl = street(3)
        X = S.at(cl[0], rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), 10.0)
        z = 10.0 ** (-7 + 3 * (i % 4) / 3)                  # 1e-7 .. 1e-4
        S.track(cl + [S.near_camera(X, z), S.near_camera(X, 5e-9)], X, cls, perturb=False)
    elif cls == "plane0":
        cl = street(3)
        X = S.at(cl[0], rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 15.0)
        e = 10.0 ** (-9 + 4 * (i % 5) / 4) * (1 if i % 2 else -1)   # |e| 1e-9 .. 1e-5
        S.track(cl, X, cls, e=e)
    elif cls == "offset":
        off = np.array([1.0, 0.3, 0.1]) * 10.0 ** (3 + 2 * (i % 3) / 2)   # 1e3 .. 1e5 m
        cl = street(4, offset=off) if cams is None else cams[:4]
        X = S.at(cl[0], rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 20.0)
        S.track(cl, X, cls)
    elif cls == "cancel":
        cl = street(2)
        for k in range(1 + i % 2):
            S.track(cl, S.at(cl[0], rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 12.0), cls)


def isolated(per_class=6, seed=7):
    """every landmark on cameras of its own (the offset landmarks' cameras translated with them), so that every S block and
    rhs row belongs to one class"""
    S = _Scene(seed)
    x0 = 0.0
    for cls in CLASSES:
        for i in range(per_class):
            _add_class(S, cls, i, x0=x0)
            x0 += 10.0
    return S.build()


def tile_and_big(seed=11):
    """a far (1 km) and a short-baseline (20 m) landmark of K = 128, 129 and 300 observations on a street of K cameras 1 cm
    apart, one street per K (its class "big K"), with a few ordinary landmarks on every street"""
    S = _Scene(seed)
    x0 = 0.0
    for K in (128, 129, 300):
        cl = S.street(x0, K, spacing=0.01)
        for D, far in ((1e3, True), (20.0, False)):
            X = S.at(cl[K // 2], 0.02 if far else -0.1, -0.03, D)
            ray = X - np.mean([S.c[k] for k in cl], 0)
            S.track(cl, X, f"big {K}", normal=_perp(ray / np.linalg.norm(ray), S.rng) if far else None)
        for i in range(3):
            c0 = int(S.rng.integers(0, K - 5))
            _add_class(S, "ordinary", i, cams=cl[c0:c0 + 5])
            S.tracks[-1] = S.tracks[-1][:3] + (f"big {K}",) + S.tracks[-1][4:]
        x0 += 10.0
    return S.build()


def shared(seed=3, M=40, per_class=3):
    """one street trajectory of M cameras 1 km from the origin, landmarks of every class on it (rotation and near_z add
    cameras of their own beside it), from a perturbed start: cameras by 2 mrad / 1 cm, landmarks by 5 cm (not the near_z ones
    or their cameras, whose cut-off views would otherwise move past the camera)"""
    S = _Scene(seed)
    off = np.array([1e3, 200.0, 10.0])
    cams = S.street(off[0], M, offset=(0.0, off[1], off[2]))
    for cls in CLASSES:
        for i in range(per_class if cls != "ordinary" else 4 * per_class):
            c0 = int(S.rng.integers(0, M - 6))
            if cls == "cancel":
                c2 = S.street(off[0] + 0.5 * c0 + 0.25, 2, offset=(0.0, off[1] + 1.0, off[2]))
                _add_class(S, cls, i, cams=c2)
            elif cls == "offset":
                _add_class(S, "ordinary", i, cams=cams[c0:c0 + 4])
                S.tracks[-1] = S.tracks[-1][:3] + ("offset",) + S.tracks[-1][4:]
            else:
                _add_class(S, cls, i, cams=cams[c0:c0 + 6])
    return S.build(perturb=True)


def fixed_mask(p, every=3):
    """a cam_fixed mask [M]: every `every`-th camera that sees a landmark of a degenerate class"""
    M = len(p["q"])
    m = np.zeros(M, bool)
    op = p["obs_ptr"]
    seen = sorted({int(c) for a in range(len(op) - 1) if p["cls"][a] != "ordinary" for c in p["obs_cam"][op[a]:op[a + 1]]})
    m[seen[::every]] = True
    return m


def distort(seed=21):
    """large Brown-Conrady coefficients (rad = 1 + k1 r^2 + k2 r^4 reaches 0 at r^2 = 2.76) and landmarks seen at
    r^2 = 0.1 .. 2.7 in their first view"""
    intr = np.array([500.0, 500.0, 640.0, 480.0, -0.5, 0.05, 0.01, -0.01])
    S = _Scene(seed, intr)
    for i, r2 in enumerate(np.linspace(0.1, 2.7, 16)):
        cl = S.street(10.0 * i, 3, spacing=0.3)
        ang = S.rng.uniform(0, 2 * np.pi)
        S.track(cl, S.at(cl[0], np.sqrt(r2) * np.cos(ang), np.sqrt(r2) * np.sin(ang), 8.0), "distort")
    p = S.build()
    return p


def _tune_s(p, a, target):
    """move the translation of observation a's (own) camera until s = |r|^2 of that observation is `target` (mpf) to within
    the rounding of t: minimum-norm Newton steps along ds/dt"""
    s_ = int(p["obs_ptr"][a]); c = int(p["obs_cam"][s_])
    for _ in range(12):
        o = vm.observation(p["q"][c], p["t"][c], p["X"][a], p["obs_uv"][s_], p["intr"], p["sigma_px"])
        s = o["r"][0] ** 2 + o["r"][1] ** 2
        g = [2 * (o["r"][0] * o["J"][0][3 + k] + o["r"][1] * o["J"][1][3 + k]) for k in range(3)]
        gg = g[0] ** 2 + g[1] ** 2 + g[2] ** 2
        if gg == 0:
            break
        p["t"][c] = [float(mpf(float(p["t"][c, k])) - (s - target) * g[k] / gg) for k in range(3)]


def huber_edge(seed=31, a=1.7):
    """Huber (a = 1.7) on the reprojection and (a = 0.7) on the plane blocks: 12 landmarks 1 km away whose first observation has
    s = a^2 (1 + k eps), k = -6 .. 5, to the rounding of its camera's t, and 8 whose observations are 5 - 500 px off (s up to
    1e6 a^2)"""
    S = _Scene(seed)
    for i in range(20):
        edge = i < 12           # 1 km deep, cameras at the origin: s moves by < 1 ulp of a^2 per ulp of t
        cl = S.street(0.0 if edge else 10.0 * i, 3)
        S.track(cl, S.at(cl[0], S.rng.uniform(-0.3, 0.3), S.rng.uniform(-0.3, 0.3), 1e3 if edge else 10.0),
                "huber_edge" if edge else "huber_far")
    p = S.build(noise_px=0.3)
    for i in range(12, 20):
        k = p["obs_ptr"][i]
        p["obs_uv"][k:k + 3] += np.float32(10.0 ** (0.7 + 0.25 * (i - 12)))
    for i in range(12):
        _tune_s(p, i, mpf(a) ** 2 * (1 + (i - 6) * mpf(vm.EPS)))
    p["loss_px"], p["loss_pl"] = (vm.HUBER, a), (vm.HUBER, 0.7)
    return p


def cauchy_far(seed=41, a=0.05):
    """Cauchy (a = 0.05) on both blocks, observations up to 800 px off: s / a^2 up to ~1e9"""
    S = _Scene(seed)
    for i in range(16):
        cl = S.street(10.0 * i, 3)
        S.track(cl, S.at(cl[0], S.rng.uniform(-0.3, 0.3), S.rng.uniform(-0.3, 0.3), 10.0), "cauchy_far")
    p = S.build()
    for i in range(16):
        k = p["obs_ptr"][i]
        p["obs_uv"][k] += np.float32(10.0 ** (-1 + 3.9 * i / 15))
    p["loss_px"], p["loss_pl"] = (vm.CAUCHY, a), (vm.CAUCHY, 0.5)
    return p
