"""Scenes and drivers shared by the tests of the coloured LiDAR map (boundary B8): the emulated device pipeline
(tests/emu/colorize_emu.cpp), the host restatement colmap_points_from_lidar (tests/emu/colmap_host.cpp) and hand-built edge cases."""
import ctypes
import os
import subprocess
from pathlib import Path

import numpy as np

from oracle import synth

ROOT = Path(__file__).resolve().parents[1]


def _ptr(a, t):
    return a.ctypes.data_as(ctypes.POINTER(t))


def compile_so(src, out, extra=()):
    san = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []
    cmd = ["g++", "-std=c++17", "-O2", *san, "-ffp-contract=off", "-Wall", "-fPIC", "-shared", "-I", str(ROOT / "include"),
           str(ROOT / "tests" / "emu" / src), "-o", str(out), *extra]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return ctypes.CDLL(str(out))


def flat(scans):
    F = len(scans)
    sp = np.zeros(F + 1, np.int64); sp[1:] = np.cumsum([len(x) for x in scans])
    xyz = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float32).reshape(-1, 3) for x in scans]) if F else np.zeros((0, 3), np.float32))
    return sp, xyz


def scene(seed, F=7, n_per_scan=2000, M=5, width=160, height=120, colour=True):
    """make_depth_scene plus a patterned RGB image per camera."""
    s = synth.make_depth_scene(seed, F=F, n_per_scan=n_per_scan, M=M, width=width, height=height)
    rng = np.random.default_rng(seed + 77)
    s["rgb"] = rng.integers(0, 256, (M, height, width, 3), dtype=np.uint8) if colour else None
    return s


def oracle_args(s):
    return (s["scans"], s["frame_ts"], s["poses"], s["image_ts"], s["cams"], s["intr"], s["width"], s["height"])


def emu_run(lib, s, leaf, half_window=0.5, batches=None, poses=None):
    """The host-policy pipeline; `batches`: images per add_images call (None: all at once).  Returns (rc, xyz, rgb, listed, stats)."""
    sp, xyz = flat(s["scans"])
    F = len(s["scans"])
    ts = np.ascontiguousarray(s["frame_ts"], np.float64)
    ps = np.ascontiguousarray(s["poses"] if poses is None else poses, np.float64)
    h = ctypes.c_void_p()
    lib.emu_color_create(ctypes.c_int32(F), _ptr(sp, ctypes.c_int64), _ptr(xyz, ctypes.c_float), _ptr(ts, ctypes.c_double), ctypes.byref(h))
    try:
        rc = lib.emu_color_begin(h, _ptr(ps, ctypes.c_double), ctypes.c_double(half_window), ctypes.c_double(leaf))
        if rc != 0:
            return rc, None, None, None, None
        cams = np.ascontiguousarray(s["cams"], np.float64); its = np.ascontiguousarray(s["image_ts"], np.float64)
        intr = np.ascontiguousarray(s["intr"], np.float64)
        M = len(cams); W, H = s["width"], s["height"]
        rgb = s.get("rgb")
        listed = np.full(M, 7, np.uint8)
        step = M if not batches else batches
        for k0 in range(0, M, max(step, 1)):
            nb = min(step, M - k0)
            img = None if rgb is None else np.ascontiguousarray(rgb[k0:k0 + nb])
            lv = np.zeros(nb, np.uint8)
            rc = lib.emu_color_add(h, ctypes.c_int64(nb), _ptr(its[k0:], ctypes.c_double), _ptr(cams[k0:], ctypes.c_double),
                                   _ptr(intr, ctypes.c_double), ctypes.c_int32(W), ctypes.c_int32(H),
                                   _ptr(img, ctypes.c_uint8) if img is not None else None, _ptr(lv, ctypes.c_uint8))
            if rc != 0:
                return rc, None, None, None, None
            listed[k0:k0 + nb] = lv
        n = ctypes.c_int64(); stats = np.zeros(5, np.int64)
        rc = lib.emu_color_finish(h, ctypes.byref(n), _ptr(stats, ctypes.c_int64))
        if rc != 0:
            return rc, None, None, None, None
        out = np.zeros((n.value, 3), np.float32); col = np.zeros((n.value, 3), np.uint8)
        lib.emu_color_export(h, _ptr(out, ctypes.c_float), _ptr(col, ctypes.c_uint8))
        return 0, out, col, listed, dict(projections=int(stats[0]), landed=int(stats[1]), survivors=int(stats[2]), peak_bytes=int(stats[3]))
    finally:
        lib.emu_color_destroy(h)


def host_points(lib, s, leaf, poses=None):
    """colmap_points_from_lidar (host/lvba_visual_offline.hpp) on the same inputs: (xyz, written)."""
    sp, xyz = flat(s["scans"])
    F = len(s["scans"])
    ps = np.ascontiguousarray(s["poses"] if poses is None else poses, np.float64); ts = np.ascontiguousarray(s["frame_ts"], np.float64)
    cams = np.ascontiguousarray(s["cams"], np.float64); its = np.ascontiguousarray(s["image_ts"], np.float64)
    intr = np.ascontiguousarray(s["intr"], np.float64)
    M = len(cams)
    f = lib.host_colmap_points
    f.restype = ctypes.c_int64
    args = [ctypes.c_int32(F), _ptr(sp, ctypes.c_int64), _ptr(xyz, ctypes.c_float), _ptr(ps, ctypes.c_double), _ptr(ts, ctypes.c_double),
            ctypes.c_int32(M), _ptr(cams, ctypes.c_double), _ptr(its, ctypes.c_double), _ptr(intr, ctypes.c_double),
            ctypes.c_int32(s["width"]), ctypes.c_int32(s["height"]), ctypes.c_double(leaf)]
    n = f(*args, None, ctypes.c_int64(-1), None)
    out = np.zeros((n, 3), np.float32); wr = np.zeros(M, np.uint8)
    f(*args, _ptr(out, ctypes.c_float), ctypes.c_int64(n), _ptr(wr, ctypes.c_uint8))
    return out, wr


def edge_scene():
    """Hand-built cases on a distortion-free camera at the origin looking down +z (fx = fy = 64, so the pixel arithmetic is exact):
    near-ties within eps at one pixel in both orders, u / v at +-0.5 rounding edges and at W - 0.5, Z <= 1e-12, NaN points, negative
    coordinates, unsorted frame timestamps, an image with an empty window."""
    W, H = 40, 30
    eps = float(np.float32(1e-6))
    pts_a, pts_b = [], []
    # pixel (u = 5, v = 5) at cx = cy = 0.5: X = Y = 4.5 / 64 * Z
    for Z, scan in [(10.0, pts_a), (10.0 + eps / 4, pts_a), (10.0 - eps / 4, pts_a), (9.0, pts_b), (9.0 - eps * 0.9, pts_b)]:
        scan.append([4.5 / 64 * Z, 4.5 / 64 * Z, Z])
    for Z, scan in [(7.0 + eps / 8, pts_a), (7.0, pts_a)]:                    # the other order, at pixel (7, 7)
        scan.append([6.5 / 64 * Z, 6.5 / 64 * Z, Z])
    for u in [0.0, -1.0, W - 1.0, W - 1.0 - 2.0 ** -16, 12.0, -0.5]:             # u = 64 X / Z + 0.5: 0.5, -0.5, W - 0.5, ... edges
        pts_a.append([u / 64 * 2.0, 3.0 / 64 * 2.0, 2.0])
        pts_b.append([3.0 / 64 * 2.0, u / 64 * 2.0, 2.0])
    pts_a += [[0.1, 0.1, 0.0], [0.1, 0.1, 1e-13], [0.1, 0.1, -3.0], [np.nan, 0.0, 5.0], [0.0, np.inf, 5.0]]
    pts_b += [[-0.05, -0.02, 4.0], [-0.05, -0.02, 4.0], [-0.3, -0.2, 6.0]]
    rng = np.random.default_rng(3)
    cloud = rng.uniform([-2, -1.5, 1.0], [2, 1.5, 8.0], (400, 3))
    scans = [np.array(pts_a, np.float32), np.array(pts_b, np.float32), cloud[:200].astype(np.float32), cloud[200:].astype(np.float32),
             np.zeros((0, 3), np.float32)]
    poses = np.zeros((5, 12)); poses[:, [0, 4, 8]] = 1.0
    poses[2, 9:] = [-0.3, 0.2, -0.1]; poses[3, 9:] = [-1.0, -0.5, 0.0]             # negative world coordinates
    frame_ts = np.array([10.3, 10.0, 10.2, 9.9, 10.1])                               # not ascending
    image_ts = np.array([10.1, 10.45, 30.0, 10.0])                                  # image 2: empty window
    cam = np.concatenate([np.eye(3).ravel(), np.zeros(3)])
    cams = np.tile(cam, (4, 1)); cams[3, 9:] = [0.05, -0.02, 0.3]
    intr = np.array([64.0, 64.0, 0.5, 0.5, 0.0, 0.0, 0.0, 0.0])
    rgb = rng.integers(0, 256, (4, H, W, 3), dtype=np.uint8)
    return dict(scans=scans, poses=poses, frame_ts=frame_ts, cams=cams, image_ts=image_ts, intr=intr, width=W, height=H, rgb=rgb)


# ------------------------------------------------------------------ the reference's own VisualizeOptComparison (tests/emu/ref_colorize_driver.cpp)
REFERENCE = Path("/root/reference")


def ref_available():
    return (REFERENCE / "src" / "lvba_system.cpp").exists()


def compile_ref(out):
    """The reference's pipeline source with the stand-ins of oracle/ref_shim/ (the flags of oracle/Makefile's `ref` target)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-pthread", "-I", str(ROOT / "oracle" / "ref_shim"), "-I", str(REFERENCE / "include"),
           f'-DREF_SYSTEM_CPP="{REFERENCE}/src/lvba_system.cpp"', f'-DREF_DATASET_CPP="{REFERENCE}/src/dataset_io.cpp"', "-shared", "-o", str(out),
           str(ROOT / "tests" / "emu" / "ref_colorize_driver.cpp"), "-l:libsqlite3.so.0"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(ROOT / "oracle"))
    assert r.returncode == 0, r.stderr[-3000:]
    lib = ctypes.CDLL(str(out))
    lib.sys_create.restype = ctypes.c_void_p
    return lib


def ref_scene(seed, F=7, n_per_scan=2000, width=160, height=120):
    """scene() with a second pose set (`before`: the odometry poses and the cameras before the optimisation), one image more whose window
    holds no LiDAR and one whose file is missing.  `loaded` marks the images whose file exists."""
    s = scene(seed, F=F, n_per_scan=n_per_scan, M=5, width=width, height=height)
    rng = np.random.default_rng(seed + 500)
    M = 7
    s["image_ts"] = np.concatenate([s["image_ts"], [s["frame_ts"][-1] + 5.0, s["image_ts"][1] + 0.01]])
    s["cams"] = np.vstack([s["cams"], s["cams"][:1], s["cams"][1:2]])
    s["rgb"] = np.concatenate([s["rgb"], rng.integers(0, 256, (2, height, width, 3), dtype=np.uint8)])
    s["loaded"] = np.array([1, 1, 1, 1, 1, 1, 0], np.uint8)
    s["poses_before"] = s["poses"].copy(); s["poses_before"][:, 9:] += rng.normal(0, 0.03, (F, 3))
    s["cams_before"] = s["cams"].copy(); s["cams_before"][:, 9:] += rng.normal(0, 0.02, (M, 3))
    return s


def ref_run(lib, s, leaf, workdir):
    """The reference on the scene: (after xyz, after rgb, before xyz, before rgb, listed) with listed from the images.txt it writes."""
    workdir = Path(workdir)
    (workdir / "all_image").mkdir(parents=True, exist_ok=True)
    lib.colz_clear_images()
    for k, t in enumerate(s["image_ts"]):
        if s["loaded"][k]:
            bgr = np.ascontiguousarray(s["rgb"][k][:, :, ::-1])
            lib.colz_add_image(f"{workdir}/all_image/{t:.6f}.png".encode(), ctypes.c_int(s["height"]), ctypes.c_int(s["width"]), _ptr(bgr, ctypes.c_uint8))
    sp, xyz = flat(s["scans"])
    f64 = lambda a: np.ascontiguousarray(a, np.float64)  # noqa: E731
    ts, pa, pb, its, ca, cb, it = (f64(s[k]) for k in ("frame_ts", "poses", "poses_before", "image_ts", "cams", "cams_before", "intr"))
    h = ctypes.c_void_p(lib.sys_create())
    try:
        na, nb = ctypes.c_int64(), ctypes.c_int64()
        lib.colz_run(h, (str(workdir) + "/").encode(), ctypes.c_int(len(s["scans"])), _ptr(sp, ctypes.c_int64), _ptr(xyz, ctypes.c_float),
                     _ptr(ts, ctypes.c_double), _ptr(pa, ctypes.c_double), _ptr(pb, ctypes.c_double), ctypes.c_int(len(its)), _ptr(its, ctypes.c_double),
                     _ptr(ca, ctypes.c_double), _ptr(cb, ctypes.c_double), _ptr(it, ctypes.c_double), ctypes.c_int(s["width"]), ctypes.c_int(s["height"]),
                     ctypes.c_double(leaf), ctypes.byref(na), ctypes.byref(nb))
        out = []
        for which, n in ((0, na.value), (1, nb.value)):
            x = np.zeros((n, 3), np.float32); c = np.zeros((n, 3), np.uint8)
            lib.colz_cloud(h, ctypes.c_int(which), _ptr(x, ctypes.c_float), _ptr(c, ctypes.c_uint8))
            out += [x, c]
    finally:
        lib.sys_destroy(h)
    lines = (workdir / "Colmap" / "sparse" / "images.txt").read_text().splitlines()
    listed = np.zeros(len(s["image_ts"]), np.uint8)
    listed[[int(ln.split()[0]) for ln in lines[0::2]]] = 1
    return (*out, listed)


def loaded_subset(s):
    """What a caller of the stage passes: the images whose file loads (the reference skips the others before anything else, :1959-1962)."""
    keep = np.nonzero(s["loaded"])[0]
    return keep, dict(s, image_ts=s["image_ts"][keep], cams=s["cams"][keep], cams_before=s["cams_before"][keep], rgb=s["rgb"][keep])


def as_set(xyz, rgb):
    return sorted(zip(map(tuple, np.asarray(xyz, np.float32).view(np.uint32).tolist()), map(tuple, np.asarray(rgb).tolist())))


def fixture():
    """tests/golden/ref_colorize.npz as a scene dict (see tests/golden/make_golden_ref_colorize.py) plus the reference's outputs."""
    z = np.load(ROOT / "tests" / "golden" / "ref_colorize.npz")
    sp, xyz = z["scan_ptr"], z["xyz"]
    s = dict(scans=[xyz[sp[j]:sp[j + 1]] for j in range(len(sp) - 1)], **{k: z[k] for k in ("frame_ts", "poses", "poses_before", "image_ts", "cams",
             "cams_before", "intr", "rgb", "loaded")}, width=int(z["width"]), height=int(z["height"]))
    ref = {k: z[k] for k in ("after_xyz", "after_rgb", "before_xyz", "before_rgb", "listed")}
    return s, float(z["leaf"]), ref
