"""CPU restatement of the coloured LiDAR map of VisualizeOptComparison — TEST INFRASTRUCTURE; nothing in the product imports it.
  window            src/lvba_system.cpp:1973-1977     frames with !(|x_buf[idx].t - id| > 0.5), a linear scan over all frames
  world points      :1983-1990                        (float)(R p + t) per coordinate, each row (r0 p0 + r1 p1) + r2 p2, then + t
  skip              :1993-1996                        an image whose window holds no point is not listed (nor in images.txt)
  z-buffer          :2037-2060, include/utils.hpp:183-205
                    projectWorldToPixel, uu = round(u), vv = round(v) (half away from zero), bounds, then in cloud order
                    `if (zc + 1e-6f < zbuf[idx]) { zbuf[idx] = (float)zc; pix[idx] = point, colour img(vv, uu) }`
  append            :2062-2069                        the kept pixels in pixel order
  thinning          include/BALM/tools.hpp:301-359    per voxel the original point nearest the centre, the first in merged order
                                                      on ties; leaf < 0.001 keeps every point
Two restatements that must agree exactly: `colorize_literal` (the per-image loop as written) and `colorize` (per image a lexsort
by pixel and the sequential rule per run; the thinning as one lexsort).  Both return the thinned cloud in ascending
(kx, ky, kz) order (the reference's unordered_map order is unspecified), or in merged order when leaf < 0.001."""
from __future__ import annotations

import numpy as np

from oracle.anchor_oracle import _keys_d2

EPS = float(np.float32(1e-6))
GREY = np.array([128, 128, 128], np.uint8)


def world_points(scan, pose):
    p = np.asarray(scan, np.float32).reshape(-1, 3).astype(np.float64)
    R = np.asarray(pose[:9], np.float64).reshape(3, 3); t = np.asarray(pose[9:], np.float64)
    w = np.empty_like(p)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(3):
            w[:, k] = ((R[k, 0] * p[:, 0] + R[k, 1] * p[:, 1]) + R[k, 2] * p[:, 2]) + t[k]
        return w.astype(np.float32)


def _round_half_away(u):
    r = np.trunc(u)
    return r + np.where(np.abs(u - r) >= 0.5, np.sign(u), 0.0)


def project(cam, intr, pts, W, H):
    """projectWorldToPixel on float32 world points: (pixel index or -1, Z in double)."""
    p = np.asarray(pts, np.float32).reshape(-1, 3).astype(np.float64)
    R = np.asarray(cam[:9], np.float64).reshape(3, 3); t = np.asarray(cam[9:], np.float64)
    fx, fy, cx, cy, k1, k2, p1, p2 = [float(v) for v in intr]
    with np.errstate(all="ignore"):
        X, Y, Z = [((R[k, 0] * p[:, 0] + R[k, 1] * p[:, 1]) + R[k, 2] * p[:, 2]) + t[k] for k in range(3)]
        ok = np.isfinite(X) & np.isfinite(Y) & np.isfinite(Z) & (Z > 1e-12)
        x = X / Z; y = Y / Z
        r2 = x * x + y * y; r4 = r2 * r2
        radial = (1.0 + k1 * r2) + k2 * r4
        x_tan = ((2.0 * p1) * x) * y + p2 * (r2 + (2.0 * x) * x)
        y_tan = p1 * (r2 + (2.0 * y) * y) + ((2.0 * p2) * x) * y
        xd = x * radial + x_tan; yd = y * radial + y_tan
        u = fx * xd + cx; v = fy * yd + cy
        ok &= np.isfinite(u) & np.isfinite(v)
        ur = _round_half_away(np.where(ok, u, -1.0)); vr = _round_half_away(np.where(ok, v, -1.0))
        ok &= (ur >= 0) & (ur < W) & (vr >= 0) & (vr < H)
    pix = np.where(ok, vr * W + ur, -1).astype(np.int64)
    return pix, Z


def image_cloud(scans, frame_ts, world, t_img, half_window):
    sel = [f for f in range(len(scans)) if not (abs(frame_ts[f] - t_img) > half_window)]
    if not sel:
        return np.zeros((0, 3), np.float32)
    return np.concatenate([world[f] for f in sel]).reshape(-1, 3)


def _colour(rgb, k, pix, W):
    if rgb is None:
        return np.tile(GREY, (len(pix), 1))
    img = np.asarray(rgb[k], np.uint8).reshape(-1, 3)
    return img[pix]


def _thin_literal(merged, colours, leaf):
    if leaf < 0.001:
        return merged, colours
    key, d2 = _keys_d2(merged, leaf)
    best = {}
    for i in range(len(merged)):
        k = (int(key[i, 0]), int(key[i, 1]), int(key[i, 2]))
        if k not in best or d2[i] < best[k][0]:
            best[k] = (d2[i], i)
    idx = np.array([best[k][1] for k in sorted(best)], np.int64)
    return merged[idx].reshape(-1, 3), colours[idx].reshape(-1, 3)


def _thin(merged, colours, leaf):
    if leaf < 0.001 or len(merged) == 0:
        return merged, colours
    key, d2 = _keys_d2(merged, leaf)
    order = np.lexsort((np.arange(len(merged)), d2, key[:, 2], key[:, 1], key[:, 0]))
    ks = key[order]
    head = np.concatenate([[True], np.any(ks[1:] != ks[:-1], axis=1)])
    return merged[order[head]], colours[order[head]]


def colorize_literal(scans, frame_ts, poses, image_ts, cams, intr, W, H, rgb=None, leaf=0.01, half_window=0.5):
    """Returns (xyz (n, 3) float32, rgb (n, 3) uint8, listed (M,) uint8)."""
    world = [world_points(s, poses[f]) for f, s in enumerate(scans)]
    merged, colours, listed = [], [], np.zeros(len(cams), np.uint8)
    for k in range(len(cams)):
        cloud = image_cloud(scans, frame_ts, world, image_ts[k], half_window)
        if len(cloud) == 0:
            continue
        listed[k] = 1
        pix, Z = project(cams[k], intr, cloud, W, H)
        zbuf = np.full(W * H, np.inf, np.float32)
        who = np.full(W * H, -1, np.int64)
        for i in range(len(cloud)):
            q = pix[i]
            if q < 0:
                continue
            if float(Z[i]) + EPS < float(zbuf[q]):
                zbuf[q] = np.float32(Z[i]); who[q] = i
        kept = np.nonzero(np.isfinite(zbuf))[0]
        merged.append(cloud[who[kept]]); colours.append(_colour(rgb, k, kept, W))
    merged = np.concatenate(merged).reshape(-1, 3) if merged else np.zeros((0, 3), np.float32)
    colours = np.concatenate(colours).reshape(-1, 3).astype(np.uint8) if colours else np.zeros((0, 3), np.uint8)
    xyz, col = _thin_literal(merged, colours, leaf)
    return xyz.astype(np.float32), col.astype(np.uint8), listed


def colorize(scans, frame_ts, poses, image_ts, cams, intr, W, H, rgb=None, leaf=0.01, half_window=0.5):
    """The same result as colorize_literal through a different route: per image the landed points lexsorted by (pixel, cloud
    order), the sequential rule per run, the thinning as one lexsort."""
    world = [world_points(s, poses[f]) for f, s in enumerate(scans)]
    merged, colours, listed = [], [], np.zeros(len(cams), np.uint8)
    for k in range(len(cams)):
        cloud = image_cloud(scans, frame_ts, world, image_ts[k], half_window)
        if len(cloud) == 0:
            continue
        listed[k] = 1
        pix, Z = project(cams[k], intr, cloud, W, H)
        idx = np.nonzero(pix >= 0)[0]
        order = idx[np.lexsort((idx, pix[idx]))]
        ps = pix[order]
        bounds = np.concatenate([[0], np.nonzero(ps[1:] != ps[:-1])[0] + 1, [len(ps)]])
        keep_pix, keep_pt = [], []
        for a, b in zip(bounds[:-1], bounds[1:]):
            zb, w = np.float32(np.inf), -1
            for i in order[a:b]:
                if float(Z[i]) + EPS < float(zb):
                    zb, w = np.float32(Z[i]), i
            if np.isfinite(zb):
                keep_pix.append(ps[a]); keep_pt.append(w)
        keep_pix = np.asarray(keep_pix, np.int64); keep_pt = np.asarray(keep_pt, np.int64)
        merged.append(cloud[keep_pt].reshape(-1, 3)); colours.append(_colour(rgb, k, keep_pix, W))
    merged = np.concatenate(merged).reshape(-1, 3) if merged else np.zeros((0, 3), np.float32)
    colours = np.concatenate(colours).reshape(-1, 3).astype(np.uint8) if colours else np.zeros((0, 3), np.uint8)
    xyz, col = _thin(merged, colours, leaf)
    return xyz.astype(np.float32), col.astype(np.uint8), listed
