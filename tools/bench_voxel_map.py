"""Boundary B3 measured on one GPU: raw scans -> device voxel map (lvba_voxel_map_create) -> plane voxels, and the
plane lookup.  Prints ONE JSON line.  bench.py runs this as a child process after its own timed region (rank 0, N = 1)
and attaches the line as `voxel_map`; it can also be run directly:

    python tools/bench_voxel_map.py [--scans 400] [--points 50000] [--voxel-size 1.0] [--repeats 3]

Workload (synthetic, seeded): a vehicle driving 0.5 m per scan along a street — ground plane, two facades 8 m to
either side, 10 % clutter — every scan sees the surfaces within 30 m.  20 M points by default (config C of the LM
bench corresponds to ~34 M).  Times: `ms_device` = CUDA events around the build passes inside the library,
`ms_call` = the whole ABI call from host memory (validation, H2D, build), best of `repeats` after one warm-up.
The CPU figure next to it is oracle/voxel_oracle.py (numpy group-by restatement, one thread) on a bounded sample."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def street_scans(n_scans, n_points, seed=0):
    rng = np.random.default_rng(seed)
    poses = np.zeros((n_scans, 12))
    scan_ptr = np.arange(n_scans + 1, dtype=np.int64) * n_points
    xyz = np.empty((n_scans * n_points, 3), np.float32)
    for i in range(n_scans):
        yaw = 0.02 * np.sin(0.05 * i)
        c, s = np.cos(yaw), np.sin(yaw)
        R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        p = np.array([0.5 * i, 0.3 * np.sin(0.02 * i), 0.0])
        poses[i, :9] = R.ravel(); poses[i, 9:] = p
        kind = rng.integers(0, 10, n_points)
        w = np.empty((n_points, 3))
        r = 30.0 * np.sqrt(rng.uniform(0, 1, n_points)); a = rng.uniform(0, 2 * np.pi, n_points)
        w[:, 0] = p[0] + r * np.cos(a); w[:, 1] = p[1] + r * np.sin(a); w[:, 2] = -1.37 + rng.normal(0, 0.01, n_points)      # ground
        wall = (kind >= 5) & (kind < 9)
        nw = int(wall.sum())
        w[wall, 0] = p[0] + rng.uniform(-30, 30, nw)
        w[wall, 1] = np.where(rng.integers(0, 2, nw) == 0, -7.73, 7.73) + rng.normal(0, 0.01, nw)
        w[wall, 2] = rng.uniform(-1.37, 4.0, nw)
        cl = kind == 9
        w[cl] = p + rng.uniform(-20, 20, (int(cl.sum()), 3))
        xyz[i * n_points:(i + 1) * n_points] = ((w - p) @ R).astype(np.float32)
    return xyz, scan_ptr, poses


def colorize_part(pkg, xyz, scan_ptr, poses, n_scans, n_cams=100, width=640, height=512, leaf=0.01):
    """Boundary B8 on the same scans: the coloured map of 100 cameras riding on every 4th pose (the 0.5 s window holds 11 scans),
    640x512 synthetic RGB, once with the poses and cameras (`after`) and once with perturbed poses and cameras (`before`).  `ms_call` is the second call
    of the size (the first pays cudaMalloc)."""
    try:
        frame_ts = 0.1 * np.arange(n_scans)
        ids = np.arange(0, n_scans, max(1, n_scans // n_cams))[:n_cams]
        Rci = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
        cams = np.zeros((len(ids), 12))
        for j, i in enumerate(ids):
            Rcw = Rci @ poses[i, :9].reshape(3, 3).T
            cams[j, :9] = Rcw.ravel(); cams[j, 9:] = -Rcw @ poses[i, 9:]
        intr = np.array([350.0, 350.0, 320.0, 256.0, -0.05, 0.01, 1e-4, -1e-4])
        yy, xx = np.mgrid[0:height, 0:width]
        rgb = np.stack([((xx * 3 + yy + 17 * k) % 256, (yy * 5 + 31 * k) % 256, (xx + yy * 2) % 256) for k in range(len(ids))])
        rgb = np.ascontiguousarray(np.moveaxis(rgb, 1, -1), np.uint8)
        rng = np.random.default_rng(5)
        before = poses.copy(); before[:, 9:] += rng.normal(0, 0.05, (n_scans, 3))
        cams_before = cams.copy(); cams_before[:, 9:] += rng.normal(0, 0.02, (len(ids), 3))     # the cameras before the optimisation
        cz = pkg.Colorizer(xyz, frame_ts, scan_ptr=scan_ptr)
        res = {}
        for name, ps, cm in (("warm-up", poses, cams), ("after", poses, cams), ("before", before, cams_before)):
            t0 = time.perf_counter()
            pts, col, listed, s = cz.run(ps, frame_ts[ids], cm, intr, width, height, rgb, leaf=leaf)
            dt = (time.perf_counter() - t0) * 1e3
            if name != "warm-up":
                res[name] = {"ms_device": s["ms_device"], "ms_call": dt, "projections": s["n_projections"],
                             "projections_per_s_device": s["n_projections"] / max(s["ms_device"], 1e-9) * 1e3,
                             "landed": s["n_landed"], "survivors": s["n_survivors"], "output_points": s["n_out"],
                             "listed": int(listed.sum()), "kernel_launches": s["kernel_launches"], "peak_device_bytes": s["peak_device_bytes"]}
        cz.close()
        return {"workload": f"{len(ids)} cameras {width}x{height} RGB over {n_scans} scans, window 0.5 s, leaf {leaf} m", **res}
    except Exception as e:          # noqa: BLE001
        return {"error": repr(e)[:300]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=400)
    ap.add_argument("--points", type=int, default=50000)
    ap.add_argument("--voxel-size", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--queries", type=int, default=200000)
    ap.add_argument("--cpu-sample-scans", type=int, default=8)
    args = ap.parse_args()
    import __graft_entry__ as graft
    pkg = graft.load_package()
    pkg.load_library()
    if pkg.device_count() < 1:
        print(json.dumps({"error": "no CUDA device (no CPU fallback)"})); return 1
    xyz, scan_ptr, poses = street_scans(args.scans, args.points)
    N = len(xyz)
    best_call, best_dev, summ, g = 1e30, 1e30, None, None
    for rep in range(args.repeats + 1):
        t0 = time.perf_counter()
        m = pkg.VoxelMap(xyz, poses, args.voxel_size, scan_ptr=scan_ptr)
        dt = (time.perf_counter() - t0) * 1e3
        if rep > 0:
            best_call = min(best_call, dt); best_dev = min(best_dev, m.summary["ms_device"])
        summ = m.summary
        if rep < args.repeats:
            m.close()
    g = m.export()
    vp, pi, cl = g["vox_ptr"], g["pose_idx"], g["clusters"]
    V = len(vp) - 1
    checks = {"every voxel seen from >= 2 poses": bool(np.all(np.diff(vp) >= 2)),
              "min_ps points per voxel": bool(np.all(np.add.reduceat(cl[:, 9], vp[:-1]) >= 15)) if V else True,
              "keys ascending": bool(np.all(np.diff(g["key"][:, 0]) >= 0)),
              "points conserved (<= input)": bool(cl[:, 9].sum() <= N)}
    rng = np.random.default_rng(1)
    X = np.column_stack([rng.uniform(0, 0.5 * args.scans, args.queries), rng.uniform(-9, 9, args.queries), rng.uniform(-2, 4, args.queries)])
    m.lookup(X)                                  # warm-up at the same size: the first call of a size pays cudaMalloc (the pool is cold)
    t0 = time.perf_counter(); nd = m.lookup(X); t_lookup = (time.perf_counter() - t0) * 1e3
    m.close()
    # CPU restatement on a bounded sample (first scans only)
    cpu = None
    if args.cpu_sample_scans > 0:
        from oracle import voxel_oracle as vox
        k = min(args.cpu_sample_scans, args.scans)
        scans = [xyz[scan_ptr[j]:scan_ptr[j + 1]] for j in range(k)]
        t0 = time.perf_counter(); vox.voxelize(scans, poses[:k], args.voxel_size); tc = time.perf_counter() - t0
        cpu = {"points_per_s": k * args.points / tc, "kind": "port (numpy, 1 thread)", "sample": f"{k} scans x {args.points} points",
               "note": "a single-thread numpy restatement: reported for orientation, not a baseline to quote a speed-up against"}
    out = {"workload": f"{args.scans} scans x {args.points} points (street scene), root voxel {args.voxel_size} m, layer_limit 2",
           "n_points": int(N), "n_voxels": int(summ["n_voxels"]), "nnz": int(summ["nnz"]), "n_nodes": summ["n_nodes"],
           "ms_device": best_dev, "ms_call": best_call, "points_per_s_device": N / (best_dev * 1e-3), "points_per_s_call": N / (best_call * 1e-3),
           "algorithmic_GBps_device": (12.0 * N + 80.0 * summ["nnz"]) / (best_dev * 1e-3) / 1e9,
           "h2d_bytes": int(summ["h2d_bytes"]), "kernel_launches": int(summ["kernel_launches"]),
           "lookup": {"queries": int(args.queries), "ms_call": t_lookup, "note": "second call of this size (the first pays cudaMalloc)", "hit_fraction": float(np.mean(np.any(nd != 0, axis=1)))},
           "checks": checks, "cpu": cpu, "depth": None}
    print(json.dumps(out), flush=True)          # B3 alone first: it survives whatever the B4 part below does
    # ---- boundary B4 on the same scans: grid of world points + depth images of cameras riding on every 25th pose
    depth = None
    try:
        frame_ts = 0.1 * np.arange(args.scans)
        t0 = time.perf_counter(); dg = pkg.DepthGrid(xyz, poses, frame_ts, 0.5, scan_ptr=scan_ptr); t_grid_cold = (time.perf_counter() - t0) * 1e3
        cold_device = dg.summary["ms_device"]
        dg.close()                                # its ~2 GB of buffers go back to the library's pool; the second build is the steady state
        t0 = time.perf_counter(); dg = pkg.DepthGrid(xyz, poses, frame_ts, 0.5, scan_ptr=scan_ptr); t_grid = (time.perf_counter() - t0) * 1e3
        ids = np.arange(0, args.scans, max(1, args.scans // 16))[:16]
        Rci = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
        cams = np.zeros((len(ids), 12))
        for j, i in enumerate(ids):
            Rcw = Rci @ poses[i, :9].reshape(3, 3).T
            cams[j, :9] = Rcw.ravel(); cams[j, 9:] = -Rcw @ poses[i, 9:]
        intr = np.array([700.0, 700.0, 640.0, 512.0, -0.05, 0.01, 1e-4, -1e-4])
        dg.render(cams[:2], frame_ts[ids[:2]], intr, 1280, 1024)
        img, info = dg.render(cams, frame_ts[ids], intr, 1280, 1024)
        uv = np.column_stack([rng.uniform(0, 1279, 160000), rng.uniform(0, 1023, 160000)]).astype(np.float32)
        kp_ptr = np.arange(len(ids) + 1, dtype=np.int64) * 10000
        _, valid, binfo = dg.backproject(cams, frame_ts[ids], intr, 1280, 1024, kp_ptr, uv)
        depth = {"grid": {"ms_call": t_grid, "ms_device": dg.summary["ms_device"], "ms_call_first": t_grid_cold, "ms_device_first": cold_device, "n_voxels": dg.summary["n_voxels"], "n_pairs": dg.summary["n_pairs"]},
                 "render": {"images": int(len(ids)), "size": "1280x1024", "ms_device": info["ms_device"], "ms_call": info["ms_total"],
                            "points_projected": int(info["work_chunks"]) * 64, "projections_per_s_device": info["work_chunks"] * 64 / max(info["ms_device"], 1e-9) * 1e3,
                            "filled_fraction": float(np.mean(img > 0)), "kernel_launches": int(info["kernel_launches"])},
                 "backproject": {"keypoints": 160000, "valid": int(valid.sum()), "ms_call": binfo["ms_total"], "ms_device": binfo["ms_device"],
                                 "d2h_bytes": int(binfo["d2h_bytes"])}}
        dg.close()
    except Exception as e:          # noqa: BLE001
        depth = {"error": repr(e)[:300]}
    out["depth"] = depth
    out["colorize"] = colorize_part(pkg, xyz, scan_ptr, poses, args.scans)
    print(json.dumps(out), flush=True)
    return 0 if all(checks.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
