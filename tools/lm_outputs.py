"""Every LM entry point of the library in deterministic mode on fixed inputs: writes each output array and every summary field
but the times to one .npz, so that two builds of the library can be compared bit for bit (LVBA_B200_DEV_LIB=<file under
global-lvba_b200/> loads another build).  Needs a GPU.

    python tools/lm_outputs.py OUT.npz
    python tools/lm_outputs.py --compare A.npz B.npz      (exit 1 unless both hold the same arrays, bit for bit)
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
import __graft_entry__ as graft  # noqa: E402
from oracle import synth  # noqa: E402
import visual_big_scene as vs  # noqa: E402

TIMES = ("ms_total", "ms_setup", "ms_build", "ms_solve", "ms_residual")
out = {}


def put(name, *arrays, sums=()):
    for i, a in enumerate(arrays):
        out[f"{name}/{i}"] = np.asarray(a)
    for j, s in enumerate(sums):
        for k, v in s.items():
            if k not in TIMES:
                out[f"{name}/sum{j}/{k}"] = np.asarray(v)


def big_voxel_problem():
    """300 poses, five voxels seen from 200-260 of them among 1500 ordinary ones (tests/test_deterministic_gpu.py)"""
    rng = np.random.Generator(np.random.Philox(key=77))
    W = 300
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp_b, pi_b, cl_b = synth.make_lidar(W, 5, R_gt, p_gt, rng, k_lo=200, k_hi=260, half=W - 1)
    vp_s, pi_s, cl_s = synth.make_lidar(W, 1500, R_gt, p_gt, rng)
    vp = np.concatenate([vp_s, vp_b[1:] + vp_s[-1]]); pi = np.concatenate([pi_s, pi_b]); cl = np.concatenate([cl_s, cl_b])
    assert np.diff(vp).max() > 128
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    return vp, pi, cl, np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1)


def noisy_scans(seed, W, n, rot, trans, noise_seed):
    scans, poses = synth.make_scan_scene(seed, W=W, n_per_scan=n)
    rng = np.random.default_rng(noise_seed)
    for i in range(1, len(poses)):
        poses[i, :9] = (poses[i, :9].reshape(3, 3) @ synth.so3_exp(rng.normal(0, rot, (1, 3)))[0]).ravel()
        poses[i, 9:] += rng.normal(0, trans, 3)
    return scans, poses


def main(path):
    pkg = graft.load_package()
    pkg.load_library()
    lo = pkg.lidar_default_opts(); lo.deterministic = 1

    vp, pi, cl, poses = big_voxel_problem()
    x, s = pkg.lidar_lm(vp, pi, cl, poses, opts=lo)
    put("lidar_lm", x, sums=[s])
    P = pkg.LidarProblem(vp, pi, cl, poses)
    P.reset_lm(lo)
    s1 = P.iterate(3); s2 = P.iterate(7)
    x = P.get_poses()
    P.reset_lm(lo)
    s3 = P.iterate(0)                      # a reset keeps the costs of the last solve until the next pass
    P.close()
    put("LidarProblem.iterate", x, sums=(s1, s2, s3))

    G = np.load(ROOT / "tests" / "golden" / "window_problem.npz")
    x, sums, tot = pkg.lidar_lm_batch(G["win_ptr"], G["vox_ptr"], G["pose_idx"], G["clusters"], G["poses"], opts=lo)
    put("lidar_lm_batch", x, sums=sums + [tot])

    scans, noisy = noisy_scans(21, 6, 4000, 0.01, 0.02, 3)
    m = pkg.VoxelMap(scans, noisy)
    x, s = m.lidar_lm(noisy, opts=lo)
    m.close()
    put("VoxelMap.lidar_lm", x, sums=[s])
    sizes = [5, 4, 1, 6]
    scans, noisy = noisy_scans(13, sum(sizes), 3000, 0.004, 0.01, 4)
    m = pkg.VoxelMap(scans, noisy, 1.0, win_ptr=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32))
    x, sums, tot = m.lidar_lm_batch(noisy, opts=lo)
    m.close()
    put("VoxelMap.lidar_lm_batch", x, sums=sums + [tot])

    p = vs.make_scene(23, M=300, n_short=250, long_tracks=((129, 0), (300, 0), (700, 100), (150, 40)))
    for name, losses in [("none", (None, None)), ("huber", ((pkg.LOSS_HUBER, 1.0), (pkg.LOSS_HUBER, 0.1))),
                         ("cauchy", ((pkg.LOSS_CAUCHY, 1.0), (pkg.LOSS_CAUCHY, 0.1)))]:
        vo = pkg.visual_default_opts(*losses); vo.deterministic = 1
        q, t, X, s = pkg.visual_lm(*vs.args(p), opts=vo)
        put(f"visual_lm/{name}", q, t, X, sums=[s])
    vo = pkg.visual_default_opts(); vo.deterministic = 1
    V = pkg.VisualProblem(*vs.args(p))
    V.reset_lm(vo)
    s1 = V.iterate(4); s2 = V.iterate(46)
    q, t, X = V.get_state()
    V.reset_lm(vo)
    s3 = V.iterate(0)
    V.close()
    put("VisualProblem.iterate", q, t, X, sums=(s1, s2, s3))
    np.savez(path, **out)
    print(f"{len(out)} arrays -> {path}")


def compare(a, b):
    A, B = np.load(a), np.load(b)
    bad = sorted(set(A.files) ^ set(B.files)) + [k for k in A.files if k in B.files and
                                                 (A[k].dtype != B[k].dtype or A[k].tobytes() != B[k].tobytes())]
    print(f"{len(A.files)} / {len(B.files)} arrays, {len(bad)} differ" + (f": {bad[:20]}" if bad else ""))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(compare(sys.argv[2], sys.argv[3]) if sys.argv[1] == "--compare" else main(sys.argv[1]))
