"""Deterministic mode of both LM paths (lvba_lidar_opts / lvba_visual_opts ::deterministic) on the GPU: identical inputs give
byte-identical systems, steps, states and summaries on fresh handles and in separate processes, and the results agree with the
default mode and the oracles.  The fixed-order tables themselves are checked without a GPU in tests/test_deterministic_emu.py."""
import os
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

from oracle import cpu_ref
from oracle import lidar_oracle as lo
from oracle import synth
from oracle import visual_oracle as vo

sys.path.insert(0, str(Path(__file__).resolve().parent))
import visual_big_scene as vs  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
# wall-clock and CUDA-event times differ from run to run; everything else in a summary must not
TIMES = ("ms_total", "ms_setup", "ms_build", "ms_solve", "ms_residual")


def _opts(pkg, det):
    o = pkg.lidar_default_opts()
    o.deterministic = int(det)
    return o


def _summary(s):
    return {k: v for k, v in s.items() if k not in TIMES}


def _run(pkg, p, det=True, u=0.01):
    """build -> system, one damped solve, then a full 10-pass LM from the same start, all on one fresh handle"""
    P = pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    try:
        P.reset_lm(_opts(pkg, det))
        r = P.build()
        g, br, bc, bl = P.get_system()
        dx = P.solve(u)
        P.reset_state()
        P.reset_lm(_opts(pkg, det))
        s = P.iterate(10)
        poses = P.get_poses()
    finally:
        P.close()
    return dict(r=np.float64(r), g=g, H=bl, dx=dx, poses=poses), _summary(s)


def _big_voxel_problem():
    """300 poses, five voxels seen from 200-260 of them among ordinary ones (as tests/test_zz_wide_gpu.py)"""
    rng = np.random.Generator(np.random.Philox(key=77))
    W = 300
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp_b, pi_b, cl_b = synth.make_lidar(W, 5, R_gt, p_gt, rng, k_lo=200, k_hi=260, half=W - 1)
    vp_s, pi_s, cl_s = synth.make_lidar(W, 1500, R_gt, p_gt, rng)
    vp = np.concatenate([vp_s, vp_b[1:] + vp_s[-1]]); pi = np.concatenate([pi_s, pi_b]); cl = np.concatenate([cl_s, cl_b])
    order = np.random.default_rng(1).permutation(len(vp) - 1)
    K = np.diff(vp); starts = vp[:-1]
    pi = np.concatenate([pi[starts[a]:starts[a] + K[a]] for a in order]); cl = np.concatenate([cl[starts[a]:starts[a] + K[a]] for a in order])
    vp = np.concatenate([[0], np.cumsum(K[order])])
    assert np.diff(vp).max() > 128
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    poses = np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1)
    return dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=poses)


@pytest.fixture(scope="module")
def cfg_c():
    return synth.make_config("C", visual=False)


@pytest.fixture(scope="module")
def big():
    return _big_voxel_problem()


VKEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


def _vopts(pkg, det):
    o = pkg.visual_default_opts()
    o.deterministic = int(det)
    return o


def _vrun(pkg, p, det=True):
    """one step (steps, S, rhs) and then a full LM from the same start, on one fresh handle"""
    args = [p[k] for k in VKEYS]
    P = pkg.VisualProblem(*args)
    try:
        P.reset_lm(_vopts(pkg, det))
        cs, ps, mc, c = P.step(1e4)
        _, rhs, _, _, S = P.get_system()
        P.reset_state()
        P.reset_lm(_vopts(pkg, det))
        s = P.iterate(50)
        q, t, X = P.get_state()
    finally:
        P.close()
    return dict(cs=cs, ps=ps, mc=np.float64(mc), c=np.float64(c), rhs=rhs, S=S, q=q, t=t, X=X), _summary(s)


def _check_visual(pkg, p):
    runs = [_vrun(pkg, p) for _ in range(3)]
    a, sa = runs[0]
    for b, sb in runs[1:]:
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert sa == sb
    d, sd = _vrun(pkg, p, det=False)
    for k in ("S", "rhs"):
        assert np.abs(a[k] - d[k]).max() <= 1e-12 * np.abs(d[k]).max(), k
    return a, sa, sd


def _check_reproducible_and_close(pkg, p):
    runs = [_run(pkg, p) for _ in range(3)]
    a, sa = runs[0]
    for b, sb in runs[1:]:
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert sa == sb
    d, sd = _run(pkg, p, det=False)
    for k in ("H", "g"):
        assert np.abs(a[k] - d[k]).max() <= 1e-12 * np.abs(d[k]).max(), k
    assert abs(a["r"] - d["r"]) <= 1e-12 * abs(d["r"])
    return a, sa, sd


def test_config_C_is_bit_reproducible(gpu_pkg, cfg_c):
    a, sa, sd = _check_reproducible_and_close(gpu_pkg, cfg_c)
    assert abs(sa["cost_last"] - sd["cost_last"]) <= 1e-6 * sd["cost_last"]
    p = cfg_c
    _, ca = cpu_ref.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], threads=16)
    assert abs(sa["cost_last"] - ca["cost_last"]) <= 1e-6 * abs(ca["cost_last"])
    # the pose system of 2000 poses takes the substructured (chunked) solve, whose separator SYRK the mode changes
    import solver_systems as ss
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    P.build()
    g, br, bc, bl = P.get_system()
    P.close()
    first, dadd = ss.damped(br, bc, bl, len(p["poses"]), 0.01)
    _, _, info = gpu_pkg.env_solve(first, bl, dadd, -g.ravel())
    assert info["path"] == gpu_pkg.SOLVE_CHUNKED, info


def test_config_C_visual_is_bit_reproducible(gpu_pkg):
    p = synth.make_config("C")
    a, sa, sd = _check_visual(gpu_pkg, p)
    assert abs(sa["cost_last"] - sd["cost_last"]) <= 1e-6 * sd["cost_last"]
    _, _, _, cb = cpu_ref.visual_lm(*[p[k] for k in VKEYS], threads=16)
    assert abs(sa["cost_last"] - cb["cost_last"]) <= 1e-6 * abs(cb["cost_last"])


def test_big_landmarks_are_bit_reproducible_and_match_the_oracle(gpu_pkg):
    p = vs.make_scene(23, M=300, n_short=250, long_tracks=((129, 0), (300, 0), (700, 100), (150, 40)))
    P = gpu_pkg.VisualProblem(*vs.args(p))
    assert P.big_counts()["n_big"] == 4
    P.close()
    a, sa, _ = _check_visual(gpu_pkg, p)
    pr, info = vo.ceres_lm(vo.VisualProblem(*vs.args(p)))
    assert sa["iterations"] == info["iters"]
    assert abs(sa["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    outs = [gpu_pkg.visual_lm(*vs.args(p), opts=_vopts(gpu_pkg, True)) for _ in range(2)]
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert x.tobytes() == y.tobytes()


def test_big_voxels_are_bit_reproducible_and_match_the_oracle(gpu_pkg, big):
    p = big
    a, sa, _ = _check_reproducible_and_close(gpu_pkg, p)
    W = len(p["poses"])
    r_ref, g_ref, blocks = lo.acc_evaluate2(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], W)
    assert abs(a["r"] - r_ref) <= 1e-8 * abs(r_ref)
    assert np.abs(a["g"] - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    ref_poses, info = lo.damping_iter(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    assert abs(sa["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"]
    assert np.abs(a["poses"] - ref_poses).max() <= 1e-6


def test_one_shot_calls_are_bit_reproducible(gpu_pkg, big):
    p = big
    outs = [gpu_pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], opts=_opts(gpu_pkg, True)) for _ in range(3)]
    for o, s in outs[1:]:
        assert o.tobytes() == outs[0][0].tobytes()
        assert _summary(s) == _summary(outs[0][1])


def test_window_batch_is_bit_reproducible_and_matches_the_oracle(gpu_pkg):
    p = synth.make_window_problem([20, 20, 14, 6, 10, 12, 2], [260, 300, 170, 90, 12, 0, 40], seed=23)
    runs = [gpu_pkg.lidar_lm_batch(p["win_ptr"], p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], opts=_opts(gpu_pkg, True))
            for _ in range(3)]
    poses, sums, _ = runs[0]
    for q, s, _ in runs[1:]:
        assert q.tobytes() == poses.tobytes()
        assert [_summary(x) for x in s] == [_summary(x) for x in sums]
    for w, win in enumerate(p["windows"]):
        lo_, hi_ = p["win_ptr"][w], p["win_ptr"][w + 1]
        if len(win["vox_ptr"]) - 1 < 3 * (hi_ - lo_):
            assert sums[w]["termination"] == 6 and np.array_equal(poses[lo_:hi_], p["poses"][lo_:hi_])
            continue
        ref, info = lo.damping_iter(win["vox_ptr"], win["pose_idx"], win["clusters"], win["poses"])
        assert abs(sums[w]["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"]
        assert np.abs(poses[lo_:hi_] - ref).max() <= 1e-6


CHILD = """
import hashlib, sys
import numpy as np
sys.path.insert(0, %r)
import __graft_entry__ as graft
from oracle import synth
pkg = graft.load_package(); pkg.load_library()
p = synth.make_config("C")
o = pkg.lidar_default_opts(); o.deterministic = 1
poses, s = pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], opts=o)
v = pkg.visual_default_opts(); v.deterministic = 1
q, t, X, sb = pkg.visual_lm(*[p[k] for k in ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")], opts=v)
h = hashlib.sha256()
for a in (poses, q, t, X):
    h.update(np.ascontiguousarray(a).tobytes())
print("DIGEST", h.hexdigest(), s["iterations"], s["accepted"], sb["iterations"], sb["accepted"])
""" % str(ROOT)


def test_two_processes_give_the_same_poses(gpu_pkg):
    digests = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", textwrap.dedent(CHILD)], capture_output=True, text=True, timeout=900,
                           cwd=str(ROOT), env=dict(os.environ))
        assert r.returncode == 0, r.stderr[-3000:]
        digests.append([ln for ln in r.stdout.splitlines() if ln.startswith("DIGEST")][0])
    assert digests[0] == digests[1], digests


def test_offline_tool_writes_the_same_trajectory_twice(gpu_pkg, tmp_path):
    """lvba_offline --deterministic --window on the synthetic dataset of tests/test_zz_offline_gpu.py: byte-identical TUM files"""
    from oracle import dataset_writer as dw
    exe = tmp_path / "lvba_offline"
    cmd = ["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
           str(gpu_pkg.LIB_PATH), f"-Wl,-rpath,{gpu_pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    scans, poses = synth.make_scan_scene(17, W=12, n_per_scan=4000)
    rng = np.random.default_rng(5)
    noisy = poses.copy()
    for i in range(1, len(noisy)):
        noisy[i, :9] = (noisy[i, :9].reshape(3, 3) @ synth.so3_exp(rng.normal(0, 0.008, (1, 3)))[0]).ravel()
        noisy[i, 9:] += rng.normal(0, 0.015, 3)
    data = tmp_path / "data"
    dw.write_lidar_dataset(data, scans, noisy)
    outs = []
    for k in range(2):
        out = tmp_path / f"opt{k}.txt"
        r = subprocess.run([str(exe), "--data", str(data), "--out", str(out), "--window", "4", "--stage1-voxel", "1.0",
                            "--stage2-voxel", "0.5", "--deterministic"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert '"stage": 2' in r.stdout
        outs.append(out.read_bytes())
    assert outs[0] == outs[1]


def test_offline_tool_visual_stage_writes_the_same_model_twice(gpu_pkg, tmp_path):
    """lvba_offline --deterministic --visual on the scene of tests/test_zz_offline_gpu.py: byte-identical trajectory, images.txt
    and points3D.txt"""
    import visual_scene
    exe = tmp_path / "lvba_offline"
    cmd = ["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
           str(gpu_pkg.LIB_PATH), f"-Wl,-rpath,{gpu_pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    data = tmp_path / "data"
    visual_scene.make(data, seed=3, W=8, n_landmarks=700)
    outs = []
    for k in range(2):
        tum = tmp_path / f"opt{k}.txt"
        r = subprocess.run([str(exe), "--data", str(data), "--config", str(data / "config.yaml"), "--visual", "--deterministic",
                            "--out", str(tum)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        assert '"stage": "visual"' in r.stdout
        sparse = data / "Colmap" / "sparse"
        outs.append([tum.read_bytes(), (sparse / "images.txt").read_bytes(), (sparse / "points3D.txt").read_bytes()])
        for f in ("images.txt", "points3D.txt"):
            (sparse / f).unlink()
    assert outs[0] == outs[1]
