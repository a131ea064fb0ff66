"""BALM2's voxel outlier removal on the H100 (lvba_lidar_voxel_residuals, lvba_lidar_remove_voxels,
lvba_lidar_remove_outliers) against the oracle of tests/lidar_outlier_oracle.py:
  * lambda_0 of every voxel on a small scene, config A, a scene with voxels seen from more than 128 poses and a reordered
    scene, and its sum against lvba_lidar_residual;
  * the device rule against the oracle rule on the device's own lambda_0, with duplicated voxels (bit-exact ties);
  * remove -> iterate in deterministic mode byte for byte against a fresh handle of the kept voxels -> reset_lm -> iterate:
    with and without constant poses, a pose_fixed change after a removal, big voxels, a voxel-map handle, two removals;
  * refused arguments leave the handle as its untouched twin;
  * damping_iter -> remove_outlier -> damping_iter on a scene with injected non-planar voxels;
  * the shim's evaluate_residual / remove_outlier (tests/shim/outliers_shim.cpp) and lvba_offline --outlier-ratio against the same
    sequence driven through the Python handle."""
import ctypes
import json
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest

import lidar_outlier_oracle as olo
from oracle import lidar_oracle as lo
from oracle import synth

pytestmark = pytest.mark.gpu
KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")
SUMMARY_KEYS = ("iterations", "accepted", "hessian_builds", "termination", "cost_first", "cost_last", "damping_last")


def _args(p):
    return [p[k] for k in KEYS]


def _opts(pkg, deterministic=0):
    o = pkg.lidar_default_opts()
    o.deterministic = deterministic
    return o


def _permute(vp, pi, cl, order):
    K = np.diff(vp); st = vp[:-1]
    pi2 = np.concatenate([pi[st[a]:st[a] + K[a]] for a in order]); cl2 = np.concatenate([cl[st[a]:st[a] + K[a]] for a in order])
    return np.concatenate([[0], np.cumsum(K[order])]).astype(np.int64), pi2, cl2


def _mixed(seed=77, W=300, n_small=1500, n_big=5):
    """ordinary voxels around a few seen from 129-260 poses, in a random voxel order"""
    rng = np.random.Generator(np.random.Philox(key=seed))
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp_b, pi_b, cl_b = synth.make_lidar(W, n_big, R_gt, p_gt, rng, k_lo=129, k_hi=260, half=W - 1)
    vp_s, pi_s, cl_s = synth.make_lidar(W, n_small, R_gt, p_gt, rng)
    vp = np.concatenate([vp_s, vp_b[1:] + vp_s[-1]]); pi = np.concatenate([pi_s, pi_b]); cl = np.concatenate([cl_s, cl_b])
    vp, pi, cl = _permute(vp, pi, cl, np.random.default_rng(seed).permutation(len(vp) - 1))
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    poses = np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1)
    return dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=poses)


_scenes = {}


def _scene(name, problem_small, problem_A):
    if name not in _scenes:
        if name == "small":
            _scenes[name] = problem_small
        elif name == "A":
            _scenes[name] = problem_A
        elif name == "big":
            _scenes[name] = _mixed()
        else:                                                         # reordered: the voxels of the small scene shuffled
            p = problem_small
            vp, pi, cl = _permute(p["vox_ptr"], p["pose_idx"], p["clusters"], np.random.default_rng(4).permutation(len(p["vox_ptr"]) - 1))
            _scenes[name] = dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=p["poses"])
    return _scenes[name]


@pytest.mark.parametrize("name", ["small", "A", "big", "reordered"])
def test_voxel_residuals_match_oracle(gpu_pkg, problem_small, problem_A, name):
    p = _scene(name, problem_small, problem_A)
    a = _args(p)
    P = gpu_pkg.LidarProblem(*a)
    lam = P.voxel_residuals()
    ref = olo.evaluate_residual(*a)
    assert lam.shape == ref.shape
    assert np.abs(lam - ref).max() <= 1e-9 * np.abs(ref).sum()
    tot = P.residual()
    assert abs(lam.sum() - tot) <= 1e-12 * abs(tot)
    moved = p["poses"].copy(); moved[:, 9:] += 0.01                       # at given poses; the handle's stay
    lam2 = P.voxel_residuals(moved)
    assert np.abs(lam2 - olo.evaluate_residual(*a[:3], moved)).max() <= 1e-9 * np.abs(ref).sum()
    assert P.voxel_residuals().tobytes() == lam.tobytes()
    P.close()


def _with_duplicates(p, n_dup=25, seed=8):
    """some voxels twice (each copy right after its original, or at the end): bit-exact ties in lambda_0"""
    vp, pi, cl = p["vox_ptr"], p["pose_idx"], p["clusters"]
    V = len(vp) - 1
    rng = np.random.default_rng(seed)
    order = list(range(V))
    for a in rng.choice(V, n_dup, replace=False):
        order.insert(order.index(a) + 1, a) if a % 2 else order.append(a)
    vp2, pi2, cl2 = _permute(vp, pi, cl, np.array(order))
    return dict(vox_ptr=vp2, pose_idx=pi2, clusters=cl2, poses=p["poses"])


@pytest.mark.parametrize("ratio", [0.0, 0.01, 0.1, 0.5, 0.9])
def test_device_rule_equals_oracle_on_device_lambda(gpu_pkg, problem_small, ratio):
    p = _with_duplicates(problem_small)
    a = _args(p)
    P = gpu_pkg.LidarProblem(*a)
    lam = P.voxel_residuals()
    assert len(np.unique(lam)) < len(lam)                                 # ties are there
    V = P.V
    removed = P.remove_outliers(ratio)
    want = olo.remove_outlier_loop(lam, ratio)
    assert np.array_equal(removed, want)
    assert P.V == V - want.sum()
    assert P.voxel_residuals().tobytes() == lam[~want].tobytes()         # the survivors, renumbered, same arithmetic
    P.close()


def _fresh_equal(pkg, P, p, removed, o, fixed=None, n_iter=6, poses=None):
    """P (a handle after its removals, at `poses`) iterates as a fresh handle of the kept voxels after reset_lm(o)"""
    vp, pi, cl = olo.kept_problem(p["vox_ptr"], p["pose_idx"], p["clusters"], removed)
    F = pkg.LidarProblem(vp, pi, cl, poses)
    F.reset_lm(o, pose_fixed=fixed)
    assert P.counts() == F.counts()
    for x, y in zip(P.structure(), F.structure()):
        assert np.array_equal(x, y)
    s = P.iterate(n_iter); t = F.iterate(n_iter)
    assert P.get_poses().tobytes() == F.get_poses().tobytes()
    assert all(s[k] == t[k] for k in SUMMARY_KEYS)
    g1, *_, b1 = P.get_system(); g2, *_, b2 = F.get_system()
    assert g1.tobytes() == g2.tobytes() and b1.tobytes() == b2.tobytes()
    F.close()


@pytest.mark.parametrize("case", ["plain", "pose_fixed", "fixed_after", "big", "only_big", "twice"])
def test_removal_equals_fresh_handle_deterministic(gpu_pkg, problem_small, case):
    p = _mixed(W=300, n_small=1500, n_big=5) if case in ("big", "only_big") else problem_small
    a = _args(p)
    W = len(p["poses"]); V = len(p["vox_ptr"]) - 1
    o = _opts(gpu_pkg, 1)
    fixed = (np.arange(W) < 3) if case == "pose_fixed" else None
    P = gpu_pkg.LidarProblem(*a)
    P.reset_lm(o, pose_fixed=fixed)
    P.iterate(2)
    now = P.get_poses()
    rng = np.random.default_rng(12)
    removed = rng.random(V) < 0.15
    if case == "big":
        K = np.diff(p["vox_ptr"])
        removed[np.nonzero(K > 128)[0][:2]] = True                        # two of the big voxels go, the others stay
    if case == "only_big":                                                # every voxel a batch CTA holds goes: no tiles left
        removed = np.diff(p["vox_ptr"]) <= 128
    if case == "twice":
        first = removed & (np.arange(V) % 2 == 0)
        P.remove_voxels(first)
        P.remove_voxels((removed & ~first)[~first])                       # in the renumbered order
    else:
        assert P.remove_voxels(removed) == V - removed.sum()
    assert P.V == V - removed.sum()
    assert P.get_poses().tobytes() == now.tobytes()
    if case == "fixed_after":
        fixed = np.arange(W) % 4 == 1
        P.reset_lm(o, pose_fixed=fixed)
    _fresh_equal(gpu_pkg, P, p, removed, o, fixed, poses=now)
    P.reset_state()
    assert P.get_poses().tobytes() == p["poses"].tobytes()                # poses0 stays
    P.close()


def test_voxel_map_handle_removal(gpu_pkg):
    scans, poses = synth.make_scan_scene(21, W=6, n_per_scan=4000)
    m = gpu_pkg.VoxelMap(scans, poses)
    g = m.export()
    P = m.lidar_problem(poses)
    o = _opts(gpu_pkg, 1)
    P.reset_lm(o)
    lam = P.voxel_residuals()
    assert np.abs(lam - olo.evaluate_residual(g["vox_ptr"], g["pose_idx"], g["clusters"], poses)).max() <= 1e-9 * np.abs(lam).sum()
    removed = P.remove_outliers(0.05)
    assert np.array_equal(removed, olo.remove_outlier_loop(lam, 0.05))
    _fresh_equal(gpu_pkg, P, dict(vox_ptr=g["vox_ptr"], pose_idx=g["pose_idx"], clusters=g["clusters"]), removed, o, poses=poses)
    P.close()
    m.close()


def test_refusals_leave_the_handle_unchanged(gpu_pkg, problem_small):
    p = problem_small
    a = _args(p)
    V = len(p["vox_ptr"]) - 1
    o = _opts(gpu_pkg, 1)
    A = gpu_pkg.LidarProblem(*a); B = gpu_pkg.LidarProblem(*a)
    for H in (A, B):
        H.reset_lm(o)
        H.iterate(1)                                                      # mid-solve: u, v and the Hessian flag carry over
    m = np.zeros(V, np.uint8); n = ctypes.c_int64(-7)
    assert A._lib.lvba_lidar_remove_voxels(A._h, None, ctypes.byref(n)) == -1      # a NULL mask
    assert n.value == -7
    for ratio in (math.nan, math.inf, 1.0, -0.1, 1.0 - 0.5 / V):
        with pytest.raises(gpu_pkg.LvbaError) as e:
            A.remove_outliers(ratio)
        assert e.value.status == -1
    with pytest.raises(gpu_pkg.LvbaError) as e:
        A.remove_voxels(np.ones(V, bool))
    assert e.value.status == -1
    bad = p["poses"].copy(); bad[0, 9] = math.nan
    A.set_poses(bad)
    with pytest.raises(gpu_pkg.LvbaError) as e:                            # a non-finite lambda_0: no threshold
        A.remove_outliers(0.1)
    assert e.value.status == -1
    A.set_poses(B.get_poses())
    assert A.V == V
    s = A.iterate(5); t = B.iterate(5)                                    # no reset: the LM state must be as it was
    assert A.get_poses().tobytes() == B.get_poses().tobytes() and all(s[k] == t[k] for k in SUMMARY_KEYS)
    A.close(); B.close()


def _injected_scene(seed=5, W=30, V=600, n_bad=25):
    """the small scene with n_bad voxels whose clusters come from a 1 m cube instead of a plane (at the true poses)"""
    p = synth.make_problem(W, V, 0, seed=seed, visual=False)
    rng = np.random.default_rng(seed)
    # fewer than reject_num at ratio 0.05, and in the first half: the walk stops after reject_num erased voxels, so the last
    # voxels at or above the threshold in walk order stay (the rule of remove_residual)
    bad = np.sort(rng.choice(V // 2, n_bad, replace=False))
    vp, pi, cl = p["vox_ptr"], p["pose_idx"], p["clusters"].copy()
    gt = p["poses_gt"]
    for a in bad:
        centre = gt[pi[vp[a]], 9:] + rng.uniform(-5, 5, 3)
        for s in range(vp[a], vp[a + 1]):
            R = gt[pi[s], :9].reshape(3, 3); t = gt[pi[s], 9:]
            n = int(cl[s, 9])
            pw = centre + rng.uniform(-0.5, 0.5, (n, 3))
            pb = (pw - t) @ R
            q = pb.T @ pb
            cl[s, :6] = (q[0, 0], q[0, 1], q[0, 2], q[1, 1], q[1, 2], q[2, 2])
            cl[s, 6:9] = pb.sum(0)
    p["clusters"] = cl
    return p, bad


def _rel_err(poses, gt):
    """gauge-free error: the translation of each pose relative to the next, against the truth"""
    def rel(x):
        R = x[:, :9].reshape(-1, 3, 3); t = x[:, 9:]
        return np.einsum("nji,nj->ni", R[:-1], t[1:] - t[:-1])
    return float(np.linalg.norm(rel(poses) - rel(gt), axis=1).mean())


def test_end_to_end_with_injected_outliers(gpu_pkg):
    p, bad = _injected_scene()
    a = _args(p)
    ratio = 0.05
    P = gpu_pkg.LidarProblem(*a)
    P.reset_lm()
    P.iterate(10)
    removed = P.remove_outliers(ratio)
    assert removed[bad].all()
    P.iterate(10)
    got = P.get_poses()
    ref, ref_removed = olo.damping_iter_with_removal(*a, ratio)
    assert np.array_equal(removed, ref_removed)
    assert np.abs(got - ref).max() <= 1e-6
    Q = gpu_pkg.LidarProblem(*a)                                           # the same chain without the removal
    Q.reset_lm(); Q.iterate(10); Q.reset_lm(); Q.iterate(10)
    assert _rel_err(got, p["poses_gt"]) < _rel_err(Q.get_poses(), p["poses_gt"])
    P.close(); Q.close()


ROOT = Path(__file__).resolve().parents[1]


def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


@pytest.mark.parametrize("ratio", [0.0, 0.1, 0.25])
def test_shim_remove_outlier_equals_oracle(gpu_pkg, tmp_path, ratio):
    exe = tmp_path / "outliers_shim"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tests" / "shim" / "outliers_shim.cpp"),
                        "-o", str(exe), *_link(gpu_pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), repr(ratio)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    d = json.loads(r.stdout.strip().splitlines()[-1])
    vp = np.array(d["vox_ptr"], np.int64); pi = np.array(d["pose_idx"], np.int32)
    cl = np.array(d["clusters"]).reshape(-1, 10); ps = np.array(d["poses"]).reshape(-1, 12)
    lam = np.array(d["lambda0"])
    ref = olo.evaluate_residual(vp, pi, cl, ps)
    assert np.abs(lam - ref).max() <= 1e-9 * np.abs(ref).sum()
    removed = olo.remove_outlier_loop(lam, ratio)                       # the oracle on the library's own lambda_0
    assert d["kept"] == np.nonzero(~removed)[0].tolist()
    assert d["n_removed"] == int(removed.sum())


def _tum_pose(line):
    from oracle import dataset_writer as dw
    v = np.array(line.split(), float)
    return np.concatenate([dw.quat_to_R(np.array([v[7], v[4], v[5], v[6]])).ravel(), v[1:4]])


def test_offline_outlier_ratio_equals_handle_sequence(gpu_pkg, tmp_path):
    """lvba_offline --deterministic --outlier-ratio R against damping_iter, remove_outliers(R), damping_iter on a handle of each
    global stage's voxel map, driven from Python with the poses the tool loaded"""
    from oracle import dataset_writer as dw
    exe = tmp_path / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(gpu_pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    W, ratio = 6, 0.05
    scans, poses = synth.make_scan_scene(23, W=W, n_per_scan=3000)
    rng = np.random.default_rng(23)
    noisy = poses.copy()
    for i in range(W):
        noisy[i, :9] = (noisy[i, :9].reshape(3, 3) @ synth.so3_exp(rng.normal(0, 0.008, (1, 3)))[0]).ravel()
        noisy[i, 9:] += rng.normal(0, 0.015, 3)
    data = tmp_path / "data"
    dw.write_lidar_dataset(data, scans, noisy)
    out = tmp_path / "opt.txt"
    r = subprocess.run([str(exe), "--data", str(data), "--out", str(out), "--stage1-voxel", "1.0", "--stage2-voxel", "1.0", "--deterministic",
                        "--outlier-ratio", repr(ratio)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    removed_tool = [json.loads(l)["outliers_removed"] for l in r.stdout.splitlines() if "outliers_removed" in l]
    assert len(removed_tool) == 2
    # the poses as the tool loads them: translation as written, rotation from the written (un-normalised) quaternion
    lines = [l for l in (data / "all_pcd_body" / "lidar_poses.txt").read_text().splitlines() if l and not l.startswith("#")]
    cur = np.array([_tum_pose(l) for l in lines if len(l.split()) == 8 and l.split()[0][0].isdigit()])
    assert cur.shape == (W, 12)
    o = gpu_pkg.lidar_default_opts(); o.deterministic = 1
    removed_py = []
    for _ in range(2):
        m = gpu_pkg.VoxelMap(scans, cur, 1.0)
        P = m.lidar_problem(cur)
        P.reset_lm(o); P.iterate(o.max_iter)
        removed_py.append(int(P.remove_outliers(ratio).sum()))
        P.iterate(o.max_iter)
        cur = P.get_poses()
        P.close(); m.close()
    assert removed_tool == removed_py and min(removed_py) > 0
    got = np.array([_tum_pose(l) for l in out.read_text().splitlines()])
    assert got.shape == (W, 12) and np.abs(got - cur).max() <= 1e-8
