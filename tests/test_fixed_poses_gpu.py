"""Constant poses in the LiDAR LM (lvba_lidar_opts::pose_fixed) on the H100, against the oracle with the same constant set
(tests/lidar_fixed_oracle.py) at the tolerances of tests/test_window_batch_gpu.py: the one-shot call for several sets and every
pose constant, NULL and all-zero masks, reproducible deterministic solves, the handle's row system and re-planning resets,
voxels seen from more than 128 poses on an any-width envelope, the batched window LM and the voxel-map entry points."""
from pathlib import Path

import numpy as np
import pytest

import lidar_fixed_oracle as lf
from oracle import lidar_oracle as lo
from oracle import synth

pytestmark = pytest.mark.gpu
REF = np.load(Path(__file__).parent / "golden" / "ref_balm.npz")
KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")
SUMMARY_KEYS = ("iterations", "accepted", "hessian_builds", "termination", "cost_first", "cost_last", "damping_last")


def _args(p):
    return [p[k] for k in KEYS]


def _opts(pkg, deterministic=0):
    o = pkg.lidar_default_opts()
    o.deterministic = deterministic
    return o


def _check_vs_oracle(got, s, ref, info, fixed, poses0):
    assert s["iterations"] == info["iters"]
    last = info["trace"][-1] if info["trace"] else None
    slack = 1 if last is not None and abs(last["r1"] - last["r2"]) <= 1e-7 * last["r1"] else 0    # test_window_batch_gpu.py
    assert abs(s["accepted"] - info["accepted"]) <= slack
    assert abs(s["cost_first"] - info["r_first"]) <= 1e-8 * info["r_first"]
    assert abs(s["cost_last"] - info["r_last"]) <= 1e-6 * info["r_last"]
    assert np.abs(got - ref).max() <= 1e-6
    assert got[fixed].tobytes() == poses0[fixed].tobytes()                      # constant poses: the same bytes


def _sets(W):
    rng = np.random.default_rng(9)
    return {"pose0": lf.mask_of(W, [0]), "first_k": np.arange(W) <= W // 4, "third": rng.random(W) < 1 / 3}


@pytest.mark.parametrize("name", ["pose0", "first_k", "third"])
def test_lm_with_constant_set_matches_oracle(gpu_pkg, problem_small, name):
    p = problem_small
    a = _args(p)
    fixed = _sets(len(p["poses"]))[name]
    got, s = gpu_pkg.lidar_lm(*a, pose_fixed=fixed)
    ref, info = lf.damping_iter_fixed(*a, fixed)
    _check_vs_oracle(got, s, ref, info, fixed, p["poses"])
    assert s["cost_last"] < s["cost_first"]


def test_every_pose_constant(gpu_pkg, problem_small):
    p = problem_small
    a = _args(p)
    fixed = np.ones(len(p["poses"]), bool)
    for det in (0, 1):
        got, s = gpu_pkg.lidar_lm(*a, opts=_opts(gpu_pkg, det), pose_fixed=fixed)
        assert got.tobytes() == p["poses"].tobytes()
        assert (s["iterations"], s["accepted"], s["hessian_builds"], s["termination"]) == (0, 0, 0, 1)   # LVBA_TERM_FUNCTION_TOL
        r = lo.only_residual(*a) / (len(p["vox_ptr"]) - 1)
        assert s["cost_first"] == s["cost_last"] and abs(s["cost_first"] - r) <= 1e-9 * r


def test_null_and_all_zero_masks_are_the_same_bits(gpu_pkg, problem_small):
    a = _args(problem_small)
    o = _opts(gpu_pkg, 1)
    x, s = gpu_pkg.lidar_lm(*a, opts=o)
    y, t = gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=np.zeros(len(a[3]), bool))
    assert x.tobytes() == y.tobytes() and all(s[k] == t[k] for k in SUMMARY_KEYS)


def test_masked_deterministic_solve_is_reproducible(gpu_pkg, problem_small):
    a = _args(problem_small)
    fixed = _sets(len(a[3]))["third"]
    o = _opts(gpu_pkg, 1)
    runs = [gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=fixed) for _ in range(2)]
    P = gpu_pkg.LidarProblem(*a)
    P.reset_lm(o, pose_fixed=fixed)
    s = P.iterate(o.max_iter)
    runs.append((P.get_poses(), s))
    P.close()
    for x, t in runs[1:]:
        assert x.tobytes() == runs[0][0].tobytes() and all(t[k] == runs[0][1][k] for k in SUMMARY_KEYS)


def _dense(br, bc, blocks, n):
    H = np.zeros((6 * n, 6 * n))
    for r, c, b in zip(br, bc, blocks):
        H[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
        if r != c:
            H[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
    return H


@pytest.mark.parametrize("level", ["L1", "L2"])
def test_handle_row_system_and_first_step(gpu_pkg, level):
    """rows / structure / get_system / solve over the free rows, against the oracle's restricted system and the first step on
    the H and g the reference's own source computed."""
    a = [REF[f"{level}_{k}"] for k in KEYS]
    W = len(a[3])
    rs, g_all, blocks = lo.acc_evaluate2(*a, W)
    H_all = lo.assemble_dense(blocks, W)
    P = gpu_pkg.LidarProblem(*a)
    assert np.array_equal(P.rows(), np.arange(W))
    for fixed in (lf.mask_of(W, [0]), np.arange(W) % 3 == 1, np.arange(W) < W // 2):
        P.reset_lm(pose_fixed=fixed)
        free = np.flatnonzero(~fixed)
        assert np.array_equal(P.rows(), free)
        r = P.build()
        assert abs(r - rs) <= 1e-9 * rs
        g, br, bc, bl = P.get_system()
        Hf, gf = lf.restricted(H_all, g_all, fixed)
        assert g.shape == (len(free), 6)
        assert np.abs(g.ravel() - gf).max() <= 1e-7 * np.abs(gf).max()
        assert np.abs(_dense(br, bc, bl, len(free)) - Hf).max() <= 1e-7 * np.abs(Hf).max()
        dx = P.solve(0.01).reshape(W, 6)
        assert np.all(dx[fixed] == 0)
        want = lf.first_step(REF[f"{level}_H"], REF[f"{level}_g"], 0.01, fixed)
        assert np.abs(dx - want).max() <= 1e-6 * np.abs(want).max()
        c = P.counts()
        assert c["n_blocks_env"] == len(br) and c["nnz"] == len(a[1])
        row = np.full(W, -1); row[free] = np.arange(len(free))             # the row system's pairs and blocks, restated
        pairs, blocks_nz = 0, set()
        vp, pi = a[0], a[1]
        for v in range(len(vp) - 1):
            rr = [int(row[q]) for q in pi[vp[v]:vp[v + 1]] if row[q] >= 0]
            pairs += len(rr) * (len(rr) - 1) // 2
            blocks_nz.update((x, y) for i, x in enumerate(rr) for y in rr[i:])
        assert c["n_pairs"] == pairs and c["n_blocks_nonzero"] == len(blocks_nz)
    P.close()


def test_replanning_reset_equals_one_shot(gpu_pkg, problem_small):
    """After a re-planning reset, iterate gives the bits of the one-shot call with that mask; a reset back to no mask gives the
    bits of the unmasked call again."""
    a = _args(problem_small)
    W = len(a[3])
    o = _opts(gpu_pkg, 1)
    P = gpu_pkg.LidarProblem(*a)
    for fixed in (_sets(W)["first_k"], _sets(W)["third"], None, np.ones(W, bool), lf.mask_of(W, [0])):
        want, ws = gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=fixed)
        P.reset_state()
        P.reset_lm(o, pose_fixed=np.zeros(W, bool) if fixed is None else fixed)
        s = P.iterate(o.max_iter)
        assert P.get_poses().tobytes() == want.tobytes()
        assert all(s[k] == ws[k] for k in ("iterations", "accepted", "termination", "cost_first", "cost_last"))
        assert len(P.rows()) == (W if fixed is None else int((~fixed).sum()))
    P.close()


def test_big_voxels_on_a_wide_envelope(gpu_pkg):
    """Voxels seen from 129-260 poses (the big-voxel passes) coupling poses far apart (the any-width solve), with a mask."""
    from test_deterministic_emu import mixed_problem
    p = mixed_problem(seed=31, W=300, n_small=1500, n_big=5)
    a = _args(p)
    W = len(p["poses"])
    assert np.diff(p["vox_ptr"]).max() > 128
    fixed = np.arange(W) % 4 == 0
    P = gpu_pkg.LidarProblem(*a)
    P.reset_lm(pose_fixed=fixed)
    _, br, bc, _ = P.get_system()
    assert (br - bc).max() > 30                                                  # taller than the register window
    P.close()
    ref, info = lf.damping_iter_fixed(*a, fixed, max_iter=4)
    o = _opts(gpu_pkg); o.max_iter = 4
    got, s = gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=fixed)
    _check_vs_oracle(got, s, ref, info, fixed, p["poses"])
    o.deterministic = 1
    x, _ = gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=fixed)
    y, _ = gpu_pkg.lidar_lm(*a, opts=o, pose_fixed=fixed)
    assert x.tobytes() == y.tobytes()


def test_batch_with_constant_poses(gpu_pkg):
    """Constant poses in some windows and one window all constant: every window equals its own masked solve; the all-constant
    window is LVBA_TERM_FUNCTION_TOL with no iteration and the skip rule still counts every pose."""
    p = synth.make_window_problem([20, 20, 14, 6, 10, 12], [260, 300, 170, 90, 12, 60], seed=23)
    wp = p["win_ptr"]
    fixed = np.zeros(len(p["poses"]), bool)
    fixed[wp[0]] = True                                                          # the first pose of window 0
    fixed[wp[1]:wp[1] + 7] = True                                                # a third of window 1
    fixed[wp[2]:wp[3]] = True                                                    # window 2 entirely
    fixed[wp[3] + 1] = True
    fixed[wp[4]:wp[5]] = True                                                    # window 4: skipped (12 voxels < 3 * 10)
    for det in (0, 1):
        o = _opts(gpu_pkg, det)
        poses, sums, _ = gpu_pkg.lidar_lm_batch(wp, *_args(p), opts=o, pose_fixed=fixed)
        ref_all, infos = lf.window_ba_fixed(wp, *_args(p), fixed)
        assert poses[fixed].tobytes() == p["poses"][fixed].tobytes()
        for w, win in enumerate(p["windows"]):
            lo_, hi_ = wp[w], wp[w + 1]
            f = fixed[lo_:hi_]
            if infos[w] is None:
                assert sums[w]["termination"] == 6 and np.array_equal(poses[lo_:hi_], p["poses"][lo_:hi_])
                continue
            if f.all():
                assert (sums[w]["iterations"], sums[w]["accepted"], sums[w]["hessian_builds"], sums[w]["termination"]) == (0, 0, 0, 1)
                assert abs(sums[w]["cost_first"] - infos[w]["r_first"]) <= 1e-9 * infos[w]["r_first"]
                assert sums[w]["cost_first"] == sums[w]["cost_last"]
                continue
            _check_vs_oracle(poses[lo_:hi_], sums[w], ref_all[lo_:hi_], infos[w], f, p["poses"][lo_:hi_])
            one, s1 = gpu_pkg.lidar_lm(*_args(win), opts=o, pose_fixed=f)
            assert s1["iterations"] == sums[w]["iterations"] and np.abs(one - poses[lo_:hi_]).max() <= 1e-9


def test_voxel_map_entry_points_with_a_mask(gpu_pkg):
    scans, poses = synth.make_scan_scene(21, W=6, n_per_scan=4000)
    rng = np.random.default_rng(3)
    noisy = poses.copy()
    for i in range(1, len(noisy)):
        noisy[i, :9] = (noisy[i, :9].reshape(3, 3) @ synth.so3_exp(rng.normal(0, 0.01, (1, 3)))[0]).ravel()
        noisy[i, 9:] += rng.normal(0, 0.02, 3)
    fixed = lf.mask_of(len(noisy), [0, 3])
    o = _opts(gpu_pkg, 1)
    m = gpu_pkg.VoxelMap(scans, noisy)
    g = m.export()
    out_dev, s = m.lidar_lm(noisy, opts=o, pose_fixed=fixed)
    out, t = gpu_pkg.lidar_lm(g["vox_ptr"], g["pose_idx"], g["clusters"], noisy, opts=o, pose_fixed=fixed)
    assert out_dev.tobytes() == out.tobytes() and s["iterations"] == t["iterations"] and s["cost_last"] == t["cost_last"]
    assert out_dev[fixed].tobytes() == noisy[fixed].tobytes() and s["cost_last"] < s["cost_first"]
    P = m.lidar_problem(noisy)                                                   # a voxel-map handle re-plans too
    P.reset_lm(o, pose_fixed=fixed)
    P.iterate(o.max_iter)
    assert P.get_poses().tobytes() == out.tobytes()
    P.close()
    m.close()
    sizes = [5, 4, 6]
    scans, poses = synth.make_scan_scene(13, W=sum(sizes), n_per_scan=3000)
    win_ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    m = gpu_pkg.VoxelMap(scans, poses, 1.0, win_ptr=win_ptr)
    fixed = np.zeros(len(poses), bool); fixed[[0, 5, 6, 7, 8]] = True          # window 1 entirely constant
    out, sums, _ = m.lidar_lm_batch(poses, min_voxels_per_pose=0, opts=o, pose_fixed=fixed)
    m.close()
    assert out[fixed].tobytes() == poses[fixed].tobytes()
    assert sums[1]["termination"] == 1 and sums[1]["iterations"] == 0


def _tool(pkg, tmp_path):
    import subprocess
    root = Path(__file__).resolve().parents[1]
    exe = tmp_path / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-I", str(root / "include"), str(root / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _offline_runs(pkg, tmp_path, W, seed, sigma, lists, extra=()):
    """the tool on one synthetic dataset, once per --fix-scans LIST; returns (start poses as loaded, {LIST: TUM lines})"""
    import subprocess
    from oracle import dataset_writer as dw
    exe = _tool(pkg, tmp_path)
    scans, poses = synth.make_scan_scene(seed, W=W, n_per_scan=3000)
    rng = np.random.default_rng(seed)
    noisy = poses.copy()
    for i in range(W):
        noisy[i, :9] = (noisy[i, :9].reshape(3, 3) @ synth.so3_exp(rng.normal(0, sigma[0], (1, 3)))[0]).ravel()
        noisy[i, 9:] += rng.normal(0, sigma[1], 3)
    data = tmp_path / "data"
    dw.write_lidar_dataset(data, scans, noisy)
    start = noisy.copy()
    for i in range(W):
        start[i, :9] = dw.quat_to_R(dw.R_to_quat(noisy[i, :9].reshape(3, 3))).ravel()
    lines = {}
    for lst in lists:
        out = tmp_path / f"opt_{lst.replace(':', '-').replace(',', '_')}.txt"
        r = subprocess.run([str(exe), "--data", str(data), "--out", str(out), "--stage1-voxel", "1.0", "--stage2-voxel", "1.0", "--deterministic",
                            "--fix-scans", lst, *extra], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        lines[lst] = out.read_text().splitlines()
        assert len(lines[lst]) == W
    return start, lines


def _pose_of(line):
    from oracle import dataset_writer as dw
    v = np.array(line.split(), float)
    return np.concatenate([dw.quat_to_R(np.array([v[7], v[4], v[5], v[6]])).ravel(), v[1:4]])


def test_shim_damping_iter_with_a_mask(gpu_pkg, tmp_path):
    """lvba_b200::damping_iter(..., &pose_fixed): the mask overrides opts->pose_fixed; constant poses keep their bits"""
    import subprocess
    from test_fixed_poses_emu import build_shim_case
    r = subprocess.run([str(build_shim_case(gpu_pkg, tmp_path))], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr


def test_offline_fix_scans(gpu_pkg, tmp_path):
    """Both global stages hold the listed scans: their TUM lines equal those of a run that lists every scan, which writes the
    input poses back; the other scans move."""
    W = 6
    start, lines = _offline_runs(gpu_pkg, tmp_path, W, 17, (0.008, 0.015), ["0,2,3", "0:5"])
    part, every = lines["0,2,3"], lines["0:5"]
    for i in (0, 2, 3):
        assert part[i] == every[i]
    for i in (1, 4, 5):
        assert part[i] != every[i]
    for i in range(W):                                                           # written back as loaded (9 decimals in the file)
        assert np.abs(_pose_of(every[i]) - start[i]).max() <= 1e-8


def test_offline_fix_scans_with_windows(gpu_pkg, tmp_path):
    """--window: the window stage holds the listed frames, a global stage the anchors whose frames are all listed; the frames
    of such anchors equal those of a run that lists every scan to 1e-12 (frames are rebuilt as anchor * rel)."""
    W = 12
    start, lines = _offline_runs(gpu_pkg, tmp_path, W, 19, (0.004, 0.01), ["0:3,8:11", "0:11"], extra=("--window", "4"))
    part, every = lines["0:3,8:11"], lines["0:11"]
    for i in list(range(4)) + list(range(8, 12)):
        assert np.abs(np.array(part[i].split(), float) - np.array(every[i].split(), float)).max() <= 1e-12
    assert any(part[i] != every[i] for i in range(4, 8))
    for i in range(W):
        assert np.abs(_pose_of(every[i]) - start[i]).max() <= 1e-8
