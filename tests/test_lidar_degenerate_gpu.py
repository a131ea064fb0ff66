"""The LiDAR plane factor on the GPU (boundary B1) on degenerate voxels, against the 50-digit oracle (oracle/balm_mp.py).

The voxel family of tests/degenerate_voxels.py drives every branch of the three device eigen solvers: the Newton fast path of
eig3_sym_plane (tile build) and sym3_smallest_eigenvalue (residual pass), their Jacobi fallbacks (strip, line), the 2 x 2
step at lambda_1 = lambda_2 (disc), exact zeros and ties in u_0 (axis), det(C) <= 0 (flat), cancellation in P/N - vbar vbar^T
(far), NN = (int)N on large and non-integral N (bulk), and the 16-sweep Jacobi of the big-voxel passes (K > 128).  Every
residual, g row and H block is held to the per-voxel bounds of tests/test_balm_mp_oracle.py (constants C_R, C_G, C_H of
balm_mp.py, calibrated there on the CPU from two float64 implementations), in the default and the deterministic mode.
"""
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import balm_mp as bm
from oracle import lidar_oracle as lo

sys.path.insert(0, str(Path(__file__).resolve().parent))
import degenerate_voxels as dv  # noqa: E402

pytestmark = pytest.mark.gpu


def _with_refs(p, poses=None):
    p = dict(p)
    if poses is not None:
        p["poses"] = poses
    p["refs"] = bm.evaluate(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    return p


@pytest.fixture(scope="module")
def iso():
    return _with_refs(dv.isolated())


@pytest.fixture(scope="module")
def tile_big():
    return _with_refs(dv.tile_and_big())


@pytest.fixture(scope="module")
def shared():
    p = dv.shared()
    return {"generating poses": _with_refs(p), "perturbed poses": _with_refs(p, p["poses0"])}


def _opts(pkg, det):
    o = pkg.lidar_default_opts()
    o.deterministic = int(det)
    return o


def _device(pkg, p, det):
    """build(), get_system() and residual() on one state; blocks {(row, col): 6x6} of the lower envelope"""
    P = pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    try:
        P.reset_lm(_opts(pkg, det))
        r_build = P.build()
        g, br, bc, bl = P.get_system()
        r_res = P.residual()
    finally:
        P.close()
    blocks = {(int(a), int(b)): bl[k] for k, (a, b) in enumerate(zip(br, bc))}
    return r_build, r_res, g, blocks


def _upper(blocks):
    return lambda i, j: blocks[(j, i)].T if i != j else blocks[(i, i)]


def _check(p, dev, by_class, capsys, label):
    """every residual, g row and H block within the bounds; per class when by_class, else for the whole problem"""
    r_build, r_res, g, blocks = dev
    W = len(p["poses"])
    whole = bm.assemble(p["vox_ptr"], p["pose_idx"], p["refs"], W)
    rows = []
    assert abs(r_build - whole["res"]) <= bm.C_R * whole["res_scale"], (label, "build", r_build, whole["res"])
    assert abs(r_res - whole["res"]) <= bm.C_R * whole["res_scale"], (label, "residual", r_res, whole["res"])
    touched = {(max(i, j), min(i, j)) for i, j in whole["H"]}
    for k, b in blocks.items():
        if k not in touched:
            assert not b.any(), (label, "a block no voxel touches", k)
    groups = sorted(set(p["cls"])) if by_class else [None]
    for c in groups:
        idx = np.arange(len(p["refs"])) if c is None else np.nonzero(p["cls"] == c)[0]
        q = dv.reorder(p, idx)
        ref = bm.assemble(q["vox_ptr"], q["pose_idx"], [p["refs"][a] for a in idx], W) if c is not None else whole
        _, rg, rh = bm.ratios(ref, 0.0, g, _upper(blocks))
        rows.append((c or "all", rg, rh))
    with capsys.disabled():
        print(f"\n{label}: residual build {abs(r_build - whole['res']) / whole['res_scale']:.3g}, "
              f"residual pass {abs(r_res - whole['res']) / whole['res_scale']:.3g} (bound {bm.C_R:g})")
        for c, rg, rh in rows:
            print(f"  {c:10s} g {rg:9.3g} (bound {bm.C_G:g})   H {rh:9.3g} (bound {bm.C_H:g})")
    for c, rg, rh in rows:
        assert rg <= bm.C_G and rh <= bm.C_H, (label, c, rg, rh)


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
def test_isolated_voxels_meet_the_bounds(gpu_pkg, iso, det, capsys):
    """every voxel on poses of its own: each g row and H block is one voxel's, checked per class"""
    _check(iso, _device(gpu_pkg, iso, det), True, capsys, f"isolated, det={det}")


@pytest.mark.parametrize("state", ["generating poses", "perturbed poses"])
@pytest.mark.parametrize("order", ["caller", "shuffled"])
def test_shared_poses_meet_the_bounds(gpu_pkg, shared, state, order, capsys):
    """the classes on one trajectory (+-4 poses): blocks sum several classes, tiles mix fast-path and fallback voxels"""
    p = shared[state]
    if order == "shuffled":
        V = len(p["vox_ptr"]) - 1
        perm = np.random.default_rng(20261016).permutation(V)
        q = dv.reorder(p, perm)
        q["refs"] = [p["refs"][a] for a in perm]
        p = q
    _check(p, _device(gpu_pkg, p, 0), False, capsys, f"shared, {state}, {order}")


def test_build_and_residual_agree_per_class(gpu_pkg, iso):
    """the LM compares the build's cost with the residual pass's: on one state they agree within the residual bound, class
    by class (strip and line take the Jacobi fallback of both, the others the Newton root)"""
    for c in sorted(set(iso["cls"])):
        idx = np.nonzero(iso["cls"] == c)[0]
        q = dv.reorder(iso, idx)
        refs = [iso["refs"][a] for a in idx]
        scale = sum(bm.delta(r) for r in refs)
        mp_sum = sum(r["res"] for r in refs)
        r_build, r_res, _, _ = _device(gpu_pkg, q, 0)
        assert abs(r_build - r_res) <= bm.C_R * scale, (c, r_build, r_res, scale)
        assert abs(r_build - mp_sum) <= bm.C_R * scale, (c, r_build, mp_sum)


@pytest.mark.parametrize("det", [0, 1], ids=["default", "deterministic"])
def test_tile_path_and_big_path_on_the_same_geometry(gpu_pkg, tile_big, det, capsys):
    """strip and line voxels from 128 poses (the tile build) and the same voxels from one pose more (lidar_big.h)"""
    assert set(np.diff(tile_big["vox_ptr"])) == {128, 129}
    _check(tile_big, _device(gpu_pkg, tile_big, det), True, capsys, f"tile / big, det={det}")


def test_lm_on_degenerate_voxels_matches_oracle(gpu_pkg, shared):
    """one damping_iter from perturbed poses on the mixed problem: the same accept / reject sequence and first cost as the
    float64 oracle, and its end cost and poses within 1e-6 or within the oracle's own sensitivity to its last input bits"""
    p = shared["perturbed poses"]
    ref_poses, info = lo.damping_iter(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    seq_ref = [t["q"] > 0 for t in info["trace"]]
    poses, s = gpu_pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    P = gpu_pkg.LidarProblem(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"])
    try:
        P.reset_lm()
        seq = []
        for _ in range(10):
            st = P.iterate(1)                       # the summary of this one pass
            seq.append(st["accepted"] > 0)
            if st["termination"] != 0:
                break
    finally:
        P.close()
    assert seq == seq_ref
    assert s["iterations"] == info["iters"] and s["accepted"] == info["accepted"]
    # the first cost (sum lambda_0 / V) carries the covariance rounding of the far voxels: both within the residual bound
    V = len(p["refs"])
    scale = bm.C_R * sum(bm.delta(r) for r in p["refs"]) / V
    mp_first = sum(r["res"] for r in p["refs"]) / V
    assert abs(s["cost_first"] - mp_first) <= scale and abs(info["r_first"] - mp_first) <= scale
    # The poles (line: 2 / (lambda_0 - lambda_1) ~ 1e6) make this LM ill-conditioned: perturbing the start poses by 1e-15
    # relative moves the float64 oracle's own end state by ~3e-4.  The device must land within 1e-6 or within 16x that spread.
    rng = np.random.default_rng(5)
    ref2, info2 = lo.damping_iter(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"] * (1 + 1e-15 * rng.standard_normal(p["poses"].shape)))
    spread_cost, spread_pose = abs(info2["r_last"] - info["r_last"]), np.abs(ref2 - ref_poses).max()
    assert abs(s["cost_last"] - info["r_last"]) <= max(1e-6 * info["r_last"], 16 * spread_cost)
    assert np.abs(poses - ref_poses).max() <= max(1e-6, 16 * spread_pose)
