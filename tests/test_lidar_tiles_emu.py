"""The tiles and destination table of the LiDAR Hessian build (global-lvba_b200/csrc/lidar_tiles.h) checked without a GPU:
the set-up steps run through the host policy (tests/emu/tiles_emu.cpp) and every property the build kernel relies on is
checked — the voxel order, the tile limits and windows, every (voxel, i < j) pair exactly once in its tile and in a run of
pairs that share one H block, and every slot in a run of its pose.  Re-run with shuffled items and under ASan/UBSan."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import synth

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu") / "libtiles_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []),
           "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "tiles_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(so))
    lib.emu_tiles_build.restype = ctypes.c_void_p
    lib.emu_tiles_get.restype = ctypes.c_int64
    lib.emu_tiles_get.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_tiles_free.argtypes = [ctypes.c_void_p]
    return lib


def envelope_of(vox_ptr, pose_idx, W):
    first = np.arange(W)
    for a in range(len(vox_ptr) - 1):
        s = pose_idx[vox_ptr[a]:vox_ptr[a + 1]]
        first[s] = np.minimum(first[s], s.min())
    for r in range(W - 2, -1, -1):
        first[r] = min(first[r], first[r + 1])
    row_start = np.zeros(W + 1, np.int64)
    row_start[1:] = np.cumsum(np.arange(W) - first + 1)
    return first.astype(np.int32), row_start


FIELDS = [("order", np.int64), ("vox_ptr", np.int32), ("pidx", np.int32), ("tile_vox", np.int32), ("pcode", np.uint32),
          ("prun", np.int64), ("ptile", np.int64), ("dcode", np.uint32), ("drun", np.int64), ("dtile", np.int64)]


def run(emu, vox_ptr, pose_idx, W, pose_grp=None, max_slots=0, max_vox=0):
    vp = np.ascontiguousarray(vox_ptr, np.int64); pi = np.ascontiguousarray(pose_idx, np.int32)
    first, row_start = envelope_of(vp, pi, W)
    n_grp = 0 if pose_grp is None else int(np.max(pose_grp)) + 1                 # pose_grp: consecutive windows 0, 1, ...
    grp_ptr = np.zeros(n_grp + 1, np.int32)
    if n_grp:
        grp_ptr[1:] = np.cumsum(np.bincount(pose_grp, minlength=n_grp))
    h = emu.emu_tiles_build(ctypes.c_int(W), ctypes.c_int64(len(vp) - 1), vp.ctypes.data_as(P(ctypes.c_int64)), pi.ctypes.data_as(P(ctypes.c_int32)),
                            ctypes.c_int(n_grp), grp_ptr.ctypes.data_as(P(ctypes.c_int32)), first.ctypes.data_as(P(ctypes.c_int)),
                            row_start.ctypes.data_as(P(ctypes.c_longlong)), ctypes.c_longlong(int(row_start[-1])), ctypes.c_int(max_slots), ctypes.c_int(max_vox))
    assert h
    out = {}
    for k, (name, dt) in enumerate(FIELDS):
        a = np.empty(emu.emu_tiles_get(h, k, None), dt)
        emu.emu_tiles_get(h, k, a.ctypes.data)
        out[name] = a
    emu.emu_tiles_free(h)
    return out, first, row_start


def check(emu, vox_ptr, pose_idx, W, pose_grp=None, max_slots=0, max_vox=0):
    S = max_slots or emu.emu_tile_slots()
    NV = max_vox or emu.emu_max_vox_per_tile()
    t, first, row_start = run(emu, vox_ptr, pose_idx, W, pose_grp, max_slots, max_vox)
    vox_ptr = np.asarray(vox_ptr, np.int64); pose_idx = np.asarray(pose_idx)
    V = len(vox_ptr) - 1
    # ---- voxel order: a stable sort by lowest pose; the local CSR is the caller's voxels in that order
    order = t["order"]
    lowest = pose_idx[vox_ptr[:-1]]
    assert np.array_equal(order, np.argsort(lowest, kind="stable"))
    K = np.diff(vox_ptr)[order]
    assert np.array_equal(np.diff(t["vox_ptr"]), K)
    assert np.array_equal(t["pidx"], np.concatenate([pose_idx[vox_ptr[a]:vox_ptr[a + 1]] for a in order]) if V else [])
    lvp, lpi = t["vox_ptr"].astype(np.int64), t["pidx"]
    # ---- tiles: consecutive voxels, <= S slots and <= NV voxels, one window each
    tv = t["tile_vox"]
    T = len(tv) - 1
    assert tv[0] == 0 and tv[-1] == V and np.all(np.diff(tv) > 0)
    assert np.all(np.diff(lvp[tv]) <= S) and np.all(np.diff(tv) <= NV)
    if pose_grp is not None:
        vgrp = np.asarray(pose_grp)[lpi[lvp[:-1]]]
        for k in range(T):
            assert len(set(vgrp[tv[k]:tv[k + 1]])) == 1
    # ---- pair runs
    pcode, prun, ptile = t["pcode"], t["prun"], t["ptile"]
    n_pairs = int((K * (K - 1) // 2).sum())
    assert len(pcode) == n_pairs and prun[0] == 0 and prun[-1] == n_pairs and np.all(np.diff(prun) > 0)
    assert len(ptile) == T + 1 and ptile[0] == 0 and ptile[-1] == len(prun) - 1 and np.all(np.diff(ptile) >= 0)
    li_all, lj_all = (pcode & 0xFFFF).astype(np.int64), (pcode >> 16).astype(np.int64)
    # ---- slot runs
    dcode, drun, dtile = t["dcode"], t["drun"], t["dtile"]
    assert len(dcode) == lvp[-1] and drun[0] == 0 and drun[-1] == lvp[-1] and np.all(np.diff(drun) > 0)
    assert len(dtile) == T + 1 and dtile[0] == 0 and dtile[-1] == len(drun) - 1
    for k in range(T):
        s0, s1 = lvp[tv[k]], lvp[tv[k + 1]]
        ns = s1 - s0
        vox_of = np.repeat(np.arange(tv[k], tv[k + 1]), K[tv[k]:tv[k + 1]])          # local voxel of every slot of the tile
        pose = lpi[s0:s1]
        # every (voxel, i < j) pair of the tile exactly once, in one of the tile's runs
        want = sorted((lvp[v] - s0 + i, lvp[v] - s0 + j) for v in range(tv[k], tv[k + 1]) for j in range(K[v]) for i in range(j))
        r0, r1 = ptile[k], ptile[k + 1]
        q0, q1 = prun[r0], prun[r1]
        got = sorted(zip(li_all[q0:q1].tolist(), lj_all[q0:q1].tolist()))
        assert got == want
        seen = set()
        for r in range(r0, r1):
            li, lj = li_all[prun[r]:prun[r + 1]], lj_all[prun[r]:prun[r + 1]]
            assert np.all(li < lj) and np.all(lj < ns) and np.all(vox_of[li] == vox_of[lj])
            blocks = set(zip(pose[lj].tolist(), pose[li].tolist()))                    # (row, col) of the lower-envelope block
            assert len(blocks) == 1
            (row, col), = blocks
            assert row > col >= first[row]
            assert (row, col) not in seen
            seen.add((row, col))
        # the tile's slots: dcode[s0:s1], a permutation, in runs of one pose each, every pose once
        assert np.array_equal(np.sort(dcode[s0:s1]), np.arange(ns))
        assert drun[dtile[k]] == s0 and drun[dtile[k + 1]] == s1
        poses = []
        for r in range(dtile[k], dtile[k + 1]):
            ps = set(pose[dcode[drun[r]:drun[r + 1]]].tolist())
            assert len(ps) == 1
            poses.append(ps.pop())
        assert len(set(poses)) == len(poses) == len(set(pose.tolist()))
    return t


def shuffled(vox_ptr, pose_idx, seed):
    rng = np.random.default_rng(seed)
    V = len(vox_ptr) - 1
    perm = rng.permutation(V)
    K = np.diff(vox_ptr)
    vp = np.zeros(V + 1, np.int64); vp[1:] = np.cumsum(K[perm])
    idx = np.concatenate([np.arange(vox_ptr[a], vox_ptr[a + 1]) for a in perm])
    return vp, np.asarray(pose_idx)[idx]


def test_table_of_synthetic_problems(emu):
    p = synth.make_problem(120, 3000 if not os.environ.get("LVBA_EMU_RERUN") else 800, 0, seed=31, visual=False)
    check(emu, p["vox_ptr"], p["pose_idx"], 120)                         # the library's tile size
    check(emu, p["vox_ptr"], p["pose_idx"], 120, max_slots=64, max_vox=8)  # many small tiles
    vp, pi = shuffled(p["vox_ptr"], p["pose_idx"], 3)
    check(emu, vp, pi, 120, max_slots=96, max_vox=48)


def test_tiles_never_hold_two_windows(emu):
    w = synth.make_window_problem([7, 0, 11, 5, 9], [60, 0, 90, 30, 70], seed=5)
    W = int(w["win_ptr"][-1])
    pose_grp = np.repeat(np.arange(len(w["win_ptr"]) - 1), np.diff(w["win_ptr"]))
    vp, pi = shuffled(w["vox_ptr"], w["pose_idx"], 8)
    for S in (0, 40):
        t = check(emu, vp, pi, W, pose_grp, max_slots=S, max_vox=S // 2)
        lvp, tv = t["vox_ptr"].astype(np.int64), t["tile_vox"]
        starts = pose_grp[t["pidx"][lvp[tv[:-1]]]]
        assert np.all(np.diff(starts) >= 0)                            # windows in order


def test_voxel_with_128_poses_and_single_slot_voxels(emu):
    """A voxel seen from 128 poses (the most a tile voxel may have) fits a tile; voxels of one slot have no pairs but still
    own a diagonal block and a gradient row."""
    rng = np.random.default_rng(9)
    W = 300
    ks = [128, 1, 1, 2, 128, 5, 1, 64, 3, 1]
    vp, pi = [0], []
    for k in ks:
        lo = int(rng.integers(0, W - k + 1))
        pi.extend(sorted(rng.choice(np.arange(lo, min(W, lo + max(k, 40))), size=k, replace=False).tolist()))
        vp.append(len(pi))
    for S, NV in ((0, 0), (128, 64), (130, 2)):
        t = check(emu, vp, pi, W, max_slots=S, max_vox=NV)
        assert len(t["tile_vox"]) >= 2


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    """The table does not depend on the order in which the items of a pass run (the device runs them concurrently), and the
    host policy finds no memory or UB error."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261015")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="7")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(ROOT), env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
