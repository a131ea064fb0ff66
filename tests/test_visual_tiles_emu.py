"""The tiles and destination table of the reduced camera system build (global-lvba_b200/csrc/visual_tiles.h) checked without a
GPU: the set-up steps run through the host policy (tests/emu/visual_tiles_emu.cpp) and every property the build kernel relies
on is checked — the landmark order, the tile limits, every camera pair of a landmark in one run of its S block with the
right hi / lo (a camera seen twice in both orders), every observation of a non-constant camera in a run of its row, and the
number of runs against a count of distinct (tile, block) pairs.  Re-run with shuffled items and under ASan/UBSan."""
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
    so = tmp_path_factory.mktemp("emu") / "libvis_tiles_emu.so"
    cmd = ["g++", "-std=c++17", "-O2", *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []),
           "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_tiles_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(so))
    lib.emu_vis_tiles_build.restype = ctypes.c_void_p
    lib.emu_vis_tiles_get.restype = ctypes.c_int64
    lib.emu_vis_tiles_get.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_vis_tiles_free.argtypes = [ctypes.c_void_p]
    return lib


def rows_of(obs_cam, M, fixed_cam):
    """System row of every camera: the active cameras in index order, -1 for the fixed camera."""
    used = np.zeros(M, bool)
    used[obs_cam] = True
    if 0 <= fixed_cam < M:
        used[fixed_cam] = False
    row_of_cam = np.full(M, -1, np.int64)
    row_of_cam[used] = np.arange(used.sum())
    return row_of_cam.astype(np.int32), int(used.sum())


def envelope_of(obs_ptr, row, n):
    first = np.arange(n)
    for a in range(len(obs_ptr) - 1):
        r = row[obs_ptr[a]:obs_ptr[a + 1]]
        r = r[r >= 0]
        if len(r):
            first[r] = np.minimum(first[r], r.min())
    for r in range(n - 2, -1, -1):
        first[r] = min(first[r], first[r + 1])
    row_start = np.zeros(n + 1, np.int64)
    row_start[1:] = np.cumsum(np.arange(n) - first + 1)
    return first.astype(np.int32), row_start


FIELDS = [("order", np.int64), ("trk_ptr", np.int32), ("row", np.int32), ("tile_trk", np.int32), ("pcode", np.uint32),
          ("prun", np.int64), ("ptile", np.int64), ("dcode", np.uint32), ("drun", np.int64), ("dtile", np.int64)]


def run(emu, obs_ptr, cam, row_of_cam, n_rows, max_slots=0, max_trk=0):
    op = np.ascontiguousarray(obs_ptr, np.int64); cm = np.ascontiguousarray(cam, np.int32); rc = np.ascontiguousarray(row_of_cam, np.int32)
    first, row_start = envelope_of(op, rc[cm], n_rows)
    h = emu.emu_vis_tiles_build(ctypes.c_int(n_rows), ctypes.c_int64(len(op) - 1), op.ctypes.data_as(P(ctypes.c_int64)),
                                cm.ctypes.data_as(P(ctypes.c_int32)), rc.ctypes.data_as(P(ctypes.c_int32)), first.ctypes.data_as(P(ctypes.c_int)),
                                row_start.ctypes.data_as(P(ctypes.c_longlong)), ctypes.c_longlong(int(row_start[-1])),
                                ctypes.c_int(max_slots), ctypes.c_int(max_trk))
    assert h
    out = {}
    for k, (name, dt) in enumerate(FIELDS):
        a = np.empty(emu.emu_vis_tiles_get(h, k, None), dt)
        emu.emu_vis_tiles_get(h, k, a.ctypes.data)
        out[name] = a
    emu.emu_vis_tiles_free(h)
    return out, first


def check(emu, obs_ptr, cam, row_of_cam, n_rows, max_slots=0, max_trk=0):
    S = max_slots or emu.emu_vis_tile_slots()
    NT = max_trk or emu.emu_vis_max_trk_per_tile()
    t, first = run(emu, obs_ptr, cam, row_of_cam, n_rows, max_slots, max_trk)
    obs_ptr = np.asarray(obs_ptr, np.int64); row = np.asarray(row_of_cam)[np.asarray(cam, np.int64)]
    T = len(obs_ptr) - 1
    # ---- landmark order: a stable sort by the lowest row >= 0 (0 when there is none); the local CSR follows it
    low = np.array([min([r for r in row[obs_ptr[a]:obs_ptr[a + 1]] if r >= 0], default=0) for a in range(T)])
    order = t["order"]
    assert np.array_equal(order, np.argsort(low, kind="stable"))
    K = np.diff(obs_ptr)[order]
    assert np.array_equal(np.diff(t["trk_ptr"]), K)
    ltp, lrow = t["trk_ptr"].astype(np.int64), t["row"]
    assert np.array_equal(lrow, np.concatenate([row[obs_ptr[a]:obs_ptr[a + 1]] for a in order]) if T else [])
    # ---- tiles: consecutive landmarks, <= S observations and <= NT landmarks
    tt = t["tile_trk"]
    NTi = len(tt) - 1
    assert tt[0] == 0 and tt[-1] == T and np.all(np.diff(tt) > 0)
    assert np.all(np.diff(ltp[tt]) <= S) and np.all(np.diff(tt) <= NT)
    # ---- pair runs: run_ptr ends at the number of contributions; the items after it have no destination
    pcode, prun, ptile = t["pcode"], t["prun"], t["ptile"]
    assert len(pcode) == int((K * (K - 1)).sum())
    assert prun[0] == 0 and np.all(np.diff(prun) > 0)
    assert len(ptile) == NTi + 1 and ptile[0] == 0 and ptile[-1] == len(prun) - 1 and np.all(np.diff(ptile) >= 0)
    hi_all, lo_all = (pcode & 0xFFFF).astype(np.int64), (pcode >> 16).astype(np.int64)
    # ---- observation runs
    dcode, drun, dtile = t["dcode"], t["drun"], t["dtile"]
    assert len(dcode) == ltp[-1] and drun[0] == 0 and drun[-1] == int((lrow >= 0).sum()) and np.all(np.diff(drun) > 0)
    assert len(dtile) == NTi + 1 and dtile[0] == 0 and dtile[-1] == len(drun) - 1
    n_contrib, blocks_all = 0, set()
    for k in range(NTi):
        s0, s1 = ltp[tt[k]], ltp[tt[k + 1]]
        rows = lrow[s0:s1]
        # every (landmark, i < j) pair with both rows >= 0 once as (hi, lo) = (larger row, smaller row); equal rows both ways
        want = []
        for a in range(tt[k], tt[k + 1]):
            for j in range(K[a]):
                for i in range(j):
                    x, y = ltp[a] - s0 + i, ltp[a] - s0 + j
                    if rows[x] < 0 or rows[y] < 0:
                        continue
                    if rows[x] == rows[y]:
                        want += [(x, y), (y, x)]
                    else:
                        want.append((x, y) if rows[x] > rows[y] else (y, x))
        want.sort()
        blocks_all |= {(k, int(rows[h]), int(rows[l])) for h, l in want}
        n_contrib += len(want)
        r0, r1 = ptile[k], ptile[k + 1]
        q0, q1 = prun[r0], prun[r1]
        assert sorted(zip(hi_all[q0:q1].tolist(), lo_all[q0:q1].tolist())) == want
        seen = set()
        for r in range(r0, r1):
            h, l = hi_all[prun[r]:prun[r + 1]], lo_all[prun[r]:prun[r + 1]]
            assert np.all(h < s1 - s0) and np.all(l < s1 - s0)
            blocks = set(zip(rows[h].tolist(), rows[l].tolist()))          # (row, col) of the lower-envelope block
            assert len(blocks) == 1
            (br, bc), = blocks
            assert br >= bc >= first[br] and bc >= 0
            assert (br, bc) not in seen
            seen.add((br, bc))
        # the tile's observations with row >= 0, each once, in runs of one row each, every row once
        d0, d1 = drun[dtile[k]], drun[dtile[k + 1]]
        assert np.array_equal(np.sort(dcode[d0:d1]), np.nonzero(rows >= 0)[0])
        rs = []
        for r in range(dtile[k], dtile[k + 1]):
            ps = set(rows[dcode[drun[r]:drun[r + 1]]].tolist())
            assert len(ps) == 1
            rs.append(ps.pop())
        assert len(set(rs)) == len(rs) == len(set(rows[rows >= 0].tolist()))
    assert prun[-1] == n_contrib
    assert len(prun) - 1 == len(blocks_all)                                 # runs = distinct (tile, block) pairs
    return t


def problem(seed, M=40, T=None, fixed_cam=0, shuffle=True):
    T = T or (400 if not os.environ.get("LVBA_EMU_RERUN") else 150)
    p = synth.make_problem(M, 10, T, seed=seed)
    op, cam = np.asarray(p["obs_ptr"], np.int64), np.asarray(p["obs_cam"]).copy()
    rng = np.random.default_rng(seed)
    if shuffle:                                                              # landmarks shuffled, cameras unsorted inside a landmark
        perm = rng.permutation(len(op) - 1)
        K = np.diff(op)[perm]
        cam = np.concatenate([rng.permutation(cam[op[a]:op[a + 1]]) for a in perm])
        op = np.zeros(len(perm) + 1, np.int64); op[1:] = np.cumsum(K)
    row_of_cam, n_rows = rows_of(cam, M, fixed_cam)
    return op, cam, row_of_cam, n_rows


@pytest.mark.parametrize("fixed_cam", [0, -1])
def test_table_of_synthetic_problems(emu, fixed_cam):
    op, cam, rc, n = problem(31, fixed_cam=fixed_cam)
    check(emu, op, cam, rc, n)                               # the library's tile size
    check(emu, op, cam, rc, n, max_slots=32, max_trk=4)      # many small tiles
    op, cam, rc, n = problem(32, fixed_cam=fixed_cam, shuffle=False)
    check(emu, op, cam, rc, n, max_slots=96, max_trk=48)


def test_camera_seen_twice_long_and_constant_landmarks(emu):
    """A landmark that sees one camera twice contributes both orders to its diagonal block; a landmark of 128 observations
    (the most one may have) fits a tile; landmarks that see only the fixed camera, or one camera, own no pair."""
    rng = np.random.default_rng(9)
    M = 60
    tracks = [[5, 5, 9], [0, 0], [0], [3], list(rng.choice(M, 128)), [7, 0, 2, 7, 7], list(rng.choice(M, 40, replace=False)), [], [11, 4]]
    op = np.zeros(len(tracks) + 1, np.int64); op[1:] = np.cumsum([len(t) for t in tracks])
    cam = np.array([c for t in tracks for c in t], np.int64)
    rc, n = rows_of(cam, M, 0)
    for S, NT in ((0, 0), (128, 64), (130, 2)):
        t = check(emu, op, cam, rc, n, max_slots=S, max_trk=NT)
        assert len(t["tile_trk"]) >= 2


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
