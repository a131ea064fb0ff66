"""Deterministic mode of both LM paths checked without a GPU.

The fixed-order sums (global-lvba_b200/csrc/lidar_tiles.h FixedSum / GatherF and the record passes of lidar_big.h and
visual_big.h) run through the host policy (tests/emu/det_emu.cpp), set up as the library sets them up: for path A the tiles'
pair and pose runs, then the slots and slot pairs of voxels seen from more than 128 poses; for path B the observations and
observation pairs of landmarks with more than 128 observations.  Checked here:
  * the destination table lists every record exactly once, under its true H block / gradient row, in ascending record order;
  * with the host policy visiting items in shuffled orders (LVBA_EMU_SHUFFLE, child processes), the deterministic build gives
    the same bits every time, while the default build's adds (the REDs of the device) do not — so the check can see order;
  * the deterministic build equals the oracle (oracle/lidar_oracle.py) and the default build within rounding;
  * the C layout of the options structs equals the ctypes layout, the defaults are 0, and without a device a deterministic
    one-shot call still returns LVBA_ERR_NO_DEVICE.
The file re-runs itself under ASan/UBSan."""
import ctypes
import hashlib
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
P = ctypes.POINTER
SEEDS = ["1", "20261015", "77"]


def _compile(out_dir):
    so = Path(out_dir) / "libdet_emu.so"
    san = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []
    cmd = ["g++", "-std=c++17", "-O2", *san, "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "det_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


def _load(so):
    lib = ctypes.CDLL(str(so))
    lib.emu_det_build.restype = ctypes.c_void_p
    lib.emu_det_get.restype = ctypes.c_int64
    lib.emu_det_get.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_det_run.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_det_free.argtypes = [ctypes.c_void_p]
    lib.emu_vdet_step.restype = None
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


FIELDS = [("vox_ptr", np.int32), ("pidx", np.int32), ("tile_vox", np.int32), ("pcode", np.uint32), ("dcode", np.uint32),
          ("prun", np.int64), ("ptile", np.int64), ("drun", np.int64), ("dtile", np.int64), ("big_vox_ptr", np.int64),
          ("big_pair_ptr", np.int64), ("big_pose", np.int32), ("H_dst", np.int64), ("H_code", np.uint32), ("H_run", np.int64),
          ("g_dst", np.int64), ("g_code", np.uint32), ("g_run", np.int64)]


class Det:
    """one emu_det_build handle; the arrays it points into live as long as this object"""

    def __init__(self, lib, p):
        self.lib = lib
        self.vp = np.ascontiguousarray(p["vox_ptr"], np.int64); self.pi = np.ascontiguousarray(p["pose_idx"], np.int32)
        self.cl = np.ascontiguousarray(p["clusters"], np.float64)
        self.W = len(p["poses"])
        self.first, self.row_start = envelope_of(self.vp, self.pi, self.W)
        self.nblocks = int(self.row_start[-1])
        self.h = lib.emu_det_build(ctypes.c_int(self.W), ctypes.c_int64(len(self.vp) - 1), self.vp.ctypes.data_as(P(ctypes.c_int64)),
                                   self.pi.ctypes.data_as(P(ctypes.c_int32)), self.cl.ctypes.data_as(P(ctypes.c_double)),
                                   self.first.ctypes.data_as(P(ctypes.c_int)), self.row_start.ctypes.data_as(P(ctypes.c_longlong)),
                                   ctypes.c_longlong(self.nblocks))
        assert self.h
        self.t = {}
        for k, (name, dt) in enumerate(FIELDS):
            a = np.empty(lib.emu_det_get(self.h, k, None), dt)
            lib.emu_det_get(self.h, k, a.ctypes.data)
            self.t[name] = a
        self.npr, self.ndr = max(len(self.t["prun"]) - 1, 0), max(len(self.t["drun"]) - 1, 0)   # no tiles: no runs table

    def run(self, tile_H, tile_g, poses, det):
        tH = np.ascontiguousarray(tile_H, np.float64); tg = np.ascontiguousarray(tile_g, np.float64)
        ps = np.ascontiguousarray(poses, np.float64)
        H = np.empty((self.nblocks, 36)); g = np.empty((self.W, 6))
        self.lib.emu_det_run(self.h, tH.ctypes.data, tg.ctypes.data, ps.ctypes.data, int(det), H.ctypes.data, g.ctypes.data)
        return H, g

    def close(self):
        if self.h:
            self.lib.emu_det_free(self.h)
            self.h = None


def mixed_problem(seed=77, W=300, n_small=1500, n_big=5):
    """ordinary voxels around a few seen from 129-260 poses (both sides of the 128-slot limit of a batch CTA)"""
    from oracle import synth
    rng = np.random.Generator(np.random.Philox(key=seed))
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp_b, pi_b, cl_b = synth.make_lidar(W, n_big, R_gt, p_gt, rng, k_lo=129, k_hi=260, half=W - 1)
    vp_s, pi_s, cl_s = synth.make_lidar(W, n_small, R_gt, p_gt, rng)
    vp = np.concatenate([vp_s, vp_b[1:] + vp_s[-1]]); pi = np.concatenate([pi_s, pi_b]); cl = np.concatenate([cl_s, cl_b])
    order = np.random.default_rng(seed).permutation(len(vp) - 1)
    K = np.diff(vp); starts = vp[:-1]
    pi = np.concatenate([pi[starts[a]:starts[a] + K[a]] for a in order]); cl = np.concatenate([cl[starts[a]:starts[a] + K[a]] for a in order])
    vp = np.concatenate([[0], np.cumsum(K[order])])
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    poses = np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1)
    return dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=poses)


def tile_sums(d, seed):
    """stand-ins for the build kernel's run sums: one record per pair run and pose run"""
    rng = np.random.default_rng(seed)
    return rng.normal(size=(d.npr + d.ndr, 36)), rng.normal(size=(d.ndr, 6))


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def visual_scene():
    """landmarks of 129-300 observations (one camera seen twice by some, constant camera 0) and short ones"""
    import visual_big_scene as vs
    p = vs.make_scene(11, M=40, n_short=30, long_tracks=((129, 0), (160, 5), (300, 0)))
    p["plane_nd"][::7, :3] = 0.0
    return p


def visual_step(lib, p, det):
    """emu_vdet_step on the library's local layout of p (tests/test_visual_big_emu.py Local)"""
    from test_visual_big_emu import Local, _ptr
    L = Local(p, 0)
    pr = L.pr
    q, t, X = (np.ascontiguousarray(a, np.float64) for a in (pr.q, pr.t, pr.X))
    n6, nb = max(L.n, 1) * 6, max(int(L.row_start[-1]), 1)
    o = dict(cam_colsq0=np.zeros(n6), pt_colsq0=np.zeros(max(L.Tv, 1) * 3), S=np.zeros(nb * 36), rhs=np.zeros(n6),
             cam_colsq=np.zeros(n6), cam_grad=np.zeros(n6))
    lib.emu_vdet_step(ctypes.c_int(L.n), ctypes.c_int64(L.Tv), *L.common(), _ptr(L.first, ctypes.c_int), _ptr(L.row_start, ctypes.c_longlong),
                      _ptr(q, ctypes.c_double), _ptr(t, ctypes.c_double), _ptr(X, ctypes.c_double), ctypes.c_int(int(det)),
                      *[_ptr(o[k], ctypes.c_double) for k in ("cam_colsq0", "pt_colsq0", "S", "rhs", "cam_colsq", "cam_grad")])
    return o


def child(so, npz_in, npz_out):
    """run in a child process, whose LVBA_EMU_SHUFFLE sets the order of the host policy's items"""
    if npz_in == "visual":
        sys.path.insert(0, str(ROOT / "tests"))
        lib = _load(so)
        p = visual_scene()
        d, a = visual_step(lib, p, True), visual_step(lib, p, False)
        np.savez(npz_out, **{f"det_{k}": v for k, v in d.items()}, **{f"def_{k}": v for k, v in a.items()})
        return
    z = np.load(npz_in)
    p = {k: z[k] for k in ("vox_ptr", "pose_idx", "clusters", "poses")}
    d = Det(_load(so), p)
    tH, tg = z["tile_H"], z["tile_g"]
    Hd, gd = d.run(tH, tg, p["poses"], True)
    Ha, ga = d.run(tH, tg, p["poses"], False)
    np.savez(npz_out, H_det=Hd, g_det=gd, H_def=Ha, g_def=ga, table=np.frombuffer(digest(*d.t.values()).encode(), np.uint8))
    d.close()


@pytest.fixture(scope="module")
def so(tmp_path_factory):
    return _compile(tmp_path_factory.mktemp("det_emu"))


@pytest.fixture(scope="module")
def lib(so):
    return _load(so)


@pytest.fixture(scope="module")
def mixed():
    return mixed_problem()


def test_table_lists_every_record_once_under_its_destination_in_order(lib, mixed):
    p = mixed
    d = Det(lib, p)
    t, first, row_start = d.t, d.first, d.row_start
    K = np.diff(p["vox_ptr"])
    assert K.max() >= 129 and (K <= 128).any()
    big = np.flatnonzero(K > 128)
    assert len(t["big_vox_ptr"]) - 1 == len(big)
    blk = lambda r, c: row_start[r] + c - first[r]          # noqa: E731  lower-envelope block (r, c), c <= r
    # ---- true destinations, restated from the tables
    dst_H = []
    for r in range(d.npr):                                    # pair runs: every pair of the run has the same block
        tt = np.searchsorted(t["ptile"], r, "right") - 1
        s0 = t["vox_ptr"][t["tile_vox"][tt]]
        codes = t["pcode"][t["prun"][r]:t["prun"][r + 1]]
        bl = {blk(t["pidx"][s0 + (c >> 16)], t["pidx"][s0 + (c & 0xffff)]) for c in codes.tolist()}
        assert len(bl) == 1
        dst_H.append(bl.pop())
    dst_g = []
    for r in range(d.ndr):                                    # pose runs: every slot of the run has the same pose
        tt = np.searchsorted(t["dtile"], r, "right") - 1
        s0 = t["vox_ptr"][t["tile_vox"][tt]]
        poses = {int(t["pidx"][s0 + c]) for c in t["dcode"][t["drun"][r]:t["drun"][r + 1]].tolist()}
        assert len(poses) == 1
        q = poses.pop()
        dst_H.append(blk(q, q)); dst_g.append(q)
    bp = t["big_pose"]
    for q in bp.tolist():                                     # big slots
        dst_H.append(blk(q, q)); dst_g.append(q)
    for b in range(len(t["big_vox_ptr"]) - 1):                # big pairs, t = j (j - 1) / 2 + i
        s = bp[t["big_vox_ptr"][b]:t["big_vox_ptr"][b + 1]]
        for j in range(1, len(s)):
            dst_H.extend(blk(s[j], s[:j]).tolist())
    assert len(t["big_pair_ptr"]) == len(t["big_vox_ptr"]) and len(dst_H) == d.npr + d.ndr + len(bp) + t["big_pair_ptr"][-1]
    assert np.array_equal(t["H_dst"], np.asarray(dst_H)) and np.array_equal(t["g_dst"], np.asarray(dst_g))
    # ---- the table: a permutation of the records, grouped by destination, ascending inside a group
    for name in ("H", "g"):
        dst, code, run = t[f"{name}_dst"], t[f"{name}_code"].astype(np.int64), t[f"{name}_run"]
        assert np.array_equal(np.sort(code), np.arange(len(dst)))
        assert run[0] == 0 and run[-1] == len(dst) and (np.diff(run) > 0).all()
        grp = np.repeat(np.arange(len(run) - 1), np.diff(run))
        first_of = code[run[:-1]]
        assert np.array_equal(dst[code], dst[first_of][grp])                   # every record under its destination
        assert (np.diff(dst[first_of]) > 0).all()                              # one group per destination
        inner = np.diff(code)[np.diff(grp) == 0]
        assert (inner > 0).all()                                               # ascending (tile, run), then item order
        assert len(np.unique(dst)) == len(run) - 1
    d.close()


def test_gather_sums_each_destination_in_record_order(lib, mixed):
    p = mixed
    d = Det(lib, p)
    tH, tg = tile_sums(d, 5)
    Hd, gd = d.run(tH, tg, p["poses"], True)
    Ha, ga = d.run(tH, tg, p["poses"], False)
    assert np.abs(Hd - Ha).max() <= 1e-12 * np.abs(Ha).max() and np.abs(gd - ga).max() <= 1e-12 * np.abs(ga).max()
    # the tile records alone (no big voxel): every element the left-to-right sum of its records
    q = mixed_problem(seed=3, W=40, n_small=300, n_big=0)
    e = Det(lib, q)
    tH, tg = tile_sums(e, 6)
    H, g = e.run(tH, tg, q["poses"], True)
    t = e.t
    want = np.zeros_like(H)
    for r in range(len(t["H_run"]) - 1):
        codes = t["H_code"][t["H_run"][r]:t["H_run"][r + 1]]
        acc = np.zeros(36)
        for c in codes:
            acc = acc + tH[c]
        want[t["H_dst"][codes[0]]] = acc
    assert want.tobytes() == H.tobytes()
    e.close(); d.close()


def test_deterministic_big_voxels_equal_the_oracle(lib):
    """voxels seen from 300 of 400 poses only: H and g are the big-voxel passes' records, gathered"""
    from oracle import lidar_oracle as lo
    from oracle import synth
    rng = np.random.Generator(np.random.Philox(key=77))
    R_gt, p_gt = synth.make_trajectory(400, rng)
    vp, pi, cl = synth.make_lidar(400, 6, R_gt, p_gt, rng, k_lo=300, k_hi=300, half=399)
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (400, 3)))
    poses = np.concatenate([R0.reshape(400, 9), p_gt + rng.normal(0, 0.02, (400, 3))], 1)
    d = Det(lib, dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=poses))
    assert d.npr == 0 and d.ndr == 0
    H, g = d.run(np.zeros((0, 36)), np.zeros((0, 6)), poses, True)
    _, g_ref, blocks = lo.acc_evaluate2(vp, pi, cl, poses, 400)
    H_ref = lo.assemble_dense(blocks, 400)
    assert np.abs(g - g_ref).max() <= 1e-7 * np.abs(g_ref).max()
    dense = np.zeros((2400, 2400))
    for r in range(400):
        for c in range(d.first[r], r + 1):
            dense[6 * r:6 * r + 6, 6 * c:6 * c + 6] = H[d.row_start[r] + c - d.first[r]].reshape(6, 6)
    mask = np.kron(np.tril(np.ones((400, 400))), np.ones((6, 6))) > 0
    assert np.abs(dense - H_ref * mask).max() <= 1e-7 * np.abs(H_ref).max()
    d.close()


def test_shuffled_items_give_the_same_bits_only_in_deterministic_mode(so, mixed, tmp_path):
    p = mixed
    d = Det(_load(so), p)
    tH, tg = tile_sums(d, 9)
    d.close()
    npz_in = tmp_path / "in.npz"
    np.savez(npz_in, tile_H=tH, tile_g=tg, **p)
    env0 = {k: v for k, v in os.environ.items() if k != "LVBA_EMU_SHUFFLE"}
    procs = {}
    for seed in [None, *SEEDS]:
        env = dict(env0, **({"LVBA_EMU_SHUFFLE": seed} if seed else {}))
        out = tmp_path / f"out_{seed}.npz"
        procs[seed] = (out, subprocess.Popen([sys.executable, __file__, "child", str(so), str(npz_in), str(out)], cwd=str(ROOT), env=env,
                                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    res = {}
    for seed, (out, proc) in procs.items():
        o, e = proc.communicate(timeout=600)
        assert proc.returncode == 0, (seed, o[-2000:], e[-3000:])
        res[seed] = dict(np.load(out))
    ref = res[None]
    for seed in SEEDS:
        assert res[seed]["table"].tobytes() == ref["table"].tobytes(), seed
        assert res[seed]["H_det"].tobytes() == ref["H_det"].tobytes(), seed
        assert res[seed]["g_det"].tobytes() == ref["g_det"].tobytes(), seed
    default = {digest(r["H_def"], r["g_def"]) for r in res.values()}
    assert len(default) > 1, "the default adds gave the same bits in every order: this check cannot see order dependence"


def test_visual_big_landmarks_give_the_same_bits_only_in_deterministic_mode(so, tmp_path):
    """the column norms, S, rhs and gradient of the visual build's big-landmark passes: bit-identical under shuffled item orders
    with records and GatherF, while the default atomics differ; both within rounding of each other (the default passes are held
    against the oracle by tests/test_visual_big_emu.py)"""
    env0 = {k: v for k, v in os.environ.items() if k != "LVBA_EMU_SHUFFLE"}
    procs = {}
    for seed in [None, *SEEDS]:
        env = dict(env0, **({"LVBA_EMU_SHUFFLE": seed} if seed else {}))
        out = tmp_path / f"vout_{seed}.npz"
        procs[seed] = (out, subprocess.Popen([sys.executable, __file__, "child", str(so), "visual", str(out)], cwd=str(ROOT), env=env,
                                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    res = {}
    for seed, (out, proc) in procs.items():
        o, e = proc.communicate(timeout=600)
        assert proc.returncode == 0, (seed, o[-2000:], e[-3000:])
        res[seed] = dict(np.load(out))
    keys = ("cam_colsq0", "pt_colsq0", "S", "rhs", "cam_colsq", "cam_grad")
    ref = res[None]
    for seed in SEEDS:
        for k in keys:
            assert res[seed][f"det_{k}"].tobytes() == ref[f"det_{k}"].tobytes(), (seed, k)
    for k in keys:
        d, a = ref[f"det_{k}"], ref[f"def_{k}"]
        assert np.abs(d - a).max() <= 1e-12 * max(np.abs(a).max(), 1e-300), k
    default = {digest(*[r[f"def_{k}"] for k in keys]) for r in res.values()}
    assert len(default) > 1, "the default adds gave the same bits in every order: this check cannot see order dependence"


def test_opts_layout_and_defaults_match_the_header(pkg, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "lvba_b200.h"
int main(void) {
  lvba_lidar_opts a; lvba_visual_opts b;
  printf("%zu %zu %zu %zu\\n", sizeof(lvba_lidar_opts), offsetof(lvba_lidar_opts, deterministic),
         sizeof(lvba_visual_opts), offsetof(lvba_visual_opts, deterministic));
  (void)a; (void)b;
  return 0;
}
""")
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(pkg.LidarOpts), pkg.LidarOpts.deterministic.offset,
                   ctypes.sizeof(pkg.VisualOpts), pkg.VisualOpts.deterministic.offset]
    assert pkg.lidar_default_opts().deterministic == 0 and pkg.visual_default_opts().deterministic == 0


def test_deterministic_one_shot_call_without_a_device(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    from oracle import synth
    p = synth.make_problem(12, 80, 0, seed=4242, visual=False)
    o = pkg.lidar_default_opts()
    o.deterministic = 1
    with pytest.raises(pkg.LvbaError) as e:
        pkg.lidar_lm(p["vox_ptr"], p["pose_idx"], p["clusters"], p["poses"], opts=o)
    assert e.value.status == -2                                                 # LVBA_ERR_NO_DEVICE


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


def test_suite_passes_under_address_and_ub_sanitizers():
    if os.environ.get("LVBA_EMU_SANITIZE"):
        pytest.skip("this is the sanitized run")
    asan = _asan()
    if not asan:
        pytest.skip("no libasan for this compiler")
    env = dict(os.environ, LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__, "-k", "not sanitizers and not header and not device"],
                       capture_output=True, text=True, cwd=str(ROOT), env=env, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout


if __name__ == "__main__" and len(sys.argv) == 5 and sys.argv[1] == "child":
    sys.path.insert(0, str(ROOT))
    child(*sys.argv[2:])
