"""Constant poses of the LiDAR LM (lvba_lidar_opts::pose_fixed) without a GPU:
  * the C and ctypes layouts of the options (pose_fixed the last field, NULL by default) and LVBA_ERR_NO_DEVICE with a mask;
  * the oracle with constant poses (tests/lidar_fixed_oracle.py): the same bits as damping_iter without a mask, and a first step
    that solves the free rows of the H and g the reference's own source computed (tests/golden/ref_balm.npz);
  * the library's set-up under masks through the host policy (tests/emu/fixed_poses_emu.cpp): the row envelope, the build's
    destination table and the deterministic record index list every pair and slot of free poses once under its true row
    destination and nothing of constant ones, and the big-voxel passes give the oracle's restricted H and g.
The table checks re-run with shuffled item orders and under ASan/UBSan."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import lidar_fixed_oracle as lf  # noqa: E402
from oracle import lidar_oracle as lo  # noqa: E402

P = ctypes.POINTER
REF = np.load(ROOT / "tests" / "golden" / "ref_balm.npz")


def test_opts_layout_and_default(pkg, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "lvba_b200.h"\n'
                   'int main(void) { lvba_lidar_opts o; lvba_lidar_default_opts(&o);\n'
                   '  printf("%zu %zu %d\\n", sizeof(lvba_lidar_opts), offsetof(lvba_lidar_opts, pose_fixed), o.pose_fixed == NULL);\n'
                   '  return 0; }\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe), str(pkg.LIB_PATH),
                        f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(pkg.LidarOpts), pkg.LidarOpts.pose_fixed.offset, 1]
    assert pkg.LidarOpts.pose_fixed.offset == ctypes.sizeof(pkg.LidarOpts) - ctypes.sizeof(ctypes.c_void_p)   # the last field
    assert not pkg.lidar_default_opts().pose_fixed


def test_no_device_with_a_mask(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    a = [REF[f"L1_{k}"] for k in ("vox_ptr", "pose_idx", "clusters", "poses")]
    W = len(a[3])
    for call in (lambda: pkg.lidar_lm(*a, pose_fixed=np.arange(W) < 3),
                 lambda: pkg.lidar_lm_batch([0, W], *a, pose_fixed=np.arange(W) < 3)):
        with pytest.raises(pkg.LvbaError) as e:
            call()
        assert e.value.status == -2
    with pytest.raises(ValueError):
        pkg.lidar_lm(*a, pose_fixed=np.ones(W - 1, bool))                   # one entry per pose


# ---- the oracle
def _ref(level):
    return [REF[f"{level}_{k}"] for k in ("vox_ptr", "pose_idx", "clusters", "poses")]


@pytest.mark.parametrize("level", ["L1", "L2"])
def test_oracle_without_mask_is_damping_iter(level):
    vp, pi, cl, ps = _ref(level)
    a, ia = lo.damping_iter(vp, pi, cl, ps, max_iter=6)
    for fixed in (None, np.zeros(len(ps), bool)):
        b, ib = lf.damping_iter_fixed(vp, pi, cl, ps, fixed, max_iter=6)
        assert np.array_equal(a, b)
        assert (ia["iters"], ia["accepted"], ia["r_first"], ia["r_last"], ia["u_last"]) == \
               (ib["iters"], ib["accepted"], ib["r_first"], ib["r_last"], ib["u_last"])


def _masks(W, rng):
    yield np.arange(W) == 0
    yield np.arange(W) < W // 2
    yield rng.random(W) < 1 / 3
    yield np.arange(W) % 3 == 2


@pytest.mark.parametrize("level", ["L1", "L2"])
def test_oracle_first_step_solves_the_reference_system_restricted(level):
    """The oracle's first step with a mask = np.linalg.solve on the free rows of the H and g the reference's source computed."""
    vp, pi, cl, ps = _ref(level)
    H_ref, g_ref = REF[f"{level}_H"], REF[f"{level}_g"]
    W = len(ps)
    rng = np.random.default_rng(3)
    for fixed in _masks(W, rng):
        free, cols = lf.free_index(fixed, W)
        Hf = H_ref[np.ix_(cols, cols)]
        want = np.zeros(6 * W)
        want[cols] = np.linalg.solve(Hf + np.diag(0.01 * np.diag(Hf)), -g_ref.ravel()[cols])
        _, info = lf.damping_iter_fixed(vp, pi, cl, ps, fixed, max_iter=1, rel_tol=-1)
        rs, g_all, blocks = lo.acc_evaluate2(vp, pi, cl, ps, W)
        got = lf.first_step(lo.assemble_sparse(blocks, W), g_all, 0.01, fixed).ravel()
        scale = np.abs(want).max()
        assert np.abs(got - want).max() <= 1e-6 * scale, (level, np.flatnonzero(fixed))
        assert np.all(got.reshape(W, 6)[fixed] == 0)
        # the trial state of the oracle's loop is the retraction of that step, constant poses untouched
        trial = lo.retract(ps, got)
        r2 = lo.only_residual(vp, pi, cl, np.where(fixed[:, None], ps, trial)) / (len(vp) - 1)
        assert np.isclose(info["trace"][0]["r2"], r2, rtol=1e-9)


def test_oracle_all_constant():
    vp, pi, cl, ps = _ref("L1")
    out, info = lf.damping_iter_fixed(vp, pi, cl, ps, np.ones(len(ps), bool))
    assert np.array_equal(out, ps) and info["iters"] == 0 and info["r_first"] == info["r_last"]
    assert info["r_first"] == lo.only_residual(vp, pi, cl, ps) / (len(vp) - 1)


# ---- the set-up through the host policy
def _compile(out_dir):
    so = Path(out_dir) / "libfixed_poses_emu.so"
    san = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []
    cmd = ["g++", "-std=c++17", "-O2", *san, "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "fixed_poses_emu.cpp"), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = ctypes.CDLL(str(_compile(tmp_path_factory.mktemp("fixed_poses_emu"))))
    lib.emu_fp_build.restype = ctypes.c_void_p
    lib.emu_fp_build.argtypes = [ctypes.c_int, ctypes.c_int64] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
    lib.emu_fp_get.restype = ctypes.c_int64
    lib.emu_fp_get.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_fp_run.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_void_p]
    lib.emu_fp_rows.argtypes = [ctypes.c_void_p]
    lib.emu_fp_nblocks.argtypes = [ctypes.c_void_p]
    lib.emu_fp_nblocks.restype = ctypes.c_longlong
    lib.emu_fp_free.argtypes = [ctypes.c_void_p]
    return lib


FIELDS = [("vox_ptr", np.int32), ("pidx", np.int32), ("tile_vox", np.int32), ("pcode", np.uint32), ("dcode", np.uint32),
          ("prun", np.int64), ("ptile", np.int64), ("drun", np.int64), ("dtile", np.int64), ("big_vox_ptr", np.int64),
          ("big_pair_ptr", np.int64), ("big_pose", np.int32), ("H_dst", np.int64), ("H_code", np.uint32), ("H_run", np.int64),
          ("g_dst", np.int64), ("g_code", np.uint32), ("g_run", np.int64), ("row_of", np.int32), ("first", np.int32),
          ("row_start", np.int64)]


class Fp:
    def __init__(self, lib, p, fixed, batch_slots=128):
        self.lib = lib
        self.vp = np.ascontiguousarray(p["vox_ptr"], np.int64); self.pi = np.ascontiguousarray(p["pose_idx"], np.int32)
        self.cl = np.ascontiguousarray(p["clusters"], np.float64)
        self.W = len(p["poses"])
        self.mask = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        self.h = lib.emu_fp_build(ctypes.c_int(self.W), ctypes.c_int64(len(self.vp) - 1), self.vp.ctypes.data, self.pi.ctypes.data,
                                  self.cl.ctypes.data, None if self.mask is None else self.mask.ctypes.data, ctypes.c_int(batch_slots))
        assert self.h
        self.t = {}
        for k, (name, dt) in enumerate(FIELDS):
            a = np.empty(lib.emu_fp_get(self.h, k, None), dt)
            lib.emu_fp_get(self.h, k, a.ctypes.data)
            self.t[name] = a
        self.n_rows, self.nblocks = lib.emu_fp_rows(self.h), lib.emu_fp_nblocks(self.h)
        self.npr, self.ndr = max(len(self.t["prun"]) - 1, 0), max(len(self.t["drun"]) - 1, 0)

    def run(self, poses, det):
        tH = np.zeros((self.npr + self.ndr, 36)); tg = np.zeros((self.ndr, 6))
        ps = np.ascontiguousarray(poses, np.float64)
        H = np.empty((max(self.nblocks, 1), 36)); g = np.empty((max(self.n_rows, 1), 6)); r = ctypes.c_double()
        self.lib.emu_fp_run(self.h, tH.ctypes.data, tg.ctypes.data, ps.ctypes.data, int(det), H.ctypes.data, g.ctypes.data,
                            ctypes.addressof(r))
        return H[:self.nblocks], g[:self.n_rows], r.value

    def close(self):
        if self.h:
            self.lib.emu_fp_free(self.h)
            self.h = None


def _problem(seed, W=40, n_vox=300):
    from oracle import synth
    rng = np.random.Generator(np.random.Philox(key=seed))
    R_gt, p_gt = synth.make_trajectory(W, rng)
    vp, pi, cl = synth.make_lidar(W, n_vox, R_gt, p_gt, rng)
    R0 = R_gt @ synth.so3_exp(rng.normal(0, 0.003, (W, 3)))
    return dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=np.concatenate([R0.reshape(W, 9), p_gt + rng.normal(0, 0.02, (W, 3))], 1))


def _all_masks(W):
    rng = np.random.default_rng(W)
    return [None, np.arange(W) == 0, rng.random(W) < 1 / 3, np.ones(W, bool), np.arange(W) >= W // 2]


def _check_tables(f, p, fixed):
    t = f.t
    W = f.W
    row_of = t["row_of"]
    want_rows = np.full(W, -1); free = np.arange(W) if fixed is None else np.flatnonzero(~fixed)
    want_rows[free] = np.arange(len(free))
    assert np.array_equal(row_of, want_rows) and f.n_rows == len(free)
    # the envelope: first[] over the free rows of every voxel, made monotone
    vp, pi = p["vox_ptr"], p["pose_idx"]
    first = np.arange(f.n_rows)
    for a in range(len(vp) - 1):
        r = row_of[pi[vp[a]:vp[a + 1]]]
        r = r[r >= 0]
        if len(r):
            first[r] = np.minimum(first[r], r.min())
    for r in range(f.n_rows - 2, -1, -1):
        first[r] = min(first[r], first[r + 1])
    assert np.array_equal(t["first"], first)
    rs = t["row_start"]
    blk = lambda r, c: rs[r] + c - first[r]          # noqa: E731
    lvp, lpi, tv = t["vox_ptr"], t["pidx"], t["tile_vox"]
    n_tiles = len(tv) - 1
    # every pair of free poses of the tiles' voxels once, under its block; nothing of a constant pose
    want_pairs, want_slots = set(), set()
    for k in range(n_tiles):
        s0 = lvp[tv[k]]
        for a in range(tv[k], tv[k + 1]):
            sl = list(range(lvp[a], lvp[a + 1]))
            for j in range(len(sl)):
                if row_of[lpi[sl[j]]] >= 0:
                    want_slots.add((k, sl[j] - s0))
                for i in range(j):
                    if row_of[lpi[sl[i]]] >= 0 and row_of[lpi[sl[j]]] >= 0:
                        want_pairs.add((k, sl[i] - s0, sl[j] - s0))
    got_pairs, got_slots = [], []
    pcode, prun, ptile = t["pcode"], t["prun"], t["ptile"]
    for k in range(n_tiles):
        s0 = lvp[tv[k]]
        for r in range(ptile[k], ptile[k + 1]):
            codes = pcode[prun[r]:prun[r + 1]]
            blocks = {blk(row_of[lpi[s0 + (c >> 16)]], row_of[lpi[s0 + (c & 0xffff)]]) for c in codes}
            assert len(blocks) == 1
            assert t["H_dst"][r] == blocks.pop()
            got_pairs += [(k, int(c & 0xffff), int(c >> 16)) for c in codes]
    dcode, drun, dtile = t["dcode"], t["drun"], t["dtile"]
    for k in range(n_tiles):
        s0 = lvp[tv[k]]
        for r in range(dtile[k], dtile[k + 1]):
            codes = dcode[drun[r]:drun[r + 1]]
            rows = {row_of[lpi[s0 + c]] for c in codes}
            assert len(rows) == 1
            row = rows.pop()
            assert row >= 0 and t["H_dst"][f.npr + r] == blk(row, row) and t["g_dst"][r] == row
            got_slots += [(k, int(c)) for c in codes]
    assert len(got_pairs) == len(set(got_pairs)) and set(got_pairs) == want_pairs
    assert len(got_slots) == len(set(got_slots)) and set(got_slots) == want_slots
    # the big voxels' records: under their row destination, or none (nblocks / W) for a constant pose
    bvp, bpose = t["big_vox_ptr"], t["big_pose"]
    h0, g0 = f.npr + f.ndr, f.ndr
    for s in range(len(bpose)):
        r = row_of[bpose[s]]
        assert t["H_dst"][h0 + s] == (blk(r, r) if r >= 0 else f.nblocks) and t["g_dst"][g0 + s] == (r if r >= 0 else W)
    q = h0 + len(bpose)
    for b in range(len(bvp) - 1):
        ps = bpose[bvp[b]:bvp[b + 1]]
        for j in range(len(ps)):
            for i in range(j):
                ri, rj = row_of[ps[i]], row_of[ps[j]]
                assert t["H_dst"][q] == (blk(rj, ri) if ri >= 0 and rj >= 0 else f.nblocks)
                q += 1
    assert q == len(t["H_dst"])
    # the record index: every record with a destination once, in ascending record order per destination
    for dst, code, run in ((t["H_dst"], t["H_code"], t["H_run"]), (t["g_dst"], t["g_code"], t["g_run"])):
        n_with = int(np.sum(dst < (f.nblocks if dst is t["H_dst"] else W)))
        assert run[-1] == n_with
        listed = code[:run[-1]]
        assert len(set(listed.tolist())) == n_with
        for r in range(len(run) - 1):
            c = code[run[r]:run[r + 1]]
            assert np.all(np.diff(c.astype(np.int64)) > 0) and len(set(dst[c].tolist())) == 1


@pytest.mark.parametrize("seed", [5, 6])
def test_table_with_constant_sets(emu, seed):
    p = _problem(seed)
    for fixed in _all_masks(len(p["poses"])):
        for bs in (128, 6):                                   # ordinary tiles; voxels of more than 6 slots through the big passes
            f = Fp(emu, p, fixed, batch_slots=bs)
            try:
                _check_tables(f, p, fixed)
            finally:
                f.close()


@pytest.mark.parametrize("level", ["L1", "L2"])
def test_table_big_passes_give_the_restricted_system(emu, level):
    """Every voxel through the big-voxel passes (batch_slots 1): H and g over the rows equal the oracle's H_ff, g_f, in both
    modes, and the residual covers every voxel."""
    vp, pi, cl, ps = _ref(level)
    p = dict(vox_ptr=vp, pose_idx=pi, clusters=cl, poses=ps)
    W = len(ps)
    assert np.diff(vp).min() >= 2
    rs, g_all, blocks = lo.acc_evaluate2(vp, pi, cl, ps, W)
    H_all = lo.assemble_dense(blocks, W)
    for fixed in _all_masks(W):
        f = Fp(emu, p, fixed, batch_slots=1)
        try:
            Hf, gf = lf.restricted(H_all, g_all, fixed)
            n = f.n_rows
            for det in (1, 0):
                H, g, r = f.run(ps, det)
                assert np.isclose(r, rs, rtol=1e-12)
                assert np.abs(g.ravel() - gf).max() <= 1e-9 * max(np.abs(gf).max(), 1e-30) if n else g.size == 0
                D = np.zeros((6 * n, 6 * n))
                rs_, fr = f.t["row_start"], f.t["first"]
                for rr in range(n):
                    for c in range(fr[rr], rr + 1):
                        B = H[rs_[rr] + c - fr[rr]].reshape(6, 6)
                        D[6 * rr:6 * rr + 6, 6 * c:6 * c + 6] = B
                        if c != rr:
                            D[6 * c:6 * c + 6, 6 * rr:6 * rr + 6] = B.T
                if n:
                    assert np.abs(D - Hf).max() <= 1e-9 * np.abs(Hf).max()
        finally:
            f.close()


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    """The tables and sums with constant poses do not depend on the order in which the items of a pass run, and the host policy
    finds no memory or UB error."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261017")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", "-k", "table", __file__],
                       capture_output=True, text=True, cwd=str(ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout


# ---- lvba_offline --fix-scans: the argument and the --check path (no GPU)
def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_fix_scans") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.fixture(scope="module")
def scan_data(tmp_path_factory):
    sys.path.insert(0, str(ROOT))
    from oracle import dataset_writer as dw, synth
    scans, poses = synth.make_scan_scene(17, W=6, n_per_scan=500)
    d = tmp_path_factory.mktemp("fix_scans_data") / "data"
    dw.write_lidar_dataset(d, scans, poses)
    return d


@pytest.mark.parametrize("value", ["", "x", "3:1", "1:", "-2", "1,,2"])
def test_offline_refuses_malformed_scan_ranges(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--fix-scans", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--fix-scans" in r.stderr, (r.returncode, r.stderr)


def test_offline_check_takes_scan_ranges_of_the_dataset(tool, scan_data):
    """--check loads the dataset and checks LIST against its scans: the last scan is fine, one past it is refused."""
    for value, rc in (("0", 0), ("0:2,5", 0), ("0:5", 0), ("6", 64), ("2:6", 64)):
        r = subprocess.run([str(tool), "--data", str(scan_data), "--fix-scans", value, "--check"], capture_output=True, text=True)
        assert r.returncode == rc, (value, r.returncode, r.stderr)
        if rc:
            assert "--fix-scans" in r.stderr and "past the last of 6" in r.stderr, r.stderr
        else:
            assert '"scans": 6' in r.stdout, r.stdout


def build_shim_case(pkg, out_dir):
    """tests/shim/fixed_poses_shim.cpp linked against the library"""
    exe = Path(out_dir) / "fixed_poses_shim"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tests" / "shim" / "fixed_poses_shim.cpp"),
                        "-o", str(exe), *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_shim_refuses_a_mask_of_the_wrong_size(pkg, tmp_path):
    r = subprocess.run([str(build_shim_case(pkg, tmp_path)), "size"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
