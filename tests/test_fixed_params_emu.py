"""Constant cameras of the visual LM (lvba_visual_opts::cam_fixed) without a GPU: the C and ctypes layouts of the options, the
NULL default, LVBA_ERR_NO_DEVICE with a mask, the index ranges of lvba_offline --fix-cameras, and the build's destination table of
tests/test_visual_tiles_emu.py (host policy, the same functors as the library) for rows planned with constant camera sets —
camera 0 only, every other camera, all but one, all of them, and a landmark of 128 observations."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_visual_tiles_emu as vt  # noqa: E402
from test_visual_tiles_emu import emu  # noqa: E402,F401  (the host-policy library, a fixture)

KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")


def test_opts_layout_and_default(pkg, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "lvba_b200.h"\n'
                   'int main(void) { lvba_visual_opts o; lvba_visual_default_opts(&o);\n'
                   '  printf("%zu %zu %d\\n", sizeof(lvba_visual_opts), offsetof(lvba_visual_opts, cam_fixed), o.cam_fixed == NULL);\n'
                   '  return 0; }\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe), str(pkg.LIB_PATH),
                        f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(pkg.VisualOpts), pkg.VisualOpts.cam_fixed.offset, 1]
    assert pkg.VisualOpts.cam_fixed.offset == ctypes.sizeof(pkg.VisualOpts) - ctypes.sizeof(ctypes.c_void_p)   # the last field
    assert not pkg.visual_default_opts().cam_fixed


def test_no_device_with_a_mask(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    from oracle import synth
    p = synth.make_problem(6, 0, 20, seed=2, lidar=False)
    args = [p[k] for k in KEYS]
    with pytest.raises(pkg.LvbaError) as e:
        pkg.visual_lm(*args, fixed_cam=-1, cam_fixed=np.arange(6) % 2 == 0)
    assert e.value.status == -2
    with pytest.raises(ValueError):
        pkg.visual_lm(*args, cam_fixed=np.ones(5, bool))                      # one entry per camera


# ---- lvba_offline --fix-cameras (global-lvba_b200/host/lvba_visual_offline.hpp parse_index_ranges)
PARSER = r'''
#include <cstdio>
#include "../global-lvba_b200/host/lvba_visual_offline.hpp"
int main(int argc, char** argv) {
  for (int i = 1; i < argc; ++i) {
    std::vector<uint8_t> m{7};
    std::string err;
    if (lvba_b200::offline::parse_index_ranges(argv[i], 12, m, &err)) { for (uint8_t v : m) std::printf("%d", v); std::printf("\n"); }
    else std::printf("ERR %zu %s\n", m.size(), err.c_str());
  }
  return 0;
}
'''
GOOD = {"0": "100000000000", "0:3": "111100000000", "0:1,5,9:11": "110001000111", "2:2,2:4": "001110000000", "11": "000000000001"}
BAD = ["", "a", "1:", ":3", "3:1", "-1", "1:-2", "0:12", "12", "1,,2", "1:2:3", "0x3", " 1", "1,"]


def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


def test_parse_index_ranges(pkg, tmp_path):
    (tmp_path / "parse.cpp").write_text(PARSER.replace("../global-lvba_b200", str(ROOT / "global-lvba_b200")))
    exe = tmp_path / "parse"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(tmp_path / "parse.cpp"), "-o", str(exe), *_link(pkg)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    args = list(GOOD) + BAD
    out = subprocess.run([str(exe), *args], capture_output=True, text=True).stdout.splitlines()
    assert len(out) == len(args)
    for a, line in zip(args, out):
        if a in GOOD:
            assert line == GOOD[a], (a, line)
        else:
            assert line.startswith("ERR 1 "), (a, line)                       # refused, mask untouched


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_fix") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("value", ["", "x", "3:1", "1:", "-2", "1,,2"])
def test_offline_refuses_malformed_camera_ranges(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--fix-cameras", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--fix-cameras" in r.stderr, (r.returncode, r.stderr)


def test_offline_accepts_camera_ranges(tool, tmp_path):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flag."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--fix-cameras", "0:3,10", "--check"], capture_output=True, text=True)
    assert "--fix-cameras" not in r.stderr and "unknown argument" not in r.stderr, r.stderr


# ---- the destination table with constant camera sets
def rows_of_mask(obs_cam, M, const):
    used = np.zeros(M, bool)
    used[obs_cam] = True
    used[const] = False
    row_of_cam = np.full(M, -1, np.int64)
    row_of_cam[used] = np.arange(used.sum())
    return row_of_cam.astype(np.int32), int(used.sum())


def masks(M, rng):
    yield np.arange(M) == 0                                                   # camera 0 only (the reference)
    yield np.arange(M) % 2 == 1                                               # every other
    yield np.arange(M) != M // 3                                              # all but one
    yield np.ones(M, bool)                                                    # all: no system row
    yield rng.random(M) < 0.3                                                 # scattered
    yield np.arange(M) < (3 * M) // 4                                         # the first 75 %


def test_table_with_constant_sets(emu):  # noqa: F811
    rng = np.random.default_rng(5)
    for seed in (41, 42):
        op, cam, _, _ = vt.problem(seed, fixed_cam=-1)
        M = 40
        for m in masks(M, rng):
            rc, n = rows_of_mask(cam, M, m)
            assert np.all(rc[m] == -1)
            t = vt.check(emu, op, cam, rc, n)
            vt.check(emu, op, cam, rc, n, max_slots=32, max_trk=4)
            # nothing of a constant camera has a destination: every observation in a row run sees a free camera
            lrow = t["row"]
            dcode, drun, ltp, tt = t["dcode"], t["drun"], t["trk_ptr"].astype(np.int64), t["tile_trk"]
            for k in range(len(tt) - 1):
                s0 = ltp[tt[k]]
                d0, d1 = drun[t["dtile"][k]], drun[t["dtile"][k + 1]]
                assert np.all(lrow[s0 + dcode[d0:d1]] >= 0)
            assert drun[-1] == int((lrow >= 0).sum())


def test_table_long_landmark_with_constant_cameras(emu):  # noqa: F811
    """A landmark of 128 observations (the most a tile takes) with half its cameras constant, and landmarks that see only
    constant cameras: the tiles' runs hold the free observations only."""
    rng = np.random.default_rng(12)
    M = 60
    tracks = [list(rng.choice(M, 128)), [1, 2, 3], [0, 0, 4], [2, 4]]
    op = np.zeros(len(tracks) + 1, np.int64); op[1:] = np.cumsum([len(t) for t in tracks])
    cam = np.array([c for t in tracks for c in t], np.int64)
    m = np.arange(M) % 2 == 0
    rc, n = rows_of_mask(cam, M, m)
    for S, NT in ((0, 0), (128, 64), (130, 2)):
        vt.check(emu, op, cam, rc, n, max_slots=S, max_trk=NT)


def _asan():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    return lib if lib and Path(lib).exists() else None


@pytest.mark.parametrize("mode", ["shuffle", "sanitize"])
def test_rerun_with_shuffled_items_and_sanitizers(mode):
    """The tables with constant cameras do not depend on the order in which the items of a pass run, and the host policy finds
    no memory or UB error."""
    if os.environ.get("LVBA_EMU_RERUN"):
        pytest.skip("this is the re-run")
    env = dict(os.environ, LVBA_EMU_RERUN="1", LVBA_EMU_SHUFFLE="20261016")
    if mode == "sanitize":
        asan = _asan()
        if not asan:
            pytest.skip("no libasan")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", "-k", "table", __file__],
                       capture_output=True, text=True, cwd=str(ROOT), env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
