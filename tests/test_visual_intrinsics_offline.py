"""`lvba_offline --refine-intrinsics LIST` (global-lvba_b200/host/lvba_visual_offline.hpp parse_intr_groups): good lists set
lvba_visual_opts::refine_intrinsics, malformed ones are refused when parsed, --check included; and one GPU run of the visual
stage with the flag on a synthetic room."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]

PARSER = r'''
#include <cstdio>
#include "../global-lvba_b200/host/lvba_visual_offline.hpp"
int main(int argc, char** argv) {
  for (int i = 1; i < argc; ++i) {
    uint32_t mask = 0xdead; std::string err;
    if (lvba_b200::offline::parse_intr_groups(argv[i], mask, &err)) std::printf("%u\n", mask);
    else std::printf("ERR %u %s\n", mask, err.c_str());
  }
  return 0;
}
'''

GOOD = {"focal": 0x03, "principal": 0x0C, "distortion": 0xF0, "focal,distortion": 0xF3, "distortion,principal,focal": 0xFF}
BAD = ["", "Focal", "focal,", ",focal", "focal,,principal", "focal,focal", "all", "k1", "focal principal"]


def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


@pytest.fixture(scope="module")
def parser(pkg, tmp_path_factory):
    d = tmp_path_factory.mktemp("intr_parse")
    (d / "parse.cpp").write_text(PARSER.replace("../global-lvba_b200", str(ROOT / "global-lvba_b200")))
    exe = d / "parse"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(d / "parse.cpp"), "-o", str(exe), *_link(pkg)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_parse_intr_groups(parser):
    args = list(GOOD) + BAD
    out = subprocess.run([str(parser), *args], capture_output=True, text=True).stdout.splitlines()
    assert len(out) == len(args)
    for a, line in zip(args, out):
        if a in GOOD:
            assert int(line) == GOOD[a], (a, line)
        else:
            assert line.startswith(f"ERR {0xdead} "), (a, line)           # refused, mask untouched


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_intr") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("value", ["bogus", "focal,focal", "focal,", ""])
def test_offline_refuses_a_malformed_list(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--refine-intrinsics", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--refine-intrinsics" in r.stderr, (r.returncode, r.stderr)


def test_offline_accepts_good_lists(tool, tmp_path):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flag."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--refine-intrinsics", "focal,distortion", "--check"], capture_output=True, text=True)
    assert "--refine-intrinsics" not in r.stderr and "unknown argument" not in r.stderr, r.stderr


@pytest.mark.gpu
def test_visual_stage_refines_intrinsics(gpu_pkg, tool, tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import visual_scene
    data = tmp_path / "data"
    visual_scene.make(data, seed=3, W=8, n_landmarks=700)
    base = [str(tool), "--data", str(data), "--config", str(data / "config.yaml"), "--visual"]

    def run(*extra):
        r = subprocess.run(base + list(extra), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        return [json.loads(x) for x in r.stdout.strip().splitlines()]
    plain = run()
    assert not [x for x in plain if x.get("stage") == "intrinsics"]
    vp = [x for x in plain if x.get("stage") == "visual"][0]
    ref = run("--refine-intrinsics", "focal", "--points3d", "lidar")
    vr = [x for x in ref if x.get("stage") == "visual"][0]
    it = [x for x in ref if x.get("stage") == "intrinsics"][0]
    vals = np.array([it[k] for k in ("fx", "fy", "cx", "cy", "d0", "d1", "d2", "d3")])
    assert np.all(np.isfinite(vals))
    # the scene is rendered with the config's intrinsics: refining the focal lengths lowers the cost a little and keeps them close
    assert vr["cost_last"] <= vp["cost_last"] * (1 + 1e-6)
    pts = np.loadtxt(data / "Colmap" / "sparse" / "points3D.txt")
    assert pts.ndim == 2 and len(pts) > 0
    held = run("--refine-intrinsics", "principal")
    ih = [x for x in held if x.get("stage") == "intrinsics"][0]
    assert ih["fx"] != it["fx"] and ih["d0"] == it["d0"] and ih["d3"] == it["d3"]     # only the listed group moves
    assert abs(it["fx"] / ih["fx"] - 1) < 0.05 and abs(it["fy"] / ih["fy"] - 1) < 0.05
