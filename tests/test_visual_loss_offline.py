"""`lvba_offline --reproj-loss KIND[:A] --plane-loss KIND[:A]` (global-lvba_b200/host/lvba_visual_offline.hpp parse_loss): good values
set the visual stage's loss and scale, malformed ones are refused with a message.  No GPU needed."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]

PARSER = r'''
#include <cstdio>
#include "../global-lvba_b200/host/lvba_visual_offline.hpp"
int main(int argc, char** argv) {
  for (int i = 1; i < argc; ++i) {
    int32_t kind = -7; double scale = -7.0; std::string err;
    if (lvba_b200::offline::parse_loss(argv[i], 0.1, kind, scale, &err)) std::printf("%d %.17g\n", kind, scale);
    else std::printf("ERR %d %g %s\n", kind, scale, err.c_str());
  }
  return 0;
}
'''

GOOD = {"none": (0, 0.1), "huber": (1, 0.1), "cauchy": (2, 0.1), "huber:1": (1, 1.0), "cauchy:2.5": (2, 2.5), "huber:1e-3": (1, 1e-3),
        "none:3": (0, 3.0)}
BAD = ["", "Huber", "huber:", "huber:0", "huber:-1", "cauchy:nan", "cauchy:inf", "huber:1x", "tukey", "huber:1:2", ":1"]


def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


@pytest.fixture(scope="module")
def parser(pkg, tmp_path_factory):
    d = tmp_path_factory.mktemp("loss_parse")
    (d / "parse.cpp").write_text(PARSER.replace("../global-lvba_b200", str(ROOT / "global-lvba_b200")))
    exe = d / "parse"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(d / "parse.cpp"), "-o", str(exe), *_link(pkg)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_parse_loss(parser):
    args = list(GOOD) + BAD
    out = subprocess.run([str(parser), *args], capture_output=True, text=True).stdout.splitlines()
    assert len(out) == len(args)
    for a, line in zip(args, out):
        if a in GOOD:
            k, s = line.split()
            assert (int(k), float(s)) == GOOD[a], (a, line)
        else:
            assert line.startswith("ERR -7 -7 "), (a, line)           # refused, kind and scale untouched


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_loss") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("flag", ["--reproj-loss", "--plane-loss"])
@pytest.mark.parametrize("value", ["bogus", "huber:0", "cauchy:-2", "huber:abc"])
def test_offline_refuses_a_malformed_loss(tool, tmp_path, flag, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), flag, value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and flag in r.stderr and value in r.stderr, (r.returncode, r.stderr)


def test_offline_accepts_good_losses(tool, tmp_path):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flags."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--reproj-loss", "huber", "--plane-loss", "cauchy:0.05", "--check"],
                       capture_output=True, text=True)
    assert "-loss" not in r.stderr and "unknown argument" not in r.stderr, r.stderr
