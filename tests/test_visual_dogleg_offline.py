"""`lvba_offline --trust-region lm|dogleg` (lvba_visual_opts::trust_region_strategy): a bad value is refused when parsed, --check
included; a good one gets past the parsing."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_dogleg") / "lvba_offline"
    link = [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *link], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("value", ["bogus", "LM", "traditional_dogleg", ""])
def test_offline_refuses_an_unknown_strategy(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--trust-region", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--trust-region" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("value", ["lm", "dogleg"])
def test_offline_accepts_both_strategies(tool, tmp_path, value):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flag."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--trust-region", value, "--check"], capture_output=True, text=True)
    assert "--trust-region" not in r.stderr and "unknown argument" not in r.stderr, r.stderr
