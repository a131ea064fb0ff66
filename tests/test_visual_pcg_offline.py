"""`lvba_offline --linear-solver dense_schur|iterative_schur` (lvba_visual_opts::linear_solver): a bad value is refused when parsed,
--check included; a good one gets past the parsing."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_pcg") / "lvba_offline"
    link = [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *link], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("value", ["bogus", "DENSE_SCHUR", "iterative", ""])
def test_offline_refuses_an_unknown_solver(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--linear-solver", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--linear-solver" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("value", ["dense_schur", "iterative_schur"])
def test_offline_accepts_both_solvers(tool, tmp_path, value):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flag."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--linear-solver", value, "--check"], capture_output=True, text=True)
    assert "--linear-solver" not in r.stderr and "unknown argument" not in r.stderr, r.stderr
