"""Order independence and memory safety of the visual outlier-removal passes (tests/test_visual_outliers_emu.py) on the host policy:
re-run with the items of every pass visited in pseudo-random orders (LVBA_EMU_SHUFFLE) and, where libasan exists, under
ASan/UBSan.  Buffers the passes allocate come back poisoned on the host policy (tests/emu/host_exec.h) in every run."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
SUITE = "tests/test_visual_outliers_emu.py"
FILTER = "host_policy"


def _run(env):
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", SUITE, "-k", FILTER],
                       capture_output=True, text=True, cwd=str(ROOT), env=dict(os.environ, **env), timeout=900)
    return r.returncode, r.stdout, r.stderr


@pytest.mark.parametrize("seed", ["3", "20261017"])
def test_visual_outlier_passes_with_shuffled_items(seed):
    rc, out, err = _run({"LVBA_EMU_SHUFFLE": seed})
    assert rc == 0, out[-3000:] + err[-2000:]
    assert "passed" in out


def test_visual_outlier_passes_under_sanitizers():
    lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not lib or not Path(lib).exists():
        pytest.skip("libasan is not installed")
    rc, out, err = _run({"LVBA_EMU_SANITIZE": "1", "LD_PRELOAD": lib, "ASAN_OPTIONS": "detect_leaks=0:abort_on_error=1", "LVBA_EMU_SHUFFLE": "7"})
    assert rc == 0, out[-3000:] + err[-2000:]
    assert "passed" in out
