"""tools/bench_visual_big.py needs a GPU for its numbers, not for its own plumbing: with the device class and calls replaced by
stand-ins of the same shape, the script must build both problems (the long tracks really longer than 128 observations) and
print two well-formed JSON lines."""
import importlib.util
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]


class _FakeProblem:
    def __init__(self, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam=0, device=-1):
        K = np.diff(obs_ptr)
        self.K = K[K > 128]
        self.M = len(q)

    def big_counts(self):
        return dict(n_big=len(self.K), n_big_obs=int(self.K.sum()), n_big_pairs=int((self.K * (self.K - 1)).sum()))

    def counts(self):
        return dict(nnz_valid=0, n_valid_tracks=0, n_blocks_env=0, n_pairs=7)

    def reset_lm(self, opts=None):
        pass

    def reset_state(self):
        pass

    def iterate(self, n):
        return dict(iterations=n, ms_build=0.4 * n, ms_solve=0.6 * n, ms_residual=0.1 * n)

    def step(self, radius):
        return None

    def get_system(self):
        return np.arange(3), np.zeros((3, 6)), np.array([0, 1, 1, 2]), np.array([0, 0, 1, 2]), np.zeros((4, 6, 6))

    def close(self):
        pass


def test_side_script_runs_to_the_end_with_stand_ins(pkg, monkeypatch, capsys):
    monkeypatch.setattr(pkg, "VisualProblem", _FakeProblem)
    monkeypatch.setattr(pkg, "visual_lm", lambda *a, **k: (None, None, None, dict(ms_setup=5.0)))
    monkeypatch.setattr(pkg, "env_solve", lambda *a, **k: (None, 0.1, dict(path=2, chunks=0, levels=0, launches=1)))
    monkeypatch.setattr(pkg, "device_count", lambda: 1)
    spec = importlib.util.spec_from_file_location("bench_visual_big", ROOT / "tools" / "bench_visual_big.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    monkeypatch.setattr(sys, "argv", ["bench_visual_big.py", "--config", "B", "--long", "4", "--kmin", "129", "--kmax", "140", "--iters", "2", "--repeats", "1"])
    assert mod.main() == 0
    lines = [json.loads(ln) for ln in capsys.readouterr().out.splitlines() if ln.startswith("{")]
    assert len(lines) == 2
    assert lines[0]["big_counts"]["n_big"] == 0 and lines[0]["big_pass_bytes"] == 0
    assert lines[1]["big_counts"]["n_big"] == 4 and lines[1]["big_pass_bytes"] > 0
    assert lines[1]["solve_path"] == "twisted" and lines[1]["ms_per_pass"]["ms_build"] == 0.4
