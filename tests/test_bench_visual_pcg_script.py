"""tools/bench_visual_pcg.py needs a GPU for its numbers, not for its own plumbing: its argument parsing, and with the device class
replaced by a stand-in of the same shape, the scenes it builds (the long tracks longer than 128 observations, the loop-closed
track) and one well-formed JSON line per scene and solver."""
import importlib.util
import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def _script():
    spec = importlib.util.spec_from_file_location("bench_visual_pcg", ROOT / "tools" / "bench_visual_pcg.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


class _FakeProblem:
    def __init__(self, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam=0, device=-1):
        self.solver = 0

    def reset_lm(self, opts=None, linear_solver=None, **kw):
        self.solver = linear_solver

    def reset_state(self):
        pass

    def iterate(self, n):
        return dict(iterations=n, ms_build=0.3 * n, ms_solve=(1.7 if self.solver else 0.6) * n, ms_total=1.1 * n, cost_last=2.0,
                    termination=1)

    def linear_stats(self):
        return dict(cg_iters_total=12, cg_iters_last=12 if self.solver else 0, term_last=0)

    def counts(self):
        return dict(nnz_valid=0, n_valid_tracks=0, n_blocks_env=10, n_pairs=7)

    def close(self):
        pass


def test_scenes_are_the_ones_described():
    m = _script()
    sc = dict(m.scenes({"long", "loop"}, "B", 5))
    assert len(sc) == 2
    long_ = [p for k, p in sc.items() if "long" in k][0]
    assert (np.diff(long_["obs_ptr"]) > 128).sum() == 5
    loop = [p for k, p in sc.items() if "loop" in k][0]
    K = np.diff(loop["obs_ptr"])
    wrapped = [np.unique(loop["obs_cam"][loop["obs_ptr"][i]:loop["obs_ptr"][i + 1]]) for i in np.nonzero(K == 20)[0]]
    assert any(c.min() < 10 and c.max() >= 390 for c in wrapped)


def test_unknown_scene_is_refused():
    with pytest.raises(SystemExit):
        _script().main(["--scenes", "config,bogus"])


def test_script_runs_to_the_end_with_stand_ins(pkg, monkeypatch, capsys):
    monkeypatch.setattr(pkg, "VisualProblem", _FakeProblem)
    monkeypatch.setattr(pkg, "device_count", lambda: 1)
    m = _script()
    assert m.main(["--config", "B", "--scenes", "loop", "--passes", "3", "--repeats", "1"]) == 0
    lines = [json.loads(x) for x in capsys.readouterr().out.strip().splitlines()]
    assert [x["solver"] for x in lines] == ["dense_schur", "iterative_schur"]
    for x in lines:
        assert {"ms_solve", "lm_passes_per_s", "cost_after_3", "passes_to_convergence", "final_cost", "n_blocks_env", "gpu"} <= set(x)
    assert lines[1]["cg_iters_mean"] == 12 and lines[1]["cg_iters_max"] == 12
