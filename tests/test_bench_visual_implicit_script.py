"""tools/bench_visual_implicit.py needs a GPU for its numbers, not for its own plumbing: its argument parsing, the street scene it
adds to tools/bench_visual_pcg.py's, and, with the device class replaced by a stand-in of the same shape, one well-formed JSON
line per scene."""
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def _script():
    spec = importlib.util.spec_from_file_location("bench_visual_implicit", ROOT / "tools" / "bench_visual_implicit.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


class _FakeProblem:
    def __init__(self, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam=0, device=-1):
        self.M = len(q)

    def reset_lm(self, opts=None, linear_solver=None, **kw):
        assert linear_solver == 1

    def reset_state(self):
        pass

    def iterate(self, n):
        return dict(iterations=n, ms_build=0.3 * n, ms_solve=1.7 * n, ms_residual=0.2 * n, ms_total=2.2 * n, cost_last=2.0, termination=1)

    def linear_stats(self):
        return dict(cg_iters_total=12, cg_iters_last=4, term_last=0)

    def schur_product(self):
        return 1

    def structure(self):
        return np.arange(self.M - 1), np.zeros(0), np.zeros(0)

    def counts(self):
        return dict(nnz_valid=100, n_valid_tracks=10, n_blocks_env=10, n_pairs=7)

    def close(self):
        pass


def test_street_scene_has_the_long_tracks():
    sc = dict(_script().scenes({"street"}, "C", 0))
    p = sc["street M=400"]
    assert sorted(np.diff(p["obs_ptr"]))[-5:] == [300, 450, 600, 800, 1000]


def test_unknown_scene_is_refused():
    with pytest.raises(SystemExit):
        _script().main(["--scenes", "config,bogus"])


def test_record_bytes():
    m = _script()
    assert m.record_bytes(10, 8, 2, 1) == 10 * 192 + 8 * 12 + 2 * 168 + (32 * 39 + 36) * 8 + 16


def test_script_runs_to_the_end_with_stand_ins(pkg, monkeypatch, capsys):
    monkeypatch.setattr(pkg, "VisualProblem", _FakeProblem)
    monkeypatch.setattr(pkg, "device_count", lambda: 1)
    m = _script()
    assert m.main(["--scenes", "loop", "--passes", "3", "--repeats", "1"]) == 0
    lines = [json.loads(x) for x in capsys.readouterr().out.strip().splitlines()]
    assert [x["scene"] for x in lines] == ["loop-closed M=400"]
    for x in lines:
        assert {"matrix_free", "ms_build", "ms_solve", "ms_residual", "lm_passes_per_s", "cg_iters_mean", "cg_iters_max",
                "record_bytes", "gpu"} <= set(x)
        assert x["matrix_free"] == 1 and x["cg_iters_max"] == 4 and abs(x["ms_build"] - 0.3) < 1e-12
