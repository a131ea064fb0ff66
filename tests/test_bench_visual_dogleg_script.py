"""tools/bench_visual_dogleg.py needs a GPU for its numbers, not for its own plumbing: its argument parsing and, with the device
class replaced by a stand-in of the same shape, its per-pass bookkeeping (rejected passes, the passes after them) and one
well-formed JSON line per strategy."""
import importlib.util
import json
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def _script():
    spec = importlib.util.spec_from_file_location("bench_visual_dogleg", ROOT / "tools" / "bench_visual_dogleg.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


class _FakeProblem:
    """Passes: accepted, rejected, reused-and-accepted, accepted with a function-tolerance stop"""
    ACC = (1, 0, 1, 0)

    def __init__(self, *a, **kw):
        self.i = 0
        self.strategy = 0

    def reset_lm(self, opts=None, trust_region_strategy=None, **kw):
        self.strategy = trust_region_strategy

    def reset_state(self):
        self.i = 0

    def iterate(self, n):
        i = self.i
        self.i += 1
        if i >= 4:
            return dict(iterations=0, accepted=0, hessian_builds=0, ms_total=0.0, cost_last=1.0, termination=1)
        reused = self.strategy == 1 and i == 2
        return dict(iterations=1, accepted=self.ACC[i], hessian_builds=0 if reused else 1, ms_total=0.5 if reused else 2.0,
                    cost_last=1.0, termination=1 if i == 3 else 0)

    def close(self):
        pass


def test_bookkeeping():
    m = _script()

    class Pkg:
        VisualProblem = _FakeProblem

    p = {k: None for k in m.VKEYS}
    lm = m.measure(Pkg, p, 0, 1)
    dg = m.measure(Pkg, p, 1, 1)
    assert lm["passes_to_stop"] == dg["passes_to_stop"] == 4 and lm["rejected"] == dg["rejected"] == 1
    assert lm["builds_per_pass"] == 1.0 and dg["builds_per_pass"] == 0.75
    assert lm["ms_after_reject"] == 2.0 and dg["ms_after_reject"] == 0.5 and dg["ms_other"] == 2.0
    assert dg["termination"] == 1
    json.dumps(dg)


def test_bad_scene_is_refused():
    with pytest.raises(SystemExit):
        _script().main(["--scenes", "config,moon"])
