"""The DOGLEG oracle of the visual LM (tests/visual_dogleg_oracle.py) on its own: it stops within 1e-6 of the LM's final cost
with and without a loss, takes every one of the three steps across the scenes, and reuses the linearisation after a rejection."""
import numpy as np
import pytest

from oracle import synth
from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_dogleg_oracle as dl
import visual_loss_oracle as vl


def _small():
    return synth.make_problem(30, 600, 300, seed=11)


def _big():
    return vs.make_scene(5, M=120, n_short=150, long_tracks=((129, 10), (300, 0)))


def _perturbed():
    p = dict(_small())
    p["X"] = p["X"] + np.random.default_rng(1).normal(0, 2.0, p["X"].shape)
    return p


@pytest.mark.parametrize("make", [_small, _big])
@pytest.mark.parametrize("loss", [None, (vl.HUBER, 1.0)])
def test_dogleg_reaches_the_lm_cost(make, loss):
    p = make()
    _, lm = vo.ceres_lm(vl.RobustProblem(*vs.args(p), loss_reproj=loss))
    _, d = dl.dogleg(vl.RobustProblem(*vs.args(p), loss_reproj=loss))
    assert d["term"] in ("function", "parameter", "gradient")
    assert abs(d["cost"] - lm["cost"]) <= 1e-6 * lm["cost"]
    assert d["builds"] == d["iters"] - d["reused"]


def test_three_cases_and_reuse():
    p = _small()
    _, d = dl.dogleg(vl.RobustProblem(*vs.args(p)), radius0=1e-2)        # small radius: Cauchy, interpolated, then Gauss-Newton
    cases = {r["case"] for r in d["trace"]}
    _, d2 = dl.dogleg(vl.RobustProblem(*vs.args(_perturbed()), loss_reproj=(vl.HUBER, 1.0)))
    cases |= {r["case"] for r in d2["trace"]}
    assert cases == {dl.GAUSS_NEWTON, dl.CAUCHY, dl.INTERPOLATED}
    tr = d2["trace"]
    rejected = [i for i, r in enumerate(tr[:-1]) if r["valid"] and not r["accepted"]]
    assert rejected
    for i in rejected:
        assert tr[i + 1]["reused"] and tr[i + 1]["radius"] == 0.5 * tr[i]["radius"]
        assert tr[i + 1]["alpha"] == tr[i]["alpha"]
    assert d2["reused"] == len(rejected) and d2["builds"] == d2["iters"] - d2["reused"]


def test_step_cases():
    """The three cases of ComputeTraditionalDoglegStep on a two-dimensional example: the step norm, the boundary point."""
    g, GN, alpha = np.array([1.0, 0.0]), np.array([-2.0, -2.0]), 0.5
    c, s, n, _ = dl.dogleg_step(g, GN, alpha, 3.0)
    assert c == dl.GAUSS_NEWTON and np.array_equal(s, GN)
    c, s, n, _ = dl.dogleg_step(g, GN, alpha, 0.25)
    assert c == dl.CAUCHY and np.allclose(s, [-0.25, 0.0]) and n == 0.25
    c, s, n, beta = dl.dogleg_step(g, GN, alpha, 1.5)
    assert c == dl.INTERPOLATED and 0 < beta < 1 and abs(np.linalg.norm(s) - 1.5) <= 1e-14
    assert np.allclose(s, -alpha * (1 - beta) * g + beta * GN)
