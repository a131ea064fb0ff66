"""The DOGLEG trust-region strategy of the visual LM (lvba_visual_opts::trust_region_strategy, global-lvba_b200/csrc/visual_dogleg.h)
on the H100: the whole solve against tests/visual_dogleg_oracle.py pass for pass (accept / reject, the case, the cost), the
build count of reused passes, determinism, the reset by a removal and by a cam_fixed re-plan, the refusals, and the default
strategy's results unchanged."""
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest

from oracle import synth
import visual_big_scene as vs
import visual_dogleg_oracle as dl
import visual_fixed_oracle as vf
import visual_loss_oracle as vl

pytestmark = pytest.mark.gpu
TR_DOGLEG = 1


def _small():
    return synth.make_problem(30, 600, 300, seed=11)


def _big():
    return vs.make_scene(5, M=120, n_short=150, long_tracks=((129, 10), (300, 0)))


def _perturbed():
    """_small with its landmarks moved by 2 m: Cauchy steps, interpolated steps, rejections and reused passes"""
    p = dict(_small())
    p["X"] = p["X"] + np.random.default_rng(1).normal(0, 2.0, p["X"].shape)
    return p


def _moved():
    """_small with its landmarks moved by 0.6 m, every one staying in front of its cameras along the path: from radius 1e4 a
    Gauss-Newton step is rejected, the next pass reuses the linearisation and is rejected again, the one after reuses it for
    an interpolated step that is accepted"""
    p = dict(_small())
    p["X"] = p["X"] + np.random.default_rng(1).normal(0, 0.6, p["X"].shape)
    return p


CAMS = (0, 3, 4)
# scene: (make, reprojection loss, constant cameras, initial radius)
SCENES = {"small": (_small, None, False, 1e4), "small_huber": (_small, (1, 1.0), False, 1e4), "big": (_big, None, False, 1e4),
          "cam_fixed": (_small, None, True, 1e4), "perturbed": (_perturbed, (1, 1.0), False, 1e4),
          "small_radius": (_small, None, False, 0.1), "big_radius": (_big, (1, 1.0), False, 0.1), "moved": (_moved, None, False, 1e4)}


def _opts(pkg, loss=None, **kw):
    o = pkg.visual_default_opts(loss)
    o.trust_region_strategy = TR_DOGLEG
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _mask(M):
    return vf.mask_of(M, CAMS)


def _device_trace(pkg, p, loss, cam_fixed, n_max=60, **kw):
    P = pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(pkg, loss, **kw), cam_fixed=_mask(len(p["q"])) if cam_fixed else None)
    trace, total = [], dict(iterations=0, hessian_builds=0, termination=0)
    for _ in range(n_max):
        s = P.iterate(1)
        total["hessian_builds"] += s["hessian_builds"]
        total["termination"] = s["termination"]
        if s["iterations"] == 0:
            break
        total["iterations"] += 1
        d = P.dogleg_state()
        trace.append(dict(accepted=s["accepted"] == 1, case=d["case"], cost=s["cost_last"], radius=d["radius"], reused=d["reused"]))
        if s["termination"] != 0:
            break
    st = P.dogleg_state()
    P.close()
    return trace, total, st


def _oracle(p, loss, cam_fixed, radius0=1e4):
    pr = vl.RobustProblem(*vs.args(p), loss_reproj=loss)
    if cam_fixed:
        vf.with_constant(pr, CAMS)
    return dl.dogleg(pr, radius0=radius0)[1]


TERM = {"max_iter": 0, "function": 1, "parameter": 2, "gradient": 3, "radius": 4, "invalid_steps": 5}


@pytest.mark.parametrize("scene", ["small", "small_huber", "big", "cam_fixed", "small_radius", "big_radius", "moved"])
def test_dogleg_matches_the_oracle_pass_for_pass(gpu_pkg, scene):
    """From radius 1e4 the first four scenes take Gauss-Newton steps; from radius 0.1 the Cauchy and the interpolated steps come
    first; the moved scene rejects steps and reuses its linearisation for them"""
    make, loss, cam_fixed, radius0 = SCENES[scene]
    p = make()
    trace, total, st = _device_trace(gpu_pkg, p, loss, cam_fixed, initial_radius=radius0)
    info = _oracle(p, loss, cam_fixed, radius0)
    ref = info["trace"]
    assert len(trace) == len(ref) == info["iters"]
    for i, (a, b) in enumerate(zip(trace, ref)):
        assert (a["accepted"], a["case"]) == (b["accepted"], b["case"]), (a, b)
        cost = b["cand"] if b["accepted"] else b["cost"]
        # the moved scene falls from 5e7 to 2e3 in a few steps: there a candidate's cost is held to 1e-9 of the cost its pass
        # started from, the scale of the rounding in the step that led to it
        scale = b["cost"] if scene == "moved" else cost
        assert abs(a["cost"] - cost) <= 1e-9 * scale, (a, b)
        if i + 1 < len(ref):                             # the radius after this pass is the one the next pass used
            assert abs(a["radius"] - ref[i + 1]["radius"]) <= 1e-9 * ref[i + 1]["radius"], (a, ref[i + 1])
            assert a["reused"] == sum(r["reused"] for r in ref[:i + 1])
    if scene == "small_radius":
        assert {b["case"] for b in ref} == {1, 2, 3}
    if scene == "moved":
        assert [b["reused"] for b in ref[:4]] == [False, False, True, True] and ref[3]["case"] == 3 and ref[3]["accepted"]
    assert total["termination"] == TERM[info["term"]]
    # a linearisation per pass that does not reuse one (+1 for a stop on the gradient tolerance, which linearises first)
    assert total["hessian_builds"] == info["builds"] == total["iterations"] - st["reused"] + (total["termination"] == 3)
    assert st["reused"] == info["reused"]


def test_reused_passes_on_the_perturbed_scene(gpu_pkg):
    """Rejections keep the linearisation: every pass after a rejected one reuses it, all three cases occur,
    and the build count falls short of the pass count by the reused passes.  Moved landmarks cross behind their cameras here,
    where the cost jumps, so the path is not compared with the oracle's pass for pass."""
    make, loss, _, _ = SCENES["perturbed"]
    trace, total, st = _device_trace(gpu_pkg, make(), loss, False, n_max=40)
    assert {a["case"] for a in trace} == {1, 2, 3}
    rejected = [i for i in range(len(trace) - 1) if not trace[i]["accepted"]]
    assert rejected
    for i in rejected:
        assert trace[i + 1]["reused"] == trace[i]["reused"] + 1
    assert st["reused"] == len(rejected) and total["hessian_builds"] == total["iterations"] - st["reused"]


def test_one_shot_dogleg(gpu_pkg):
    p = _small()
    _, _, _, s = gpu_pkg.visual_lm(*vs.args(p), trust_region_strategy=TR_DOGLEG)
    info = _oracle(p, None, False)
    assert (s["iterations"], s["accepted"], s["hessian_builds"]) == (info["iters"], info["accepted"], info["builds"])
    assert abs(s["cost_last"] - info["cost"]) <= 1e-9 * info["cost"]


@pytest.mark.parametrize("scene", ["small", "perturbed"])
def test_deterministic_runs_are_bit_identical(gpu_pkg, scene):
    make, loss, _, _ = SCENES[scene]
    p = make()
    runs = []
    for _ in range(2):
        P = gpu_pkg.VisualProblem(*vs.args(p))
        P.reset_lm(_opts(gpu_pkg, loss, deterministic=1))
        s = P.iterate(10)
        runs.append((P.get_state(), {k: v for k, v in s.items() if not k.startswith("ms_")}, P.dogleg_state()))
        P.close()
    (a, sa, da), (b, sb, db) = runs
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert sa == sb and da == db


def test_removal_and_replan_reset_the_state(gpu_pkg):
    make, loss, _, _ = SCENES["perturbed"]
    p = make()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, loss))
    P.iterate(40)
    assert P.dogleg_state()["reused"] > 0
    P.remove_outliers(1e3, 2)
    d = P.dogleg_state()
    assert (d["reused"], d["case"], d["mu"], d["radius"]) == (0, 0, 1e-8, 1e4)
    P.iterate(8)
    assert P.dogleg_state()["case"] != 0
    P.reset_lm(_opts(gpu_pkg, loss), cam_fixed=_mask(len(p["q"])))
    d = P.dogleg_state()
    assert (d["reused"], d["case"], d["mu"], d["alpha"]) == (0, 0, 1e-8, 0.0)
    s = P.iterate(3)                                  # the state has converged by now: one pass may end the solve
    assert s["iterations"] >= 1 and P.dogleg_state()["case"] != 0
    P.reset_lm(gpu_pkg.visual_default_opts())
    with pytest.raises(gpu_pkg.LvbaError):
        P.dogleg_state()
    P.close()


def test_refusals_leave_the_handle_unchanged(gpu_pkg):
    p = _small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg))
    P.iterate(2)
    state, ds = P.get_state(), P.dogleg_state()
    bad = [(dict(trust_region_strategy=2), -1), (dict(trust_region_strategy=-1), -1), (dict(linear_solver=1), -1),
           (dict(refine_intrinsics=0x03), -4)]
    for kw, code in bad:
        with pytest.raises(gpu_pkg.LvbaError) as e:
            P.reset_lm(_opts(gpu_pkg, **kw))
        assert e.value.status == code, kw
        with pytest.raises(gpu_pkg.LvbaError) as e:
            gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, **kw))
        assert e.value.status == code, kw
    assert all(np.array_equal(x, y) for x, y in zip(state, P.get_state()))
    assert P.dogleg_state() == ds
    s = P.iterate(1)
    assert s["iterations"] == 1
    P.close()


@pytest.mark.parametrize("change", ["none", "set_state", "reset_state", "set_intrinsics", "step_rescale"])
def test_state_changes_end_the_reuse(gpu_pkg, change):
    """On the moved scene the second pass is rejected, so the third would reuse its linearisation.  A call that changes the
    state, the intrinsics or the Jacobi scale in between makes the third pass linearise again at what the handle now holds."""
    p = _moved()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg))
    s = P.iterate(2)
    assert (s["iterations"], s["accepted"]) == (2, 1)
    reused = P.dogleg_state()["reused"]
    if change == "set_state":
        q, t, _ = P.get_state()
        P.set_state(q, t, _small()["X"])
    elif change == "reset_state":
        P.reset_state()
    elif change == "set_intrinsics":
        intr = np.array(p["intr"], np.float64)
        intr[0] *= 1.001
        P.set_intrinsics(intr)
    elif change == "step_rescale":
        P.step(1e4, recompute_scale=True)
    cost = P.cost()
    s = P.iterate(1)
    assert s["iterations"] == 1
    if change == "none":
        assert s["hessian_builds"] == 0 and P.dogleg_state()["reused"] == reused + 1
    else:
        assert s["hessian_builds"] == 1 and P.dogleg_state()["reused"] == reused
        # the pass took the cost at the handle's state: a rejected step keeps it, an accepted one lowers it
        if s["accepted"]:
            assert s["cost_last"] < cost
        else:
            assert abs(s["cost_last"] - cost) <= 1e-12 * cost      # the build's sum of the cost, in another order
    P.close()


def test_default_strategy_unchanged(gpu_pkg):
    """lvba_visual_lm with the default options in deterministic mode gives the bits of the build before the trust-region
    strategy option (tests/golden/visual_default_lm.json, tests/golden/make_golden_visual_default.py)."""
    golden = Path(__file__).resolve().parent / "golden"
    spec = importlib.util.spec_from_file_location("make_golden_visual_default", golden / "make_golden_visual_default.py")
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    want = json.loads((golden / "visual_default_lm.json").read_text())
    for name, (p, loss) in mg.scenes().items():
        got = mg.digest(gpu_pkg, p, loss)
        assert got == want[name], name
