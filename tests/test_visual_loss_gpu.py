"""Robust losses on the visual LM on the H100 (the kLoss instantiations of global-lvba_b200/csrc/visual.cuh and visual_big.h):
cost, step and reduced camera system against tests/visual_loss_oracle.py on a tile-only scene and on the mixed scene of
tests/test_visual_big_gpu.py (landmarks beyond 128 observations), both with wrong matches; the whole LM on the tile-only scene and
on a scene of long landmarks; the robust solve against ground truth; deterministic mode with a loss; the handle's loss rules."""
import numpy as np
import pytest

from oracle import synth
import visual_big_scene as vs
import visual_loss_oracle as vl
from test_visual_big_gpu import _mixed

pytestmark = pytest.mark.gpu

HUBER = ((vl.HUBER, 1.0), (vl.HUBER, 0.1))
CAUCHY = ((vl.CAUCHY, 1.0), (vl.CAUCHY, 0.1))
SUMMARY_KEYS = ("iterations", "accepted", "hessian_builds", "termination", "cost_first", "cost_last", "damping_last")


def _tiles():
    p = synth.make_problem(30, 0, 300, seed=11, lidar=False)
    return vl.with_outliers(p, 0.05, 20.0, 50.0, 11)[0]


def _mixed_outliers():
    return vl.with_outliers(_mixed(), 0.05, 20.0, 50.0, 17)[0]


def _long_lm():
    """The scene of test_visual_big_gpu.test_full_lm_matches_oracle: landmarks of 129 to 700 observations whose LM converges
    within 50 passes (the mixed scene with wrong matches does not, and two runs that differ in rounding part within them)."""
    p = vs.make_scene(23, M=300, n_short=250, long_tracks=((129, 0), (300, 0), (700, 100), (150, 40)))
    p["plane_nd"][::13, :3] = 0.0
    return p


SCENES = {"tiles": _tiles, "mixed": _mixed_outliers}
LM_SCENES = {"tiles": _tiles, "long": _long_lm}


def _opts(pkg, losses, deterministic=0):
    lr, lp = losses
    o = pkg.visual_default_opts(reproj_loss=lr, plane_loss=lp)
    o.deterministic = deterministic
    return o


@pytest.mark.parametrize("fixed_cam", [0, -1])
@pytest.mark.parametrize("losses", [HUBER, CAUCHY], ids=["huber", "cauchy"])
@pytest.mark.parametrize("scene", ["tiles", "mixed"])
def test_cost_and_step_match_oracle(gpu_pkg, scene, losses, fixed_cam):
    p = SCENES[scene]()
    P = gpu_pkg.VisualProblem(*vs.args(p), fixed_cam=fixed_cam)
    pr = vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam, loss_reproj=losses[0], loss_plane=losses[1])
    if scene == "mixed":
        assert P.big_counts()["n_big"] == 3
    plain = P.cost()                                              # a new handle has no loss
    assert abs(plain - vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam).cost()) <= 1e-10 * plain
    P.reset_lm(_opts(gpu_pkg, losses))
    c = P.cost()
    assert abs(c - pr.cost()) <= 1e-10 * pr.cost() and c < plain
    cs, ps, model, cost = P.step(1e4)
    ref = vl.single_step(pr, 1e4, True)
    assert abs(cost - ref["cost"]) <= 1e-10 * ref["cost"]
    assert abs(model - ref["model"]) <= 1e-7 * abs(ref["model"])
    assert np.abs(cs - ref["cam_step"]).max() <= 1e-6 * np.abs(ref["cam_step"]).max()
    assert np.abs(ps - ref["pt_step"]).max() <= 1e-6 * np.abs(ref["pt_step"]).max()
    cam, rhs, br, bc, bl = P.get_system()
    S = gpu_pkg.env_blocks_to_dense(br, bc, bl, len(cam))
    assert np.abs(S - ref["S_nodamp"]).max() <= 1e-8 * np.abs(ref["S_nodamp"]).max()
    assert np.abs(rhs.ravel() - ref["rhs"]).max() <= 1e-8 * np.abs(ref["rhs"]).max()
    # the candidate cost through lvba_visual_cost at the oracle's candidate state
    qn, tn, Xn = pr.plus(np.concatenate([ref["cam_step"][pr.cam_active].ravel(), ref["pt_step"][pr.tv].ravel()]))
    P.set_state(qn, tn, Xn)
    c2 = pr.cost(qn, tn, Xn)
    assert abs(P.cost() - c2) <= 1e-10 * c2
    # reset_lm without opts: plain again
    P.reset_lm()
    c3 = vl.RobustProblem(*vs.args(p), fixed_cam=fixed_cam).cost(qn, tn, Xn)
    assert abs(P.cost() - c3) <= 1e-10 * c3
    P.close()


@pytest.mark.parametrize("scene,losses", [("tiles", HUBER), ("tiles", CAUCHY), ("long", HUBER)],
                         ids=["tiles-huber", "tiles-cauchy", "long-huber"])
def test_full_lm_matches_oracle(gpu_pkg, scene, losses):
    """(Cauchy on the long scene runs ~50 passes and one of them sits on the acceptance threshold: the device and the oracle,
    which differ in rounding, then accept one step apart.  Its cost and step are checked above on the mixed scene.)"""
    p = LM_SCENES[scene]()
    q, t, X, s = gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, losses))
    pr, info = vl.ceres_lm(vl.RobustProblem(*vs.args(p), loss_reproj=losses[0], loss_plane=losses[1]))
    assert s["iterations"] == info["iters"]
    assert s["accepted"] == info["accepted"]
    assert s["termination"] == vl.TERM[info["term"]]
    assert abs(s["cost_first"] - info["cost0"]) <= 1e-10 * info["cost0"]
    assert abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"]
    assert np.array_equal(q[0], p["q"][0]) and np.array_equal(t[0], p["t"][0])


def _cam_error(p, q, t):
    R = vl.vo.quat_to_rot(q); Rg = vl.vo.quat_to_rot(p["q_gt"])
    c = -np.einsum("nji,nj->ni", R, t); cg = -np.einsum("nji,nj->ni", Rg, p["t_gt"])
    return float(np.sqrt(((c - cg) ** 2).sum(1)).mean())


def test_robust_solve_is_closer_to_ground_truth(gpu_pkg):
    """The reference's losses on the scene with wrong matches.  (Cauchy at 1 sigma also discounts the inliers' 1-sigma noise; on
    this scene its cameras are not closer than the plain solve's, so it is not asserted here.)"""
    p = _tiles()
    q0, t0, _, _ = gpu_pkg.visual_lm(*vs.args(p))
    q1, t1, _, _ = gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, HUBER))
    assert _cam_error(p, q1, t1) < _cam_error(p, q0, t0)


def _bytes(q, t, X, s):
    return q.tobytes() + t.tobytes() + X.tobytes() + repr([s[k] for k in SUMMARY_KEYS]).encode()


@pytest.mark.parametrize("scene", ["tiles", "long"])
def test_deterministic_with_huber_is_bit_reproducible(gpu_pkg, scene):
    p = LM_SCENES[scene]()
    o = _opts(gpu_pkg, HUBER, deterministic=1)
    runs = []
    for _ in range(2):
        P = gpu_pkg.VisualProblem(*vs.args(p))
        P.reset_lm(o)
        s = P.iterate(50)
        runs.append(_bytes(*P.get_state(), s))
        P.close()
    for _ in range(2):
        runs.append(_bytes(*gpu_pkg.visual_lm(*vs.args(p), opts=o)))
    assert runs[1] == runs[0] and runs[2] == runs[0] and runs[3] == runs[0]
    # and it is the robust solve: the same iterations as the default mode with the same loss, costs within the oracle's tolerance
    q, t, X, s = gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, HUBER))
    _, _, _, sd = gpu_pkg.visual_lm(*vs.args(p), opts=o)
    assert sd["iterations"] == s["iterations"] and abs(sd["cost_last"] - s["cost_last"]) <= 1e-6 * s["cost_last"]


def test_explicit_none_equals_default_opts(gpu_pkg):
    p = _mixed_outliers()
    d = gpu_pkg.visual_default_opts(); d.deterministic = 1
    e = gpu_pkg.visual_default_opts(); e.deterministic = 1
    e.reproj_loss = gpu_pkg.LOSS_NONE; e.reproj_loss_scale = 7.0
    e.plane_loss = gpu_pkg.LOSS_NONE; e.plane_loss_scale = 0.0
    assert _bytes(*gpu_pkg.visual_lm(*vs.args(p), opts=d)) == _bytes(*gpu_pkg.visual_lm(*vs.args(p), opts=e))


def test_reset_lm_refuses_a_bad_loss_and_keeps_the_handle(gpu_pkg):
    p = _tiles()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, HUBER))
    c_huber = P.cost()
    for field, kind, scale in (("reproj_loss", 5, 1.0), ("plane_loss", 1, 0.0), ("plane_loss", 2, float("nan"))):
        o = _opts(gpu_pkg, HUBER)
        setattr(o, field, kind); setattr(o, field + "_scale", scale)
        with pytest.raises(gpu_pkg.LvbaError) as e:
            P.reset_lm(o)
        assert e.value.status == -1
        assert P.cost() == c_huber                                  # the handle keeps its losses
    P.close()
