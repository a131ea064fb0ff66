"""The matrix-free product of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_implicit.h) on the H100: which scenes the rule moves,
the operator rebuilt through lvba_visual_apply_system against the oracle's S + diag(dadd) and the device's CG against the oracle's
cg on it, the tight step against DENSE_SCHUR's, the whole LM against the oracle's, determinism, composition with removal,
solver switches and re-plans, and lvba_visual_get_system on a handle without S."""
import ctypes as C

import numpy as np
import pytest

from oracle import synth
from oracle import visual_oracle as vo
import visual_big_scene as vs
import visual_outlier_oracle as voo
import visual_pcg_oracle as vp

pytestmark = pytest.mark.gpu
HUBER = ((1, 1.0), (1, 0.1))


def _small():
    return synth.make_problem(14, 0, 80, seed=5, lidar=False)


def _mixed():
    return vs.make_scene(17, M=400, n_short=300, long_tracks=((128, 5), (129, 20), (300, 60), (1000, 0)), extra_tracks=([3, 3, 4, 3, 5],))


def _loop():
    return vs.make_scene(11, M=400, long_tracks=[(20, 390)])


def _long_small():
    """60 cameras, a 200-observation track over all of them (each seen three or four times) and a repeated-camera track."""
    return vs.make_scene(5, M=60, n_short=60, long_tracks=((200, 0),), extra_tracks=([3, 3, 4, 3, 5],))


def _rows_300():
    """A 300-observation track over cameras 0-299 of 400 and 1500 short tracks: moved; with cameras 1-299 constant it is not."""
    return vs.make_scene(7, M=400, n_short=1500, long_tracks=((300, 0),))


def _opts(pkg, losses=None, **kw):
    o = pkg.visual_default_opts(*(losses or (None, None)))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _rhs(P):
    n = len(P.structure()[0])
    rhs = np.empty(6 * n)
    st = P._lib.lvba_visual_get_system(P._h, rhs.ctypes.data_as(C.POINTER(C.c_double)), None)
    assert st == 0
    return rhs


def _operator(P):
    n6 = 6 * len(P.structure()[0])
    return np.stack([P.apply_system(e) for e in np.eye(n6)], axis=1)


@pytest.mark.parametrize("make,moved", [(_small, 0), (_mixed, 1), (_loop, 1), (_long_small, 1), (_rows_300, 1)],
                         ids=["small", "mixed", "loop_closed", "long_small", "rows_300"])
def test_the_rule_moves_the_long_track_scenes(gpu_pkg, make, moved):
    P = gpu_pkg.VisualProblem(*vs.args(make()))
    assert P.schur_product() == moved
    P.reset_lm(linear_solver=1)
    assert P.schur_product() == moved
    P.close()


@pytest.mark.parametrize("radius", [1e4, 3.0])
def test_operator_and_cg_match_the_oracle(gpu_pkg, radius):
    p = _long_small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    assert P.schur_product() == 1
    with pytest.raises(gpu_pkg.LvbaError) as e:
        P.apply_system(np.zeros(6 * len(P.structure()[0])))
    assert e.value.status == -1                                       # no step yet
    P.reset_lm(linear_solver=1)
    cs, _, _, _ = P.step(radius)
    st = P.linear_stats()
    A = _operator(P)
    ref = vp.single_step(vo.VisualProblem(*vs.args(p)), radius)
    assert _rel(A, ref["S"]) <= 1e-9                                  # S + diag(dadd), damped
    x, it, term = vp.cg(A, _rhs(P))
    assert (st["cg_iters_last"], st["term_last"]) == (it, term)
    pr = vo.VisualProblem(*vs.args(p))
    n = A.shape[0] // 6
    assert _rel(cs[pr.cam_active], (x * ref["scale"][:6 * n]).reshape(n, 6)) <= 1e-10
    P.close()


# Huber on the 60-camera scene: on the mixed scene with Huber the oracle's own CG (dense, explicit S), run as long, ends 1.6e-6
# from the direct solution, past the 400-camera tolerance whatever the product
SCENES = {"plain": (_mixed, {}), "huber": (_long_small, {"losses": HUBER}), "cam_fixed": (_mixed, {"mask": [0, 3, 4, 100]}),
          "repeated_camera": (_long_small, {})}


@pytest.mark.parametrize("scene", list(SCENES))
def test_tight_step_matches_dense_schur(gpu_pkg, scene):
    make, kw = SCENES[scene]
    p = make()
    mask = None
    if "mask" in kw:
        mask = np.zeros(len(p["q"]), bool); mask[kw["mask"]] = True
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, kw.get("losses")), cam_fixed=mask)
    cs0, ps0, m0, _ = P.step(1e4)
    n = len(P.structure()[0])
    P.reset_lm(_opts(gpu_pkg, kw.get("losses")), cam_fixed=mask, linear_solver=1, eta=1e-14, min_linear_iter=6 * n,
               max_linear_iter=6 * n)
    assert P.schur_product() == 1
    cs1, ps1, m1, _ = P.step(1e4)
    st = P.linear_stats()
    assert st["cg_iters_last"] == 6 * n and st["term_last"] in (0, 1)
    tol = 1e-6 if n > 100 else 1e-8                                   # tests/test_visual_pcg_gpu.py's tolerances
    assert _rel(cs1, cs0) <= tol and _rel(ps1, ps0) <= tol, (_rel(cs1, cs0), _rel(ps1, ps0))
    assert abs(m1 - m0) <= tol * abs(m0)
    P.close()


def test_lm_matches_the_oracle(gpu_pkg):
    p = _long_small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    assert P.schur_product() == 1
    P.close()
    _, _, _, s = gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, linear_solver=1))
    _, info = vp.ceres_lm(vo.VisualProblem(*vs.args(p)))
    assert (s["iterations"], s["accepted"]) == (info["iters"], info["accepted"])
    assert abs(s["cost_last"] - info["cost"]) <= 1e-8 * info["cost"]


@pytest.mark.parametrize("det", [0, 1])
def test_two_runs_are_bit_identical(gpu_pkg, det):
    p = _mixed()
    o = _opts(gpu_pkg, linear_solver=1, deterministic=det)
    runs = []
    for _ in range(2):
        P = gpu_pkg.VisualProblem(*vs.args(p))
        P.reset_lm(o)
        s = P.iterate(8)
        runs.append((P.get_state(), {k: v for k, v in s.items() if not k.startswith("ms_")}, P.linear_stats()))
        P.close()
    (a, sa, la), (b, sb, lb) = runs
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and sa == sb and la == lb
    assert la["cg_iters_total"] > 0


def test_remove_outliers_then_iterate_equals_a_fresh_handle(gpu_pkg):
    p = _long_small()
    o = _opts(gpu_pkg, linear_solver=1)
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(o)
    P.iterate(3)
    tr = voo.Tracker(p)
    q, t, X = P.get_state()
    tr.remove_outliers(q, t, X, 1.0)
    P.remove_outliers(1.0)
    s = P.iterate(4)
    k = tr.kept_problem()
    k["q"], k["t"], k["X"] = q, t, X
    F = gpu_pkg.VisualProblem(*vs.args(k))
    F.reset_lm(o)
    sf = F.iterate(4)
    assert P.schur_product() == F.schur_product() == 1
    assert all(np.array_equal(x, y) for x, y in zip(P.get_state(), F.get_state()))
    assert (s["iterations"], s["accepted"], s["cost_last"]) == (sf["iterations"], sf["accepted"], sf["cost_last"])
    assert P.linear_stats() == F.linear_stats()
    P.close(); F.close()


def test_switching_solvers_on_one_handle_equals_fresh_handles(gpu_pkg):
    p = _long_small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    for solver in (1, 0, 1):
        o = _opts(gpu_pkg, linear_solver=solver, deterministic=1)
        P.reset_lm(o); P.reset_state()
        s = P.iterate(5)
        F = gpu_pkg.VisualProblem(*vs.args(p))
        F.reset_lm(o)
        sf = F.iterate(5)
        assert all(np.array_equal(x, y) for x, y in zip(P.get_state(), F.get_state())), solver
        assert s["cost_last"] == sf["cost_last"] and P.linear_stats() == F.linear_stats()
        F.close()
    P.close()


def test_cam_fixed_replan_evaluates_the_rule_again(gpu_pkg):
    p = _rows_300()
    mask = np.zeros(len(p["q"]), bool); mask[1:300] = True
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(linear_solver=1)
    assert P.schur_product() == 1
    P.reset_lm(linear_solver=1, cam_fixed=mask)
    assert P.schur_product() == 0
    s = P.iterate(3)
    assert s["iterations"] == 3 and P.linear_stats()["cg_iters_total"] > 0
    P.reset_lm(linear_solver=1)
    assert P.schur_product() == 1
    P.close()


def test_get_system_without_s(gpu_pkg):
    p = _long_small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(linear_solver=1)
    P.step(1e4)
    rhs = _rhs(P)
    cam, br, bc = P.structure()
    blocks = np.full((len(br), 6, 6), 7.0)
    st = P._lib.lvba_visual_get_system(P._h, None, blocks.ctypes.data_as(C.POINTER(C.c_double)))
    assert st == -4 and (blocks == 7.0).all()                         # LVBA_ERR_UNSUPPORTED, nothing written
    P.reset_lm()                                                       # DENSE_SCHUR at the same state
    P.step(1e4)
    assert _rel(rhs, _rhs(P)) <= 1e-12
    with pytest.raises(gpu_pkg.LvbaError):
        P.apply_system(np.zeros(6 * len(cam)))                         # the last pass did not run CG
    P.close()
