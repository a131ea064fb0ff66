"""ITERATIVE_SCHUR for the visual LM (lvba_visual_opts::linear_solver, global-lvba_b200/csrc/visual_pcg.h) on the H100: the step
with a tight forcing tolerance against DENSE_SCHUR's, the device's CG against tests/visual_pcg_oracle.py on the device's own
system, the whole LM against the oracle's, determinism, composition with removal and solver switches, and the refusals."""
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


def _cam_fixed(p):
    m = np.zeros(len(p["q"]), bool); m[[0, 3, 4]] = True
    return m


SCENES = {"small": (_small, {}), "mixed": (_mixed, {}), "huber": (_small, {"losses": HUBER}), "cam_fixed": (_small, {"mask": True}),
          "loop_closed": (_loop, {})}


def _opts(pkg, losses=None, **kw):
    o = pkg.visual_default_opts(*(losses or (None, None)))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("scene", list(SCENES))
def test_tight_step_matches_dense_schur(gpu_pkg, scene):
    make, kw = SCENES[scene]
    p = make()
    mask = _cam_fixed(p) if kw.get("mask") else None
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, kw.get("losses")), cam_fixed=mask)
    cs0, ps0, m0, _ = P.step(1e4)
    n = len(P.structure()[0])
    if scene == "loop_closed":                                # AUTO takes the any-width path for the direct solve
        cam, rhs, br, bc, blocks = P.get_system()
        first = np.arange(n); np.minimum.at(first, br, bc)
        assert gpu_pkg.env_solve(first, blocks, np.ones(6 * n), rhs.ravel())[2]["path"] == 5
    P.reset_lm(_opts(gpu_pkg, kw.get("losses")), cam_fixed=mask, linear_solver=1, eta=1e-14, min_linear_iter=6 * n,
               max_linear_iter=6 * n)
    cs1, ps1, m1, _ = P.step(1e4)
    st = P.linear_stats()
    assert st["cg_iters_last"] == 6 * n and st["term_last"] in (0, 1)
    # the 400-camera scenes have the worst conditioned camera systems here, and by default S is summed by atomics: over four runs
    # on an H100 the two solves agreed to at most 3.1e-7 (mixed) and 2.8e-8 (loop-closed), the small scenes to 1e-8
    tol = 1e-6 if scene in ("mixed", "loop_closed") else 1e-8
    assert _rel(cs1, cs0) <= tol and _rel(ps1, ps0) <= tol, (_rel(cs1, cs0), _rel(ps1, ps0))
    assert abs(m1 - m0) <= tol * abs(m0)
    P.close()


@pytest.mark.parametrize("radius", [1e4, 3.0])
def test_device_cg_is_the_rule_on_the_device_system(gpu_pkg, radius):
    p = _small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(linear_solver=1)
    cs, _, _, _ = P.step(radius)
    st = P.linear_stats()
    cam, rhs, br, bc, blocks = P.get_system()
    n = len(cam)
    S = np.zeros((6 * n, 6 * n))
    for b, r, c in zip(blocks, br, bc):
        S[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
        if r != c:
            S[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
    ref = vp.single_step(vo.VisualProblem(*vs.args(p)), radius)
    x, it, term = vp.cg(vp.sym_lower(S) + np.diag(ref["dadd"]), rhs.ravel())
    assert (st["cg_iters_last"], st["term_last"]) == (it, term)
    pr = vo.VisualProblem(*vs.args(p))
    step = (x * ref["scale"][:6 * n]).reshape(n, 6)
    assert _rel(cs[pr.cam_active], step) <= 1e-10
    P.close()


def test_lm_matches_the_oracle(gpu_pkg):
    p = _small()
    _, _, _, s = gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, linear_solver=1))
    _, info = vp.ceres_lm(vo.VisualProblem(*vs.args(p)))
    assert (s["iterations"], s["accepted"]) == (info["iters"], info["accepted"])
    assert abs(s["cost_last"] - info["cost"]) <= 1e-8 * info["cost"]


@pytest.mark.parametrize("make", [_small, _mixed], ids=["small", "mixed"])
def test_deterministic_mode_is_bit_reproducible(gpu_pkg, make):
    p = make()
    o = _opts(gpu_pkg, linear_solver=1, deterministic=1)
    runs = []
    for _ in range(2):
        P = gpu_pkg.VisualProblem(*vs.args(p))
        P.reset_lm(o)
        s = P.iterate(8)
        runs.append((P.get_state(), {k: v for k, v in s.items() if not k.startswith("ms_")}, P.linear_stats()))
        P.close()
    (a, sa, la), (b, sb, lb) = runs
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and sa == sb and la == lb
    o.max_iter = 8
    q, t, X, s1 = gpu_pkg.visual_lm(*vs.args(p), opts=o)
    assert np.array_equal(q, a[0]) and np.array_equal(t, a[1]) and np.array_equal(X, a[2])


def test_remove_outliers_then_iterate_equals_a_fresh_handle(gpu_pkg):
    p = _small()
    o = _opts(gpu_pkg, linear_solver=1, deterministic=1)
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(o)
    P.iterate(3)
    tr = voo.Tracker(p)
    q, t, X = P.get_state()
    tr.remove_outliers(q, t, X, 1.0)
    P.remove_outliers(1.0)
    assert P.linear_stats() == dict(cg_iters_total=0, cg_iters_last=0, term_last=0)
    s = P.iterate(4)
    k = tr.kept_problem()
    k["q"], k["t"], k["X"] = q, t, X
    F = gpu_pkg.VisualProblem(*vs.args(k))
    F.reset_lm(o)
    sf = F.iterate(4)
    assert all(np.array_equal(x, y) for x, y in zip(P.get_state(), F.get_state()))
    assert (s["iterations"], s["accepted"], s["cost_last"]) == (sf["iterations"], sf["accepted"], sf["cost_last"])
    assert P.linear_stats() == F.linear_stats()
    P.close(); F.close()


def test_switching_solvers_on_one_handle_equals_fresh_handles(gpu_pkg):
    p = _small()
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


def test_refusals_leave_the_handle_unchanged(gpu_pkg):
    p = _small()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, linear_solver=1, deterministic=1))
    P.iterate(2)
    state, stats = P.get_state(), P.linear_stats()
    bad = [(dict(linear_solver=2), -1), (dict(linear_solver=-1), -1), (dict(linear_solver=1, eta=0.0), -1),
           (dict(linear_solver=1, eta=float("nan")), -1), (dict(linear_solver=1, eta=float("inf")), -1),
           (dict(linear_solver=1, min_linear_iter=-1), -1), (dict(linear_solver=1, max_linear_iter=0), -1),
           (dict(linear_solver=1, min_linear_iter=9, max_linear_iter=8), -1), (dict(linear_solver=1, refine_intrinsics=3), -4)]
    for kw, status in bad:
        with pytest.raises(gpu_pkg.LvbaError) as e:
            P.reset_lm(_opts(gpu_pkg, **kw))
        assert e.value.status == status, kw
        if kw.get("refine_intrinsics") is None:
            q = p["q"].copy()
            with pytest.raises(gpu_pkg.LvbaError) as e:
                gpu_pkg.visual_lm(*vs.args(dict(p, q=q)), opts=_opts(gpu_pkg, **kw))
            assert e.value.status == status and np.array_equal(q, p["q"]), kw
    assert P.linear_stats() == stats and all(np.array_equal(x, y) for x, y in zip(P.get_state(), state))
    # the handle still iterates with its previous options
    s = P.iterate(1)
    assert s["iterations"] == 1 and P.linear_stats()["cg_iters_total"] > stats["cg_iters_total"]
    P.close()
