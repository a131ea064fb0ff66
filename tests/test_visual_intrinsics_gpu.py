"""The intrinsics block of the visual LM (lvba_visual_opts::refine_intrinsics) on the H100: one lvba_visual_step against the
bordered system of tests/visual_intr_oracle.py (border, corner, rhs and every step), the whole LM against the oracle's, mask 0
bit for bit as a handle without the block, deterministic mode, constant cameras, losses and landmarks beyond 128 observations,
outlier removal between two solves, reset_state, and the refusals."""
import numpy as np
import pytest

from oracle import synth
import visual_big_scene as vs
import visual_fixed_oracle as vf
import visual_intr_oracle as vi
import visual_loss_oracle as vl
from test_visual_big_gpu import _mixed

pytestmark = pytest.mark.gpu

INVALID_ARG = -1


def _tiles():
    return vi.miscalibrated(synth.make_problem(30, 0, 300, seed=11, lidar=False))


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


def _opts(pkg, mask, losses=(None, None), deterministic=0):
    o = pkg.visual_default_opts(reproj_loss=losses[0], plane_loss=losses[1])
    o.refine_intrinsics = mask
    o.deterministic = deterministic
    return o


CASES = {
    "tiles-focal": (_tiles, vi.FOCAL, (None, None), None),
    "tiles-all": (_tiles, 0xFF, (None, None), None),
    "tiles-k1-huber": (lambda: vl.with_outliers(_tiles(), 0.05, 20.0, 50.0, 3)[0], 0x10, ((vl.HUBER, 1.0), (vl.HUBER, 0.1)), None),
    "tiles-dist-cauchy-fixed": (_tiles, vi.DISTORTION, ((vl.CAUCHY, 1.0), None), [0, 4, 5, 9]),
    "tiles-principal-allfixed": (_tiles, vi.PRINCIPAL, (None, None), "all"),
    "mixed-focal-dist": (lambda: vi.miscalibrated(_mixed()), vi.FOCAL | vi.DISTORTION, (None, None), None),
}


@pytest.mark.parametrize("case", list(CASES))
def test_step_matches_oracle(gpu_pkg, case):
    make, mask, losses, cams = CASES[case]
    p = make()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    pr = vi.IntrProblem(*vs.args(p), mask=mask, loss_reproj=losses[0], loss_plane=losses[1])
    cam_fixed = None
    if cams is not None:
        fixed = range(pr.M) if cams == "all" else cams
        cam_fixed = vf.mask_of(pr.M, fixed)
        vf.with_constant(pr, fixed)
    P.reset_lm(_opts(gpu_pkg, mask, losses), cam_fixed=cam_fixed)
    cs, ps, model, cost = P.step(1e4)
    ref = vi.step_bordered(pr, 1e4)
    s = ref["system"]
    assert abs(cost - pr.cost_k()) <= 1e-10 * cost
    got = P.intrinsics_system()
    cam = P.structure()[0]
    assert len(cam) == pr.nc
    rows = np.concatenate([6 * pr.cam_col[c] + np.arange(6) for c in cam]).astype(np.int64) if len(cam) else np.zeros(0, np.int64)
    if len(cam):
        assert _rel(got["border"], s["B"][rows]) <= 1e-8
    assert _rel(got["corner"], s["C"]) <= 1e-8
    assert _rel(got["rhs"], s["rhs_k"]) <= 1e-8
    d = ref["delta"]
    step = np.zeros(8); step[pr.free] = d[pr.nb:]
    assert _rel(got["step"], step) <= 1e-8
    ca = np.nonzero(pr.cam_active)[0]
    if len(ca):
        assert _rel(cs[ca], d[:6 * pr.nc].reshape(-1, 6)[pr.cam_col[ca]]) <= 1e-8
    assert not cs[~pr.cam_active].any()
    assert _rel(ps[pr.tv], d[6 * pr.nc:pr.nb].reshape(-1, 3)) <= 1e-8
    assert abs(model - ref["model"]) <= 1e-8 * abs(ref["model"])


@pytest.mark.parametrize("mask", [vi.FOCAL | 0x10, 0xFF])
def test_full_lm_matches_oracle(gpu_pkg, mask):
    p = _tiles()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, mask))
    s = P.iterate(50)
    pr, info = vi.ceres_lm(vi.IntrProblem(*vs.args(p), mask=mask))
    assert abs(s["cost_last"] - info["cost"]) <= 1e-6 * info["cost"], (s, info)
    got = P.get_intrinsics()
    assert np.abs(got / pr.intr - 1).max() <= 1e-6, (got, pr.intr)
    held = [i for i in range(8) if not (mask >> i) & 1]
    assert np.array_equal(got[held], p["intr"][held])
    assert abs(P.cost() - s["cost_last"]) <= 1e-10 * s["cost_last"]


def _run(pkg, p, opts, n=12):
    P = pkg.VisualProblem(*vs.args(p))
    P.reset_lm(opts)
    s = P.iterate(n)
    return P, s, P.get_state(), P.get_intrinsics()


@pytest.mark.parametrize("scene", ["tiles", "mixed"])
def test_mask_zero_is_bit_identical_to_a_handle_without_the_block(gpu_pkg, scene):
    p = _tiles() if scene == "tiles" else _mixed()
    plain = gpu_pkg.visual_default_opts(); plain.deterministic = 1
    _, s0, st0, in0 = _run(gpu_pkg, p, plain)
    # a handle that refined, was restored, and is reset with mask 0 runs the plain passes again
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, 0xFF, deterministic=1))
    P.iterate(3)
    assert not np.array_equal(P.get_intrinsics(), p["intr"])
    P.reset_state()
    P.reset_lm(_opts(gpu_pkg, 0, deterministic=1))
    s1 = P.iterate(12)
    st1 = P.get_state()
    for a, b in zip(st0, st1):
        assert np.array_equal(a, b)
    assert np.array_equal(in0, p["intr"]) and np.array_equal(P.get_intrinsics(), p["intr"])
    assert (s0["cost_last"], s0["iterations"]) == (s1["cost_last"], s1["iterations"])


@pytest.mark.parametrize("scene", ["tiles", "mixed"])
def test_deterministic_mode_repeats_bits(gpu_pkg, scene):
    p = _tiles() if scene == "tiles" else vi.miscalibrated(_mixed())
    o = _opts(gpu_pkg, vi.FOCAL | vi.DISTORTION, ((vl.HUBER, 1.0), None), deterministic=1)
    _, s0, st0, in0 = _run(gpu_pkg, p, o)
    _, s1, st1, in1 = _run(gpu_pkg, p, o)
    for a, b in zip(st0 + (in0,), st1 + (in1,)):
        assert np.array_equal(a, b)
    assert s0["cost_last"] == s1["cost_last"]


def test_outlier_removal_keeps_intrinsics_and_mask(gpu_pkg):
    p, _ = vl.with_outliers(_tiles(), 0.05, 20.0, 50.0, 5)
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, vi.FOCAL, ((vl.HUBER, 1.0), None)))
    P.iterate(50)
    k1 = P.get_intrinsics()
    removed, _ = P.remove_outliers(3.0, 2)
    assert removed.any()
    assert np.array_equal(P.get_intrinsics(), k1)
    # the handle still refines after its re-plan: its next step matches the oracle of the kept observations
    keep = ~removed
    ptr = p["obs_ptr"]
    c = np.concatenate([[0], np.cumsum(keep)])
    L = c[ptr[1:]] - c[ptr[:-1]]
    qq, tt, XX = P.get_state()
    q = dict(p, q=qq, t=tt, X=XX, intr=k1, obs_ptr=np.concatenate([[0], np.cumsum(L)]), obs_cam=p["obs_cam"][keep],
             obs_uv=p["obs_uv"][keep], plane_nd=np.where((L >= 2)[:, None], p["plane_nd"], 0.0))
    pr = vi.IntrProblem(*vs.args(q), mask=vi.FOCAL, loss_reproj=(vl.HUBER, 1.0))
    _, _, model, cost = P.step(1e4)
    ref = vi.step_bordered(pr, 1e4)
    assert abs(cost - pr.cost_k()) <= 1e-10 * cost
    assert _rel(P.intrinsics_system()["step"][:2], ref["delta"][pr.nb:]) <= 1e-8
    assert abs(model - ref["model"]) <= 1e-8 * abs(ref["model"])


def test_reset_state_and_set_intrinsics(gpu_pkg):
    p = _tiles()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    c0 = P.cost()
    P.reset_lm(_opts(gpu_pkg, 0xFF))
    P.iterate(10)
    assert not np.array_equal(P.get_intrinsics(), p["intr"])
    P.reset_state()
    assert np.array_equal(P.get_intrinsics(), p["intr"])
    assert P.cost() == c0
    truth = synth.INTR.copy()
    P.set_intrinsics(truth)
    assert np.array_equal(P.get_intrinsics(), truth)
    assert P.cost() != c0
    bad = truth.copy(); bad[5] = np.nan
    with pytest.raises(gpu_pkg.LvbaError) as e:
        P.set_intrinsics(bad)
    assert e.value.status == INVALID_ARG
    assert np.array_equal(P.get_intrinsics(), truth)


def test_no_stale_system_after_a_reset(gpu_pkg):
    p = _tiles()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    P.reset_lm(_opts(gpu_pkg, 0xFF))
    P.step(1e4)
    assert P.intrinsics_system()["step"].any()
    for reset in (lambda: P.reset_lm(_opts(gpu_pkg, vi.FOCAL)), P.reset_state):
        reset()
        got = P.intrinsics_system()
        assert not got["step"].any() and not got["corner"].any() and not got["rhs"].any() and not got["border"].any()
        P.step(1e4)
        assert P.intrinsics_system()["corner"].any()


def test_refusals(gpu_pkg):
    p = _tiles()
    P = gpu_pkg.VisualProblem(*vs.args(p))
    with pytest.raises(gpu_pkg.LvbaError) as e:
        P.reset_lm(_opts(gpu_pkg, 0x100))
    assert e.value.status == INVALID_ARG
    q0 = p["q"].copy()
    with pytest.raises(gpu_pkg.LvbaError) as e:
        gpu_pkg.visual_lm(*vs.args(p), opts=_opts(gpu_pkg, vi.FOCAL))
    assert e.value.status == INVALID_ARG
    assert np.array_equal(p["q"], q0)
