"""Per-observation reprojection errors and reprojection-outlier removal of the visual handle (lvba_visual_obs_residuals,
lvba_visual_remove_observations, lvba_visual_remove_outliers) without a GPU:
  * the oracle (tests/visual_outlier_oracle.py): the literal per-landmark loop and the vectorised form agree on random scenes
    and on exact ties s == tau, +inf, NaN, min_track_len above every track and landmarks without a plane;
  * s_q of oracle/visual_oracle.reproj_eval against the 50-digit forward model of oracle/visual_mp.py, within its first-order
    error scale;
  * the library's rule, compaction and caller-index passes with the re-plan's source (global-lvba_b200/csrc/visual_outliers.h)
    through the host policy (tests/emu/visual_outliers_emu.cpp): the removed mask equals the oracle's, and the plan after one
    or two removals equals a fresh plan of the caller-compacted problem: a landmark crossing 129 -> 128, 300-observation
    tracks, a camera losing all its observations, landmarks dropped by min_track_len;
  * the three calls refuse a NULL handle before any device work, and without a device there is no handle."""
import ctypes
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import degenerate_landmarks as dl  # noqa: E402
import visual_big_scene as vs  # noqa: E402
import visual_outlier_oracle as voo  # noqa: E402
from oracle import visual_mp as vm  # noqa: E402
from oracle import visual_oracle as vo  # noqa: E402


def _tracker_case(seed, T=60, max_len=9, frac_bad=0.15):
    """random in_problem / landmark states and s values with every special case mixed in"""
    rng = np.random.default_rng(seed)
    L = rng.integers(0, max_len, T)
    obs_ptr = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    N = int(obs_ptr[-1])
    lm_in = rng.random(T) > 0.1
    trk = np.repeat(np.arange(T), L)
    obs_in = lm_in[trk] & (rng.random(N) > 0.1)
    tau = 4.0
    sq = rng.random(N) * 8.0
    sq[rng.random(N) < frac_bad] = tau                                  # exact ties: kept
    sq[rng.random(N) < 0.05] = np.inf                                   # behind the camera: removed
    sq[rng.random(N) < 0.05] = np.nan                                   # not finite: removed
    sq[~obs_in] = np.nan
    mask = rng.random(N) < 0.3
    return obs_ptr, obs_in, lm_in, sq, tau, mask


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("min_len", [1, 2, 3, 100])
def test_loop_and_vectorised_rule_agree(seed, min_len):
    obs_ptr, obs_in, lm_in, sq, tau, mask = _tracker_case(seed)
    for kw in (dict(sq=sq, tau=tau), dict(mask=mask)):
        a = voo.rule_loop(obs_ptr, obs_in, lm_in, min_len, **kw)
        b = voo.rule_vec(obs_ptr, obs_in, lm_in, min_len, **kw)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert not (a[0] & ~obs_in).any()                               # nothing out of the problem is removed again
        assert not (a[1] & ~lm_in).any()
    if min_len == 100:                                                  # above every track: everything in the problem goes
        rm, dr = voo.rule_vec(obs_ptr, obs_in, lm_in, min_len, sq=sq, tau=tau)
        assert np.array_equal(rm, obs_in) and np.array_equal(dr, lm_in)


def test_rule_edge_cases():
    obs_ptr = np.array([0, 3, 5, 5, 8], np.int64)                       # landmark 2 has a plane and no observation
    lm_in = np.array([True, True, True, False])                         # landmark 3 has no plane
    obs_in = np.array([1, 1, 1, 1, 1, 0, 0, 0], bool)
    sq = np.array([4.0, np.nextafter(4.0, 5.0), np.inf, np.nan, 0.0, np.nan, np.nan, np.nan])
    rm, dr = voo.rule_loop(obs_ptr, obs_in, lm_in, 1, sq=sq, tau=4.0)
    assert rm.tolist() == [False, True, True, True, False, False, False, False]
    assert dr.tolist() == [False, False, True, False]                   # no observation left: dropped
    rm, dr = voo.rule_loop(obs_ptr, obs_in, lm_in, 2, sq=sq, tau=4.0)
    assert rm.tolist() == [True, True, True, True, True, False, False, False]
    assert dr.tolist() == [True, True, True, False]
    assert voo.tau_of(1e300, 1e-300) == np.finfo(np.float64).max       # +inf stays above an overflowing threshold


# ---- s_q against the 50-digit forward model.  The error scale of s = r0^2 + r1^2 is E = 2 (|r0| pix0 + |r1| pix1) amp, with
# pix and amp the first-order scales of visual_mp.observation; the constant is the smallest power of two at least 4x the worst
# ratio |s - s_50| / (eps E) of the float64 oracle over the degenerate family, every observation (measured on the CPU:
# tile_and_big 1.73, isolated 1.04, shared 0.45, distort 0.18).
C_SQ = 8.0


def _family():
    for name, fn in (("isolated", dl.isolated), ("tile_and_big", dl.tile_and_big), ("distort", dl.distort), ("shared", dl.shared)):
        yield name, fn()


@pytest.mark.parametrize("name,p", list(_family()), ids=[n for n, _ in _family()])
def test_sq_meets_the_extended_precision_forward_model(name, p):
    tr = voo.Tracker(p)
    sq = tr.sq(p["q"], p["t"], p["X"])
    op = np.asarray(p["obs_ptr"]); trk = np.repeat(np.arange(len(op) - 1), np.diff(op))
    uv = np.asarray(p["obs_uv"], np.float32).reshape(-1, 2)
    n_inf = 0
    for qi in np.nonzero(tr.obs_in)[0]:
        c = int(p["obs_cam"][qi])
        o = vm.observation(p["q"][c], p["t"][c], p["X"][trk[qi]], uv[qi], p["intr"], p["sigma_px"])
        if not o["valid"]:
            assert sq[qi] == np.inf
            n_inf += 1
            continue
        r0, r1 = o["r"]
        ref = float(r0 * r0 + r1 * r1)
        E = float(2 * (abs(r0) * o["pix"][0] + abs(r1) * o["pix"][1]) * o["amp"]) + ref
        assert abs(sq[qi] - ref) <= C_SQ * vm.EPS * E, (name, qi, sq[qi], ref)
    if name == "isolated":
        assert n_inf > 0                                                # the family reaches the cut-off


# ---- the library's passes through the host policy
def _compile(out_dir):
    so = Path(out_dir) / "libvisual_outliers_emu.so"
    san = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []
    r = subprocess.run(["g++", "-std=c++17", "-O2", *san, "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "visual_outliers_emu.cpp"),
                        "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = ctypes.CDLL(str(_compile(tmp_path_factory.mktemp("visual_outliers_emu"))))
    lib.emu_vo_run.restype = ctypes.c_int64
    lib.emu_vo_run.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int] + [ctypes.c_void_p] * 11
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _scene():
    p = vs.make_scene(5, M=60, n_short=80, long_tracks=((129, 0), (300, 7), (140, 20)))
    p["plane_nd"][3] = 0.0                                              # a landmark without a plane
    return p


def _run(emu, p, rounds, fixed_cam=0):
    """rounds: list of (kind, arg, min_len); kind 'mask' (arg: bool [N]) or 'tau' (arg: max_err_px at the scene's state).
    Returns (bad, removed per round, left per round, tracker)."""
    tr = voo.Tracker(p)
    N = int(p["obs_ptr"][-1]); T = len(p["obs_ptr"]) - 1
    masks = np.zeros((len(rounds), N), np.uint8); sq = np.full((len(rounds), N), np.nan); taus = np.full(len(rounds), -1.0)
    want = []
    for r, (kind, arg, ml) in enumerate(rounds):
        if kind == "mask":
            masks[r] = arg
            want.append(tr.remove_observations(arg, ml))
        elif kind == "tau_exact":                                       # arg: the threshold tau itself
            sq[r] = tr.sq(p["q"], p["t"], p["X"])
            taus[r] = arg
            want.append(voo.rule_vec(tr.obs_ptr, tr.obs_in, tr.lm_in, ml, sq=sq[r], tau=arg))
            tr.apply(*want[-1])
        else:
            sq[r] = tr.sq(p["q"], p["t"], p["X"])
            taus[r] = voo.tau_of(arg, p["sigma_px"])
            want.append(tr.remove_outliers(p["q"], p["t"], p["X"], arg, ml))
    k = tr.kept_problem()
    kvalid = np.ascontiguousarray(vo.valid_tracks(k["plane_nd"]), np.uint8)
    kidx = np.ascontiguousarray(np.nonzero(tr.obs_in)[0], np.int64)
    valid = np.ascontiguousarray(vo.valid_tracks(np.asarray(p["plane_nd"])), np.uint8)
    removed = np.zeros((len(rounds), N), np.uint8); left = np.zeros(2 * len(rounds), np.int64)
    op = np.ascontiguousarray(p["obs_ptr"], np.int64); oc = np.ascontiguousarray(p["obs_cam"], np.int32)
    uv = np.ascontiguousarray(p["obs_uv"], np.float32)
    ml = np.array([r[2] for r in rounds], np.int32)
    bad = emu.emu_vo_run(len(p["q"]), T, fixed_cam, _ptr(valid), _ptr(op), _ptr(oc), _ptr(uv), len(rounds), _ptr(masks), _ptr(sq), _ptr(taus),
                         _ptr(ml), _ptr(removed), _ptr(left), _ptr(kvalid), _ptr(k["obs_ptr"]), _ptr(k["obs_cam"]), _ptr(k["obs_uv"]), _ptr(kidx))
    for r, (rm, _) in enumerate(want):
        if bad >= 0:
            assert np.array_equal(removed[r].astype(bool), rm), r
    return bad, left, tr


def test_host_policy_crossing_129_to_128(emu):
    p = _scene()
    op = p["obs_ptr"]; L = np.diff(op)
    a = int(np.nonzero(L == 129)[0][0])
    m = np.zeros(int(op[-1]), bool); m[op[a] + 60] = True
    bad, left, tr = _run(emu, p, [("mask", m, 3)])
    assert bad == 0
    assert left[0] == int(tr.obs_in.sum())


def test_host_policy_camera_loses_all_observations(emu):
    p = _scene()
    m = np.asarray(p["obs_cam"]) == 11
    bad, _, _ = _run(emu, p, [("mask", m, 3)])
    assert bad == 0
    bad, _, _ = _run(emu, p, [("mask", m, 3)], fixed_cam=-1)
    assert bad == 0


def test_host_policy_drops_short_tracks(emu):
    p = _scene()
    rng = np.random.default_rng(2)
    m = rng.random(int(p["obs_ptr"][-1])) < 0.2
    for ml in (1, 3, 5, 200):
        bad, left, tr = _run(emu, p, [("mask", m, ml)])
        assert bad == 0, ml
        assert left[1] == int(tr.lm_in.sum())
    assert (tr.lm_in.sum() < vo.valid_tracks(p["plane_nd"]).sum())


def test_host_policy_outlier_rule_with_cutoff_and_exact_tie(emu):
    p = _scene()
    N = int(p["obs_ptr"][-1])
    rng = np.random.default_rng(4)
    bad_obs = rng.choice(N, N // 50, replace=False)
    p["obs_uv"] = p["obs_uv"].copy(); p["obs_uv"][bad_obs] += 40.0      # gross outliers
    p["X"] = p["X"].copy()
    vs.put_behind(p, 10)                                                # the cut-off: s = +inf
    sq = voo.Tracker(p).sq(p["q"], p["t"], p["X"])
    f = np.nonzero(np.isfinite(sq))[0]
    tie = int(f[np.argsort(sq[f])[len(f) // 2]])                      # tau = the median s exactly: that observation is kept
    bad, _, tr = _run(emu, p, [("tau_exact", float(sq[tie]), 1)])
    assert bad == 0
    assert tr.obs_in[tie]
    assert not tr.obs_in[p["obs_ptr"][10]:p["obs_ptr"][11]].any()
    assert not tr.obs_in[bad_obs].any()


def test_host_policy_two_successive_removals(emu):
    p = _scene()
    N = int(p["obs_ptr"][-1])
    rng = np.random.default_rng(6)
    bad, left, _ = _run(emu, p, [("mask", rng.random(N) < 0.1, 3), ("tau", 2.0, 2)])
    assert bad == 0
    bad, left, _ = _run(emu, p, [("tau", 3.0, 1), ("mask", rng.random(N) < 0.1, 4)])
    assert bad == 0
    assert left[0] >= left[2]


def test_host_policy_refuses_an_empty_problem(emu):
    p = _scene()
    N = int(p["obs_ptr"][-1])
    bad, _, _ = _run(emu, p, [("mask", np.ones(N, bool), 1)])
    assert bad == -1


# ---- ABI without a device
def test_calls_refuse_a_null_handle_before_device_work(pkg):
    lib = pkg.load_library()
    sq = np.zeros(4); m = np.zeros(4, np.uint8); a, b = ctypes.c_int64(), ctypes.c_int64()
    assert lib.lvba_visual_obs_residuals(None, _ptr(sq)) == -1
    assert lib.lvba_visual_remove_observations(None, _ptr(m), ctypes.c_int32(3), ctypes.byref(a), ctypes.byref(b)) == -1
    assert lib.lvba_visual_remove_outliers(None, ctypes.c_double(3.0), ctypes.c_int32(3), _ptr(m), ctypes.byref(a), ctypes.byref(b)) == -1


def test_no_device_means_no_handle(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    p = vs.make_scene(1, M=10, n_short=20)
    with pytest.raises(pkg.LvbaError) as e:
        pkg.VisualProblem(*vs.args(p))
    assert e.value.status == -2


# ---- the C++ callers without a GPU: the shim compiles, lvba_offline checks --reproj-filter / --min-track-len when it parses them
def _link(pkg):
    return [str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"]


def test_shim_solve_visual_remove_outliers_compiles(pkg, tmp_path):
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tests" / "shim" / "visual_outliers_shim.cpp"),
                        "-o", str(tmp_path / "visual_outliers_shim"), *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_reproj_filter") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        *_link(pkg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("flag,value", [("--reproj-filter", v) for v in ("0", "-1", "nan", "inf", "abc", "3x", "")]
                         + [("--min-track-len", v) for v in ("0", "-2", "1.5", "x", "")])
def test_offline_refuses_bad_filter_arguments(tool, tmp_path, flag, value):
    for extra in ([], ["--check"]):
        r = subprocess.run([str(tool), "--data", str(tmp_path), flag, value, *extra], capture_output=True, text=True)
        assert r.returncode == 64 and flag in r.stderr, (extra, r.returncode, r.stderr)


def test_offline_takes_good_filter_arguments(tool, tmp_path):
    """Past the argument parsing: the run fails later, on the empty dataset directory, not on the flags."""
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--reproj-filter", "2.5", "--min-track-len", "2", "--check"], capture_output=True, text=True)
    assert "--reproj-filter" not in r.stderr and "--min-track-len" not in r.stderr and "unknown argument" not in r.stderr, r.stderr
