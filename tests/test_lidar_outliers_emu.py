"""BALM2's voxel outlier removal (lvba_lidar_voxel_residuals / _remove_voxels / _remove_outliers) without a GPU:
  * the oracle (tests/lidar_outlier_oracle.py): the literal walk with erase of remove_residual and the k* form of the device
    passes agree on random lambda arrays, ties at the threshold, outliers first / last / adjacent, ratio 0, the largest ratio
    the rule accepts, and V = 1;
  * per-voxel lambda_0 of the oracle equals the reference's own evaluate_only_residual, voxel by voxel
    (tests/golden/ref_balm.npz, where oracle/_ref/ is built);
  * the library's rule passes and re-plan (global-lvba_b200/csrc/lidar_outliers.h) through the host policy
    (tests/emu/outliers_emu.cpp): the mask equals the oracle rule, and the gathered records and layout of the kept voxels equal
    those of a fresh handle of the kept CSR, with and without big voxels, in one removal or several;
  * the three calls refuse a NULL handle before any device work;
  * lvba_offline --outlier-ratio is checked when it is parsed, --check included."""
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
import lidar_outlier_oracle as olo  # noqa: E402
from oracle import balm_ref, synth  # noqa: E402

REF = np.load(ROOT / "tests" / "golden" / "ref_balm.npz")
KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")


def _cases():
    rng = np.random.default_rng(5)
    base = rng.random(40)
    yield "random", rng.random(200)
    yield "ties", np.round(rng.random(120) * 6) / 6                  # many exact ties at any threshold
    yield "all_equal", np.full(30, 0.25)
    yield "first", np.concatenate(([9.0, 8.0], base))
    yield "last", np.concatenate((base, [8.0, 9.0]))
    yield "adjacent", np.concatenate((base[:20], [7.0, 9.0, 8.0], base[20:]))
    yield "negative", rng.standard_normal(50) * 1e-6
    yield "single", np.array([0.3])
    yield "two", np.array([0.5, 0.1])


RATIOS = [0.0, 0.01, 0.05, 0.1, 0.25, 0.5, 0.9]


def _ratios(V):
    rs = list(RATIOS)
    top = np.nextafter(1.0 - 1.0 / V, 2.0) if V > 1 else None          # just inside floor((1 - r) V) >= 1 ...
    while top is not None and olo.rule_params(top, V) is None:
        top = np.nextafter(top, 0.0)
    if top is not None:
        rs.append(float(top))
    return [r for r in rs if olo.rule_params(r, V) is not None]


@pytest.mark.parametrize("name,lam", list(_cases()), ids=[c[0] for c in _cases()])
def test_loop_and_k_star_form_agree(name, lam):
    V = len(lam)
    for r in _ratios(V):
        a = olo.remove_outlier_loop(lam, r)
        b = olo.remove_outlier_mask(lam, r)
        assert np.array_equal(a, b), (name, r)
        k = olo.rule_params(r, V)[1]
        thr = np.sort(lam)[olo.rule_params(r, V)[0]]
        assert k <= a.sum() <= (lam >= thr).sum() or a.sum() == V
    for r in (1.0, -0.1, math.nan, math.inf):
        assert olo.rule_params(r, V) is None
    if V == 1:
        assert olo.rule_params(0.0, 1) == (0, 0) and olo.rule_params(0.5, 1) is None


def test_rule_counts_without_ties():
    rng = np.random.default_rng(3)
    for V in (10, 37, 100):
        for r in (0.1, 0.13, 0.3):
            lam = rng.random(V)
            lam[np.argsort(lam)[-V // 2:]] += 10.0                    # high voxels spread everywhere
            k_thr, reject = olo.rule_params(r, V)
            thr = np.sort(lam)[k_thr]
            n_ge = int((lam >= thr).sum())
            x = r * V
            assert n_ge == (math.ceil(x) + 1 if x == int(x) else math.floor(x) + 2) or abs(x - round(x)) < 1e-9
            assert reject <= olo.remove_outlier_loop(lam, r).sum() <= n_ge


def test_ratio_zero():
    # reject_num = 0: the walk stops at the first kept voxel only when nothing was erased before it
    lam = np.array([5.0, 5.0, 1.0, 5.0, 2.0])
    assert olo.remove_outlier_loop(lam, 0.0).tolist() == [True, True, False, True, False]
    assert not olo.remove_outlier_loop(lam[2:], 0.0).any()


@pytest.mark.skipif(not balm_ref.available(), reason="oracle/_ref/libbalm_ref.so needs the reference sources")
@pytest.mark.parametrize("level", ["L1", "L2"])
def test_per_voxel_lambda0_pinned_to_reference(level):
    vp, pi, cl, ps = (REF[f"{level}_{k}"] for k in KEYS)
    lam = olo.evaluate_residual(vp, pi, cl, ps)
    for a in range(len(vp) - 1):
        one_vp = np.array([0, vp[a + 1] - vp[a]], np.int64)
        ref = balm_ref.lidar_residual(one_vp, pi[vp[a]:vp[a + 1]], cl[vp[a]:vp[a + 1]], ps)
        assert abs(lam[a] - ref) <= 1e-9 * max(1.0, abs(ref)), (level, a)


# ---- the library's passes through the host policy
def _compile(out_dir):
    so = Path(out_dir) / "liboutliers_emu.so"
    san = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"] if os.environ.get("LVBA_EMU_SANITIZE") else []
    r = subprocess.run(["g++", "-std=c++17", "-O2", *san, "-Wall", "-fPIC", "-shared", str(ROOT / "tests" / "emu" / "outliers_emu.cpp"),
                        "-o", str(so)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = ctypes.CDLL(str(_compile(tmp_path_factory.mktemp("outliers_emu"))))
    lib.emu_ol_rule.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_ol_gather.restype = ctypes.c_int64
    lib.emu_ol_gather.argtypes = [ctypes.c_int, ctypes.c_int64] + [ctypes.c_void_p] * 4 + [ctypes.c_int64] + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("name,lam", list(_cases()), ids=[c[0] for c in _cases()])
def test_host_policy_rule_equals_oracle(emu, name, lam):
    lam = np.ascontiguousarray(lam, np.float64)
    V = len(lam)
    for r in _ratios(V):
        got = np.zeros(V, np.uint8); thr = ctypes.c_double()
        assert emu.emu_ol_rule(V, _ptr(lam), r, _ptr(got), ctypes.byref(thr)) == 0
        assert np.array_equal(got.astype(bool), olo.remove_outlier_loop(lam, r)), (name, r)
        assert thr.value == np.sort(lam)[olo.rule_params(r, V)[0]]
    got = np.zeros(V, np.uint8); thr = ctypes.c_double()
    assert emu.emu_ol_rule(V, _ptr(lam), 1.0, _ptr(got), ctypes.byref(thr)) == -1
    assert emu.emu_ol_rule(V, _ptr(lam), math.nan, _ptr(got), ctypes.byref(thr)) == -1
    bad = lam.copy(); bad[V // 2] = math.nan
    assert emu.emu_ol_rule(V, _ptr(bad), 0.0, _ptr(got), ctypes.byref(thr)) == 1


def _problem(seed, W=24, V=300):
    p = synth.make_problem(W, V, 1, seed=seed)
    return [np.ascontiguousarray(p[k]) for k in KEYS]


@pytest.mark.parametrize("batch_slots", [128, 3])
@pytest.mark.parametrize("n_removals", [1, 2])
def test_host_policy_gather_equals_fresh_layout(emu, batch_slots, n_removals):
    vp, pi, cl, ps = _problem(21)
    V = len(vp) - 1
    rng = np.random.default_rng(batch_slots + n_removals)
    cases = [rng.random(V) < 0.1, np.arange(V) < 7, np.arange(V) >= V - 5, olo.remove_outlier_loop(rng.random(V), 0.2)]
    if batch_slots < 128:
        cases.append(np.diff(vp) <= batch_slots)                          # only big voxels left: a plan without tiles
    for removed in cases:
        kvp, kpi, kcl = olo.kept_problem(vp, pi, cl, removed)
        kvp = np.ascontiguousarray(kvp, np.int64); kpi = np.ascontiguousarray(kpi, np.int32); kcl = np.ascontiguousarray(kcl)
        rm = np.ascontiguousarray(removed, np.uint8)
        bad = emu.emu_ol_gather(len(ps), V, _ptr(vp), _ptr(pi), _ptr(cl), _ptr(rm), len(kvp) - 1, _ptr(kvp), _ptr(kpi), _ptr(kcl),
                                batch_slots, n_removals)
        assert bad == 0


def test_calls_refuse_a_null_handle_before_device_work(pkg):
    lib = pkg.load_library()
    lam = np.zeros(4); m = np.zeros(4, np.uint8); n = ctypes.c_int64()
    assert lib.lvba_lidar_voxel_residuals(None, None, _ptr(lam)) == -1
    assert lib.lvba_lidar_remove_voxels(None, _ptr(m), ctypes.byref(n)) == -1
    assert lib.lvba_lidar_remove_outliers(None, ctypes.c_double(0.1), _ptr(m), ctypes.byref(n)) == -1


def test_no_device_means_no_handle(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    vp, pi, cl, ps = _problem(4, V=40)
    with pytest.raises(pkg.LvbaError) as e:
        pkg.LidarProblem(vp, pi, cl, ps)
    assert e.value.status == -2


# ---- lvba_offline --outlier-ratio: the argument (no GPU)
@pytest.fixture(scope="module")
def tool(pkg, tmp_path_factory):
    exe = tmp_path_factory.mktemp("offline_outliers") / "lvba_offline"
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tools" / "lvba_offline.cpp"), "-o", str(exe),
                        str(pkg.LIB_PATH), f"-Wl,-rpath,{pkg.LIB_PATH.parent}", "-L/usr/local/cuda/lib64", "-lcudart", "-ldl"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("value", ["1", "1.0", "-0.1", "nan", "inf", "abc", "0.1x", ""])
def test_offline_refuses_a_bad_outlier_ratio(tool, tmp_path, value):
    r = subprocess.run([str(tool), "--data", str(tmp_path), "--outlier-ratio", value, "--check"], capture_output=True, text=True)
    assert r.returncode == 64 and "--outlier-ratio" in r.stderr, (r.returncode, r.stderr)


def test_offline_check_takes_an_outlier_ratio(tool, tmp_path):
    from oracle import dataset_writer as dw
    scans, poses = synth.make_scan_scene(17, W=4, n_per_scan=300)
    dw.write_lidar_dataset(tmp_path / "data", scans, poses)
    for value in ("0", "0.05", "0.999"):
        r = subprocess.run([str(tool), "--data", str(tmp_path / "data"), "--outlier-ratio", value, "--check"], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
