"""The coloured LiDAR map (global-lvba_b200/csrc/color_pipeline.h — boundary B8: VisualizeOptComparison's z-buffer, colouring and
thinning) checked WITHOUT a GPU: the pass functors the CUDA kernels run, instantiated with the sequential host policy
(tests/emu/, test infrastructure only), against oracle/colorize_oracle.py — points, colours, order and listed flags EXACTLY —
and the oracle against the host restatement colmap_points_from_lidar that `lvba_offline --check --points3d lidar` runs.
The suite is re-run here with the items of every pass shuffled and under ASan/UBSan (the device runs them in no order)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import colorize_scene as cs
from oracle import colorize_oracle as co


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return cs.compile_so("colorize_emu.cpp", tmp_path_factory.mktemp("emu") / "libcolorize_emu.so")


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return cs.compile_so("colmap_host.cpp", tmp_path_factory.mktemp("host") / "libcolmap_host.so", ["-ldl"])


def _check(emu, s, leaf, batches=None, half_window=0.5):
    rc, xyz, rgb, listed, st = cs.emu_run(emu, s, leaf, half_window=half_window, batches=batches)
    assert rc == 0
    ref = co.colorize(*cs.oracle_args(s), rgb=s.get("rgb"), leaf=leaf, half_window=half_window)
    assert np.array_equal(xyz.view(np.uint32), ref[0].view(np.uint32))
    assert np.array_equal(rgb, ref[1]) and np.array_equal(listed, ref[2])
    return xyz, rgb, listed, st


@pytest.mark.parametrize("seed,leaf", [(1, 0.01), (2, 0.05), (3, 0.2), (4, 0.0005)])
def test_device_passes_equal_oracle_exactly(emu, seed, leaf):
    s = cs.scene(seed)
    xyz, rgb, listed, st = _check(emu, s, leaf)
    assert len(xyz) > 300 and st["survivors"] >= len(xyz) and st["landed"] >= st["survivors"]
    if leaf < 0.001:
        assert len(xyz) == st["survivors"]


def test_two_oracles_agree(emu):
    s = cs.scene(5, F=5, n_per_scan=700, M=3)
    for leaf in (0.02, 0.0):
        a = co.colorize(*cs.oracle_args(s), rgb=s["rgb"], leaf=leaf)
        b = co.colorize_literal(*cs.oracle_args(s), rgb=s["rgb"], leaf=leaf)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("leaf", [0.01, 0.0])
def test_edge_cases(emu, leaf):
    s = cs.edge_scene()
    xyz, rgb, listed, st = _check(emu, s, leaf)
    lit = co.colorize_literal(*cs.oracle_args(s), rgb=s["rgb"], leaf=leaf)
    assert np.array_equal(xyz, lit[0]) and np.array_equal(rgb, lit[1])
    assert listed.tolist() == [1, 1, 0, 1]                    # image 2 has no frame within 0.5 s


def test_near_ties_keep_the_first_point_within_eps(emu):
    """`zc + 1e-6f < zbuf` is not a minimum: a later point nearer by less than eps (one float ulp at 10 m is 0.95e-6) does not
    replace the kept one, one nearer by two ulps does."""
    s = cs.edge_scene()
    f32 = np.float32
    down = lambda z, n: float(f32(z) - f32(n) * np.spacing(f32(z)))              # noqa: E731  n ulps below z
    at = lambda u, Z: [u / 64 * Z, u / 64 * Z, Z]                                  # noqa: E731  pixel (u + 0.5 rounded) on the diagonal
    a = np.array([at(4.5, 10.0), at(4.5, down(10.0, 1)), at(6.5, 10.0), at(6.5, down(10.0, 2))], np.float32)
    b = np.array([at(4.5, down(10.0, 1)), at(8.5, 8.0), at(8.5, down(8.0, 1))], np.float32)
    poses = np.zeros((2, 12)); poses[:, [0, 4, 8]] = 1.0
    t = dict(s, scans=[a, b], poses=poses, frame_ts=np.array([10.0, 10.0]), cams=s["cams"][:1], image_ts=np.array([10.0]), rgb=s["rgb"][:1])
    xyz, rgb, listed, _ = _check(emu, t, 0.0)
    assert xyz[:, 2].tolist() == [f32(10.0), f32(down(10.0, 2)), f32(8.0)]       # pixels (5, 5), (7, 7), (9, 9) in pixel order
    W = s["width"]
    img = s["rgb"][0].reshape(-1, 3)
    assert rgb.tolist() == [img[5 * W + 5].tolist(), img[7 * W + 7].tolist(), img[9 * W + 9].tolist()]


def test_batches_give_identical_output(emu):
    s = cs.scene(6, M=6)
    outs = [cs.emu_run(emu, s, 0.02, batches=b)[1:4] for b in (1, 2, None)]
    for o in outs[1:]:
        assert all(np.array_equal(x, y) for x, y in zip(outs[0], o))
    ref = co.colorize(*cs.oracle_args(s), rgb=s["rgb"], leaf=0.02)
    assert np.array_equal(outs[0][0], ref[0]) and np.array_equal(outs[0][1], ref[1])


def test_grey_equals_the_host_restatement(emu, host):
    """Without images every point is (128, 128, 128) and the points, their order and the listed images are those of
    colmap_points_from_lidar — the code behind today's grey points3D.txt."""
    for seed, leaf in [(7, 0.01), (8, 0.1), (9, 0.0)]:
        s = cs.scene(seed, colour=False)
        rc, xyz, rgb, listed, _ = cs.emu_run(emu, s, leaf)
        hx, hw = cs.host_points(host, s, leaf)
        assert rc == 0 and np.array_equal(xyz.view(np.uint32), hx.view(np.uint32)) and np.array_equal(listed, hw)
        assert (rgb == 128).all()
    s = cs.edge_scene(); s["rgb"] = None
    rc, xyz, _, listed, _ = cs.emu_run(emu, s, 0.01)
    hx, hw = cs.host_points(host, s, 0.01)
    assert rc == 0 and np.array_equal(xyz.view(np.uint32), hx.view(np.uint32)) and np.array_equal(listed, hw)


def test_far_points_are_refused_and_empty_inputs(emu):
    s = cs.edge_scene()
    far = [x.copy() for x in s["scans"]]
    far[2][0] = [3.0e7, 0.0, 5.0]                            # 3e9 leaf voxels of 1 cm: beyond 2^30
    rc = cs.emu_run(emu, dict(s, scans=far), 0.01)[0]
    assert rc == -1
    assert cs.emu_run(emu, dict(s, scans=far), 0.0)[0] == 0   # no thinning: no voxel key to refuse
    empty = dict(s, scans=[np.zeros((0, 3), np.float32)] * 5)
    rc, xyz, rgb, listed, _ = cs.emu_run(emu, empty, 0.01)
    assert rc == 0 and len(xyz) == 0 and listed.tolist() == [0, 0, 0, 0]


def test_memory_is_bounded_by_table_and_batch(emu):
    """Many images of the same few frames: the pending survivors are folded into the table whenever they outnumber it, so the
    stage's footprint does not grow with the number of images."""
    s = cs.scene(10, F=4, n_per_scan=1500, M=4)
    many = dict(s, cams=np.tile(s["cams"], (12, 1)), image_ts=np.tile(s["image_ts"], 12), rgb=np.tile(s["rgb"], (12, 1, 1, 1)))
    few = dict(s, cams=np.tile(s["cams"], (3, 1)), image_ts=np.tile(s["image_ts"], 3), rgb=np.tile(s["rgb"], (3, 1, 1, 1)))
    pk_many = cs.emu_run(emu, many, 0.02, batches=4)[4]["peak_bytes"]
    pk_few = cs.emu_run(emu, few, 0.02, batches=4)[4]["peak_bytes"]
    assert pk_many <= 1.25 * pk_few


@pytest.mark.skipif(bool(os.environ.get("LVBA_EMU_RERUN")), reason="already a re-run")
@pytest.mark.parametrize("mode", ["shuffle-1", "shuffle-20260923", "asan"])
def test_rerun_shuffled_and_sanitized(mode):
    env = dict(os.environ, LVBA_EMU_RERUN="1")
    if mode == "asan":
        lib = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
        if not lib or not os.path.exists(lib):
            pytest.skip("libasan not available")
        env.update(LVBA_EMU_SANITIZE="1", LD_PRELOAD=lib, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", LVBA_EMU_SHUFFLE="7")
    else:
        env["LVBA_EMU_SHUFFLE"] = mode.split("-")[1]
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", __file__], capture_output=True, text=True,
                       cwd=str(cs.ROOT), env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
