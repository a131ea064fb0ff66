"""The coloured LiDAR map (boundary B8) on the device through the C ABI: bit for bit the oracle (oracle/colorize_oracle.py) and,
without images, the host restatement colmap_points_from_lidar behind today's grey points3D.txt; batch-size invariance; a
bench-size street for invariants and a device footprint that does not grow with the number of images."""
import numpy as np
import pytest

import colorize_scene as cs
from oracle import colorize_oracle as co

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return cs.compile_so("colmap_host.cpp", tmp_path_factory.mktemp("host") / "libcolmap_host.so", ["-ldl"])


def dev_run(pkg, s, leaf, batch=None, poses=None):
    cz = pkg.Colorizer(s["scans"], s["frame_ts"])
    try:
        return cz.run(s["poses"] if poses is None else poses, s["image_ts"], s["cams"], s["intr"], s["width"], s["height"], s.get("rgb"),
                      leaf=leaf, batch=batch)
    finally:
        cz.close()


@pytest.mark.parametrize("seed,leaf", [(1, 0.01), (2, 0.05), (3, 0.2), (4, 0.0005)])
def test_device_equals_oracle_bit_for_bit(gpu_pkg, seed, leaf):
    s = cs.scene(seed)
    xyz, rgb, listed, summ = dev_run(gpu_pkg, s, leaf)
    ref = co.colorize(*cs.oracle_args(s), rgb=s["rgb"], leaf=leaf)
    assert np.array_equal(xyz.view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(rgb, ref[1]) and np.array_equal(listed, ref[2])
    assert summ["n_out"] == len(xyz) > 300 and summ["n_survivors"] >= summ["n_out"] and summ["kernel_launches"] > 0


@pytest.mark.parametrize("leaf", [0.01, 0.0])
def test_edge_cases_on_the_device(gpu_pkg, leaf):
    s = cs.edge_scene()
    xyz, rgb, listed, _ = dev_run(gpu_pkg, s, leaf)
    ref = co.colorize_literal(*cs.oracle_args(s), rgb=s["rgb"], leaf=leaf)
    assert np.array_equal(xyz.view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(rgb, ref[1]) and listed.tolist() == [1, 1, 0, 1]


def test_grey_device_equals_the_host_restatement(gpu_pkg, host):
    for seed, leaf in [(7, 0.01), (8, 0.1), (9, 0.0)]:
        s = cs.scene(seed, colour=False)
        xyz, rgb, listed, _ = dev_run(gpu_pkg, s, leaf)
        hx, hw = cs.host_points(host, s, leaf)
        assert np.array_equal(xyz.view(np.uint32), hx.view(np.uint32)) and np.array_equal(listed, hw) and (rgb == 128).all()
        # the rows of points3D.txt as the grey writer formats them are therefore the same bytes
        fmt = lambda p: "".join(f"{i} {x:.6f} {y:.6f} {z:.6f} 128 128 128 0\n" for i, (x, y, z) in enumerate(p.astype(np.float64)))  # noqa: E731
        assert fmt(xyz) == fmt(hx)


def test_batch_size_invariance(gpu_pkg):
    s = cs.scene(6, M=6)
    outs = [dev_run(gpu_pkg, s, 0.02, batch=b)[:3] for b in (1, 2, None)]
    for o in outs[1:]:
        assert all(np.array_equal(x, y) for x, y in zip(outs[0], o))
    ref = co.colorize(*cs.oracle_args(s), rgb=s["rgb"], leaf=0.02)
    assert np.array_equal(outs[0][0], ref[0]) and np.array_equal(outs[0][1], ref[1])


def test_bench_size_street_invariants_and_flat_footprint(gpu_pkg):
    import sys
    sys.path.insert(0, str(cs.ROOT / "tools"))
    from bench_voxel_map import street_scans
    xyz, scan_ptr, poses = street_scans(400, 50000)
    frame_ts = 0.1 * np.arange(400)
    Rci = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
    W, H = 640, 512
    intr = np.array([350.0, 350.0, 320.0, 256.0, -0.05, 0.01, 1e-4, -1e-4])

    def cams_for(ids):
        cams = np.zeros((len(ids), 12))
        for j, i in enumerate(ids):
            Rcw = Rci @ poses[i, :9].reshape(3, 3).T
            cams[j, :9] = Rcw.ravel(); cams[j, 9:] = -Rcw @ poses[i, 9:]
        return cams

    cz = gpu_pkg.Colorizer(xyz, frame_ts, scan_ptr=scan_ptr)
    try:
        peaks = {}
        for n in (50, 200):
            ids = np.linspace(0, 399, n).astype(int)
            out, col, listed, s = cz.run(poses, frame_ts[ids], cams_for(ids), intr, W, H, None, leaf=0.1, batch=25)
            peaks[n] = s["peak_device_bytes"]
            assert listed.all() and s["n_listed"] == n and (col == 128).all() and np.isfinite(out).all()
            assert s["n_survivors"] <= W * H * n and s["n_out"] <= s["n_survivors"]
        assert peaks[200] <= 1.2 * peaks[50], peaks
        # without thinning: the survivors in merged order; those of the first image each round to a distinct pixel of it
        ids = np.array([100])
        out, _, _, s = cz.run(poses, frame_ts[ids], cams_for(ids), intr, W, H, None, leaf=0.0)
        pix, _ = co.project(cams_for(ids)[0], intr, out, W, H)
        assert (pix >= 0).all() and len(np.unique(pix)) == len(pix) == s["n_survivors"] <= W * H
        assert np.all(np.diff(pix) > 0)                       # pixel order
    finally:
        cz.close()
