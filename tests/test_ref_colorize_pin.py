"""The colour half of boundary B8 held against the reference's own VisualizeOptComparison (src/lvba_system.cpp:1932-2143): the oracle
(oracle/colorize_oracle.py), which the device passes equal exactly (tests/test_colorize_emu.py, tests/test_zz_colorize_gpu.py), reproduces
both clouds the reference keeps — `after` (x_buf_ under Rcw_all_optimized_ / tcw_all_optimized_) and `before` (x_buf_before_ under
Rcw_all_ / tcw_all_) — point, channel order and colour, and the images it lists.  Always against the committed fixture
(tests/golden/ref_colorize.npz); where the reference source exists, also live on more seeded scenes.  Compared as sets of
(x, y, z, r, g, b): the reference returns the thinned cloud in unordered_map order."""
import numpy as np
import pytest

import colorize_scene as cs
from oracle import colorize_oracle as co


def oracle_both(s, leaf):
    keep, sub = cs.loaded_subset(s)
    a = co.colorize(*cs.oracle_args(sub), rgb=sub["rgb"], leaf=leaf)
    b = co.colorize(sub["scans"], sub["frame_ts"], sub["poses_before"], sub["image_ts"], sub["cams_before"], sub["intr"], sub["width"], sub["height"],
                    rgb=sub["rgb"], leaf=leaf)
    listed = np.zeros(len(s["image_ts"]), np.uint8); listed[keep] = a[2]
    return a, b, listed


def test_oracle_equals_the_reference_fixture():
    s, leaf, ref = cs.fixture()
    a, b, listed = oracle_both(s, leaf)
    assert len(ref["after_xyz"]) > 2000 and not np.array_equal(ref["after_xyz"], ref["before_xyz"])
    assert cs.as_set(a[0], a[1]) == cs.as_set(ref["after_xyz"], ref["after_rgb"])
    assert cs.as_set(b[0], b[1]) == cs.as_set(ref["before_xyz"], ref["before_rgb"])
    assert listed.tolist() == ref["listed"].tolist() == [1, 1, 1, 1, 1, 0, 0]     # no LiDAR in its window; file missing


@pytest.mark.skipif(not cs.ref_available(), reason="the reference source is not present")
@pytest.mark.parametrize("seed,leaf", [(22, 0.02), (23, 0.0)])
def test_oracle_equals_the_reference_live(tmp_path, seed, leaf):
    lib = cs.compile_ref(tmp_path / "libref_colorize.so")
    s = cs.ref_scene(seed)
    ax, ac, bx, bc, listed = cs.ref_run(lib, s, leaf, tmp_path / "data")
    a, b, mine = oracle_both(s, leaf)
    assert len(ax) > 2000
    assert cs.as_set(a[0], a[1]) == cs.as_set(ax, ac) and cs.as_set(b[0], b[1]) == cs.as_set(bx, bc)
    assert mine.tolist() == listed.tolist()
