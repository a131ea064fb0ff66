"""Boundary B8 on the device against the reference's own VisualizeOptComparison, through the committed fixture
tests/golden/ref_colorize.npz (tests/golden/make_golden_ref_colorize.py): both clouds — after and before — equal the reference's as sets of
(x, y, z, r, g, b), and the listed images are the ones its images.txt holds."""
import numpy as np
import pytest

import colorize_scene as cs

pytestmark = pytest.mark.gpu


def test_device_equals_the_reference_fixture(gpu_pkg):
    s, leaf, ref = cs.fixture()
    keep, sub = cs.loaded_subset(s)
    cz = gpu_pkg.Colorizer(sub["scans"], sub["frame_ts"])
    try:
        ax, ac, la, _ = cz.run(sub["poses"], sub["image_ts"], sub["cams"], sub["intr"], sub["width"], sub["height"], sub["rgb"], leaf=leaf)
        bx, bc, lb, _ = cz.run(sub["poses_before"], sub["image_ts"], sub["cams_before"], sub["intr"], sub["width"], sub["height"], sub["rgb"], leaf=leaf)
    finally:
        cz.close()
    assert cs.as_set(ax, ac) == cs.as_set(ref["after_xyz"], ref["after_rgb"])
    assert cs.as_set(bx, bc) == cs.as_set(ref["before_xyz"], ref["before_rgb"])
    listed = np.zeros(len(s["image_ts"]), np.uint8); listed[keep] = la
    assert listed.tolist() == ref["listed"].tolist() and la.tolist() == lb.tolist()
