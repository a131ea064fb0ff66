"""Writes tests/golden/ref_colorize.npz: the reference's own VisualizeOptComparison (src/lvba_system.cpp:1932-2143, compiled where it lies
through tests/emu/ref_colorize_driver.cpp) on a seeded scene with patterned images — five images at the working size, one whose window holds
no LiDAR, one whose file is missing — under two pose sets.  Holds the inputs, both clouds it keeps (after / before, R G B) and the images it
lists in images.txt.  Run where the reference source exists:  python tests/golden/make_golden_ref_colorize.py"""
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent)); sys.path.insert(0, str(HERE.parents[1]))
import colorize_scene as cs  # noqa: E402

SEED, LEAF = 21, 0.01


def main():
    with tempfile.TemporaryDirectory() as tmp:
        lib = cs.compile_ref(Path(tmp) / "libref_colorize.so")
        s = cs.ref_scene(SEED)
        ax, ac, bx, bc, listed = cs.ref_run(lib, s, LEAF, Path(tmp) / "data")
    sp, xyz = cs.flat(s["scans"])
    np.savez_compressed(HERE / "ref_colorize.npz", scan_ptr=sp, xyz=xyz, frame_ts=s["frame_ts"], poses=s["poses"], poses_before=s["poses_before"],
                        image_ts=s["image_ts"], cams=s["cams"], cams_before=s["cams_before"], intr=s["intr"], width=s["width"], height=s["height"],
                        rgb=s["rgb"], loaded=s["loaded"], leaf=LEAF, after_xyz=ax, after_rgb=ac, before_xyz=bx, before_rgb=bc, listed=listed)


if __name__ == "__main__":
    main()
