"""Pins the window-BA oracle (oracle.lidar_oracle.window_ba — LvbaSystem::runWindowBA, reference
src/lvba_system.cpp:232-302) without a GPU: committed golden fixture (regression) and agreement of the two
independent restatements (numpy vs the C++ port) window by window."""
from pathlib import Path

import numpy as np

from oracle import cpu_ref
from oracle import lidar_oracle as lo

GOLD = np.load(Path(__file__).parent / "golden" / "window_problem.npz")


def test_window_golden_regression():
    poses, infos = lo.window_ba(GOLD["win_ptr"], GOLD["vox_ptr"], GOLD["pose_idx"], GOLD["clusters"], GOLD["poses"])
    assert [i is None for i in infos] == list(GOLD["W_skipped"])
    assert [0 if i is None else i["iters"] for i in infos] == list(GOLD["W_iters"])
    assert [0 if i is None else i["accepted"] for i in infos] == list(GOLD["W_accepted"])
    assert np.abs(poses - GOLD["W_poses"]).max() <= 1e-12
    for w, i in enumerate(infos):
        if i is not None:
            assert abs(i["r_last"] - GOLD["W_cost_last"][w]) <= 1e-12 * GOLD["W_cost_last"][w]


def test_skip_rule_and_untouched_windows():
    """:262-266 — a window with fewer than 3 voxels per pose keeps its poses; the threshold is the caller's."""
    wp, n = GOLD["win_ptr"], len(GOLD["win_ptr"]) - 1
    for w in range(n):
        if GOLD["W_skipped"][w]:
            assert np.array_equal(GOLD["W_poses"][wp[w]:wp[w + 1]], GOLD["poses"][wp[w]:wp[w + 1]])
    poses, infos = lo.window_ba(GOLD["win_ptr"], GOLD["vox_ptr"], GOLD["pose_idx"], GOLD["clusters"], GOLD["poses"],
                                min_voxels_per_pose=1000)
    assert all(i is None for i in infos) and np.array_equal(poses, GOLD["poses"])


def test_cpp_port_agrees_window_by_window():
    """The port sums H, g and the residual per thread, so its last bits follow the thread count: it runs with the reference's
    own 16 (bavoxel.hpp:25), not the host's core count."""
    wp = GOLD["win_ptr"]
    first = GOLD["pose_idx"][GOLD["vox_ptr"][:-1]]
    win_of_vox = np.searchsorted(wp, first, side="right") - 1
    for w in range(len(wp) - 1):
        if GOLD["W_skipped"][w]:
            continue
        vs = np.nonzero(win_of_vox == w)[0]
        sl = [np.arange(GOLD["vox_ptr"][a], GOLD["vox_ptr"][a + 1]) for a in vs]
        vp = np.zeros(len(vs) + 1, np.int64); vp[1:] = np.cumsum([len(x) for x in sl])
        idx = np.concatenate(sl)
        poses, s = cpu_ref.lidar_lm(vp, (GOLD["pose_idx"][idx] - wp[w]).astype(np.int32), GOLD["clusters"][idx],
                                    GOLD["poses"][wp[w]:wp[w + 1]], threads=16)
        assert s["iterations"] == GOLD["W_iters"][w] and s["accepted"] == GOLD["W_accepted"][w]
        assert abs(s["cost_last"] - GOLD["W_cost_last"][w]) <= 1e-9 * GOLD["W_cost_last"][w]
        assert np.abs(poses - GOLD["W_poses"][wp[w]:wp[w + 1]]).max() <= 1e-9
