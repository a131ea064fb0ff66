"""Regenerates tests/golden/visual_default_lm.json: SHA-256 digests of what lvba_visual_lm returns with the default options in
deterministic mode (q, t, X and the summary's counts, termination and costs) on three seeded scenes, recorded with the build
that preceded the trust-region strategy option (lvba_visual_opts::trust_region_strategy).  tests/test_visual_dogleg_gpu.py holds
the default strategy's output to these bits.  Needs a GPU:

    python tests/golden/make_golden_visual_default.py [--root TREE] [--out FILE]

--root: the repository tree whose build to run (default: this one)."""
import argparse
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parents[2]


def scenes():
    from oracle import synth
    import visual_big_scene as vs
    return {"small": (synth.make_problem(30, 600, 300, seed=11), None),
            "small_huber": (synth.make_problem(30, 600, 300, seed=11), 1),
            "big": (vs.make_scene(5, M=120, n_short=150, long_tracks=((129, 10), (300, 0))), None)}


def digest(pkg, p, loss):
    import visual_big_scene as vs
    o = pkg.visual_default_opts(loss)
    o.deterministic = 1
    q, t, X, s = pkg.visual_lm(*vs.args(p), opts=o)
    h = hashlib.sha256()
    for a in (q, t, X):
        h.update(np.ascontiguousarray(a, np.float64).tobytes())
    h.update(np.array([s["iterations"], s["accepted"], s["hessian_builds"], s["termination"]], np.int64).tobytes())
    h.update(np.array([s["cost_first"], s["cost_last"]], np.float64).tobytes())
    return {"sha256": h.hexdigest(), "iterations": s["iterations"], "cost_last": s["cost_last"]}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=str(HERE))
    ap.add_argument("--out", default=str(HERE / "tests" / "golden" / "visual_default_lm.json"))
    a = ap.parse_args(argv)
    root = Path(a.root).resolve()
    sys.path[:0] = [str(root), str(root / "tests")]
    import __graft_entry__ as graft
    pkg = graft.load_package()
    pkg.load_library()
    out = {name: digest(pkg, p, loss) for name, (p, loss) in scenes().items()}
    Path(a.out).write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
