"""Constant cameras under an active communicator (run under torchrun): lvba_visual_opts::cam_fixed runs on one GPU, so a mask with a
nonzero entry is LVBA_ERR_UNSUPPORTED, in the one-shot call and in lvba_visual_reset_lm, with the caller's buffers untouched, while
an all-zero mask is the same as none.
    python -m torch.distributed.run --nproc-per-node 2 tools/mgpu_fixed_check.py"""
import os
import sys

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import __graft_entry__ as g  # noqa: E402
from oracle import synth  # noqa: E402

KEYS = ("q", "t", "X", "plane_nd", "obs_ptr", "obs_cam", "obs_uv", "intr", "sigma_px", "sigma_plane")
UNSUPPORTED = -4

rank = int(os.environ.get("RANK", 0)); lrank = int(os.environ.get("LOCAL_RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
torch.cuda.set_device(lrank)
dist.init_process_group("nccl", device_id=torch.device("cuda", lrank))
pkg = g.load_package(); pkg.load_library()
uid = [pkg.comm_unique_id() if rank == 0 else None]; dist.broadcast_object_list(uid, src=0)
pkg.comm_init(world, rank, uid[0], lrank)
p = synth.make_problem(30, 0, 300, seed=11, lidar=False)
args = [p[k] for k in KEYS]
M = len(p["q"])
mask = np.zeros(M, bool); mask[[3, 7]] = True
ok = True
try:
    pkg.visual_lm(*args, fixed_cam=0, cam_fixed=mask)
    ok = False; print("one-shot with a mask was accepted")
except pkg.LvbaError as e:
    ok &= e.status == UNSUPPORTED; print("one-shot with a mask:", e.status)
q, t, X, s = pkg.visual_lm(*args, fixed_cam=0, cam_fixed=np.zeros(M, bool))       # all zero = no mask
ref = pkg.visual_lm(*args, fixed_cam=0)
ok &= s["iterations"] == ref[3]["iterations"] and abs(s["cost_last"] - ref[3]["cost_last"]) <= 1e-9 * ref[3]["cost_last"]
P = pkg.VisualProblem(*args, fixed_cam=0)
try:
    P.reset_lm(cam_fixed=mask)
    ok = False; print("reset with a mask was accepted")
except pkg.LvbaError as e:
    ok &= e.status == UNSUPPORTED; print("reset with a mask:", e.status)
P.reset_lm(cam_fixed=np.zeros(M, bool))
s2 = P.iterate(50)
ok &= s2["iterations"] == ref[3]["iterations"]
P.close()
print(f"MGPU_FIXED {'PASS' if ok else 'FAIL'} rank {rank} world {world}", flush=True)
pkg.comm_destroy(); dist.destroy_process_group()
sys.exit(0 if ok else 1)
