"""Constant LiDAR poses under an active communicator (run under torchrun): lvba_lidar_opts::pose_fixed runs on one GPU, so a mask
with a nonzero entry is LVBA_ERR_UNSUPPORTED, in lvba_lidar_lm and in lvba_lidar_reset_lm, while an all-zero mask is the same as
none.
    python -m torch.distributed.run --nproc-per-node 2 tools/mgpu_fixed_lidar_check.py"""
import os
import sys

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import __graft_entry__ as g  # noqa: E402
from oracle import synth  # noqa: E402

KEYS = ("vox_ptr", "pose_idx", "clusters", "poses")
UNSUPPORTED = -4

rank = int(os.environ.get("RANK", 0)); lrank = int(os.environ.get("LOCAL_RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
torch.cuda.set_device(lrank)
dist.init_process_group("nccl", device_id=torch.device("cuda", lrank))
pkg = g.load_package(); pkg.load_library()
uid = [pkg.comm_unique_id() if rank == 0 else None]; dist.broadcast_object_list(uid, src=0)
pkg.comm_init(world, rank, uid[0], lrank)
p = synth.make_problem(30, 600, 0, seed=11, visual=False)
args = [p[k] for k in KEYS]
W = len(p["poses"])
mask = np.zeros(W, bool); mask[[0, 7]] = True
ok = True
try:
    pkg.lidar_lm(*args, pose_fixed=mask)
    ok = False; print("one-shot with a mask was accepted")
except pkg.LvbaError as e:
    ok &= e.status == UNSUPPORTED; print("one-shot with a mask:", e.status)
x, s = pkg.lidar_lm(*args, pose_fixed=np.zeros(W, bool))                    # all zero = no mask
y, ref = pkg.lidar_lm(*args)
ok &= s["iterations"] == ref["iterations"] and abs(s["cost_last"] - ref["cost_last"]) <= 1e-9 * ref["cost_last"]
P = pkg.LidarProblem(*args)
try:
    P.reset_lm(pose_fixed=mask)
    ok = False; print("reset with a mask was accepted")
except pkg.LvbaError as e:
    ok &= e.status == UNSUPPORTED; print("reset with a mask:", e.status)
P.reset_lm(pose_fixed=np.zeros(W, bool))
s2 = P.iterate(10)
ok &= s2["iterations"] == ref["iterations"]
P.close()
print(f"MGPU_FIXED_LIDAR {'PASS' if ok else 'FAIL'} rank {rank} world {world}", flush=True)
pkg.comm_destroy(); dist.destroy_process_group()
sys.exit(0 if ok else 1)
