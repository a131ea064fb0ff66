"""global-lvba_b200 — host-side mirror (Python/ctypes) of the C ABI in include/lvba_b200.h.

The product is `liblvba_b200.so` (CUDA, sm_90a) built from `csrc/`; this module only
binds it.  It is what tests/ and bench.py use to drive the library exactly as a C++
caller would (plain pointers and sizes).  There is NO CPU fallback here: if the shared
library is missing, or no CUDA device is present, every compute call raises.

The directory name contains a hyphen (it mirrors the reference repo name), so import it
through `__graft_entry__.load_package()` / `tests/conftest.py`, which register it as the
module `global_lvba_b200`.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "liblvba_b200.so"
_lib = None

# names every build of the library must export (kept in sync with include/lvba_b200.h;
# tests/test_abi.py cross-checks this list against the header)
EXPORTS = [
    "lvba_version", "lvba_device_count", "lvba_status_string", "lvba_last_error", "lvba_release_cached_memory",
    "lvba_lidar_default_opts", "lvba_visual_default_opts",
    "lvba_lidar_lm", "lvba_lidar_lm_batch", "lvba_lidar_create", "lvba_lidar_destroy", "lvba_lidar_set_poses",
    "lvba_lidar_get_poses", "lvba_lidar_build", "lvba_lidar_residual", "lvba_lidar_solve",
    "lvba_lidar_structure", "lvba_lidar_get_system", "lvba_lidar_reset_lm", "lvba_lidar_reset_state", "lvba_lidar_iterate",
    "lvba_lidar_counts", "lvba_lidar_rows",
    "lvba_lidar_voxel_residuals", "lvba_lidar_remove_voxels", "lvba_lidar_remove_outliers",
    "lvba_visual_lm", "lvba_visual_create", "lvba_visual_destroy", "lvba_visual_set_state",
    "lvba_visual_get_state", "lvba_visual_cost", "lvba_visual_step", "lvba_visual_structure",
    "lvba_visual_get_system", "lvba_visual_reset_lm", "lvba_visual_reset_state", "lvba_visual_iterate", "lvba_visual_counts",
    "lvba_visual_big_counts", "lvba_visual_obs_residuals", "lvba_visual_remove_observations", "lvba_visual_remove_outliers",
    "lvba_visual_get_intrinsics", "lvba_visual_set_intrinsics", "lvba_visual_get_intrinsics_system", "lvba_visual_linear_stats",
    "lvba_visual_schur_product", "lvba_visual_apply_system", "lvba_visual_dogleg_state",
    "lvba_voxel_default_opts", "lvba_voxel_map_create", "lvba_voxel_map_create_windows", "lvba_voxel_map_windows",
    "lvba_voxel_map_lidar_lm_batch", "lvba_voxel_map_summary", "lvba_voxel_map_export",
    "lvba_voxel_map_lookup", "lvba_voxel_map_lidar_create", "lvba_voxel_map_lidar_lm", "lvba_voxel_map_destroy",
    "lvba_depth_grid_create", "lvba_depth_render", "lvba_depth_backproject", "lvba_depth_grid_destroy",
    "lvba_tracks_triangulate", "lvba_tracks_mean_reproj",
    "lvba_fuse_default_opts", "lvba_tracks_fuse_create", "lvba_tracks_fuse_summary", "lvba_tracks_fuse_export", "lvba_tracks_fuse_destroy",
    "lvba_anchor_clouds_create", "lvba_anchor_clouds_export", "lvba_anchor_clouds_destroy",
    "lvba_colorizer_create", "lvba_colorizer_begin", "lvba_colorizer_add_images", "lvba_colorizer_finish",
    "lvba_colorizer_export", "lvba_colorizer_destroy",
    "lvba_env_solve", "lvba_lidar_owned_rows", "lvba_visual_owned_rows", "lvba_comm_bytes_sent",
    "lvba_comm_unique_id", "lvba_comm_init", "lvba_comm_destroy", "lvba_comm_info", "lvba_shard_owner",
]


class LvbaError(RuntimeError):
    def __init__(self, status, detail):
        super().__init__(f"lvba status {status}: {detail}")
        self.status = status


class LidarOpts(C.Structure):
    _fields_ = [("u0", C.c_double), ("v0", C.c_double), ("max_iter", C.c_int32), ("rel_tol", C.c_double),
                ("device", C.c_int32), ("verbose", C.c_int32), ("deterministic", C.c_int32),
                ("pose_fixed", C.POINTER(C.c_uint8))]


class VisualOpts(C.Structure):
    _fields_ = [("max_iter", C.c_int32), ("refine_intrinsics", C.c_uint32), ("initial_radius", C.c_double), ("max_radius", C.c_double),
                ("min_radius", C.c_double), ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double),
                ("min_relative_decrease", C.c_double), ("function_tolerance", C.c_double),
                ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
                ("jacobi_scaling", C.c_int32), ("device", C.c_int32), ("verbose", C.c_int32),
                ("deterministic", C.c_int32),
                ("reproj_loss", C.c_int32), ("reproj_loss_scale", C.c_double),
                ("plane_loss", C.c_int32), ("plane_loss_scale", C.c_double),
                ("linear_solver", C.c_int32), ("eta", C.c_double), ("min_linear_iter", C.c_int32), ("max_linear_iter", C.c_int32),
                ("trust_region_strategy", C.c_int32),
                ("cam_fixed", C.POINTER(C.c_uint8))]


# lvba_linear_solver: the solver of the reduced camera system (VisualOpts.linear_solver)
LINEAR_DENSE_SCHUR, LINEAR_ITERATIVE_SCHUR = 0, 1
# the termination of one conjugate-gradients solve (VisualProblem.linear_stats)
CG_SUCCESS, CG_NO_CONVERGENCE, CG_FAILURE = 0, 1, 2
# lvba_trust_region: the trust-region strategy (VisualOpts.trust_region_strategy)
TR_LEVENBERG_MARQUARDT, TR_DOGLEG = 0, 1
# lvba_dogleg_case: the step of the last dogleg pass (VisualProblem.dogleg_state)
DOGLEG_NONE, DOGLEG_GAUSS_NEWTON, DOGLEG_CAUCHY, DOGLEG_INTERPOLATED = 0, 1, 2, 3

# lvba_visual_opts::refine_intrinsics: bit i frees intr[i] of (fx fy cx cy k1 k2 p1 p2)
INTR_FOCAL, INTR_PRINCIPAL, INTR_DISTORTION = 0x03, 0x0C, 0xF0

# lvba_loss_kind: the robust loss of the reprojection / plane residual blocks (VisualOpts.reproj_loss / plane_loss)
LOSS_NONE, LOSS_HUBER, LOSS_CAUCHY = 0, 1, 2


class Summary(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("accepted", C.c_int32), ("hessian_builds", C.c_int32),
                ("termination", C.c_int32), ("cost_first", C.c_double), ("cost_last", C.c_double),
                ("damping_last", C.c_double), ("ms_total", C.c_double), ("ms_setup", C.c_double),
                ("ms_build", C.c_double), ("ms_solve", C.c_double), ("ms_residual", C.c_double),
                ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class VoxelOpts(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("eigen_ratio", C.c_float * 4), ("layer_limit", C.c_int32),
                ("min_points", C.c_int32), ("device", C.c_int32)]


class VoxelSummary(C.Structure):
    _fields_ = [("n_points", C.c_int64), ("n_voxels", C.c_int64), ("nnz", C.c_int64), ("n_nodes", C.c_int64 * 3),
                ("ms_total", C.c_double), ("ms_upload", C.c_double), ("ms_device", C.c_double),
                ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["n_nodes"] = list(self.n_nodes)
        return d


class DepthSummary(C.Structure):
    _fields_ = [("n_points", C.c_int64), ("n_voxels", C.c_int64), ("n_pairs", C.c_int64),
                ("ms_total", C.c_double), ("ms_upload", C.c_double), ("ms_device", C.c_double),
                ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("work_pairs", C.c_int64), ("work_chunks", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def build_library(force=False, quiet=True):
    """Compile csrc/ for sm_90a with nvcc (cross-compiles without a GPU)."""
    if LIB_PATH.exists() and not force:
        src_m = max(p.stat().st_mtime for p in list((_HERE / "csrc").glob("*.cu*")) + list((_HERE / "csrc").glob("*.h")) + [(_HERE.parent / "include" / "lvba_b200.h")])
        if LIB_PATH.stat().st_mtime >= src_m:
            return LIB_PATH
    r = subprocess.run(["make", "-C", str(_HERE / "csrc")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building liblvba_b200.so failed:\n" + r.stdout + r.stderr)
    if not quiet:
        print(r.stdout)
    return LIB_PATH


def load_library():
    """dlopen liblvba_b200.so; raises (never falls back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = LIB_PATH
    if os.environ.get("LVBA_B200_DEV_LIB"):          # another build of the same library (e.g. an older one to compare against): tools/ only
        path = _HERE / os.environ["LVBA_B200_DEV_LIB"]
    if not path.exists():
        raise LvbaError(-2, f"{path} not built: run __graft_entry__.build(); there is no CPU fallback")
    lib = C.CDLL(str(path), mode=C.RTLD_GLOBAL)
    lib.lvba_status_string.restype = C.c_char_p
    lib.lvba_last_error.restype = C.c_char_p
    lib.lvba_shard_owner.restype = C.c_int32
    _lib = lib
    return lib


def _chk(rc):
    if rc != 0:
        lib = load_library()
        raise LvbaError(rc, (lib.lvba_last_error() or b"").decode() or lib.lvba_status_string(rc).decode())


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def device_count():
    return int(load_library().lvba_device_count())


def shard_owner(min_pose, n_rows, n_ranks):
    return int(load_library().lvba_shard_owner(int(min_pose), int(n_rows), int(n_ranks)))


def lidar_default_opts():
    o = LidarOpts()
    load_library().lvba_lidar_default_opts(C.byref(o))
    return o


def visual_default_opts(reproj_loss=None, plane_loss=None):
    """lvba_visual_default_opts; reproj_loss / plane_loss: None (no loss), a kind (LOSS_*, the default scale) or (kind, scale)."""
    o = VisualOpts()
    load_library().lvba_visual_default_opts(C.byref(o))
    for loss, kind, scale in ((reproj_loss, "reproj_loss", "reproj_loss_scale"), (plane_loss, "plane_loss", "plane_loss_scale")):
        if loss is None:
            continue
        if isinstance(loss, tuple):
            setattr(o, kind, int(loss[0])); setattr(o, scale, float(loss[1]))
        else:
            setattr(o, kind, int(loss))
    return o


# ------------------------------------------------------------------ B1: LiDAR
def _with_pose_fixed(opts, pose_fixed, W):
    """opts (None: the defaults) with pose_fixed set from a boolean mask of W poses; returns (opts, the mask array the
    pointer refers to, which the caller keeps alive for the call).  pose_fixed None leaves opts as they are."""
    if pose_fixed is None:
        return opts, None
    m = np.ascontiguousarray(np.asarray(pose_fixed, bool), np.uint8)
    if m.shape != (W,):
        raise ValueError(f"pose_fixed has shape {m.shape}, expected ({W},)")
    o = lidar_default_opts() if opts is None else LidarOpts.from_buffer_copy(opts)
    o.pose_fixed = _p(m, C.c_uint8)
    return o, m


def lidar_lm(vox_ptr, pose_idx, clusters, poses, opts=None, pose_fixed=None):
    """One-shot drop-in for BALM2::damping_iter (bavoxel.hpp:662).  pose_fixed: boolean mask [W] of constant poses
    (lvba_lidar_opts::pose_fixed), or None.  Returns (poses, summary dict)."""
    lib = load_library()
    vp = np.ascontiguousarray(vox_ptr, np.int64); pi = np.ascontiguousarray(pose_idx, np.int32)
    cl = _f64(clusters); ps = _f64(poses).copy()
    opts, mask = _with_pose_fixed(opts, pose_fixed, ps.shape[0])
    s = Summary()
    _chk(lib.lvba_lidar_lm(C.c_int32(ps.shape[0]), C.c_int64(len(vp) - 1), _p(vp, C.c_int64), _p(pi, C.c_int32),
                           _p(cl, C.c_double), _p(ps, C.c_double), C.byref(opts) if opts is not None else None,
                           C.byref(s)))
    return ps, s.as_dict()


def lidar_lm_batch(win_ptr, vox_ptr, pose_idx, clusters, poses, min_voxels_per_pose=3, opts=None, pose_fixed=None):
    """Every window of LvbaSystem::runWindowBA (src/lvba_system.cpp:232-302) in one call.  pose_fixed: boolean mask over
    the concatenated poses, or None.  Returns (poses, [per-window summary dict], total summary dict)."""
    lib = load_library()
    wp = np.ascontiguousarray(win_ptr, np.int32)
    vp = np.ascontiguousarray(vox_ptr, np.int64); pi = np.ascontiguousarray(pose_idx, np.int32)
    cl = _f64(clusters); ps = _f64(poses).copy()
    opts, mask = _with_pose_fixed(opts, pose_fixed, ps.shape[0])
    nw = len(wp) - 1
    sums = (Summary * max(nw, 1))()
    tot = Summary()
    _chk(lib.lvba_lidar_lm_batch(C.c_int32(nw), _p(wp, C.c_int32), C.c_int64(len(vp) - 1), _p(vp, C.c_int64),
                                 _p(pi, C.c_int32), _p(cl, C.c_double), _p(ps, C.c_double),
                                 C.c_int32(min_voxels_per_pose), C.byref(opts) if opts is not None else None,
                                 sums, C.byref(tot)))
    return ps, [sums[i].as_dict() for i in range(nw)], tot.as_dict()


class LidarProblem:
    """Device-resident handle (lvba_lidar_create ...)."""

    def __init__(self, vox_ptr, pose_idx, clusters, poses, device=-1):
        lib = load_library()
        self._lib = lib
        self.vp = np.ascontiguousarray(vox_ptr, np.int64); self.pi = np.ascontiguousarray(pose_idx, np.int32)
        cl = _f64(clusters); ps = _f64(poses)
        self.W = ps.shape[0]; self.V = len(self.vp) - 1
        self._h = C.c_void_p()
        _chk(lib.lvba_lidar_create(C.c_int32(self.W), C.c_int64(self.V), _p(self.vp, C.c_int64), _p(self.pi, C.c_int32),
                                   _p(cl, C.c_double), _p(ps, C.c_double), C.c_int32(device), C.byref(self._h)))

    @classmethod
    def _from_handle(cls, h, W, V):
        self = cls.__new__(cls)
        self._lib = load_library(); self._h = h; self.W = W; self.V = V; self.vp = None; self.pi = None
        return self

    def close(self):
        if self._h:
            self._lib.lvba_lidar_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_poses(self, poses):
        ps = _f64(poses); _chk(self._lib.lvba_lidar_set_poses(self._h, _p(ps, C.c_double)))

    def get_poses(self):
        out = np.empty((self.W, 12)); _chk(self._lib.lvba_lidar_get_poses(self._h, _p(out, C.c_double))); return out

    def build(self):
        r = C.c_double(); _chk(self._lib.lvba_lidar_build(self._h, C.byref(r))); return r.value

    def residual(self, poses=None):
        r = C.c_double()
        if poses is None:
            _chk(self._lib.lvba_lidar_residual(self._h, None, C.byref(r)))
        else:
            ps = _f64(poses); _chk(self._lib.lvba_lidar_residual(self._h, _p(ps, C.c_double), C.byref(r)))
        return r.value

    def solve(self, u):
        dx = np.empty(self.W * 6); _chk(self._lib.lvba_lidar_solve(self._h, C.c_double(u), _p(dx, C.c_double))); return dx

    def rows(self):
        """pose_of_row [n_rows] (lvba_lidar_rows): the free poses, one row of the pose system each, ascending."""
        n = C.c_int32(); _chk(self._lib.lvba_lidar_rows(self._h, C.byref(n), None))
        out = np.empty(n.value, np.int32)
        _chk(self._lib.lvba_lidar_rows(self._h, C.byref(n), _p(out, C.c_int32)))
        return out

    def structure(self):
        nb = C.c_int64(); _chk(self._lib.lvba_lidar_structure(self._h, C.byref(nb), None, None))
        br = np.empty(nb.value, np.int32); bc = np.empty(nb.value, np.int32)
        _chk(self._lib.lvba_lidar_structure(self._h, C.byref(nb), _p(br, C.c_int32), _p(bc, C.c_int32)))
        return br, bc

    def get_system(self):
        """(g [n_rows, 6], brow, bcol, blocks): the system over the rows (rows())."""
        br, bc = self.structure()
        g = np.empty((len(self.rows()), 6)); blocks = np.empty((len(br), 6, 6))
        _chk(self._lib.lvba_lidar_get_system(self._h, _p(g, C.c_double), _p(blocks, C.c_double)))
        return g, br, bc, blocks

    def reset_lm(self, opts=None, pose_fixed=None):
        """lvba_lidar_reset_lm; pose_fixed: boolean mask [W] of constant poses (a mask that differs from the handle's
        re-plans it), or None for what opts.pose_fixed says."""
        opts, mask = _with_pose_fixed(opts, pose_fixed, self.W)
        _chk(self._lib.lvba_lidar_reset_lm(self._h, C.byref(opts) if opts is not None else None))

    def reset_state(self):
        _chk(self._lib.lvba_lidar_reset_state(self._h))

    def iterate(self, n):
        s = Summary(); _chk(self._lib.lvba_lidar_iterate(self._h, C.c_int32(n), C.byref(s))); return s.as_dict()

    def owned_rows(self):
        """(row_begin, row_end, sharded): block rows of H this rank holds (multi-GPU, include/lvba_b200.h)"""
        a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
        _chk(self._lib.lvba_lidar_owned_rows(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, bool(c.value)

    def counts(self, nonzero=True):
        a, b, c, d = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        _chk(self._lib.lvba_lidar_counts(self._h, C.byref(a), C.byref(b), C.byref(c) if nonzero else None, C.byref(d)))
        return dict(nnz=a.value, n_blocks_env=b.value, n_blocks_nonzero=c.value if nonzero else None, n_pairs=d.value)

    def voxel_residuals(self, poses=None):
        """lambda0 [V] of every voxel (lvba_lidar_voxel_residuals, VOX_HESS::evaluate_residual) at `poses`, or at the
        handle's poses when None; in the handle's voxel order (the caller's, minus the voxels removed so far)."""
        out = np.empty(self.V)
        ps = None if poses is None else _f64(poses)
        _chk(self._lib.lvba_lidar_voxel_residuals(self._h, None if ps is None else _p(ps, C.c_double), _p(out, C.c_double)))
        return out

    def remove_voxels(self, mask):
        """Erase the voxels where mask [V] is true (lvba_lidar_remove_voxels); returns the number of voxels left."""
        m = np.ascontiguousarray(np.asarray(mask, bool), np.uint8)
        if m.shape != (self.V,):
            raise ValueError(f"mask has shape {m.shape}, expected ({self.V},)")
        n = C.c_int64()
        _chk(self._lib.lvba_lidar_remove_voxels(self._h, _p(m, C.c_uint8), C.byref(n)))
        self.V = n.value
        return self.V

    def remove_outliers(self, ratio):
        """BALM2::remove_outlier at the handle's poses (lvba_lidar_remove_outliers); returns the boolean mask [V before the
        call] of the removed voxels."""
        out = np.zeros(self.V, np.uint8)
        n = C.c_int64()
        _chk(self._lib.lvba_lidar_remove_outliers(self._h, C.c_double(ratio), _p(out, C.c_uint8), C.byref(n)))
        self.V -= n.value
        return out.astype(bool)


SOLVE_AUTO, SOLVE_ONE_CTA, SOLVE_TWISTED, SOLVE_CHUNKED, SOLVE_SHARED_WINDOW, SOLVE_ANY_WIDTH = range(6)


def env_layout(first_raw):
    """Monotone first[] and row offsets of the block envelope (Envelope::build, csrc/runtime.cuh)."""
    n = len(first_raw)
    first = np.minimum(np.asarray(first_raw, np.int64), np.arange(n))
    first = np.minimum.accumulate(first[::-1])[::-1]
    row_start = np.zeros(n + 1, np.int64)
    row_start[1:] = np.cumsum(np.arange(n) - first + 1)
    return first.astype(np.int32), row_start


def env_solve(first, blocks, dadd, rhs, path=SOLVE_AUTO, chunks=0, reps=1, device=-1):
    """lvba_env_solve: (A + diag(dadd)) x = rhs through one of the block LDL^T paths; returns x, ms, info dict."""
    lib = load_library()
    first = np.ascontiguousarray(first, np.int32)
    n = len(first)
    blocks = _f64(blocks); dadd = _f64(dadd); rhs = _f64(rhs)
    x = np.zeros(6 * n)
    ms = C.c_double(0.0)
    info = np.zeros(4, np.int32)
    _chk(lib.lvba_env_solve(C.c_int32(n), _p(first, C.c_int32), _p(blocks, C.c_double), _p(dadd, C.c_double), _p(rhs, C.c_double),
                            _p(x, C.c_double), C.c_int32(path), C.c_int32(chunks), C.c_int32(reps), C.c_int32(device),
                            C.byref(ms), _p(info, C.c_int32)))
    return x, ms.value, {"path": int(info[0]), "chunks": int(info[1]), "levels": int(info[2]), "launches": int(info[3])}


def env_blocks_to_dense(br, bc, blocks, n):
    """Expand lower-envelope 6x6 blocks into a dense symmetric matrix (test helper)."""
    H = np.zeros((6 * n, 6 * n))
    for r, c, b in zip(br, bc, blocks):
        H[6 * r:6 * r + 6, 6 * c:6 * c + 6] = b
        if r != c:
            H[6 * c:6 * c + 6, 6 * r:6 * r + 6] = b.T
    return H


# ------------------------------------------------------------------ B2: visual
def _with_cam_fixed(opts, cam_fixed, M):
    """opts (None: the defaults) with cam_fixed set from a boolean mask of M cameras; returns (opts, the mask array the
    pointer refers to, which the caller keeps alive for the call).  cam_fixed None leaves opts as they are."""
    if cam_fixed is None:
        return opts, None
    m = np.ascontiguousarray(np.asarray(cam_fixed, bool), np.uint8)
    if m.shape != (M,):
        raise ValueError(f"cam_fixed has shape {m.shape}, expected ({M},)")
    o = visual_default_opts() if opts is None else VisualOpts.from_buffer_copy(opts)
    o.cam_fixed = _p(m, C.c_uint8)
    return o, m


def _with_linear(opts, linear_solver, eta, min_linear_iter, max_linear_iter, trust_region_strategy=None):
    """opts (None: the defaults) with those of the linear-solver and trust-region fields that are not None set
    (lvba_visual_opts::linear_solver, eta, min_linear_iter, max_linear_iter, trust_region_strategy); opts as they are when all
    are None."""
    kw = dict(linear_solver=linear_solver, eta=eta, min_linear_iter=min_linear_iter, max_linear_iter=max_linear_iter,
              trust_region_strategy=trust_region_strategy)
    if all(v is None for v in kw.values()):
        return opts
    o = visual_default_opts() if opts is None else VisualOpts.from_buffer_copy(opts)
    for k, v in kw.items():
        if v is not None:
            setattr(o, k, v)
    return o


def visual_lm(q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam=0, opts=None, cam_fixed=None,
              linear_solver=None, eta=None, min_linear_iter=None, max_linear_iter=None, trust_region_strategy=None):
    """One-shot drop-in for the Ceres block of optimizeCameraPoses (lvba_system.cpp:1571-1656).  cam_fixed: boolean mask
    [M] of further constant cameras (lvba_visual_opts::cam_fixed), or None.  linear_solver (LINEAR_*), eta, min_linear_iter,
    max_linear_iter: the solver of the reduced camera system, trust_region_strategy (TR_*): LM or dogleg; None for what opts
    says."""
    lib = load_library()
    opts = _with_linear(opts, linear_solver, eta, min_linear_iter, max_linear_iter, trust_region_strategy)
    q = _f64(q).copy(); t = _f64(t).copy(); X = _f64(X).copy(); pl = _f64(plane_nd)
    op = np.ascontiguousarray(obs_ptr, np.int64); oc = np.ascontiguousarray(obs_cam, np.int32)
    uv = np.ascontiguousarray(obs_uv, np.float32); it = _f64(intr)
    opts, mask = _with_cam_fixed(opts, cam_fixed, q.shape[0])
    s = Summary()
    _chk(lib.lvba_visual_lm(C.c_int32(q.shape[0]), C.c_int64(X.shape[0]), _p(q, C.c_double), _p(t, C.c_double),
                            _p(X, C.c_double), _p(pl, C.c_double), _p(op, C.c_int64), _p(oc, C.c_int32),
                            _p(uv, C.c_float), _p(it, C.c_double), C.c_double(sigma_px), C.c_double(sigma_plane),
                            C.c_int32(fixed_cam), C.byref(opts) if opts is not None else None, C.byref(s)))
    del mask
    return q, t, X, s.as_dict()


class VisualProblem:
    def __init__(self, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam=0, device=-1):
        lib = load_library()
        self._lib = lib
        q = _f64(q); t = _f64(t); X = _f64(X); pl = _f64(plane_nd)
        op = np.ascontiguousarray(obs_ptr, np.int64); oc = np.ascontiguousarray(obs_cam, np.int32)
        uv = np.ascontiguousarray(obs_uv, np.float32); it = _f64(intr)
        self.M, self.T = q.shape[0], X.shape[0]
        self.n_obs = int(op[-1])
        self._h = C.c_void_p()
        _chk(lib.lvba_visual_create(C.c_int32(self.M), C.c_int64(self.T), _p(q, C.c_double), _p(t, C.c_double),
                                    _p(X, C.c_double), _p(pl, C.c_double), _p(op, C.c_int64), _p(oc, C.c_int32),
                                    _p(uv, C.c_float), _p(it, C.c_double), C.c_double(sigma_px),
                                    C.c_double(sigma_plane), C.c_int32(fixed_cam), C.c_int32(device), C.byref(self._h)))

    def close(self):
        if self._h:
            self._lib.lvba_visual_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_state(self, q, t, X):
        q = _f64(q); t = _f64(t); X = _f64(X)
        _chk(self._lib.lvba_visual_set_state(self._h, _p(q, C.c_double), _p(t, C.c_double), _p(X, C.c_double)))

    def get_state(self):
        q = np.empty((self.M, 4)); t = np.empty((self.M, 3)); X = np.empty((self.T, 3))
        _chk(self._lib.lvba_visual_get_state(self._h, _p(q, C.c_double), _p(t, C.c_double), _p(X, C.c_double)))
        return q, t, X

    def cost(self):
        c = C.c_double(); _chk(self._lib.lvba_visual_cost(self._h, C.byref(c))); return c.value

    def step(self, radius, jacobi_scaling=True, recompute_scale=True):
        cs = np.empty((self.M, 6)); ps = np.empty((self.T, 3)); mc = C.c_double(); c = C.c_double()
        _chk(self._lib.lvba_visual_step(self._h, C.c_double(radius), C.c_int32(int(jacobi_scaling)),
                                        C.c_int32(int(recompute_scale)), _p(cs, C.c_double), _p(ps, C.c_double),
                                        C.byref(mc), C.byref(c)))
        return cs, ps, mc.value, c.value

    def structure(self):
        na = C.c_int32(); nb = C.c_int64()
        _chk(self._lib.lvba_visual_structure(self._h, C.byref(na), None, C.byref(nb), None, None))
        cam = np.empty(na.value, np.int32); br = np.empty(nb.value, np.int32); bc = np.empty(nb.value, np.int32)
        _chk(self._lib.lvba_visual_structure(self._h, C.byref(na), _p(cam, C.c_int32), C.byref(nb), _p(br, C.c_int32), _p(bc, C.c_int32)))
        return cam, br, bc

    def get_system(self):
        cam, br, bc = self.structure()
        rhs = np.empty((len(cam), 6)); blocks = np.empty((len(br), 6, 6))
        _chk(self._lib.lvba_visual_get_system(self._h, _p(rhs, C.c_double), _p(blocks, C.c_double)))
        return cam, rhs, br, bc, blocks

    def reset_lm(self, opts=None, cam_fixed=None, refine_intrinsics=None, linear_solver=None, eta=None, min_linear_iter=None,
                 max_linear_iter=None, trust_region_strategy=None):
        """lvba_visual_reset_lm; cam_fixed: boolean mask [M] of further constant cameras (a mask that differs from the
        handle's re-plans it), or None for what opts.cam_fixed says; refine_intrinsics: the mask of free intrinsics
        (INTR_* bits), or None for what opts.refine_intrinsics says; linear_solver (LINEAR_*), eta, min_linear_iter,
        max_linear_iter: the solver of the reduced camera system, trust_region_strategy (TR_*): LM or dogleg; None for what
        opts says."""
        opts = _with_linear(opts, linear_solver, eta, min_linear_iter, max_linear_iter, trust_region_strategy)
        opts, mask = _with_cam_fixed(opts, cam_fixed, self.M)
        if refine_intrinsics is not None:
            opts = visual_default_opts() if opts is None else VisualOpts.from_buffer_copy(opts)
            opts.refine_intrinsics = int(refine_intrinsics)
        _chk(self._lib.lvba_visual_reset_lm(self._h, C.byref(opts) if opts is not None else None))
        del mask

    def reset_state(self):
        _chk(self._lib.lvba_visual_reset_state(self._h))

    def get_intrinsics(self):
        """The handle's current (fx fy cx cy k1 k2 p1 p2) (lvba_visual_get_intrinsics)."""
        out = np.empty(8); _chk(self._lib.lvba_visual_get_intrinsics(self._h, _p(out, C.c_double))); return out

    def set_intrinsics(self, intr):
        it = _f64(intr)
        if it.shape != (8,):
            raise ValueError(f"intr has shape {it.shape}, expected (8,)")
        _chk(self._lib.lvba_visual_set_intrinsics(self._h, _p(it, C.c_double)))

    def intrinsics_system(self):
        """The intrinsics block of the last step (lvba_visual_get_intrinsics_system): dict(border [n_active*6, k],
        corner [k, k], rhs [k], step [8])."""
        k = C.c_int32()
        _chk(self._lib.lvba_visual_get_intrinsics_system(self._h, C.byref(k), None, None, None, None))
        n6 = 6 * len(self.structure()[0])
        B = np.zeros((n6, k.value)); Cc = np.zeros((k.value, k.value)); r = np.zeros(k.value); st = np.zeros(8)
        _chk(self._lib.lvba_visual_get_intrinsics_system(self._h, C.byref(k), _p(B, C.c_double), _p(Cc, C.c_double),
                                                         _p(r, C.c_double), _p(st, C.c_double)))
        return dict(border=B, corner=Cc, rhs=r, step=st)

    def linear_stats(self):
        """lvba_visual_linear_stats: dict(cg_iters_total (since the last reset_lm or removal), cg_iters_last, term_last (CG_*))."""
        a, b, c = C.c_int64(), C.c_int32(), C.c_int32()
        _chk(self._lib.lvba_visual_linear_stats(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(cg_iters_total=a.value, cg_iters_last=b.value, term_last=c.value)

    def dogleg_state(self):
        """lvba_visual_dogleg_state: dict(radius, mu, alpha, grad_norm, gn_norm, case (DOGLEG_*), reused (passes since the
        last reset_lm or removal that reused a linearisation)).  LvbaError unless the last reset_lm chose TR_DOGLEG."""
        d = [C.c_double() for _ in range(5)]
        c, r = C.c_int32(), C.c_int64()
        _chk(self._lib.lvba_visual_dogleg_state(self._h, *[C.byref(v) for v in d], C.byref(c), C.byref(r)))
        return dict(radius=d[0].value, mu=d[1].value, alpha=d[2].value, grad_norm=d[3].value, gn_norm=d[4].value, case=c.value,
                    reused=r.value)

    def schur_product(self):
        """lvba_visual_schur_product: 1 when ITERATIVE_SCHUR runs on the matrix-free product for this plan, 0 on the explicit S."""
        m = C.c_int32(); _chk(self._lib.lvba_visual_schur_product(self._h, C.byref(m))); return m.value

    def apply_system(self, x):
        """lvba_visual_apply_system: (S + D) x of the last ITERATIVE_SCHUR pass, x and the result [n_active*6]."""
        x = _f64(x).ravel()
        n6 = 6 * len(self.structure()[0])
        if x.shape != (n6,):
            raise ValueError(f"x has shape {x.shape}, expected ({n6},)")
        y = np.empty(n6)
        _chk(self._lib.lvba_visual_apply_system(self._h, _p(x, C.c_double), _p(y, C.c_double)))
        return y

    def iterate(self, n):
        s = Summary(); _chk(self._lib.lvba_visual_iterate(self._h, C.c_int32(n), C.byref(s))); return s.as_dict()

    def owned_rows(self):
        a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
        _chk(self._lib.lvba_visual_owned_rows(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, bool(c.value)

    def counts(self):
        a, b, c, d = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        _chk(self._lib.lvba_visual_counts(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(nnz_valid=a.value, n_valid_tracks=b.value, n_blocks_env=c.value, n_pairs=d.value)

    def big_counts(self):
        """Landmarks with more than 128 observations, which take their own device passes: dict(n_big, n_big_obs, n_big_pairs)."""
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        _chk(self._lib.lvba_visual_big_counts(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(n_big=a.value, n_big_obs=b.value, n_big_pairs=c.value)

    def obs_residuals(self):
        """s_q = r0^2 + r1^2 [N_obs] of every observation at the current state (lvba_visual_obs_residuals), indexed as the
        obs_cam / obs_uv given at create: +inf where the camera-frame depth fails z > 1e-8, NaN for observations not in the
        problem (landmark without a plane or dropped, observation removed)."""
        out = np.empty(self.n_obs)
        _chk(self._lib.lvba_visual_obs_residuals(self._h, _p(out, C.c_double)))
        return out

    def remove_observations(self, mask, min_track_len=3):
        """Erase the observations where mask [N_obs] is true, then drop the landmarks left with fewer than min_track_len
        observations (lvba_visual_remove_observations); returns (observations left, landmarks left)."""
        m = np.ascontiguousarray(np.asarray(mask, bool), np.uint8)
        if m.shape != (self.n_obs,):
            raise ValueError(f"mask has shape {m.shape}, expected ({self.n_obs},)")
        a, b = C.c_int64(), C.c_int64()
        _chk(self._lib.lvba_visual_remove_observations(self._h, _p(m, C.c_uint8), C.c_int32(min_track_len), C.byref(a), C.byref(b)))
        return a.value, b.value

    def remove_outliers(self, max_err_px, min_track_len=3):
        """Remove every observation whose reprojection error is not <= max_err_px, then the landmarks left with fewer than
        min_track_len observations (lvba_visual_remove_outliers); returns the boolean mask [N_obs] of the observations this
        call took out, and the number of landmarks it dropped."""
        out = np.zeros(self.n_obs, np.uint8)
        a, b = C.c_int64(), C.c_int64()
        _chk(self._lib.lvba_visual_remove_outliers(self._h, C.c_double(max_err_px), C.c_int32(min_track_len), _p(out, C.c_uint8),
                                                   C.byref(a), C.byref(b)))
        return out.astype(bool), b.value


# ------------------------------------------------------------------ B3: adaptive voxel map
def voxel_default_opts():
    o = VoxelOpts()
    load_library().lvba_voxel_default_opts(C.byref(o))
    return o


class VoxelMap:
    """Device-resident adaptive voxel map (cut_voxel + recut + tras_opt, bavoxel.hpp:799-836, 420-474).
    scans: list of (n_i, 3) float32 body-frame clouds (or one (N, stride) float32 array with scan_ptr); poses (W, 12)."""

    def __init__(self, scans, poses, voxel_size=1.0, eigen_ratio=None, layer_limit=2, min_points=15, device=-1,
                 scan_ptr=None, win_ptr=None):
        lib = load_library()
        self._lib = lib
        ps = _f64(poses)
        if scan_ptr is None:
            W = len(scans)
            sp = np.zeros(W + 1, np.int64)
            sp[1:] = np.cumsum([len(s) for s in scans])
            xyz = (np.concatenate([np.asarray(s, np.float32).reshape(-1, 3) for s in scans]) if W else np.zeros((0, 3), np.float32))
        else:
            sp = np.ascontiguousarray(scan_ptr, np.int64); W = len(sp) - 1
            xyz = np.asarray(scans, np.float32)
        xyz = np.ascontiguousarray(xyz, np.float32)
        stride = xyz.shape[1] if xyz.ndim == 2 else 3
        o = voxel_default_opts()
        o.voxel_size = float(voxel_size); o.layer_limit = int(layer_limit); o.min_points = int(min_points); o.device = int(device)
        if eigen_ratio is not None:
            for k in range(4):
                o.eigen_ratio[k] = float(eigen_ratio[k])
        self._h = C.c_void_p()
        s = VoxelSummary()
        self.win_ptr = None if win_ptr is None else np.ascontiguousarray(win_ptr, np.int32)
        if self.win_ptr is None:
            _chk(lib.lvba_voxel_map_create(C.c_int32(W), _p(sp, C.c_int64), _p(xyz, C.c_float), C.c_int32(stride),
                                           _p(ps, C.c_double), C.byref(o), C.byref(self._h), C.byref(s)))
        else:       # one independent map per window of scans (runWindowBA)
            _chk(lib.lvba_voxel_map_create_windows(C.c_int32(len(self.win_ptr) - 1), _p(self.win_ptr, C.c_int32), _p(sp, C.c_int64),
                                                   _p(xyz, C.c_float), C.c_int32(stride), _p(ps, C.c_double), C.byref(o),
                                                   C.byref(self._h), C.byref(s)))
        self.summary = s.as_dict()

    def close(self):
        if self._h:
            self._lib.lvba_voxel_map_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def export(self):
        """dict: vox_ptr, pose_idx, clusters (arguments of lidar_lm) + key, path, centre, normal, eigenvalues per voxel."""
        V, nnz = self.summary["n_voxels"], self.summary["nnz"]
        o = dict(vox_ptr=np.zeros(V + 1, np.int64), pose_idx=np.zeros(nnz, np.int32), clusters=np.zeros((nnz, 10)),
                 key=np.zeros((V, 3), np.int64), path=np.zeros((V, 3), np.int8), centre=np.zeros((V, 3)),
                 normal=np.zeros((V, 3)), eigenvalues=np.zeros((V, 3)))
        _chk(self._lib.lvba_voxel_map_export(self._h, _p(o["vox_ptr"], C.c_int64), _p(o["pose_idx"], C.c_int32),
                                             _p(o["clusters"], C.c_double), _p(o["key"], C.c_int64), _p(o["path"], C.c_int8),
                                             _p(o["centre"], C.c_double), _p(o["normal"], C.c_double),
                                             _p(o["eigenvalues"], C.c_double)))
        return o

    def lidar_lm(self, poses, min_voxels_per_pose=0, opts=None, pose_fixed=None):
        """tras_opt + BALM2::damping_iter on the map's voxels without the clusters leaving the device.  pose_fixed: boolean
        mask [W] of constant poses, or None.  Returns (poses, summary dict)."""
        ps = _f64(poses).copy()
        opts, mask = _with_pose_fixed(opts, pose_fixed, ps.shape[0])
        s = Summary()
        _chk(self._lib.lvba_voxel_map_lidar_lm(self._h, _p(ps, C.c_double), C.c_int32(min_voxels_per_pose),
                                               C.byref(opts) if opts is not None else None, C.byref(s)))
        return ps, s.as_dict()

    def windows(self):
        """Window index of every voxel (windowed maps)."""
        w = np.zeros(self.summary["n_voxels"], np.int32)
        n = C.c_int32()
        _chk(self._lib.lvba_voxel_map_windows(self._h, C.byref(n), _p(w, C.c_int32)))
        return w

    def lidar_lm_batch(self, poses, min_voxels_per_pose=3, opts=None, pose_fixed=None):
        """runWindowBA's window stage from a windowed map.  pose_fixed: boolean mask over the concatenated poses, or None.
        Returns (poses, [per-window summary], total)."""
        ps = _f64(poses).copy()
        opts, mask = _with_pose_fixed(opts, pose_fixed, ps.shape[0])
        nw = len(self.win_ptr) - 1
        sums = (Summary * max(nw, 1))()
        tot = Summary()
        _chk(self._lib.lvba_voxel_map_lidar_lm_batch(self._h, _p(ps, C.c_double), C.c_int32(min_voxels_per_pose),
                                                     C.byref(opts) if opts is not None else None, sums, C.byref(tot)))
        return ps, [sums[i].as_dict() for i in range(nw)], tot.as_dict()

    def lidar_problem(self, poses):
        """Device-resident LidarProblem of the map's voxels (lvba_voxel_map_lidar_create)."""
        ps = _f64(poses)
        h = C.c_void_p()
        _chk(self._lib.lvba_voxel_map_lidar_create(self._h, _p(ps, C.c_double), C.byref(h)))
        return LidarProblem._from_handle(h, ps.shape[0], self.summary["n_voxels"])

    def lookup(self, X):
        """recompute_local_planes (lvba_system.cpp:1529-1566): (n, 4) plane (n, d) per world point, zeros when none."""
        X = _f64(X).reshape(-1, 3)
        out = np.zeros((len(X), 4))
        _chk(self._lib.lvba_voxel_map_lookup(self._h, C.c_int64(len(X)), _p(X, C.c_double), _p(out, C.c_double)))
        return out


# ------------------------------------------------------------------ B4: depth rendering
class DepthGrid:
    """Device-resident grid of world points (buildGridMapFromOptimized, lvba_system.cpp:1266-1338) that renders depth
    images (generateDepthWithVoxel, :835-919).  scans: list of (n_i, 3) float32 clouds or one (N, stride) array + scan_ptr."""

    def __init__(self, scans, poses, frame_ts, voxel_size=0.5, device=-1, scan_ptr=None):
        lib = load_library()
        self._lib = lib
        ps = _f64(poses); ts = _f64(frame_ts)
        if scan_ptr is None:
            F = len(scans)
            sp = np.zeros(F + 1, np.int64)
            sp[1:] = np.cumsum([len(s) for s in scans])
            xyz = (np.concatenate([np.asarray(s, np.float32).reshape(-1, 3) for s in scans]) if F else np.zeros((0, 3), np.float32))
        else:
            sp = np.ascontiguousarray(scan_ptr, np.int64); F = len(sp) - 1
            xyz = np.asarray(scans, np.float32)
        xyz = np.ascontiguousarray(xyz, np.float32)
        stride = xyz.shape[1] if xyz.ndim == 2 else 3
        self._h = C.c_void_p()
        s = DepthSummary()
        _chk(lib.lvba_depth_grid_create(C.c_int32(F), _p(sp, C.c_int64), _p(xyz, C.c_float), C.c_int32(stride), _p(ps, C.c_double),
                                        _p(ts, C.c_double), C.c_double(voxel_size), C.c_int32(device), C.byref(self._h), C.byref(s)))
        self.summary = s.as_dict()

    def close(self):
        if self._h:
            self._lib.lvba_depth_grid_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def render(self, cams, image_ts, intr, width, height, half_window=0.5):
        """cams (M, 12) = Rcw row-major, tcw.  Returns ((M, height, width) float32, summary dict)."""
        cams = _f64(cams).reshape(-1, 12); its = _f64(image_ts); it = _f64(intr)
        M = len(cams)
        out = np.zeros((M, height, width), np.float32)
        s = DepthSummary()
        _chk(self._lib.lvba_depth_render(self._h, C.c_int32(M), _p(cams, C.c_double), _p(its, C.c_double), C.c_double(half_window),
                                         _p(it, C.c_double), C.c_int32(width), C.c_int32(height), _p(out, C.c_float), C.byref(s)))
        return out, s.as_dict()


    def backproject(self, cams, image_ts, intr, width, height, kp_ptr, kp_uv, half_window=0.5):
        """Depth-fused 3-D candidates (lvba_system.cpp:1020-1038) of every keypoint; images never leave the device.
        Returns (Xw (n, 3), valid (n,) uint8, summary dict)."""
        cams = _f64(cams).reshape(-1, 12); its = _f64(image_ts); it = _f64(intr)
        kp = np.ascontiguousarray(kp_ptr, np.int64); uv = np.ascontiguousarray(kp_uv, np.float32).reshape(-1, 2)
        Xw = np.zeros((len(uv), 3)); valid = np.zeros(len(uv), np.uint8)
        s = DepthSummary()
        _chk(self._lib.lvba_depth_backproject(self._h, C.c_int32(len(cams)), _p(cams, C.c_double), _p(its, C.c_double), C.c_double(half_window),
                                              _p(it, C.c_double), C.c_int32(width), C.c_int32(height), _p(kp, C.c_int64), _p(uv, C.c_float),
                                              _p(Xw, C.c_double), _p(valid, C.c_uint8), C.byref(s)))
        return Xw, valid, s.as_dict()


# ------------------------------------------------------------------ B8: coloured LiDAR map
class ColorizeSummary(C.Structure):
    _fields_ = [(k, C.c_int64) for k in ("n_points", "n_images", "n_listed", "n_projections", "n_landed", "n_survivors", "n_out")] + \
               [("ms_device", C.c_double), ("ms_total", C.c_double)] + \
               [(k, C.c_int64) for k in ("kernel_launches", "h2d_bytes", "d2h_bytes", "peak_device_bytes")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Colorizer:
    """The coloured LiDAR map of VisualizeOptComparison (lvba_system.cpp:1932-2143) on the device: scans uploaded once, then one
    begin() .. add_images() .. finish() per pose set (the optimised poses, then the poses from before the optimisation)."""

    def __init__(self, scans, frame_ts, device=-1, scan_ptr=None):
        lib = load_library()
        self._lib = lib
        ts = _f64(frame_ts)
        if scan_ptr is None:
            F = len(scans)
            sp = np.zeros(F + 1, np.int64)
            sp[1:] = np.cumsum([len(s) for s in scans])
            xyz = (np.concatenate([np.asarray(s, np.float32).reshape(-1, 3) for s in scans]) if F else np.zeros((0, 3), np.float32))
        else:
            sp = np.ascontiguousarray(scan_ptr, np.int64); F = len(sp) - 1
            xyz = np.asarray(scans, np.float32)
        xyz = np.ascontiguousarray(xyz, np.float32)
        stride = xyz.shape[1] if xyz.ndim == 2 else 3
        self.F = F
        self._h = C.c_void_p()
        _chk(lib.lvba_colorizer_create(C.c_int32(F), _p(sp, C.c_int64), _p(xyz, C.c_float), C.c_int32(stride), _p(ts, C.c_double),
                                       C.c_int32(device), C.byref(self._h)))

    def close(self):
        if self._h:
            self._lib.lvba_colorizer_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def begin(self, frame_poses, leaf, half_window=0.5):
        ps = _f64(frame_poses).reshape(-1, 12)
        _chk(self._lib.lvba_colorizer_begin(self._h, _p(ps, C.c_double), C.c_double(half_window), C.c_double(leaf)))

    def add_images(self, image_ts, cams, intr, width, height, rgb=None):
        """cams (n, 12) = Rcw row-major, tcw; rgb (n, height, width, 3) uint8 in R, G, B order or None (grey).
        Returns listed (n,) uint8: 1 where the image has LiDAR in its window."""
        cams = _f64(cams).reshape(-1, 12); its = _f64(image_ts); it = _f64(intr)
        n = len(cams)
        listed = np.zeros(n, np.uint8)
        img = None
        if rgb is not None:
            img = np.ascontiguousarray(rgb, np.uint8)
            if img.shape != (n, height, width, 3):
                raise ValueError(f"rgb has shape {img.shape}, expected {(n, height, width, 3)}")
        _chk(self._lib.lvba_colorizer_add_images(self._h, C.c_int32(n), _p(its, C.c_double), _p(cams, C.c_double), _p(it, C.c_double),
                                                 C.c_int32(width), C.c_int32(height), _p(img, C.c_uint8) if img is not None else None,
                                                 _p(listed, C.c_uint8)))
        return listed

    def finish(self):
        """Returns (xyz (n, 3) float32, rgb (n, 3) uint8, summary dict)."""
        n = C.c_int64(); s = ColorizeSummary()
        _chk(self._lib.lvba_colorizer_finish(self._h, C.byref(n), C.byref(s)))
        xyz = np.zeros((n.value, 3), np.float32); rgb = np.zeros((n.value, 3), np.uint8)
        _chk(self._lib.lvba_colorizer_export(self._h, _p(xyz, C.c_float), _p(rgb, C.c_uint8)))
        return xyz, rgb, s.as_dict()

    def run(self, frame_poses, image_ts, cams, intr, width, height, rgb=None, leaf=0.01, half_window=0.5, batch=None):
        """One pose set end to end; `batch` images per add_images call (None: all at once).  Returns (xyz, rgb, listed, summary)."""
        self.begin(frame_poses, leaf, half_window)
        cams = _f64(cams).reshape(-1, 12); its = _f64(image_ts)
        n = len(cams); step = n if not batch else int(batch)
        listed = [np.zeros(0, np.uint8)]
        for k0 in range(0, n, max(step, 1)):
            sl = slice(k0, k0 + step)
            listed.append(self.add_images(its[sl], cams[sl], intr, width, height, None if rgb is None else rgb[sl]))
        xyz, col, s = self.finish()
        return xyz, col, np.concatenate(listed), s


# ------------------------------------------------------------------ B5: per-track numerics of the track fusion
def _track_args(obs_ptr, obs_cam, obs_uv, cams, intr):
    return (np.ascontiguousarray(obs_ptr, np.int64), np.ascontiguousarray(obs_cam, np.int32), np.ascontiguousarray(obs_uv, np.float32).reshape(-1, 2),
            _f64(cams).reshape(-1, 12), _f64(intr))


def tracks_triangulate(obs_ptr, obs_cam, obs_uv, cams, intr, device=-1):
    """TriangulateTrackDLT (lvba_system.cpp:52-111) of every track.  Returns (Xw (T, 3), mean_reproj, count, ok)."""
    op, oc, uv, cm, it = _track_args(obs_ptr, obs_cam, obs_uv, cams, intr)
    T = len(op) - 1
    Xw = np.zeros((T, 3)); mean = np.zeros(T); cnt = np.zeros(T, np.int32); ok = np.zeros(T, np.uint8)
    _chk(load_library().lvba_tracks_triangulate(C.c_int64(T), _p(op, C.c_int64), _p(oc, C.c_int32), _p(uv, C.c_float), C.c_int32(len(cm)),
                                                _p(cm, C.c_double), _p(it, C.c_double), C.c_int32(device), _p(Xw, C.c_double),
                                                _p(mean, C.c_double), _p(cnt, C.c_int32), _p(ok, C.c_uint8)))
    return Xw, mean, cnt, ok


def tracks_mean_reproj(obs_ptr, obs_cam, obs_uv, cams, intr, Xw, min_count, device=-1):
    """ComputeMeanReproj (lvba_system.cpp:8-50) of one 3-D point per track.  Returns (mean_reproj, count, ok)."""
    op, oc, uv, cm, it = _track_args(obs_ptr, obs_cam, obs_uv, cams, intr)
    T = len(op) - 1
    X = _f64(Xw).reshape(-1, 3); mean = np.zeros(T); cnt = np.zeros(T, np.int32); ok = np.zeros(T, np.uint8)
    _chk(load_library().lvba_tracks_mean_reproj(C.c_int64(T), _p(op, C.c_int64), _p(oc, C.c_int32), _p(uv, C.c_float), C.c_int32(len(cm)),
                                                _p(cm, C.c_double), _p(it, C.c_double), C.c_int32(device), _p(X, C.c_double),
                                                C.c_int32(min_count), _p(mean, C.c_double), _p(cnt, C.c_int32), _p(ok, C.c_uint8)))
    return mean, cnt, ok


# ------------------------------------------------------------------ B6: anchor clouds
class FuseOpts(C.Structure):
    _fields_ = [("obser_thr", C.c_int32), ("min_view_angle_deg", C.c_double), ("reproj_mean_thr_px", C.c_double),
                ("depth_gate_m", C.c_double), ("device", C.c_int32), ("map_order", C.c_int32)]


FUSE_ORDER_ASCENDING, FUSE_ORDER_LIBSTDCXX = 0, 1


class FuseSummary(C.Structure):
    _fields_ = [(k, C.c_int64) for k in ("n_keypoints", "n_components", "n_candidates", "n_tracks", "n_depth_selected", "n_tri_selected",
                                         "n_rounds", "n_attempts", "n_obs", "n_inliers", "kernel_launches")] + [("ms_total", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def tracks_fuse(kp_ptr, kp_uv, matches, cams, intr, kp_Xw, kp_valid, obser_thr=3, min_view_angle_deg=8.0, reproj_thr=3.0, depth_gate=0.12, device=-1,
                map_order=None):
    """lvba_tracks_fuse_create + export (boundary B7: BuildTracksAndFuse3D).  matches: (m, 4) int (img_a, kp_a, img_b, kp_b) in the
    reference's visiting order.  map_order: None = the library's default (FUSE_ORDER_LIBSTDCXX: the container order of a g++ build of the reference),
    or FUSE_ORDER_ASCENDING (library independent).  Returns dict(obs_ptr, img, kp, inlier, Xw, source, mean, summary)."""
    lib = load_library()
    kp_ptr = np.ascontiguousarray(kp_ptr, np.int64); uv = np.ascontiguousarray(kp_uv, np.float32)
    m = np.ascontiguousarray(matches, np.int32).reshape(-1, 4)
    cols = [np.ascontiguousarray(m[:, q]) for q in range(4)]
    cams = _f64(cams); intr = _f64(intr); X = _f64(kp_Xw); va = np.ascontiguousarray(kp_valid, np.uint8)
    o = FuseOpts(); lib.lvba_fuse_default_opts(C.byref(o))
    o.obser_thr = obser_thr; o.min_view_angle_deg = min_view_angle_deg; o.reproj_mean_thr_px = reproj_thr; o.depth_gate_m = depth_gate; o.device = device
    if map_order is not None:
        o.map_order = map_order
    h = C.c_void_p(); s = FuseSummary()
    _chk(lib.lvba_tracks_fuse_create(C.c_int32(len(kp_ptr) - 1), _p(kp_ptr, C.c_int64), _p(uv, C.c_float), C.c_int64(len(m)),
                                     _p(cols[0], C.c_int32), _p(cols[1], C.c_int32), _p(cols[2], C.c_int32), _p(cols[3], C.c_int32),
                                     _p(cams, C.c_double), _p(intr, C.c_double), _p(X, C.c_double), _p(va, C.c_uint8), C.byref(o),
                                     C.byref(h), C.byref(s)))
    try:
        n, no = s.n_tracks, s.n_obs
        obs_ptr = np.zeros(n + 1, np.int64); img = np.zeros(no, np.int32); kp = np.zeros(no, np.int32); inl = np.zeros(no, np.uint8)
        Xw = np.zeros((n, 3)); src = np.zeros(n, np.uint8); mean = np.zeros(n)
        _chk(lib.lvba_tracks_fuse_export(h, _p(obs_ptr, C.c_int64), _p(img, C.c_int32), _p(kp, C.c_int32), _p(inl, C.c_uint8),
                                         _p(Xw, C.c_double), _p(src, C.c_uint8), _p(mean, C.c_double)))
    finally:
        lib.lvba_tracks_fuse_destroy(h)
    return dict(obs_ptr=obs_ptr, img=img, kp=kp, inlier=inl, Xw=Xw, source=src, mean=mean, summary=s.as_dict())


def anchor_clouds(scans, rel_poses, win_ptr, leaf=0.1, device=-1):
    """Tail of runWindowBA's window loop (lvba_system.cpp:284-301): returns [one (n_w, 3) float32 cloud per window]."""
    lib = load_library()
    S = len(scans)
    sp = np.zeros(S + 1, np.int64)
    sp[1:] = np.cumsum([len(s) for s in scans])
    xyz = np.ascontiguousarray(np.concatenate([np.asarray(s, np.float32).reshape(-1, 3) for s in scans]) if S else np.zeros((0, 3)), np.float32)
    wp = np.ascontiguousarray(win_ptr, np.int32); rl = _f64(rel_poses)
    h = C.c_void_p(); n = C.c_int64()
    _chk(lib.lvba_anchor_clouds_create(C.c_int32(len(wp) - 1), _p(wp, C.c_int32), _p(sp, C.c_int64), _p(xyz, C.c_float), C.c_int32(3),
                                       _p(rl, C.c_double), C.c_double(leaf), C.c_int32(device), C.byref(h), C.byref(n)))
    cp = np.zeros(len(wp), np.int64); out = np.zeros((n.value, 3), np.float32)
    try:
        _chk(lib.lvba_anchor_clouds_export(h, _p(cp, C.c_int64), _p(out, C.c_float), None))
    finally:
        lib.lvba_anchor_clouds_destroy(h)
    return [out[cp[w]:cp[w + 1]] for w in range(len(wp) - 1)]


# ------------------------------------------------------------------ multi-GPU
def comm_unique_id():
    buf = (C.c_ubyte * 128)(); _chk(load_library().lvba_comm_unique_id(buf)); return bytes(buf)


def comm_init(n_ranks, rank, uid, device):
    buf = (C.c_ubyte * 128).from_buffer_copy(uid) if uid is not None else None
    _chk(load_library().lvba_comm_init(C.c_int32(n_ranks), C.c_int32(rank), buf, C.c_int32(device)))


def comm_bytes_sent():
    lib = load_library()
    lib.lvba_comm_bytes_sent.restype = C.c_int64
    return int(lib.lvba_comm_bytes_sent())


def comm_destroy():
    _chk(load_library().lvba_comm_destroy())
