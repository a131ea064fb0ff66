/*
 * lvba_b200.h — C ABI of the H100-native (sm_90a) LiDAR-visual bundle-adjustment hot path.
 *
 * This is the drop-in boundary for the two solver call sites of xuankuzcr/Global-LVBA
 * (SURVEY.md §8b).  The reference has no FFI of its own: both call sites are plain C++
 * inside one translation unit, so every entry point below cites the reference code it
 * replaces.  All buffers are HOST pointers owned by the caller; the library copies in
 * at call time, keeps its own device memory, writes results back before returning and
 * retains no caller pointer.  Nothing throws across this boundary: every function
 * returns LVBA_OK (0) or a negative lvba_status, and on error in/out buffers are left
 * untouched.  There is no CPU fallback: without a CUDA device every compute entry
 * point returns LVBA_ERR_NO_DEVICE.
 *
 * Conventions shared with the reference:
 *   pose           12 doubles: R (3x3 row-major, body->world) then p      IMUST.R/.p   include/BALM/tools.hpp:147-153
 *   cluster        10 doubles: Pxx Pxy Pxz Pyy Pyz Pzz vx vy vz N          PointCluster include/BALM/tools.hpp:407-424
 *   tangent order  (dphi, dp) per pose, R <- R*Exp(dphi), p <- p + dp      include/BALM/bavoxel.hpp:722-727
 *   quaternion     {w,x,y,z} (memory order of qs[k])                      src/lvba_system.cpp:1513-1516
 *   intr[8]        fx fy cx cy k1 k2 p1 p2 (Brown-Conrady)                 include/utils.hpp:53-58
 */
#ifndef LVBA_B200_H
#define LVBA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LVBA_B200_VERSION 100   /* 0.1.0 */

typedef enum lvba_status {
  LVBA_OK = 0,
  LVBA_ERR_INVALID_ARG = -1,   /* null pointer, negative size, index out of range, non-monotone CSR */
  LVBA_ERR_NO_DEVICE = -2,     /* no CUDA device / driver: the product path has no CPU fallback */
  LVBA_ERR_CUDA = -3,          /* a CUDA runtime call failed; see lvba_last_error() */
  LVBA_ERR_UNSUPPORTED = -4,   /* problem shape outside what this build handles */
  LVBA_ERR_NUMERIC = -5,       /* non-finite step / zero pivot and no recovery possible */
  LVBA_ERR_COMM = -6,          /* NCCL not loadable or a collective failed */
  LVBA_ERR_NOMEM = -7
} lvba_status;

/* ---- path A options: BALM2::damping_iter constants, include/BALM/bavoxel.hpp:664,686,760 */
typedef struct lvba_lidar_opts {
  double u0;           /* 0.01  initial damping            (bavoxel.hpp:664) */
  double v0;           /* 2.0   initial damping growth     (bavoxel.hpp:664) */
  int32_t max_iter;    /* 10                               (bavoxel.hpp:686) */
  double rel_tol;      /* 1e-6  |r1-r2|/r1 stop            (bavoxel.hpp:760); <0 disables the test */
  int32_t device;      /* CUDA device ordinal; -1 = current */
  int32_t verbose;     /* 1: print one line per LM iteration to stderr */
  int32_t deterministic; /* 0; 1: every device sum in a fixed order, so that identical inputs give bit-identical
                          * results on every run and in every process on the same GPU model and library build.
                          * Costs device memory for one record per summed contribution (allocated when a call or
                          * lvba_lidar_reset_lm first asks for the mode) and build / solve time.  One GPU only: with an
                          * active communicator (lvba_comm_init) the call returns LVBA_ERR_UNSUPPORTED. */
  /* Constant poses (ceres::Problem::SetParameterBlockConstant applied to damping_iter, e.g. the first scan as the gauge, or
   * the scans of a map already optimised): NULL (the default) or W bytes, nonzero = pose held constant; for the batched
   * calls W covers the concatenated poses.  A constant pose gets no row in the pose system (the free poses get rows in
   * ascending pose order, see lvba_lidar_rows) and comes back bit-identical.  Every voxel still enters the cost through all
   * of its slots, constant ones included, and the AVG_THR divisor stays V.  D = diag(H) of the free rows.  With no free
   * pose (in a batch: no free pose in a window) there is nothing to solve: the residual is evaluated once, the summary has
   * 0 iterations, 0 builds, cost_first = cost_last and LVBA_TERM_FUNCTION_TOL (a window that min_voxels_per_pose skips is
   * still LVBA_TERM_SKIPPED).  Read by lvba_lidar_lm, lvba_lidar_lm_batch, lvba_voxel_map_lidar_lm and
   * lvba_voxel_map_lidar_lm_batch, which plan their problem with it, and by lvba_lidar_reset_lm (a new handle has none):
   * a reset whose mask differs from the handle's current one re-plans the rows, the envelope, the solver and the build's
   * tables before it returns (the clusters stay on the device).  If that re-plan fails, the reset returns the error and
   * the handle keeps its previous constant poses with deterministic mode off (reset again to turn it on); should restoring
   * the previous plan fail as well, every later call on the handle but lvba_lidar_destroy and the pose copies returns
   * LVBA_ERR_INVALID_ARG.  An all-zero mask is the same as NULL; any nonzero entry with an active communicator is
   * LVBA_ERR_UNSUPPORTED.  The library keeps no copy of the pointer. */
  const uint8_t* pose_fixed;
} lvba_lidar_opts;

/* ---- path B robust losses: the ceres::LossFunction of a residual block (src/lvba_system.cpp:1585-1586, :1630, :1639).
 *      A block with squared whitened norm s = |r|^2 (the 2-vector of a reprojection, r_p^2 of a plane) costs 1/2 rho(s);
 *      with scale a, b = a^2:
 *        LVBA_LOSS_HUBER   s <= b: rho = s;  else rho = 2 a sqrt(s) - b, rho' = max(DBL_MIN, a / sqrt(s))   (ceres::HuberLoss)
 *        LVBA_LOSS_CAUCHY  rho = b log(1 + s / b), rho' = max(DBL_MIN, 1 / (1 + s / b))                    (ceres::CauchyLoss)
 *      Both have rho'' <= 0 everywhere, so Ceres' Corrector only scales the residual and the Jacobian by sqrt(rho') (no
 *      second-order term); losses whose rho'' can be positive are not offered.  The loss acts on the whitened residual:
 *      Huber 1.0 on the reprojection is 1 sigma_px, Huber 0.1 on the plane is 0.1 sigma_plane.  The loss is applied per
 *      residual block, before any sum; it has not been run on more than one GPU. */
typedef enum lvba_loss_kind {
  LVBA_LOSS_NONE = 0,
  LVBA_LOSS_HUBER = 1,
  LVBA_LOSS_CAUCHY = 2
} lvba_loss_kind;

/* ---- path B options: the ceres::Solver::Options in force at src/lvba_system.cpp:1572-1576
 *      (ceres-solver 2.1.0 defaults everywhere else, SURVEY.md Q10) */
typedef struct lvba_visual_opts {
  int32_t max_iter;              /* 50      options.max_num_iterations (:1573) */
  /* Refined intrinsics (a variable ceres::Problem parameter block of size 8 in every ReprojErrorWhitenedDistorted, held by a
   * SubsetManifold): 0 (the default: the intr given at create stay constant, and every pass is the one without this field) or a
   * mask whose bit i frees intr[i] of (fx fy cx cy k1 k2 p1 p2); LVBA_INTR_FOCAL, LVBA_INTR_PRINCIPAL, LVBA_INTR_DISTORTION
   * name the groups.  One block shared by every camera.  The free entries get their Jacobi scale, LM diagonal and gradient
   * entries; the reduced camera system gains a border that is solved with the camera system (one more solve per free entry)
   * and a k x k corner; the parameter tolerance takes ||x|| over all 8 entries and the step over the free ones (Ceres).  As
   * `deterministic`: a handle takes it from lvba_visual_reset_lm, and lvba_visual_step / _iterate / _cost then follow the handle's
   * current intrinsics (lvba_visual_get_intrinsics).  The sums of the block run in a fixed order whatever `deterministic` says.
   * Refused before any device work: bits above 7 (LVBA_ERR_INVALID_ARG), a nonzero mask with an active communicator
   * (LVBA_ERR_UNSUPPORTED), a nonzero mask in the one-shot lvba_visual_lm, whose intr is const (LVBA_ERR_INVALID_ARG). */
  uint32_t refine_intrinsics;     /* 0; in the padding after max_iter, so that the struct keeps its size and the offsets of
                                  * every other field.  A caller that fills the struct field by field instead of starting from
                                  * lvba_visual_default_opts must set it too: what the padding held before is read as a mask */
  double initial_radius;         /* 1e4  */
  double max_radius;             /* 1e16 */
  double min_radius;             /* 1e-32 */
  double min_lm_diagonal;        /* 1e-6 */
  double max_lm_diagonal;        /* 1e32 */
  double min_relative_decrease;  /* 1e-3 */
  double function_tolerance;     /* 1e-6;  <0 disables */
  double gradient_tolerance;     /* 1e-10; <0 disables */
  double parameter_tolerance;    /* 1e-8;  <0 disables */
  int32_t jacobi_scaling;        /* 1 */
  int32_t device;
  int32_t verbose;
  int32_t deterministic;         /* 0; 1: every device sum in a fixed order, as lvba_lidar_opts::deterministic (the
                                  * same bits on every run on one GPU model and library build, memory allocated when a
                                  * call or lvba_visual_reset_lm first asks for it, LVBA_ERR_UNSUPPORTED with an active
                                  * communicator) */
  /* Robust losses (lvba_loss_kind), as `deterministic`: the one-shot call takes them from its opts, a handle from
   * lvba_visual_reset_lm (lvba_visual_cost / lvba_visual_step then follow the handle; a new handle has none).  An unknown
   * kind, or a kind other than LVBA_LOSS_NONE whose scale is not finite and > 0, is LVBA_ERR_INVALID_ARG before any
   * device work.  The default scales are the reference's HuberLoss(1.0) / HuberLoss(0.1) (src/lvba_system.cpp:1585-1586). */
  int32_t reproj_loss;           /* LVBA_LOSS_NONE (loss_function = nullptr, :1630) */
  double reproj_loss_scale;      /* 1.0 */
  int32_t plane_loss;            /* LVBA_LOSS_NONE (:1639) */
  double plane_loss_scale;       /* 0.1 */
  /* The solver of the damped reduced camera system (Ceres' linear_solver_type), lvba_linear_solver:
   *   LVBA_LINEAR_DENSE_SCHUR (the default, the reference's choice, src/lvba_system.cpp:1574): the envelope LDL^T.
   *   LVBA_LINEAR_ITERATIVE_SCHUR: Ceres' ITERATIVE_SCHUR with the explicit Schur complement and the SCHUR_JACOBI
   *     preconditioner, restated from ceres-solver 2.1.0: conjugate gradients on (S + D) y = rhs preconditioned by the inverses
   *     of its 6x6 diagonal blocks, stopped by the inexact-Newton test on the quadratic model, zeta < eta after at least
   *     min_linear_iter iterations, or after max_linear_iter.  An inexact step is a different algorithm: iterates, iteration
   *     counts and the final cost differ from DENSE_SCHUR's within the forcing tolerance.  A solve that fails (a preconditioner
   *     pivot that is not finite and > 0, a rho, beta or alpha that is 0 or not finite) is an invalid LM step; one that stops
   *     on a non-positive curvature p.Ap or at the iteration limit gives its current step.  Its envelope need not be narrow:
   *     long tracks and loop closures, where the LDL^T fills the whole envelope, cost only their nonzero blocks per iteration.
   *     In deterministic mode the solve adds no records: given S it has the same bits on every run.
   * As `deterministic`: the one-shot call takes these from its opts, a handle from lvba_visual_reset_lm.  Refused before any
   * device work: an unknown solver, and for ITERATIVE_SCHUR an eta that is not finite and > 0, min_linear_iter < 0 or
   * max_linear_iter < max(1, min_linear_iter) (LVBA_ERR_INVALID_ARG); ITERATIVE_SCHUR with refine_intrinsics != 0 or an active
   * communicator (LVBA_ERR_UNSUPPORTED).  lvba_visual_linear_stats reports the iterations.  The four fields sit before
   * cam_fixed, which stays the last field. */
  int32_t linear_solver;         /* LVBA_LINEAR_DENSE_SCHUR */
  double eta;                    /* 0.1   Solver::Options::eta */
  int32_t min_linear_iter;       /* 0     min_linear_solver_iterations */
  int32_t max_linear_iter;       /* 500   max_linear_solver_iterations */
  /* The trust-region strategy (Ceres' trust_region_strategy_type), lvba_trust_region:
   *   LVBA_TR_LEVENBERG_MARQUARDT (the default, the reference's choice): initial_radius, max_radius, min_lm_diagonal and
   *     max_lm_diagonal as documented above.
   *   LVBA_TR_DOGLEG: Ceres' TRADITIONAL_DOGLEG, restated from ceres-solver 2.1.0 (csrc/visual_dogleg.h): the Gauss-Newton step
   *     (the DENSE_SCHUR solve with the small regularisation mu D^2), the Cauchy point and the dogleg between them inside the
   *     radius, which starts at initial_radius (max_radius does not bound it, as in Ceres).  A rejected step keeps the
   *     linearisation and only moves the dogleg point, so a rejected pass costs no build and no solve: hessian_builds is then
   *     lower than iterations.  lvba_visual_set_state, _reset_state, _set_intrinsics and an lvba_visual_step that recomputes the
   *     Jacobi scale change what that linearisation was taken at: the next pass linearises again.
   * As linear_solver: the one-shot call takes it from its opts, a handle from lvba_visual_reset_lm.  Refused before any device
   * work: an unknown value, and DOGLEG with ITERATIVE_SCHUR (LVBA_ERR_INVALID_ARG: the dogleg needs an exact Gauss-Newton step);
   * DOGLEG with refine_intrinsics != 0 or an active communicator (LVBA_ERR_UNSUPPORTED).  lvba_visual_dogleg_state reports the
   * state.  Sits before cam_fixed, which stays the last field. */
  int32_t trust_region_strategy; /* LVBA_TR_LEVENBERG_MARQUARDT */
  /* Constant cameras (ceres::Problem::SetParameterBlockConstant, which the reference calls on camera 0 at
   * src/lvba_system.cpp:1582-1583): NULL (the default) or M bytes, nonzero = camera held constant.  The constant cameras are
   * fixed_cam and every camera c with cam_fixed[c] != 0; they get no row in the reduced camera system and come back
   * bit-identical.  Their observations still enter their landmarks' blocks and every cost, which covers all residual blocks;
   * Jacobi scaling, the LM diagonal and the gradient and parameter tolerances cover the free parameters only (Ceres).  With
   * every camera constant only the landmarks move: lvba_visual_structure reports n_active = 0 and no blocks, lvba_visual_step
   * writes cam_step as zeros and the landmark step of the eliminated point blocks alone.  Landmarks are never constant.
   * As `deterministic`: the one-shot call plans its problem with the mask; a handle takes it from lvba_visual_reset_lm (a new
   * handle has none), and a reset whose mask differs from the handle's current one re-plans the rows, the landmark layout
   * and the build's tables before it returns (observations and state stay on the device).  If that re-plan fails, the reset
   * returns the error and the handle keeps its previous constant cameras with deterministic mode off (reset again to turn it
   * on); should restoring the previous plan fail as well, every later call on the handle but lvba_visual_destroy and the state
   * copies returns LVBA_ERR_INVALID_ARG.  An all-zero mask is the same as
   * NULL; any nonzero entry with an active communicator is LVBA_ERR_UNSUPPORTED.  The library keeps no copy of the pointer. */
  const uint8_t* cam_fixed;
} lvba_visual_opts;

typedef enum lvba_linear_solver {
  LVBA_LINEAR_DENSE_SCHUR = 0,
  LVBA_LINEAR_ITERATIVE_SCHUR = 1
} lvba_linear_solver;

typedef enum lvba_trust_region {
  LVBA_TR_LEVENBERG_MARQUARDT = 0,
  LVBA_TR_DOGLEG = 1              /* Ceres' TRADITIONAL_DOGLEG */
} lvba_trust_region;

/* the step of the last dogleg pass (lvba_visual_dogleg_state) */
typedef enum lvba_dogleg_case {
  LVBA_DOGLEG_NONE = 0,           /* no step since the last reset */
  LVBA_DOGLEG_GAUSS_NEWTON = 1,   /* the Gauss-Newton step lies inside the radius */
  LVBA_DOGLEG_CAUCHY = 2,         /* the gradient step cut at the radius */
  LVBA_DOGLEG_INTERPOLATED = 3    /* the point between the Cauchy point and the Gauss-Newton step on the radius */
} lvba_dogleg_case;

#define LVBA_INTR_FOCAL      0x03u   /* fx fy */
#define LVBA_INTR_PRINCIPAL  0x0Cu   /* cx cy */
#define LVBA_INTR_DISTORTION 0xF0u   /* k1 k2 p1 p2 */

typedef enum lvba_termination {
  LVBA_TERM_MAX_ITER = 0,
  LVBA_TERM_FUNCTION_TOL = 1,   /* A: bavoxel.hpp:760 ; B: Ceres function tolerance */
  LVBA_TERM_PARAMETER_TOL = 2,
  LVBA_TERM_GRADIENT_TOL = 3,
  LVBA_TERM_RADIUS = 4,
  LVBA_TERM_INVALID_STEPS = 5,
  LVBA_TERM_SKIPPED = 6         /* window BA: fewer than min_voxels_per_pose * W voxels, poses untouched */
} lvba_termination;

typedef struct lvba_summary {
  int32_t iterations;        /* LM loop passes executed (accepted + rejected) */
  int32_t accepted;          /* accepted steps */
  int32_t hessian_builds;    /* passes that rebuilt H/g (A) or J/S (B) */
  int32_t termination;       /* lvba_termination */
  double cost_first;         /* A: sum(lambda0)/V at entry ; B: 1/2 sum rho(|r|^2) over the residual blocks at entry
                              *    (rho(s) = s without a loss: 1/2 sum r^2) */
  double cost_last;          /* same quantity at the returned state */
  double damping_last;       /* A: u ; B: trust-region radius */
  double ms_total;           /* wall time inside the call (host clock) */
  double ms_setup;           /* host symbolic analysis + H2D upload */
  double ms_build;           /* CUDA-event time in Hessian / Jacobian+Schur build kernels */
  double ms_solve;           /* CUDA-event time in factorisation + substitution */
  double ms_residual;        /* CUDA-event time in residual-only passes + retraction */
  int64_t kernel_launches;   /* launches of this library's own kernels during the call */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
} lvba_summary;

/* ---- misc ------------------------------------------------------------------------------ */
int         lvba_version(void);
int         lvba_device_count(void);          /* 0 when no usable GPU; never fails */
const char* lvba_status_string(int status);
const char* lvba_last_error(void);            /* thread-local detail of the last failure */
/* Device buffers of destroyed problems are cached for reuse by later calls (cudaMalloc/cudaFree cost
 * milliseconds each); this returns the cached memory to the driver. */
int         lvba_release_cached_memory(void);
void        lvba_lidar_default_opts(lvba_lidar_opts* o);
void        lvba_visual_default_opts(lvba_visual_opts* o);

/* ======================================================================================
 * B1  LiDAR LM — replaces  void BALM2::damping_iter(vector<IMUST>& x_stats, VOX_HESS& voxhess)
 *     include/BALM/bavoxel.hpp:662-767, called at src/lvba_system.cpp:264 and :386.
 *
 *   W          number of poses (BALM2::win_size)
 *   V          number of plane voxels (VOX_HESS::plvec_voxels.size())
 *   vox_ptr    [V+1] CSR offsets; voxel a owns slots vox_ptr[a]..vox_ptr[a+1]
 *   pose_idx   [nnz] pose index i of every slot with (*plvec_voxels[a])[i].N != 0, ascending inside a voxel
 *   clusters   [nnz*10] body-frame PointCluster of that slot
 *   poses      [W*12] in/out
 * ====================================================================================== */
int lvba_lidar_lm(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                  const double* clusters, double* poses, const lvba_lidar_opts* opts,
                  lvba_summary* summary);

/* B1 batched — every window of LvbaSystem::runWindowBA (src/lvba_system.cpp:232-302: consecutive windows of
 * `window_size` poses, one BALM2::damping_iter each, :264) in ONE call: one block-diagonal system, one CTA per
 * window in the factorisation, per-window u / v / accept-reject / stop test.  Results equal n_windows separate
 * lvba_lidar_lm calls.
 *   win_ptr    [n_windows+1] window w owns poses win_ptr[w] .. win_ptr[w+1]-1 of the concatenated `poses`
 *   pose_idx   indices into the concatenated pose array; every voxel lies inside ONE window
 *   min_voxels_per_pose   windows with fewer than this many voxels per pose are skipped and their poses left
 *              untouched (3 in the reference, :262-266); their summary carries LVBA_TERM_SKIPPED
 *   summaries  [n_windows] per-window LM summary (iterations, accepted, costs, damping, termination); may be NULL
 *   total      timing / traffic of the whole call; may be NULL
 * Windows of more than 31 poses return LVBA_ERR_UNSUPPORTED (solve those with lvba_lidar_lm). */
int lvba_lidar_lm_batch(int32_t n_windows, const int32_t* win_ptr, int64_t V, const int64_t* vox_ptr,
                        const int32_t* pose_idx, const double* clusters, double* poses,
                        int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                        lvba_summary* summaries, lvba_summary* total);
/* Device-resident handle for the same problem: lets a caller (bench, parity tests, a ROS
 * node that re-solves after outlier removal: lvba_lidar_remove_outliers) run single phases with inputs already in HBM. */
typedef struct lvba_lidar_problem lvba_lidar_problem;

int lvba_lidar_create(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                      const double* clusters, const double* poses, int32_t device,
                      lvba_lidar_problem** out);
int lvba_lidar_destroy(lvba_lidar_problem* p);
int lvba_lidar_set_poses(lvba_lidar_problem* p, const double* poses);     /* H2D, W*12 */
int lvba_lidar_get_poses(lvba_lidar_problem* p, double* poses);           /* D2H, W*12 */
/* VOX_HESS::acc_evaluate2 + divide_thread (bavoxel.hpp:68-174, 597-639) at the current poses:
 * builds H and g on the device, returns sum_v lambda0 (NOT divided by V). */
int lvba_lidar_build(lvba_lidar_problem* p, double* residual_sum);
/* VOX_HESS::evaluate_only_residual (bavoxel.hpp:176-203) at `poses` (host, W*12) or at the
 * current device poses when poses == NULL. */
int lvba_lidar_residual(lvba_lidar_problem* p, const double* poses, double* residual_sum);
/* (H + u*diag(H)) dx = -g  (bavoxel.hpp:692-710) over the free rows; dx [W*6] to host, zeros for constant poses. */
int lvba_lidar_solve(lvba_lidar_problem* p, double u, double* dx);
/* The rows of the pose system: n_rows free poses (W without lvba_lidar_opts::pose_fixed) and pose_of_row [n_rows], the
 * pose of every row, ascending (the identity without a mask).  Either pointer may be NULL. */
int lvba_lidar_rows(lvba_lidar_problem* p, int32_t* n_rows, int32_t* pose_of_row);
/* Block structure of the lower-triangular envelope that stores H over the rows: nblocks and per block (row, col). */
int lvba_lidar_structure(lvba_lidar_problem* p, int64_t* nblocks, int32_t* brow, int32_t* bcol);
/* Copy out g [n_rows*6] and the envelope blocks [nblocks*36, row-major 6x6, block (r,c) = H[6r.., 6c..]], by rows. */
int lvba_lidar_get_system(lvba_lidar_problem* p, double* g, double* blocks);
/* n LM passes of damping_iter starting from the handle's state (u, v, poses carried in the
 * handle; call lvba_lidar_reset_lm to restart).  Device-resident: no problem data crosses PCIe.  The reset also takes the
 * handle's constant poses (lvba_lidar_opts::pose_fixed), which build, solve, iterate and get_system then follow. */
int lvba_lidar_reset_lm(lvba_lidar_problem* p, const lvba_lidar_opts* opts);
/* restore the poses passed to lvba_lidar_create (device-to-device; nothing crosses PCIe) */
int lvba_lidar_reset_state(lvba_lidar_problem* p);
int lvba_lidar_iterate(lvba_lidar_problem* p, int32_t n_iter, lvba_summary* summary);
/* exact algorithmic byte / flop counters of SURVEY.md §8(d) for this problem instance (nnz: every slot; the blocks and
 * pose pairs: those of the row system) */
int lvba_lidar_counts(lvba_lidar_problem* p, int64_t* nnz, int64_t* n_blocks_env,
                      int64_t* n_blocks_nonzero, int64_t* n_pairs);

/* ---- voxel outlier removal: BALM2's own rule, which the reference carries commented out in include/BALM/bavoxel.hpp.
 * The three calls run on one GPU (an active communicator is LVBA_ERR_UNSUPPORTED) on a handle from lvba_lidar_create or
 * lvba_voxel_map_lidar_create.  The handle's voxel order is the caller's order minus the voxels removed so far.
 *
 * VOX_HESS::evaluate_residual (bavoxel.hpp:205-234): lambda0 of every voxel at `poses` (host, W*12), or at the current
 * device poses when NULL.  lambda0 [V] is in the handle's voxel order.  The values come from the arithmetic of
 * lvba_lidar_residual, whose sum they give up to summation order. */
int lvba_lidar_voxel_residuals(lvba_lidar_problem* p, const double* poses, double* lambda0);
/* plvec_voxels.erase for every voxel with remove[a] != 0 (remove [V], handle order).  Survivors keep their relative order
 * and are renumbered 0..n_left-1 (n_left may be NULL).  Afterwards the handle is planned as lvba_lidar_create on the kept
 * voxels with the current poses and the handle's constant poses would be: the AVG_THR divisor is the kept count, and counts,
 * structure, get_system and residual follow the kept voxels.  The poses and the poses lvba_lidar_reset_state restores stay as
 * they are; removal is one-way.  The LM state is reset as lvba_lidar_reset_lm with the handle's options would reset it
 * (deterministic mode stays on, its records set up again).  A NULL mask or one that removes every voxel is
 * LVBA_ERR_INVALID_ARG with nothing removed.  A failed re-plan (deterministic mode's record set-up included) keeps the
 * previous voxels with deterministic mode off and writes nothing to n_left, or, if restoring them fails too, leaves a handle
 * that refuses every call but destroy and the pose copies. */
int lvba_lidar_remove_voxels(lvba_lidar_problem* p, const uint8_t* remove, int64_t* n_left);
/* BALM2::remove_outlier(x_stats, voxhess, ratio) (bavoxel.hpp:650-660 with VOX_HESS::remove_residual :236-268) at the
 * current poses, then the re-plan of lvba_lidar_remove_voxels.  The rule is the reference's, in double, quirks included:
 *   thr = sorted(lambda0)[floor((1 - ratio) V) - 1],  reject_num = floor(ratio V);
 *   the voxels are walked in order, every voxel with lambda0 >= thr is erased, and the walk stops after the first KEPT voxel
 *   at which the count of erased voxels equals reject_num.
 * So it removes between reject_num and #{lambda0 >= thr} voxels, depending on where they sit: without ties that count is
 * ceil(ratio V) + 1 when ratio V is an integer and floor(ratio V) + 2 otherwise.  With ratio = 0 (reject_num = 0) the walk
 * can only stop at a first voxel that is kept: ratio = 0 removes nothing when the first voxel is below the maximum, and
 * every maximal voxel when it is not.  removed [V before the call] (may be NULL): 1 for every erased voxel;
 * n_removed (may be NULL).  LVBA_ERR_INVALID_ARG with the handle unchanged when ratio is not finite or outside [0, 1), when
 * floor((1 - ratio) V) < 1, when some lambda0 is not finite, or when the rule would erase every voxel. */
int lvba_lidar_remove_outliers(lvba_lidar_problem* p, double ratio, uint8_t* removed, int64_t* n_removed);

/* ======================================================================================
 * B2  visual LM — replaces the Ceres block of LvbaSystem::optimizeCameraPoses(),
 *     src/lvba_system.cpp:1571-1656 (problem build :1578-1640, ceres::Solve :1643,
 *     write-back :1651-1665).  Residual functors: include/utils.hpp:51-147.
 *
 *   M, T        cameras, landmarks
 *   q_wxyz      [M*4] in/out   qs[k]   (:1513-1516)
 *   t           [M*3] in/out   ts[k]
 *   X           [T*3] in/out   Xs[pi]  (:1521-1525); landmarks without a valid plane are left untouched
 *   plane_nd    [T*4] (n, d); n == 0 marks "no valid plane" => landmark and its observations are skipped (:1598-1603)
 *   obs_ptr     [T+1] CSR; obs_cam [nnz] camera of each inlier observation; obs_uv [nnz*2] float pixel (:1624-1625).
 *               A landmark may have any number of observations, and may see one camera more than once.
 *   fixed_cam   camera held constant (0 in the reference, :1582-1583); -1 = none.  lvba_visual_opts::cam_fixed adds any
 *               set of further constant cameras.
 * ====================================================================================== */
int lvba_visual_lm(int32_t M, int64_t T, double* q_wxyz, double* t, double* X,
                   const double* plane_nd, const int64_t* obs_ptr, const int32_t* obs_cam,
                   const float* obs_uv, const double intr[8], double sigma_px, double sigma_plane,
                   int32_t fixed_cam, const lvba_visual_opts* opts, lvba_summary* summary);

typedef struct lvba_visual_problem lvba_visual_problem;

int lvba_visual_create(int32_t M, int64_t T, const double* q_wxyz, const double* t, const double* X,
                       const double* plane_nd, const int64_t* obs_ptr, const int32_t* obs_cam,
                       const float* obs_uv, const double intr[8], double sigma_px, double sigma_plane,
                       int32_t fixed_cam, int32_t device, lvba_visual_problem** out);
int lvba_visual_destroy(lvba_visual_problem* p);
int lvba_visual_set_state(lvba_visual_problem* p, const double* q_wxyz, const double* t, const double* X);
int lvba_visual_get_state(lvba_visual_problem* p, double* q_wxyz, double* t, double* X);
/* 1/2 sum rho(|r|^2) over all residual blocks at the current device state, with the losses of the last
 * lvba_visual_reset_lm (1/2 sum r^2 without) */
int lvba_visual_cost(lvba_visual_problem* p, double* cost);
/* One linearisation + Schur elimination + reduced solve + back-substitution at the current state
 * with the given trust-region radius; writes the (unscaled) tangent step: cam_step [M*6] (zeros for
 * inactive cameras), pt_step [T*3] (zeros for skipped landmarks), and the model cost change. */
int lvba_visual_step(lvba_visual_problem* p, double radius, int32_t jacobi_scaling, int32_t recompute_scale,
                     double* cam_step, double* pt_step, double* model_cost_change, double* cost);
/* Reduced camera system of the last lvba_visual_step: block structure + values + rhs (for parity tests). */
int lvba_visual_structure(lvba_visual_problem* p, int32_t* n_active, int32_t* cam_of_row /* [n_active] */,
                          int64_t* nblocks, int32_t* brow, int32_t* bcol);
/* After a pass of ITERATIVE_SCHUR on the matrix-free product (lvba_visual_schur_product) there is no S: a call with blocks !=
 * NULL returns LVBA_ERR_UNSUPPORTED and writes nothing; with blocks == NULL it writes rhs as after any pass. */
int lvba_visual_get_system(lvba_visual_problem* p, double* rhs /* [n_active*6] */, double* blocks /* [nblocks*36] */);
int lvba_visual_reset_lm(lvba_visual_problem* p, const lvba_visual_opts* opts);
/* restore q, t, X and the intrinsics passed to lvba_visual_create (device-to-device) */
int lvba_visual_reset_state(lvba_visual_problem* p);
/* The handle's current intrinsics (fx fy cx cy k1 k2 p1 p2): those given at create until an accepted step of a refining
 * solve (lvba_visual_opts::refine_intrinsics) or lvba_visual_set_intrinsics changes them.  Set refuses a non-finite entry
 * with LVBA_ERR_INVALID_ARG and leaves the handle unchanged. */
int lvba_visual_get_intrinsics(lvba_visual_problem* p, double intr[8]);
int lvba_visual_set_intrinsics(lvba_visual_problem* p, const double intr[8]);
/* The intrinsics block of the last lvba_visual_step (for parity tests, beside lvba_visual_get_system), k = the number of free
 * entries, in ascending order of their index.  border [n_active*6*k]: B, row 6 r + a of camera row r, column j of free entry
 * j; corner [k*k]: C = sum J_k^T J_k - sum E V^-1 E^T, without the LM diagonal (as the blocks of lvba_visual_get_system);
 * rhs [k]: -(g_k - sum E V^-1 g_X), these three with the Jacobi scaling applied, as the camera system; step [8]: the change of
 * the intrinsics, zeros in the held entries.  Any pointer may be NULL.  Until the first lvba_visual_step after create,
 * lvba_visual_reset_lm, lvba_visual_reset_state or a removal, only k and step (all zeros) are written. */
int lvba_visual_get_intrinsics_system(lvba_visual_problem* p, int32_t* k, double* border, double* corner, double* rhs,
                                      double* step);
/* The conjugate gradients of LVBA_LINEAR_ITERATIVE_SCHUR: cg_iters_total, the iterations of every solve since the last
 * lvba_visual_reset_lm or removal; cg_iters_last and term_last, the iteration count and termination of the last solve
 * (0 SUCCESS, 1 NO_CONVERGENCE, 2 FAILURE).  All zero until a solve has run.  Any pointer may be NULL. */
int lvba_visual_linear_stats(lvba_visual_problem* p, int64_t* cg_iters_total, int32_t* cg_iters_last, int32_t* term_last);
/* The product ITERATIVE_SCHUR runs its conjugate gradients on, chosen for the handle's plan from its structure at create and at
 * every re-plan (a new cam_fixed, a removal), whatever the linear solver: *matrix_free = 0 for the explicit reduced camera
 * system S in envelope storage, 1 for the matrix-free product through the Jacobian blocks, which never forms S.  The
 * matrix-free product costs O(observations) per product where the explicit S costs O(sum of squared track lengths) to build:
 * long tracks and loop closures take it.  The two are the same algorithm (the same CG on the same S + D, with sums in another
 * order); DENSE_SCHUR always builds S. */
int lvba_visual_schur_product(lvba_visual_problem* p, int32_t* matrix_free);
/* y = (S + D) x [n_active*6] for the damped reduced camera system of the last lvba_visual_step or iteration, through the product
 * its conjugate gradients used (for parity tests).  LVBA_ERR_INVALID_ARG unless that pass ran ITERATIVE_SCHUR: before any pass,
 * after lvba_visual_reset_lm or a re-plan, and under DENSE_SCHUR. */
int lvba_visual_apply_system(lvba_visual_problem* p, const double* x, double* y);
/* The dogleg state of a handle whose last lvba_visual_reset_lm chose LVBA_TR_DOGLEG (else LVBA_ERR_INVALID_ARG): the radius
 * Delta and mu as the next pass will use them; alpha, |g| and |GN| of the current linearisation and the lvba_dogleg_case of the
 * last step (all 0 before the first pass); the passes since the last reset that reused a linearisation.  In the D-scaled
 * space of csrc/visual_dogleg.h.  Any pointer may be NULL.  A reset, a removal and a cam_fixed re-plan start it again. */
int lvba_visual_dogleg_state(lvba_visual_problem* p, double* radius, double* mu, double* alpha, double* grad_norm,
                             double* gn_norm, int32_t* step_case, int64_t* reused);
int lvba_visual_iterate(lvba_visual_problem* p, int32_t n_iter, lvba_summary* summary);
int lvba_visual_counts(lvba_visual_problem* p, int64_t* nnz_valid, int64_t* n_valid_tracks,
                       int64_t* n_blocks_env, int64_t* n_pairs);
/* Landmarks with more than 128 observations (this rank's, with a valid plane) do not fit the build tiles and take their own
 * device passes: their number, their observations and their ordered observation pairs (sum of K (K - 1)). */
int lvba_visual_big_counts(lvba_visual_problem* p, int64_t* n_big, int64_t* n_big_obs, int64_t* n_big_pairs);

/* ---- per-observation reprojection errors and reprojection-outlier removal: the solve, filter, solve-again loop of a Ceres
 * bundle adjustment (COLMAP: FilterPoints3DWithLargeReprojectionError, then another BA).  The three calls run on one GPU (an
 * active communicator is LVBA_ERR_UNSUPPORTED: a rank holds only its own landmarks).
 *
 * Observations are named by the caller's arrays: entry q of the [N_obs] arrays below, N_obs = obs_ptr[T] as given to
 * lvba_visual_create, is obs_cam[q] / obs_uv[q].  No index map is needed, and removals compose.  An observation is IN THE
 * PROBLEM while its landmark has a valid plane and has not been dropped, and it has not been removed.  For each one
 * s_q = r0^2 + r1^2, the squared whitened reprojection norm that lvba_visual_cost sums before any loss, from the same device
 * function.
 *
 * The rule, in double, at the current device state:
 *   1. tau = (max_err_px / sigma_px)^2, once on the host (DBL_MAX should it overflow);
 *   2. an observation in the problem is removed iff !(z > 1e-8 && s_q <= tau), z its camera-frame depth: the cut-off case,
 *      NaN and s_q > tau are removed, s_q == tau is kept;
 *   3. a landmark left with fewer than min_track_len observations in the problem is DROPPED: its remaining observations are
 *      removed too, its plane term leaves the cost, and its X stays as it is, as for a landmark without a plane.
 *
 * After a removal the handle has the plan lvba_visual_create would make from the kept observations (dropped landmarks without
 * a plane), with the handle's fixed_cam, cam_fixed, losses and deterministic flag: rows, landmark layout, tiles, big
 * landmarks, tables, counts and big_counts.  A camera that loses every observation loses its row (lvba_visual_step writes
 * zeros for it); a landmark may move from the big path to the tiles (129 -> 128 observations).  The state and the restore
 * point of lvba_visual_reset_state do not change: removal is one-way.  The LM state is reset as lvba_visual_reset_lm with the
 * handle's options would reset it (radius, a fresh Jacobi scale; deterministic mode's records are set up again before the call
 * returns).  A later cam_fixed change re-plans from the kept observations.
 * Refused with LVBA_ERR_INVALID_ARG and the handle unchanged: a NULL mask, min_track_len < 1, max_err_px not finite or not > 0,
 * a removal that would leave no observation in the problem.  A failed re-plan restores the previous plan with deterministic
 * mode off (or, if that fails too, leaves a handle that refuses every call but destroy and the state copies); then nothing is
 * removed and no output is written. */

/* s_q of every observation in the problem at the current state into sq_res [N_obs]: +inf where z > 1e-8 fails (the residual
 * and the cost are 0 there), NaN for every observation not in the problem.  1/2 the sum of the finite entries plus the plane
 * terms is lvba_visual_cost without losses, up to summation order. */
int lvba_visual_obs_residuals(lvba_visual_problem* p, double* sq_res);
/* Removes every observation with remove[q] != 0 (remove [N_obs]; flags on observations already out of the problem are
 * ignored), then step 3 of the rule, then the re-plan.  n_obs_left, n_tracks_left (may be NULL): observations and landmarks
 * left in the problem. */
int lvba_visual_remove_observations(lvba_visual_problem* p, const uint8_t* remove, int32_t min_track_len, int64_t* n_obs_left,
                                    int64_t* n_tracks_left);
/* The rule above, then the re-plan of lvba_visual_remove_observations.  removed [N_obs] (may be NULL): 1 for every observation
 * this call took out, those of dropped landmarks included; n_removed_obs, n_removed_tracks (may be NULL): their numbers and the
 * number of dropped landmarks. */
int lvba_visual_remove_outliers(lvba_visual_problem* p, double max_err_px, int32_t min_track_len, uint8_t* removed,
                                int64_t* n_removed_obs, int64_t* n_removed_tracks);

/* ======================================================================================
 * B3  adaptive voxel map (set-up stage) — replaces the cut_voxel / recut / tras_opt sequence in front of every
 *     LiDAR solve and the plane lookup in front of the visual solve:
 *       cut_voxel per scan       include/BALM/bavoxel.hpp:799-836   src/lvba_system.cpp:248-251, 366-369, 1499-1502
 *       recut + tras_opt         include/BALM/bavoxel.hpp:420-474   src/lvba_system.cpp:255-258, 374-377, 1504-1506
 *       recompute_local_planes   src/lvba_system.cpp:1529-1566 with findCorrespondPoint, bavoxel.hpp:320-333
 *     The map is built on the device from the raw scans (sort-based, no hash table, no per-point allocation) and
 *     stays there; the plane voxels come back in exactly the layout lvba_lidar_lm takes.
 *
 *   W                  number of scans = poses of the window (win_size)
 *   scan_ptr           [W+1] CSR offsets into the point array; scan j owns points scan_ptr[j] .. scan_ptr[j+1]-1
 *   xyz                body-frame points, x y z as float at the start of every record
 *   xyz_stride_floats  record size in floats: 3 for packed xyz, 12 for an array of pcl::PointXYZINormal (48 B)
 *   poses              [W*12] pose of every scan (x_buf / anchor_poses)
 *   Voxel order: ascending (root key x, y, z), then octant path — the reference's unordered_map order is unspecified.
 *   A non-finite point, or one more than 2^30 root voxels from the origin, is LVBA_ERR_INVALID_ARG (the reference's
 *   float -> int64 cast is undefined there).
 * ====================================================================================== */
typedef struct lvba_voxel_opts {
  double voxel_size;       /* root voxel edge: stage1_root_voxel_size_ / stage2_root_voxel_size_ (lvba_system.cpp:344-345) */
  float eigen_ratio[4];    /* eigen_ratio_array per layer, bavoxel.hpp:17-22 (set_eigen_ratio_array, lvba_system.cpp:360) */
  int32_t layer_limit;     /* 2   bavoxel.hpp:13; 0..2 supported */
  int32_t min_points;      /* 15  min_ps, bavoxel.hpp:24 */
  int32_t device;          /* CUDA device ordinal; -1 = current */
} lvba_voxel_opts;

typedef struct lvba_voxel_summary {
  int64_t n_points;
  int64_t n_voxels;        /* plane voxels seen from >= 2 poses (VOX_HESS::plvec_voxels.size()) */
  int64_t nnz;             /* (voxel, pose) clusters */
  int64_t n_nodes[3];      /* octree nodes per layer that hold points (layers never reached are 0) */
  double ms_total;         /* wall time inside lvba_voxel_map_create (host clock) */
  double ms_upload;        /* validation + packing + H2D enqueue */
  double ms_device;        /* CUDA-event time of the build passes */
  int64_t kernel_launches; /* launches of this library's own kernels (the cub sorts / scans are not counted) */
  int64_t h2d_bytes;
} lvba_voxel_summary;

typedef struct lvba_voxel_map lvba_voxel_map;

void lvba_voxel_default_opts(lvba_voxel_opts* o);
int lvba_voxel_map_create(int32_t W, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats,
                          const double* poses, const lvba_voxel_opts* opts, lvba_voxel_map** out,
                          lvba_voxel_summary* summary /* may be NULL */);
/* One INDEPENDENT map per window of consecutive scans, all built together — the surf_map that runWindowBA creates, recuts
 * and deletes once per window (src/lvba_system.cpp:232-258).  win_ptr [n_windows+1]: window w owns scans
 * win_ptr[w] .. win_ptr[w+1]-1; W = win_ptr[n_windows].  Voxels never merge across windows, pose indices are those of the
 * concatenated scans, voxels are ordered by (window, key, path): the export is the input of lvba_lidar_lm_batch as it
 * stands.  lvba_voxel_map_lookup is not defined on a windowed map (LVBA_ERR_UNSUPPORTED). */
int lvba_voxel_map_create_windows(int32_t n_windows, const int32_t* win_ptr, const int64_t* scan_ptr, const float* xyz,
                                  int32_t xyz_stride_floats, const double* poses, const lvba_voxel_opts* opts,
                                  lvba_voxel_map** out, lvba_voxel_summary* summary /* may be NULL */);
/* n_windows (0 for a single map) and, when vox_window != NULL, the window of every voxel [V]. */
int lvba_voxel_map_windows(lvba_voxel_map* m, int32_t* n_windows, int32_t* vox_window);
int lvba_voxel_map_summary(const lvba_voxel_map* m, lvba_voxel_summary* summary);
/* Copy out the plane voxels (sizes from the summary).  Any pointer may be NULL.
 *   vox_ptr [V+1], pose_idx [nnz], clusters [nnz*10]   the arguments of lvba_lidar_lm / lvba_lidar_create
 *   root_key [V*3] int64 voxel key; path [V*3] int8 (layer, octant1 or -1, octant2 or -1)
 *   centre, normal, eigenvalues [V*3]   judge_eigen's center / direct / value_vector (bavoxel.hpp:346-349); the sign
 *   of `normal` is not defined (nor is it by Eigen's solver) */
int lvba_voxel_map_export(lvba_voxel_map* m, int64_t* vox_ptr, int32_t* pose_idx, double* clusters, int64_t* root_key,
                          int8_t* path, double* centre, double* normal, double* eigenvalues);
/* recompute_local_planes: for n world points X [n*3] the plane (n, d) [n*4] of the PLANE node each one falls in,
 * zeros when there is none — the plane_nd argument of lvba_visual_lm. */
int lvba_voxel_map_lookup(lvba_voxel_map* m, int64_t n, const double* X, double* plane_nd);
/* tras_opt straight into B1: the map's plane voxels as a device-resident LiDAR problem (handle API above).  The cluster
 * records never leave HBM; only the CSR index arrays (12 B per cluster) visit the host for the symbolic analysis.
 * poses [W*12]: the linearisation point (normally the poses the map was built with). */
int lvba_voxel_map_lidar_create(lvba_voxel_map* m, const double* poses, lvba_lidar_problem** out);
/* ... and solved: cut_voxel + recut (the map) -> tras_opt + BALM2::damping_iter (this call), poses [W*12] in/out.
 * Fewer than min_voxels_per_pose * W voxels (the caller-side rule of src/lvba_system.cpp:262-266; pass 0 for
 * runLidarBA, which has none) or an empty map: LVBA_OK, LVBA_TERM_SKIPPED, poses untouched. */
int lvba_voxel_map_lidar_lm(lvba_voxel_map* m, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                            lvba_summary* summary);
/* The window stage of runWindowBA (src/lvba_system.cpp:232-266) from a windowed map: tras_opt + damping_iter of EVERY window
 * in one batched solve (see lvba_lidar_lm_batch for summaries / total / the skip rule), clusters never leaving the device. */
int lvba_voxel_map_lidar_lm_batch(lvba_voxel_map* m, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                                  lvba_summary* summaries, lvba_summary* total);
int lvba_voxel_map_destroy(lvba_voxel_map* m);

/* ======================================================================================
 * B6  anchor clouds — replaces the tail of the window loop of runWindowBA, src/lvba_system.cpp:284-301 (and its twin at
 *     :1474-1491): every scan of a window transformed into the window's anchor frame (pl_transform, include/BALM/tools.hpp:385-395:
 *     the result is stored back as float), merged, and down-sampled with down_sampling_voxel2 (tools.hpp:301-359): per voxel of
 *     edge `leaf` the ORIGINAL point closest to the voxel centre, the first in cloud order among equally close ones.
 *   win_ptr [n_windows+1] over scans; scan_ptr / xyz / xyz_stride_floats as for B3
 *   rel_poses [S*12]   pose of every scan in its anchor frame: rel.R = anchor.R^T x.R, rel.p = anchor.R^T (x.p - anchor.p) (:286-289)
 *   leaf               anchor_leaf_size_ (window_ba/anchor_leaf_size, 0.1); < 0.001 returns the transformed points unsampled (:303)
 *   export: cloud_ptr [n_windows+1], xyz [n_points*3] float — the anchor_clouds; points of a window are ordered by voxel key
 *   (the reference's unordered_map order is unspecified)
 * ====================================================================================== */
typedef struct lvba_anchor_clouds lvba_anchor_clouds;
int lvba_anchor_clouds_create(int32_t n_windows, const int32_t* win_ptr, const int64_t* scan_ptr, const float* xyz,
                              int32_t xyz_stride_floats, const double* rel_poses, double leaf, int32_t device,
                              lvba_anchor_clouds** out, int64_t* n_points_out);
int lvba_anchor_clouds_export(lvba_anchor_clouds* a, int64_t* cloud_ptr, float* xyz, double* ms_device /* may be NULL */);
int lvba_anchor_clouds_destroy(lvba_anchor_clouds* a);

/* ======================================================================================
 * B4  depth rendering — replaces the world point grid and the per-image z-buffer in front of the track fusion:
 *       buildGridMapFromOptimized   src/lvba_system.cpp:1266-1338   (0.5 m voxels of ALL world points, per-frame voxel sets,
 *                                                                    per image the voxels of the frames within +-0.5 s)
 *       generateDepthWithVoxel      src/lvba_system.cpp:835-919     (project every point of those voxels, (int) pixel,
 *                                                                    `if (d == 0 || Z < d) d = (float)Z`)
 *     The z-buffer is float(min Z) whatever the visiting order, so the images are reproducible bit for bit.
 *
 *   n_frames, scan_ptr, xyz, xyz_stride_floats, poses   as for B3: pl_fulls_ / x_buf_ (dataset_io_)
 *   frame_ts     [n_frames] LiDAR frame timestamps x_buf_[i].t, ascending (the reference binary-searches them, :1318-1319)
 *   voxel_size   0.5 in the reference (:1277)
 *   cams         [n_images*12] Rcw (row-major) then tcw per image: Rcw_all_optimized_ / tcw_all_optimized_ (:861-864)
 *   image_ts     [n_images] image timestamps; NaN = an image name that does not parse (:1309-1314) -> empty image
 *   half_window  0.5 s in the reference (:1299)
 *   intr         fx fy cx cy k1 k2 p1 p2
 *   depth        [n_images * height * width] float, row-major per image (cv::Mat CV_32FC1), 0 = no point
 * ====================================================================================== */
typedef struct lvba_depth_summary {
  int64_t n_points, n_voxels;
  int64_t n_pairs;          /* distinct (frame, voxel) pairs = sum of the per_frame_voxels set sizes */
  double ms_total, ms_upload, ms_device;
  int64_t kernel_launches, h2d_bytes, d2h_bytes;
  int64_t work_pairs;       /* render: (image, frame-in-window, voxel) triples examined */
  int64_t work_chunks;      /* render: 64-point chunks projected (every voxel of a window once) */
} lvba_depth_summary;

typedef struct lvba_depth_grid lvba_depth_grid;

int lvba_depth_grid_create(int32_t n_frames, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats,
                           const double* poses, const double* frame_ts, double voxel_size, int32_t device,
                           lvba_depth_grid** out, lvba_depth_summary* summary /* may be NULL */);
int lvba_depth_render(lvba_depth_grid* g, int32_t n_images, const double* cams, const double* image_ts, double half_window,
                      const double intr[8], int32_t width, int32_t height, float* depth,
                      lvba_depth_summary* summary /* may be NULL */);
/* The depth-fused 3-D candidates of the track fusion — the loop at src/lvba_system.cpp:1020-1038 of BuildTracksAndFuse3D
 * (fetchDepthBilinear include/utils.hpp:246-275 -> backProjectPixelDepthDistorted :235-243 -> camToWorld :277-283) for
 * EVERY keypoint of every image; a pure function of (image, keypoint), so the caller indexes the result by
 * (component[t].first, component[t].second).  The depth images are rendered and sampled on the device and never copied out.
 *   kp_ptr  [n_images+1] CSR over images; kp_uv [n_kp*2] float pixel (all_keypoints_[im][kp].x / .y)
 *   Xw      [n_kp*3] out: points3d (zeros where invalid); valid [n_kp] out: valid_mask */
int lvba_depth_backproject(lvba_depth_grid* g, int32_t n_images, const double* cams, const double* image_ts, double half_window,
                           const double intr[8], int32_t width, int32_t height, const int64_t* kp_ptr, const float* kp_uv,
                           double* Xw, uint8_t* valid, lvba_depth_summary* summary /* may be NULL */);
int lvba_depth_grid_destroy(lvba_depth_grid* g);

/* ======================================================================================
 * B8  coloured LiDAR map — the numeric part of VisualizeOptComparison, src/lvba_system.cpp:1932-2143:
 *     per image (in the order given): the scans with |x_buf[idx].t - id| <= half_window (a linear scan over all frames, any
 *     timestamp order, :1973-1977), every point moved to the world as (float)(R p + t) (:1983-1990); an image whose window holds
 *     no point is not listed (:1993-1996, the skip precedes its images.txt line); a z-buffer in cloud order (scan, then point):
 *     projectWorldToPixel (include/utils.hpp:183-205), round() to the pixel, `if (zc + 1e-6f < zbuf) { zbuf = (float)zc; keep }`
 *     (:2037-2060, order dependent); the kept points in pixel order coloured from the image (:2051-2055, :2062-2069); after
 *     all images down_sampling_voxel2(merged, leaf) (include/BALM/tools.hpp:301-359; leaf < 0.001 keeps every point).
 *   create: the scans once (n_frames, scan_ptr, xyz, xyz_stride_floats as for B3; frame_ts [n_frames] = x_buf[i].t)
 *   begin:  one pose set: frame_poses [n_frames*12], half_window 0.5, leaf colmap_output/filter_size_points3D.  The two
 *           clouds of the reference pair poses and cameras as follows (:1983-1990, :1998-2001, :2041, :2079):
 *             after  (points3D.txt, colored_merged_after.pcd):  frame_poses = x_buf_,         cams = Rcw_all_optimized_ / tcw_all_optimized_
 *             before (colored_merged_before.pcd):               frame_poses = x_buf_before_,  cams = Rcw_all_ / tcw_all_
 *           With leaf >= 0.001 every FINITE world point of every scan — not only those in some image's window — must lie within
 *           2^30 leaf voxels of the origin, else LVBA_ERR_INVALID_ARG (the rule of B6); the voxel-key range is taken over them too.
 *           Non-finite pose or camera entries are LVBA_ERR_INVALID_ARG.  The reference would instead drop the points they touch
 *           (projectWorldToPixel's allFinite) and still list the image; this stage refuses such input rather than guess.
 *   add_images (any number of calls): image_ts [n], cams [n*12] Rcw row-major then tcw, intr fx fy cx cy k1 k2 p1 p2, the
 *           image size after any resize, rgb [n][height][width][3] in R, G, B order (NULL: every point (128, 128, 128)),
 *           listed [n] out: 1 when the image has LiDAR in its window.  The library cuts the images into device batches itself.
 *   finish: n_out; export: xyz [n_out*3] float, rgb [n_out*3], in ascending (kx, ky, kz) leaf-voxel order (x-major, signed)
 *           — the reference's unordered_map order is unspecified — or, with leaf < 0.001, in merged order.
 *   Device memory is bounded by the scans, the thinned table and one batch, not by the number of images.
 * ====================================================================================== */
typedef struct lvba_colorize_summary {
  int64_t n_points;          /* LiDAR points of the scans */
  int64_t n_images, n_listed;
  int64_t n_projections;     /* (image, window point) pairs projected */
  int64_t n_landed;          /* of those, inside their image */
  int64_t n_survivors;       /* z-buffer survivors of all images = size of the merged cloud before thinning */
  int64_t n_out;
  double ms_device, ms_total;
  int64_t kernel_launches, h2d_bytes, d2h_bytes;
  int64_t peak_device_bytes; /* the stage's own device buffers at their largest (sort scratch aside) */
} lvba_colorize_summary;

typedef struct lvba_colorizer lvba_colorizer;
int lvba_colorizer_create(int32_t n_frames, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats,
                          const double* frame_ts, int32_t device, lvba_colorizer** out);
int lvba_colorizer_begin(lvba_colorizer* c, const double* frame_poses, double half_window, double leaf);
int lvba_colorizer_add_images(lvba_colorizer* c, int32_t n_images, const double* image_ts, const double* cams, const double intr[8],
                              int32_t width, int32_t height, const uint8_t* rgb /* may be NULL */, uint8_t* listed);
int lvba_colorizer_finish(lvba_colorizer* c, int64_t* n_out, lvba_colorize_summary* summary /* may be NULL */);
int lvba_colorizer_export(lvba_colorizer* c, float* xyz, uint8_t* rgb);
int lvba_colorizer_destroy(lvba_colorizer* c);

/* ======================================================================================
 * B5  per-track numerics of the track fusion (BuildTracksAndFuse3D, src/lvba_system.cpp:921-1263), many tracks at once:
 *       TriangulateTrackDLT   src/lvba_system.cpp:52-111    lvba_tracks_triangulate
 *       ComputeMeanReproj     src/lvba_system.cpp:8-50      lvba_tracks_mean_reproj
 *     The caller keeps what is inherently sequential there — connected components over the match graph, one observation
 * per image, the greedy view-angle filter (its result depends on the iteration order of std::unordered_map) — and passes the
 * SELECTED observations of every track (`selected_ids`) as a CSR list.
 *   obs_ptr [n_tracks+1]; obs_cam [n_obs] image id of each selected observation (ids outside [0, n_cams) are skipped, :74-78);
 *   obs_uv [n_obs*2] float keypoint; cams [n_cams*12] Rcw row-major + tcw (Rcw_all_optimized_ / tcw_all_optimized_)
 *   triangulate: Xw [n_tracks*3], mean_reproj, count, ok (the function's bool) out; fewer than 4 observations / 8 rows -> ok = 0
 *   mean_reproj: Xw in (e.g. the depth-fused candidate), min_count = obser_thr_ (:1098) or 4 (:108)
 * ====================================================================================== */
int lvba_tracks_triangulate(int64_t n_tracks, const int64_t* obs_ptr, const int32_t* obs_cam, const float* obs_uv, int32_t n_cams,
                            const double* cams, const double intr[8], int32_t device, double* Xw, double* mean_reproj,
                            int32_t* count, uint8_t* ok);
int lvba_tracks_mean_reproj(int64_t n_tracks, const int64_t* obs_ptr, const int32_t* obs_cam, const float* obs_uv, int32_t n_cams,
                            const double* cams, const double intr[8], int32_t device, const double* Xw, int32_t min_count,
                            double* mean_reproj, int32_t* count, uint8_t* ok);

/* ======================================================================================
 * Boundary B7 (SURVEY.md 8f N3): track fusion — LvbaSystem::BuildTracksAndFuse3D
 * (reference src/lvba_system.cpp:921-1263) as one call.  In: the keypoints of all images
 * (CSR), the pairwise matches as four parallel arrays in the order the reference visits them
 * (image pairs (i < j) by ascending i then j, the matches of a pair in stored order), camera
 * poses [n_images][12] = Rcw row-major then tcw, intrinsics fx fy cx cy k1 k2 p1 p2, and the
 * depth-fused 3-D candidate of every keypoint with its validity flag (what
 * lvba_depth_backproject returns: the loop at :1020-1038).  Out: the tracks in the order the
 * reference appends them; Track::observations = the whole connected component in BFS order,
 * Track::inlier_indices as one flag per observation, Xw_fused, which candidate was chosen
 * (1 depth, 2 triangulation) and its mean reprojection error.  The (image, keypoint, inlier)
 * lists are the observation CSR of lvba_visual_lm once the inliers are kept (:1610-1617).
 * Where the reference iterates std::unordered_map<int,int> (unspecified order: the greedy
 * view-angle filter depends on it, and with it which tracks survive) the images of a component are
 * visited in the order GNU libstdc++'s container has after the reference's reserve() / insert calls
 * (map_order = LVBA_FUSE_ORDER_LIBSTDCXX, the default: what a g++ build of the reference does; with
 * it the stage reproduces the reference's own source track for track, tests/test_ref_system_pin.py,
 * tests/test_zzz_ref_gpu.py) or in ascending id (LVBA_FUSE_ORDER_ASCENDING: independent of any C++
 * library).
 * ====================================================================================== */
typedef struct lvba_fuse_opts {
  int32_t obser_thr;              /* minimum members / images / survivors (lvba_system.h:139: 3) */
  double min_view_angle_deg;      /* track_fusion/min_view_angle (8) */
  double reproj_mean_thr_px;      /* track_fusion/reproj_mean_thr (3) */
  double depth_gate_m;            /* distance to the anchor's depth point (0.12, :1050) */
  int32_t device;                 /* -1: current */
  int32_t map_order;              /* LVBA_FUSE_ORDER_*: visiting order of the three unordered_map loops (:1057, :1069, :1124) */
} lvba_fuse_opts;
#define LVBA_FUSE_ORDER_ASCENDING 0
#define LVBA_FUSE_ORDER_LIBSTDCXX 1
typedef struct lvba_fuse_summary {
  int64_t n_keypoints, n_components, n_candidates, n_tracks, n_depth_selected, n_tri_selected;
  int64_t n_rounds, n_attempts;   /* retries: a failed component is tried again from its next keypoint as BFS seed (:1199) */
  int64_t n_obs, n_inliers;       /* totals over the tracks: sizes of the export arrays */
  int64_t kernel_launches;
  double ms_total;
} lvba_fuse_summary;
typedef struct lvba_track_set lvba_track_set;
void lvba_fuse_default_opts(lvba_fuse_opts* o);
int lvba_tracks_fuse_create(int32_t n_images, const int64_t* kp_ptr /* [n_images+1] */, const float* kp_uv /* [n_kp][2] */,
                            int64_t n_matches, const int32_t* match_img_a, const int32_t* match_kp_a, const int32_t* match_img_b,
                            const int32_t* match_kp_b, const double* cams, const double intr[8], const double* kp_Xw /* [n_kp][3] */,
                            const uint8_t* kp_valid /* [n_kp] */, const lvba_fuse_opts* opts /* NULL: defaults */,
                            lvba_track_set** out, lvba_fuse_summary* summary /* may be NULL */);
int lvba_tracks_fuse_summary(const lvba_track_set* s, lvba_fuse_summary* summary);
/* arrays sized from the summary: obs_ptr [n_tracks+1], obs_* [n_obs], Xw [n_tracks][3], source / mean_reproj [n_tracks]; any but obs_ptr may be NULL */
int lvba_tracks_fuse_export(lvba_track_set* s, int64_t* obs_ptr, int32_t* obs_img, int32_t* obs_kp, uint8_t* obs_inlier, double* Xw,
                            uint8_t* source, double* mean_reproj);
int lvba_tracks_fuse_destroy(lvba_track_set* s);

/* ======================================================================================
 * The block LDL^T of the pose / camera system on its own (diagnostics, solver tests and the
 * solver line of bench.py).  Solves (A + diag(dadd)) x = rhs for a symmetric matrix of 6x6
 * blocks stored as a block envelope: row r keeps the blocks of columns first[r]..r
 * contiguously, row after row, each block row-major; first[] must be non-decreasing (what the
 * library builds from the voxel / track structure); only the lower triangle of the diagonal
 * blocks is read.  LDL^T without pivoting (A may be indefinite), as Eigen::SimplicialLDLT in
 * BALM2::damping_iter (reference include/BALM/bavoxel.hpp:695-710) and the DENSE_SCHUR
 * Cholesky of ceres::Solve (src/lvba_system.cpp:1573-1575).
 *   path  LVBA_SOLVE_AUTO: what lvba_lidar_lm / lvba_visual_lm pick for this structure;
 *         the other values pin one path and fail with LVBA_ERR_UNSUPPORTED if the structure
 *         does not allow it.  chunks: for LVBA_SOLVE_CHUNKED (0 = library default).
 *   reps  >= 1 solves; ms (may be NULL) = fastest of them, device time by CUDA events.
 *   info  (may be NULL) int32[4]: path taken, chunks, tree levels, kernel launches per solve.
 * ====================================================================================== */
#define LVBA_SOLVE_AUTO 0
#define LVBA_SOLVE_ONE_CTA 1        /* one register-window factorisation (columns of <= 30 blocks) */
#define LVBA_SOLVE_TWISTED 2        /* two-ended elimination on two SMs, joined at one separator */
#define LVBA_SOLVE_CHUNKED 3        /* substructured: chunk interiors + tree of separators, one CTA per node */
#define LVBA_SOLVE_SHARED_WINDOW 4  /* shared-memory window (columns of <= 320 blocks) */
#define LVBA_SOLVE_ANY_WIDTH 5      /* device-wide passes, any envelope */
int lvba_env_solve(int32_t n, const int32_t* first, const double* blocks, const double* dadd, const double* rhs,
                   double* x, int32_t path, int32_t chunks, int32_t reps, int32_t device, double* ms, int32_t* info);

/* ======================================================================================
 * Multi-GPU (one process per GPU).  The path shards by contiguous pose-block rows
 * (SURVEY.md §8e): voxel / track -> owner of its lowest pose / camera index.  Every rank
 * passes the FULL problem to *_create; after lvba_comm_init each rank keeps only its shard
 * of voxels / tracks on its GPU.  The pose / camera system is ROW-OWNED: the substructured
 * solver's chunks are the multi-GPU unit, a rank builds and factorises the rows of its own
 * chunks, only the <= band-width block rows a rank's voxels reach into its right neighbour's
 * range travel (ncclSend/ncclRecv), the ranks' separator complements meet in one
 * ncclAllGather (~0.8 MB per rank), the small top tree is solved redundantly and the update
 * is assembled by an all-reduce of 48 bytes per pose; g, the right-hand sides, diagonals
 * and the scalar costs (O(poses) data) use ncclAllReduce.  Structures the solver cannot
 * cut per rank fall back to an all-reduce of the full matrix.  NCCL is dlopen()ed
 * (libnccl.so.2) on first use.
 * ====================================================================================== */
#define LVBA_NCCL_ID_BYTES 128
int lvba_comm_unique_id(void* id_out /* LVBA_NCCL_ID_BYTES */);
/* Row ownership of a problem created after lvba_comm_init: this rank holds the block rows [row_begin, row_end) of H (pose rows)
 * / of the reduced camera system; *sharded = 1 when the system is row-owned and solved by the substructured solver with its
 * chunks spread over the ranks (only <= band-width boundary rows travel between neighbours, SURVEY.md 8(e)), 0 when every rank
 * holds the all-reduced full system (one GPU, or a structure that cannot be cut per rank).  lvba_*_get_system returns the
 * owned rows only when sharded. */
int lvba_lidar_owned_rows(lvba_lidar_problem* p, int32_t* row_begin, int32_t* row_end, int32_t* sharded);
int lvba_visual_owned_rows(lvba_visual_problem* p, int32_t* row_begin, int32_t* row_end, int32_t* sharded);
/* NCCL payload (bytes handed to send-type calls by this rank) since the previous call of this function */
int64_t lvba_comm_bytes_sent(void);
int lvba_comm_init(int32_t n_ranks, int32_t rank, const void* id /* LVBA_NCCL_ID_BYTES */, int32_t device);
int lvba_comm_destroy(void);
int lvba_comm_info(int32_t* n_ranks, int32_t* rank);
/* Host-only shard rule (no GPU needed; used by the gloo CPU tests): owner rank of a unit whose
 * lowest pose index is `min_pose` when `n_rows` pose-block rows are split over `n_ranks`. */
int32_t lvba_shard_owner(int32_t min_pose, int32_t n_rows, int32_t n_ranks);

#ifdef __cplusplus
}
#endif
#endif /* LVBA_B200_H */
