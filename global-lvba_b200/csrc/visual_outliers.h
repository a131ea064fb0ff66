// visual_outliers.h — per-observation reprojection errors and reprojection-outlier removal on the visual problem handle
// (lvba_visual_obs_residuals, lvba_visual_remove_observations, lvba_visual_remove_outliers): the solve, filter, solve-again
// loop of a Ceres bundle adjustment (COLMAP's FilterPoints3DWithLargeReprojectionError between two solves).
// Plain C++ with no CUDA: the rule and the compaction are item passes run by an execution policy (CudaExec of exec.cuh in the
// library, the host policy of tests/emu in the CPU tests), and the re-plan's host side (the kept landmarks and their CSR) is
// shared by visual_api.cuh and the CPU tests the same way.
//
// Observations are named by the caller's index q (obs_cam[q] / obs_uv[q] as given to lvba_visual_create).  Every local
// observation w of the handle carries it in obs_src[w].  An observation is in the problem while its landmark has a valid plane
// and has not been dropped, and it has not been removed.  The rule, in double:
//   keep_w     = !remove[obs_src[w]]                       (lvba_visual_remove_observations)
//              = s_w <= tau,  s_w = r0^2 + r1^2 (+inf where the depth fails z > 1e-8),  tau = (max_err_px / sigma_px)^2
//                                                          (lvba_visual_remove_outliers: NaN, +inf and s > tau are removed,
//                                                          s == tau is kept)
//   a landmark with fewer than min_track_len kept observations is dropped: its kept observations are removed too and its
//   plane term leaves the cost.
#pragma once
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "visual_plan.h"

namespace lvba {
namespace voutliers {

struct NanFillF {              // out[q] = NaN: every caller observation not in the problem
  double* out;
  LVBA_HD void operator()(int64_t q) const { out[q] = NAN; }
};

// The caller index of every local observation while nothing has been removed: the observations of local landmark k are those of
// the caller's landmark trk_id[k], in the caller's order.  One item per local landmark.
struct DeriveSrcF {
  const int* trk_id; const int* trk_ptr; const int64_t* caller_ptr; int64_t* src;
  LVBA_HD void operator()(int64_t k) const {
    const int64_t q0 = caller_ptr[trk_id[k]];
    for (int w = trk_ptr[k]; w < trk_ptr[k + 1]; ++w) src[w] = q0 + (w - trk_ptr[k]);
  }
};

// keep[w] (item w < nnz) by the caller's mask (remove != null) or by the threshold on s (sq, caller-indexed); keep[nnz] = 0, so
// that the exclusive scan of keep [nnz + 1] ends with the kept count.
struct KeepF {
  int64_t nnz; const int64_t* src; const uint8_t* remove; const double* sq; double tau; int32_t* keep;
  LVBA_HD void operator()(int64_t w) const {
    if (w == nnz) { keep[w] = 0; return; }
    keep[w] = remove ? (remove[src[w]] == 0) : (sq[src[w]] <= tau);
  }
};

// One item per local landmark k (and item Tv for the scan's end): its kept count; a landmark left with fewer than min_len is
// dropped and its observations' keep flags cleared.  kcnt[k]: the kept observations of k (0 when dropped), tkeep[k] = !dropped.
struct TrackF {
  int64_t Tv; const int* trk_ptr; int32_t min_len; int32_t* keep; int32_t* kcnt; int32_t* tkeep;
  LVBA_HD void operator()(int64_t k) const {
    if (k == Tv) { tkeep[k] = 0; return; }
    int32_t c = 0;
    for (int w = trk_ptr[k]; w < trk_ptr[k + 1]; ++w) c += keep[w];
    const bool drop = c < min_len;
    if (drop)
      for (int w = trk_ptr[k]; w < trk_ptr[k + 1]; ++w) keep[w] = 0;
    kcnt[k] = drop ? 0 : c;
    tkeep[k] = !drop;
  }
};

struct KeepBytesF {            // the keep flags as bytes, for the copy to the host
  const int32_t* keep; uint8_t* out;
  LVBA_HD void operator()(int64_t w) const { out[w] = (uint8_t)keep[w]; }
};

struct RemovedF {              // removed[obs_src[w]] = 1 for every observation this removal takes out (removed zeroed before)
  const int32_t* keep; const int64_t* src; uint8_t* removed;
  LVBA_HD void operator()(int64_t w) const { if (!keep[w]) removed[src[w]] = 1; }
};

// The kept observations' camera, pixel and caller index at their scanned positions (the local order, compacted).
struct CompactF {
  const int32_t* keep; const int32_t* pos; const int* cam; const float2* uv; const int64_t* src;
  int* cam_out; float2* uv_out; int64_t* src_out;
  LVBA_HD void operator()(int64_t w) const {
    if (!keep[w]) return;
    const int32_t p = pos[w];
    cam_out[p] = cam[w]; uv_out[p] = uv[w]; src_out[p] = src[w];
  }
};

// The caller indices of a new plan from its source landmarks (visual_plan's per-observation gather, for obs_src): one item per
// new local landmark k, source landmark src_trk[k] with observations src_obs[src_ptr[i] ..).
struct GatherSrcF {
  const int* src_trk; const int* trk_ptr; const long long* src_ptr; const int64_t* in; int64_t* out;
  LVBA_HD void operator()(int64_t k) const {
    const long long q0 = src_ptr[src_trk[k]];
    for (int w = trk_ptr[k]; w < trk_ptr[k + 1]; ++w) out[w] = in[q0 + (w - trk_ptr[k])];
  }
};

// The rule's buffers, in the policy's memory
template <class Ex>
struct RuleBufs {
  typename Ex::template Buf<int32_t> keep, pos, kcnt, tkeep, tpos;   // [nnz + 1] [nnz + 1] [Tv] [Tv + 1] [Tv + 1]
};

// keep [nnz] and kcnt [Tv] by the rule above over the local CSR (trk_ptr [Tv + 1], obs_src [nnz]), pos [nnz + 1] the exclusive
// scan of keep; *n_obs_left, *n_trk_left: the observations and landmarks kept.  remove (caller mask) or sq / tau as KeepF.
// Returns a policy status.
template <class Ex>
int keep_rule(Ex& ex, int64_t nnz, int64_t Tv, const int* trk_ptr, const int64_t* obs_src, const uint8_t* remove, const double* sq,
              double tau, int32_t min_len, RuleBufs<Ex>& B, int64_t* n_obs_left, int64_t* n_trk_left) {
  LVBA_PLAN_TRY(B.keep.alloc((size_t)nnz + 1));
  LVBA_PLAN_TRY(B.pos.alloc((size_t)nnz + 1));
  LVBA_PLAN_TRY(B.kcnt.alloc((size_t)std::max<int64_t>(Tv, 1)));
  LVBA_PLAN_TRY(B.tkeep.alloc((size_t)Tv + 1));
  LVBA_PLAN_TRY(B.tpos.alloc((size_t)Tv + 1));
  LVBA_PLAN_TRY(ex.for_each(nnz + 1, KeepF{nnz, obs_src, remove, sq, tau, B.keep.p}));
  LVBA_PLAN_TRY(ex.for_each(Tv + 1, TrackF{Tv, trk_ptr, min_len, B.keep.p, B.kcnt.p, B.tkeep.p}));
  LVBA_PLAN_TRY(ex.exclusive_scan(B.keep.p, B.pos.p, nnz + 1));
  LVBA_PLAN_TRY(ex.exclusive_scan(B.tkeep.p, B.tpos.p, Tv + 1));
  int32_t a = 0, b = 0;
  LVBA_PLAN_TRY(ex.fetch(&a, B.pos.p + nnz, 1));
  LVBA_PLAN_TRY(ex.fetch(&b, B.tpos.p + Tv, 1));
  *n_obs_left = a;
  *n_trk_left = b;
  return 0;
}

// ---------------------------------------------------------------- the re-plan's source
// The source landmarks of a re-plan from the handle's own arrays (visual_replan): the local landmarks of the current plan
// (trk_id [Tv] the caller's landmark, trk_ptr [Tv + 1], cam [nnz]), taken in the caller's order, with the host CSR of their
// observations.  keep / kcnt (host copies of the rule's, null: every observation) leave out the removed observations and the
// dropped landmarks, so that the plan is the one lvba_visual_create makes from the kept observations.
struct ReplanSource {
  std::vector<int64_t> valid;          // source landmarks in ascending caller order
  std::vector<int64_t> src_ptr;        // [Tv + 1] CSR of every source landmark's (kept) observations
  std::vector<int32_t> cam;            // their cameras
};

inline void replan_source(int64_t Tv, const int* trk_id, const int* trk_ptr, const int* cam, const uint8_t* keep, const int32_t* kcnt,
                          ReplanSource& S) {
  S.valid.clear();
  S.src_ptr.assign((size_t)Tv + 1, 0);
  for (int64_t k = 0; k < Tv; ++k) {
    S.src_ptr[k + 1] = S.src_ptr[k] + (kcnt ? kcnt[k] : trk_ptr[k + 1] - trk_ptr[k]);
    if (!kcnt || kcnt[k] > 0) S.valid.push_back(k);
  }
  std::sort(S.valid.begin(), S.valid.end(), [&](int64_t a, int64_t b) { return trk_id[a] < trk_id[b]; });
  const int64_t nnz = Tv > 0 ? trk_ptr[Tv] : 0;
  if (!keep) { S.cam.assign(cam, cam + nnz); return; }
  S.cam.clear();
  S.cam.reserve((size_t)S.src_ptr[Tv]);
  for (int64_t w = 0; w < nnz; ++w) if (keep[w]) S.cam.push_back(cam[w]);
}

}  // namespace voutliers
}  // namespace lvba
