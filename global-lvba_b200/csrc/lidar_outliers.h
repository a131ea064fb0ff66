// lidar_outliers.h — BALM2's voxel outlier removal on the LiDAR problem handle (lvba_lidar_voxel_residuals,
// lvba_lidar_remove_voxels, lvba_lidar_remove_outliers).  The reference carries it commented out in include/BALM/bavoxel.hpp:
//   VOX_HESS::evaluate_residual  :205-234   lambda_0 of every voxel ("for outlier removal usage")
//   VOX_HESS::remove_residual    :236-268   the walk that erases voxels from plvec_voxels
//   BALM2::remove_outlier        :650-660   the threshold and the number of voxels to reject
// Plain C++ with no CUDA: the rule is item passes run by an execution policy (CudaExec of exec.cuh in the library, the host
// policy of tests/emu in the CPU tests), and the re-plan's host side (which voxels are kept, and where each kept voxel's records
// are on the device) is shared by lidar_api.cuh and the CPU tests the same way.
//
// The rule, in double as the reference computes it (V voxels, lambda in handle order):
//   thr        = sorted(lambda)[floor((1 - ratio) V) - 1]
//   reject_num = floor(ratio V)
//   walk the voxels in order; a voxel with lambda >= thr is erased; the walk stops after the first KEPT voxel at which the
//   count of erased voxels equals reject_num.
// Equivalently removed_i = (lambda_i >= thr) && i < k*, where k* is the first i with lambda_i < thr and
// #{j < i : lambda_j >= thr} = reject_num (V when there is none).  That is what the passes below compute.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "lidar_plan.h"

namespace lvba {
namespace outliers {

// an order-preserving integer key of a finite double (-0.0 sorts just below +0.0; they compare equal as thresholds)
LVBA_BHD uint64_t order_key(double x) {
  uint64_t b;
  memcpy(&b, &x, sizeof b);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}
LVBA_BHD double key_value(uint64_t k) {
  const uint64_t b = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
  double x;
  memcpy(&x, &b, sizeof x);
  return x;
}

struct KeyF {                  // key and index of every voxel for the sort; bad[i] = lambda_i is not finite
  const double* lam; uint64_t* key; uint32_t* idx; int32_t* bad;
  LVBA_BHD void operator()(int64_t i) const {
    const double x = lam[i];
    bad[i] = !isfinite(x);
    key[i] = order_key(x);
    idx[i] = (uint32_t)i;
  }
};
struct FlagF {                 // flag[i] = lambda_i >= thr
  const double* lam; double thr; int32_t* flag;
  LVBA_BHD void operator()(int64_t i) const { flag[i] = lam[i] >= thr; }
};
struct StopF {                 // cand[i] = i where the walk stops after voxel i (kept, reject_num erased before it), else V
  const double* lam; double thr; const int32_t* erased_before; int64_t reject_num; int32_t V; int32_t* cand;
  LVBA_BHD void operator()(int64_t i) const { cand[i] = (lam[i] < thr && erased_before[i] == reject_num) ? (int32_t)i : V; }
};
struct MaskF {                 // removed[i] = lambda_i >= thr && i < k*
  const int32_t* flag; int64_t k_star; uint8_t* removed;
  LVBA_BHD void operator()(int64_t i) const { removed[i] = (uint8_t)(flag[i] && i < k_star); }
};

// the rule's two numbers (remove_outlier :655-656); false for a ratio outside [0, 1) or not finite, or floor((1 - ratio) V) < 1
inline bool rule_params(double ratio, int64_t V, int64_t* k_thr, int64_t* reject_num) {
  if (!(ratio >= 0.0 && ratio < 1.0)) return false;          // also refuses NaN
  const double n = (double)V;
  const double k = floor((1.0 - ratio) * n);
  if (!(k >= 1.0)) return false;
  *k_thr = (int64_t)k;
  *reject_num = (int64_t)floor(ratio * n);
  return true;
}

struct RuleOut {
  bool non_finite = false;     // some lambda_0 is not finite: no threshold (std::sort would be undefined), nothing computed
  double thr = 0.0;
  int64_t reject_num = 0, k_star = 0;
};

// removed [V] (policy memory) from lambda [V] (policy memory); ratio already checked by rule_params.  Returns a policy status.
template <class Ex>
int remove_rule(Ex& ex, const double* lam, int64_t V, double ratio, uint8_t* removed, RuleOut& out) {
  int64_t k_thr = 0;
  out = RuleOut{};
  if (!rule_params(ratio, V, &k_thr, &out.reject_num)) return -1;
  typename Ex::template Buf<uint64_t> key, key_sorted;
  typename Ex::template Buf<uint32_t> idx, idx_sorted;
  typename Ex::template Buf<int32_t> flag, before;
  LVBA_PLAN_TRY(key.alloc((size_t)V));
  LVBA_PLAN_TRY(key_sorted.alloc((size_t)V));
  LVBA_PLAN_TRY(idx.alloc((size_t)V));
  LVBA_PLAN_TRY(idx_sorted.alloc((size_t)V));
  LVBA_PLAN_TRY(flag.alloc((size_t)V));
  LVBA_PLAN_TRY(before.alloc((size_t)V));
  // 1. non-finite check (flag holds the bad bits)
  LVBA_PLAN_TRY(ex.for_each(V, KeyF{lam, key.p, idx.p, flag.p}));
  int32_t mn = 0, mx = 0;
  LVBA_PLAN_TRY(ex.min_max(flag.p, V, &mn, &mx));
  if (mx != 0) { out.non_finite = true; return 0; }
  // 2-3. the stable radix sort of the keys; thr = the (k_thr - 1)-th smallest lambda
  LVBA_PLAN_TRY(ex.sort_pairs(key.p, key_sorted.p, idx.p, idx_sorted.p, V, 64));
  uint64_t kt = 0;
  LVBA_PLAN_TRY(ex.fetch(&kt, key_sorted.p + (k_thr - 1), 1));
  out.thr = key_value(kt);
  // 4. flags in handle order, their exclusive scan (voxels erased before i) and the first stop: k*
  LVBA_PLAN_TRY(ex.for_each(V, FlagF{lam, out.thr, flag.p}));
  LVBA_PLAN_TRY(ex.exclusive_scan(flag.p, before.p, V));
  int32_t* cand = reinterpret_cast<int32_t*>(idx.p);          // idx is free again: V int32 candidates
  LVBA_PLAN_TRY(ex.for_each(V, StopF{lam, out.thr, before.p, out.reject_num, (int32_t)V, cand}));
  LVBA_PLAN_TRY(ex.min_max(cand, V, &mn, &mx));
  out.k_star = mn;
  // 5. the mask
  return ex.for_each(V, MaskF{flag.p, out.k_star, removed});
}

// ---------------------------------------------------------------- the re-plan after a removal
// Where every handle-order voxel's records are on the device: a local voxel of the SoA records (cl, in the order of lidar_layout)
// or a big voxel (the AoS big_cl).  Built from the plan's layout; removal never moves a voxel between the two (a voxel keeps its
// slots).
struct VoxelHome {
  std::vector<int64_t> where;          // [V] >= 0: local voxel; < 0: big voxel -1 - where
  std::vector<int> local_vox;          // [V_local] handle voxel of every local voxel; empty when the layout is the identity
  std::vector<int> l_vox_ptr;          // [V_local + 1] first SoA slot of every local voxel
  std::vector<int64_t> big_vox_ptr;    // [n_big + 1] first big_cl slot of every big voxel
  std::vector<int> big_vox;            // [n_big] handle voxel of every big voxel
};

inline void voxel_home(int64_t V, const int64_t* vox_ptr, const LidarLayout& L, VoxelHome& H) {
  const int64_t Vl = (int64_t)L.slot0.size();
  H.where.assign((size_t)V, 0);
  H.local_vox.clear();
  if (!L.identity) {
    // the caller voxel of a first slot: one mark per voxel over the slots (no search)
    std::vector<int> voxel_at((size_t)vox_ptr[V]);
    for (int64_t a = 0; a < V; ++a) voxel_at[(size_t)vox_ptr[a]] = (int)a;
    H.local_vox.resize((size_t)Vl);
    for (int64_t i = 0; i < Vl; ++i) H.local_vox[i] = voxel_at[(size_t)L.slot0[i]];
  }
  for (int64_t i = 0; i < Vl; ++i) H.where[L.identity ? i : H.local_vox[i]] = i;
  for (size_t b = 0; b < L.big_vox.size(); ++b) H.where[(size_t)L.big_vox[b]] = -1 - (int64_t)b;
  H.l_vox_ptr = L.l_vox_ptr;
  H.big_vox_ptr = L.big_vox_ptr;
  H.big_vox.assign(L.big_vox.begin(), L.big_vox.end());
}

// The kept voxels' CSR and their plan: layout, home and, for the gather, the old device position of every new record.
struct KeptPlan {
  int64_t V = 0;
  std::vector<int64_t> vox_ptr{0};
  std::vector<int32_t> pose_idx;
  LidarLayout L;
  VoxelHome home;
  std::vector<int> src0;               // [V_local] first old SoA slot of every new local voxel
  std::vector<int> big_src;            // [n_big_slots] old big_cl slot of every new big slot
};

// remove [V] (handle order, nonzero = erase) over the handle's CSR (vox_ptr, pose_idx) and its home.  Returns a LidarLayout error
// (never one for a CSR a single-GPU handle was planned with).
inline int plan_kept(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const VoxelHome& old, const uint8_t* remove,
                     KeptPlan& K, int batch_slots = tiles::kSlots) {
  std::vector<int64_t> old_of;         // new handle voxel -> old handle voxel
  for (int64_t a = 0; a < V; ++a) {
    if (remove[a]) continue;
    old_of.push_back(a);
    K.pose_idx.insert(K.pose_idx.end(), pose_idx + vox_ptr[a], pose_idx + vox_ptr[a + 1]);
    K.vox_ptr.push_back((int64_t)K.pose_idx.size());
  }
  K.V = (int64_t)old_of.size();
  const int rc = lidar_layout(W, K.V, K.vox_ptr.data(), K.pose_idx.data(), nullptr, 0, nullptr, K.L, tiles::kTileSlots, tiles::kMaxVoxPerTile,
                              batch_slots);
  if (rc != kLayoutOk) return rc;
  voxel_home(K.V, K.vox_ptr.data(), K.L, K.home);
  const int64_t Vl = (int64_t)K.L.slot0.size();
  K.src0.resize((size_t)Vl);
  for (int64_t i = 0; i < Vl; ++i) {
    const int64_t c = K.L.identity ? i : K.home.local_vox[i];
    K.src0[i] = old.l_vox_ptr[(size_t)old.where[(size_t)old_of[(size_t)c]]];
  }
  K.big_src.clear();
  for (size_t b = 0; b < K.L.big_vox.size(); ++b) {
    const int64_t ob = -1 - old.where[(size_t)old_of[(size_t)K.L.big_vox[b]]];
    for (int64_t s = old.big_vox_ptr[ob]; s < old.big_vox_ptr[ob + 1]; ++s) K.big_src.push_back((int)s);
  }
  return kLayoutOk;
}

// The gather of the new SoA records and slot poses from the old ones, one item per new slot (the SoA as doubles:
// pair k of slot w at 2 (k nnz_pad + w)).  Local voxel i of w by binary search in the new local CSR.
struct GatherSoaF {
  int32_t n_vox; const int* l_vox_ptr; const int* src0;
  const double* old_cl; int64_t old_pad; const int* old_pidx;
  double* cl; int64_t pad; int* pidx;
  LVBA_BHD void operator()(int64_t w) const {
    int lo = 0, hi = n_vox;
    while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (l_vox_ptr[m] <= w) lo = m; else hi = m; }
    const int64_t q = src0[lo] + (w - l_vox_ptr[lo]);
    pidx[w] = old_pidx[q];
    for (int k = 0; k < 5; ++k) {
      cl[2 * (k * pad + w)] = old_cl[2 * (k * old_pad + q)];
      cl[2 * (k * pad + w) + 1] = old_cl[2 * (k * old_pad + q) + 1];
    }
  }
};
struct GatherAosF {            // the big voxels' 10-double records: out[i] = in[src[i]]
  const int* src; const double* in; double* out;
  LVBA_BHD void operator()(int64_t i) const {
    for (int k = 0; k < 10; ++k) out[10 * i + k] = in[10 * (int64_t)src[i] + k];
  }
};
struct ScatterF {              // out[id[b]] = in[b]: the big voxels' lambda_0 to their handle positions
  const double* in; const int* id; double* out;
  LVBA_BHD void operator()(int64_t b) const { out[id[b]] = in[b]; }
};

}  // namespace outliers
}  // namespace lvba
