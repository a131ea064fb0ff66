// visual_outliers_emu.cpp — TEST INFRASTRUCTURE: the reprojection-outlier removal of visual_outliers.h run through the host
// policy, so that tests/test_visual_outliers_emu.py can check it without a GPU.  It calls the library's own rule passes
// (keep_rule), compaction (CompactF, RemovedF), caller-index passes (DeriveSrcF, GatherSrcF) and re-plan source
// (replan_source) with the symbolic set-up of visual_plan.h, and does itself only what visual_plan and visual_gather_kernel do
// on the device: the row map, the layout, and the gather of every new local observation from its source landmark.  Never part
// of the product.
#include <cstring>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_outliers.h"
#include "host_exec.h"

using namespace lvba;

namespace {

// the per-observation arrays of a plan, as the handle holds them on the device
struct Plan {
  std::vector<int> row_of_cam, cam_of_row;
  VisualLayout L;
  std::vector<int> trk_id, obs_cam;           // trk_id: the caller's landmark
  std::vector<float2> obs_uv;
  HostExec::Buf<int64_t> obs_src;
  HostExec::Buf<int> trk_ptr;
};

// visual_plan on one GPU: source landmarks valid of n_src (host CSR src_ptr / src_cam), src_id the caller's landmark of a source
// landmark (null: the source landmarks are the caller's), the device arrays cam / uv and, when given, the caller index src
// (else it is derived from the caller's obs_ptr as visual_obs_src does).
void plan(int M, int fixed_cam, const std::vector<int64_t>& valid, int64_t n_src, const int64_t* src_ptr, const int32_t* src_cam, const int* src_id,
          const int* cam, const float2* uv, const int64_t* src, const int64_t* caller_ptr, Plan& P) {
  HostExec ex;
  std::vector<char> used((size_t)M, 0);
  for (int64_t i : valid)
    for (int64_t q = src_ptr[i]; q < src_ptr[i + 1]; ++q) used[src_cam[q]] = 1;
  visual_row_map(M, used, fixed_cam, nullptr, P.row_of_cam, P.cam_of_row);
  std::vector<int> min_row, min_sys_row;
  visual_first_rows((int)P.cam_of_row.size(), valid.data(), (int64_t)valid.size(), src_ptr, src_cam, P.row_of_cam.data(), min_row, min_sys_row);
  P.L = VisualLayout{};
  visual_layout((int)P.cam_of_row.size(), valid.data(), (int64_t)valid.size(), nullptr, min_sys_row.data(), src_ptr, src_cam, P.row_of_cam.data(), P.L);
  const int64_t Tv = P.L.Tv, nnz = P.L.nnz;
  P.trk_id.resize((size_t)Tv);
  P.obs_cam.resize((size_t)nnz);
  P.obs_uv.resize((size_t)nnz);
  P.trk_ptr.alloc((size_t)Tv + 1);
  std::memcpy(P.trk_ptr.p, P.L.trk_ptr.data(), ((size_t)Tv + 1) * sizeof(int));
  for (int64_t k = 0; k < Tv; ++k) {                           // visual_gather_kernel
    const int64_t i = P.L.trk_id[k];
    P.trk_id[k] = src_id ? src_id[i] : (int)i;
    for (int64_t w = P.L.trk_ptr[k], q = src_ptr[i]; q < src_ptr[i + 1]; ++q, ++w) { P.obs_cam[w] = cam[q]; P.obs_uv[w] = uv[q]; }
  }
  P.obs_src.alloc((size_t)nnz);
  if (src) {
    HostExec::Buf<long long> sp;
    sp.alloc((size_t)n_src + 1);
    for (size_t i = 0; i < sp.n; ++i) sp.p[i] = src_ptr[i];
    ex.for_each(Tv, voutliers::GatherSrcF{P.L.trk_id.data(), P.trk_ptr.p, sp.p, src, P.obs_src.p});
  } else {
    ex.for_each(Tv, voutliers::DeriveSrcF{P.trk_id.data(), P.trk_ptr.p, caller_ptr, P.obs_src.p});
  }
}

template <class A, class B>
int64_t diff(const A& a, const B& b) { return a.size() == b.size() && std::equal(a.begin(), a.end(), b.begin()) ? 0 : 1; }

}  // namespace

// The caller's problem (M cameras, T landmarks, the landmarks with a valid plane in `valid_lm` [T], CSR obs_ptr / obs_cam /
// obs_uv [N][2]) through n_rounds removals: round r removes by mask masks[r N ..] when taus[r] < 0, else by s_q <= taus[r] with
// sq[r N ..] (caller-indexed, NaN out of the problem), with min_lens[r].  removed [n_rounds N] and left [2 n_rounds]
// (observations, landmarks) come back per round.  The final plan is compared with a fresh plan of the kept problem (kvalid,
// kptr, kcam, kuv, and kidx: the caller index of every kept observation); returns the number of differing arrays (0: equal), -1 when a round would leave no observation.
extern "C" int64_t emu_vo_run(int M, int64_t T, int fixed_cam, const uint8_t* valid_lm, const int64_t* obs_ptr, const int32_t* obs_cam,
                              const float* obs_uv, int n_rounds, const uint8_t* masks, const double* sq, const double* taus,
                              const int32_t* min_lens, uint8_t* removed, int64_t* left, const uint8_t* kvalid, const int64_t* kptr,
                              const int32_t* kcam, const float* kuv, const int64_t* kidx) {
  HostExec ex;
  const int64_t N = obs_ptr[T];
  std::vector<int64_t> valid;
  for (int64_t i = 0; i < T; ++i) if (valid_lm[i]) valid.push_back(i);
  const float2* uv = reinterpret_cast<const float2*>(obs_uv);
  Plan cur;
  plan(M, fixed_cam, valid, T, obs_ptr, obs_cam, nullptr, obs_cam, uv, nullptr, obs_ptr, cur);
  for (int r = 0; r < n_rounds; ++r) {
    const int64_t Tv = cur.L.Tv, nnz = cur.L.nnz;
    voutliers::RuleBufs<HostExec> B;
    int64_t kept_obs = 0, kept_trk = 0;
    const bool by_mask = taus[r] < 0;
    voutliers::keep_rule(ex, nnz, Tv, cur.trk_ptr.p, cur.obs_src.p, by_mask ? masks + r * N : nullptr, by_mask ? nullptr : sq + r * N,
                         by_mask ? 0.0 : taus[r], min_lens[r], B, &kept_obs, &kept_trk);
    if (kept_obs == 0) return -1;
    std::memset(removed + r * N, 0, (size_t)N);
    ex.for_each(nnz, voutliers::RemovedF{B.keep.p, cur.obs_src.p, removed + r * N});
    left[2 * r] = kept_obs;
    left[2 * r + 1] = kept_trk;
    HostExec::Buf<int> ccam;
    HostExec::Buf<float2> cuv;
    HostExec::Buf<int64_t> csrc;
    ccam.alloc((size_t)kept_obs); cuv.alloc((size_t)kept_obs); csrc.alloc((size_t)kept_obs);
    ex.for_each(nnz, voutliers::CompactF{B.keep.p, B.pos.p, cur.obs_cam.data(), cur.obs_uv.data(), cur.obs_src.p, ccam.p, cuv.p, csrc.p});
    HostExec::Buf<uint8_t> keep8;
    keep8.alloc((size_t)nnz);
    ex.for_each(nnz, voutliers::KeepBytesF{B.keep.p, keep8.p});
    voutliers::ReplanSource S;
    voutliers::replan_source(Tv, cur.trk_id.data(), cur.trk_ptr.p, cur.obs_cam.data(), keep8.p, B.kcnt.p, S);
    Plan nx;
    plan(M, fixed_cam, S.valid, Tv, S.src_ptr.data(), S.cam.data(), cur.trk_id.data(), ccam.p, cuv.p, csrc.p, obs_ptr, nx);
    std::swap(cur.row_of_cam, nx.row_of_cam); std::swap(cur.cam_of_row, nx.cam_of_row); std::swap(cur.L, nx.L);
    std::swap(cur.trk_id, nx.trk_id); std::swap(cur.obs_cam, nx.obs_cam); std::swap(cur.obs_uv, nx.obs_uv);
    cur.obs_src.swap(nx.obs_src); cur.trk_ptr.swap(nx.trk_ptr);
  }
  std::vector<int64_t> kv;
  for (int64_t i = 0; i < T; ++i) if (kvalid[i]) kv.push_back(i);
  Plan ref;
  plan(M, fixed_cam, kv, T, kptr, kcam, nullptr, kcam, reinterpret_cast<const float2*>(kuv), nullptr, kptr, ref);
  int64_t bad = 0;
  bad += diff(cur.cam_of_row, ref.cam_of_row) + diff(cur.row_of_cam, ref.row_of_cam);
  bad += diff(cur.L.trk_ptr, ref.L.trk_ptr) + diff(cur.trk_id, ref.trk_id) + (cur.L.Tv_small != ref.L.Tv_small);
  bad += diff(cur.L.batch_trk, ref.L.batch_trk) + diff(cur.L.tile_trk, ref.L.tile_trk) + diff(cur.L.big_pair_ptr, ref.L.big_pair_ptr);
  bad += (cur.L.n_ordered != ref.L.n_ordered) + (cur.L.big_pairs != ref.L.big_pairs);
  bad += diff(cur.obs_cam, ref.obs_cam);
  bad += cur.obs_uv.size() != ref.obs_uv.size() ||
         (!cur.obs_uv.empty() && std::memcmp(cur.obs_uv.data(), ref.obs_uv.data(), cur.obs_uv.size() * sizeof(float2)) != 0);
  // the caller index of the kept problem's observation j is kidx[j]
  std::vector<int64_t> ref_src((size_t)ref.obs_src.n);
  for (size_t w = 0; w < ref_src.size(); ++w) ref_src[w] = kidx[ref.obs_src.p[w]];
  bad += diff(std::vector<int64_t>(cur.obs_src.p, cur.obs_src.p + cur.obs_src.n), ref_src);
  // and every survivor's caller index names an observation with the same camera and pixel
  for (int64_t w = 0; w < (int64_t)cur.obs_cam.size(); ++w) {
    const int64_t q = cur.obs_src.p[w];
    bad += (q < 0 || q >= N || obs_cam[q] != cur.obs_cam[w] || std::memcmp(&uv[q], &cur.obs_uv[w], sizeof(float2)) != 0) ? 1 : 0;
    if (bad > 1000) break;
  }
  return bad;
}
