// outliers_emu.cpp — TEST INFRASTRUCTURE: the voxel outlier removal of lidar_outliers.h run through the host policy, so that
// tests/test_lidar_outliers_emu.py can check it without a GPU.  It calls the library's own rule passes (remove_rule) and
// re-plan (voxel_home, plan_kept, GatherSoaF, GatherAosF), and does itself only what lidar_create_impl does on the device for a
// fresh handle: the caller's AoS records transposed to the SoA in the layout's order.  batch_slots sets which voxels go to the
// big-voxel passes.  Never part of the product.
#include <cstring>
#include <vector>

#include "../../global-lvba_b200/csrc/lidar_outliers.h"
#include "host_exec.h"

using namespace lvba;

// removed [V]; thr_out: the threshold.  Returns 0, 1 for a non-finite lambda, -1 for refused parameters.
extern "C" int emu_ol_rule(int64_t V, const double* lam, double ratio, uint8_t* removed, double* thr_out) {
  HostExec ex;
  HostExec::Buf<double> d_lam;
  HostExec::Buf<uint8_t> d_rm;
  d_lam.alloc((size_t)V);
  d_rm.alloc((size_t)V);
  std::memcpy(d_lam.p, lam, (size_t)V * sizeof(double));
  outliers::RuleOut r;
  if (outliers::remove_rule(ex, d_lam.p, V, ratio, d_rm.p, r) != 0) return -1;
  if (r.non_finite) return 1;
  std::memcpy(removed, d_rm.p, (size_t)V);
  *thr_out = r.thr;
  return 0;
}

// the records of a fresh handle (lidar_create_impl): SoA (as doubles, [5][pad][2]) and slot poses of the local voxels, AoS of the
// big voxels, zero padding
struct Records {
  LidarLayout L;
  int64_t pad = 0;
  HostExec::Buf<double> cl, big_cl;
  HostExec::Buf<int> pidx;
};
static void fresh(int W, int64_t V, const int64_t* vp, const int32_t* pi, const double* aos, int batch_slots, Records& R) {
  lidar_layout(W, V, vp, pi, nullptr, 0, nullptr, R.L, tiles::kTileSlots, tiles::kMaxVoxPerTile, batch_slots);
  R.pad = ((R.L.nnz + 31) / 32) * 32 + 32;
  R.cl.alloc((size_t)10 * R.pad);
  std::memset(R.cl.p, 0, R.cl.n * sizeof(double));
  R.pidx.alloc((size_t)R.L.nnz);
  for (size_t i = 0; i + 1 < R.L.l_vox_ptr.size(); ++i)
    for (int w = R.L.l_vox_ptr[i]; w < R.L.l_vox_ptr[i + 1]; ++w) {
      const int64_t q = R.L.slot0[i] + (w - R.L.l_vox_ptr[i]);
      R.pidx.p[w] = pi[q];
      for (int k = 0; k < 10; ++k) R.cl.p[2 * ((k / 2) * R.pad + w) + (k & 1)] = aos[10 * q + k];
    }
  R.big_cl.alloc(R.L.big_src.size() * 10);
  for (size_t s = 0; s < R.L.big_src.size(); ++s) std::memcpy(R.big_cl.p + 10 * s, aos + 10 * (int64_t)R.L.big_src[s], 10 * sizeof(double));
}

template <class A, class B>
static int64_t diff(const A& a, const B& b) { return a.size() == b.size() && std::equal(a.begin(), a.end(), b.begin()) ? 0 : 1; }

// Removes `remove` [V] from the fresh records of the caller's problem with the library's re-plan and gathers, and compares the
// result with a fresh layout of the kept CSR (kvp, kpi, kaos: the kept voxels, in order).  n_removals > 1: the removal is split in
// that many steps, each over the result of the previous (renumbered) one.  Returns the number of differing items (0: equal).
extern "C" int64_t emu_ol_gather(int W, int64_t V, const int64_t* vp, const int32_t* pi, const double* aos, const uint8_t* remove,
                                 int64_t KV, const int64_t* kvp, const int32_t* kpi, const double* kaos, int batch_slots, int n_removals) {
  HostExec ex;
  Records cur;
  fresh(W, V, vp, pi, aos, batch_slots, cur);
  outliers::VoxelHome home;
  outliers::voxel_home(V, vp, cur.L, home);
  std::vector<int64_t> cvp(vp, vp + V + 1);
  std::vector<int32_t> cpi(pi, pi + vp[V]);
  std::vector<uint8_t> rm(remove, remove + V);
  std::vector<int64_t> orig((size_t)V);                          // original index of every current voxel
  for (int64_t a = 0; a < V; ++a) orig[a] = a;
  for (int step = 0; step < n_removals; ++step) {
    std::vector<uint8_t> part(orig.size(), 0);                   // this step's share: every n_removals-th removed voxel
    for (size_t a = 0; a < orig.size(); ++a) part[a] = rm[orig[a]] && ((int)(orig[a] % n_removals) == step || step + 1 == n_removals);
    outliers::KeptPlan K;
    if (outliers::plan_kept(W, (int64_t)orig.size(), cvp.data(), cpi.data(), home, part.data(), K, batch_slots) != kLayoutOk) return -1;
    Records nx;
    nx.L = K.L;
    nx.pad = ((K.L.nnz + 31) / 32) * 32 + 32;
    nx.cl.alloc((size_t)10 * nx.pad);
    ex.fill_zero(nx.cl.p, nx.cl.n);
    nx.pidx.alloc((size_t)K.L.nnz);
    ex.for_each(K.L.nnz, outliers::GatherSoaF{(int32_t)K.L.slot0.size(), K.L.l_vox_ptr.data(), K.src0.data(), cur.cl.p, cur.pad, cur.pidx.p,
                                              nx.cl.p, nx.pad, nx.pidx.p});
    nx.big_cl.alloc(K.big_src.size() * 10);
    ex.for_each((int64_t)K.big_src.size(), outliers::GatherAosF{K.big_src.data(), cur.big_cl.p, nx.big_cl.p});
    std::vector<int64_t> orig2;
    for (size_t a = 0; a < orig.size(); ++a) if (!part[a]) orig2.push_back(orig[a]);
    orig.swap(orig2);
    cvp = K.vox_ptr; cpi = K.pose_idx; home = K.home;
    cur.L = nx.L; cur.pad = nx.pad; cur.cl.swap(nx.cl); cur.pidx.swap(nx.pidx); cur.big_cl.swap(nx.big_cl);
  }
  Records ref;
  fresh(W, KV, kvp, kpi, kaos, batch_slots, ref);
  outliers::VoxelHome ref_home;
  outliers::voxel_home(KV, kvp, ref.L, ref_home);
  int64_t bad = 0;
  bad += (int64_t)orig.size() != KV;
  bad += diff(cvp, std::vector<int64_t>(kvp, kvp + KV + 1)) + diff(cpi, std::vector<int32_t>(kpi, kpi + kvp[KV]));
  bad += diff(cur.L.l_vox_ptr, ref.L.l_vox_ptr) + diff(cur.L.slot0, ref.L.slot0) + diff(cur.L.batch_vox, ref.L.batch_vox);
  bad += diff(cur.L.tile_vox, ref.L.tile_vox) + diff(cur.L.big_vox, ref.L.big_vox) + diff(cur.L.big_pose, ref.L.big_pose);
  bad += diff(cur.L.big_vox_ptr, ref.L.big_vox_ptr) + diff(cur.L.big_pair_ptr, ref.L.big_pair_ptr) + (cur.L.identity != ref.L.identity);
  bad += diff(home.where, ref_home.where) + diff(home.local_vox, ref_home.local_vox) + diff(home.big_vox, ref_home.big_vox);
  if (cur.cl.n != ref.cl.n || cur.pidx.n != ref.pidx.n || cur.big_cl.n != ref.big_cl.n) return bad + 1;
  auto same = [](const void* a, const void* b, size_t bytes) { return bytes == 0 || std::memcmp(a, b, bytes) == 0; };
  bad += !same(cur.cl.p, ref.cl.p, cur.cl.n * sizeof(double));
  bad += !same(cur.pidx.p, ref.pidx.p, cur.pidx.n * sizeof(int));
  bad += !same(cur.big_cl.p, ref.big_cl.p, cur.big_cl.n * sizeof(double));
  return bad;
}
