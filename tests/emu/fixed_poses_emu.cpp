// fixed_poses_emu.cpp — TEST INFRASTRUCTURE: the LiDAR set-up under constant poses (lvba_lidar_opts::pose_fixed) run through the
// host policy, so that tests/test_fixed_poses_emu.py can check it without a GPU.  It calls the library's own set-up
// (global-lvba_b200/csrc/lidar_plan.h: lidar_row_map, lidar_first_rows, lidar_layout, lidar_tables, lidar_det_index) with the row
// map, and the big-voxel passes of lidar_big.h with it; it does only the per-slot gathers of poses and cluster records itself,
// which the library does on the device.  batch_slots sets which voxels go to the big-voxel passes (1: every voxel of two or more
// slots, so that H and g come from the library's own arithmetic).  Never part of the product.
#include <cmath>
#include <cstring>
#include <vector>

#include "../../global-lvba_b200/csrc/lidar_plan.h"
#include "host_exec.h"

using namespace lvba;

struct FpOut {
  int W = 0, n_rows = 0;
  std::vector<int> row_of, pose_of_row, first;
  std::vector<long long> row_start;
  long long nblocks = 0;
  LidarLayout L;
  std::vector<int> pidx;                 // pose of every local slot of the tiles
  std::vector<double> big_cl;            // AoS records of the big voxels' slots
  tiles::Runs<HostExec> prun, drun;
  tiles::FixedSum<HostExec> H, g;
  big::View view() const {
    return big::View{(int64_t)L.big_vox.size(), L.big_vox_ptr.data(), L.big_pose.data(), big_cl.data(), L.big_pair_ptr.data(),
                     first.data(), row_start.data(), row_of.data(), nblocks, W};
  }
};

// mask: W bytes (nonzero = constant) or null
extern "C" void* emu_fp_build(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const double* clusters,
                              const uint8_t* mask, int batch_slots) {
  FpOut* o = new FpOut;
  o->W = W;
  o->n_rows = lidar_row_map(W, mask, o->row_of, o->pose_of_row);
  o->first = lidar_first_rows(W, V, vox_ptr, pose_idx, o->row_of.data(), o->n_rows);
  const int n = o->n_rows;                                     // Envelope::build
  for (int r = 0; r < n; ++r) o->first[r] = std::min(o->first[r], r);
  for (int r = n - 2; r >= 0; --r) o->first[r] = std::min(o->first[r], o->first[r + 1]);
  o->row_start.assign((size_t)n + 1, 0);
  for (int r = 0; r < n; ++r) o->row_start[r + 1] = o->row_start[r] + (r - o->first[r] + 1);
  o->nblocks = o->row_start[n];
  LidarLayout& L = o->L;
  lidar_layout(W, V, vox_ptr, pose_idx, nullptr, 0, nullptr, L, tiles::kTileSlots, tiles::kMaxVoxPerTile, batch_slots);
  for (size_t i = 0; i + 1 < L.l_vox_ptr.size(); ++i)
    for (int q = 0; q < L.l_vox_ptr[i + 1] - L.l_vox_ptr[i]; ++q) o->pidx.push_back(pose_idx[L.slot0[i] + q]);
  for (int q : L.big_src) o->big_cl.insert(o->big_cl.end(), clusters + 10 * (int64_t)q, clusters + 10 * (int64_t)q + 10);
  HostExec ex;
  const tiles::TableIn in{(int64_t)L.tile_vox.size() - 1, W, o->nblocks, L.tile_vox.data(), L.l_vox_ptr.data(), o->pidx.data(), nullptr,
                          o->first.data(), o->row_start.data(), o->row_of.data()};
  if (lidar_tables(ex, in, (int64_t)L.slot0.size(), L.n_pairs, L.nnz, o->prun, o->drun) ||
      lidar_det_index(ex, in, o->prun, o->drun, o->view(), (int64_t)L.big_src.size(), L.big_pair_ptr.back(), o->H, o->g)) {
    delete o;
    return nullptr;
  }
  return o;
}

// which: 0 local vox_ptr, 1 local pidx, 2 tile_vox (int32); 3 pair codes, 4 slot codes (uint32); 5 pair run_ptr, 6 pair tile_run,
// 7 slot run_ptr, 8 slot tile_run (int64); 9 big_vox_ptr, 10 big_pair_ptr (int64), 11 big_pose (int32); H records: 12 dst (int64),
// 13 code (uint32), 14 run_ptr (int64); g records: 15 dst, 16 code, 17 run_ptr; 18 row_of, 19 first (int32), 20 row_start (int64)
extern "C" int64_t emu_fp_get(void* h, int which, void* dst) {
  FpOut* o = static_cast<FpOut*>(h);
  auto out = [&](const auto* p, size_t n) {
    if (dst && n) std::memcpy(dst, p, n * sizeof(*p));
    return (int64_t)n;
  };
  switch (which) {
    case 0: return out(o->L.l_vox_ptr.data(), o->L.l_vox_ptr.size());
    case 1: return out(o->pidx.data(), o->pidx.size());
    case 2: return out(o->L.tile_vox.data(), o->L.tile_vox.size());
    case 3: return out(o->prun.code.p, o->prun.code.n);
    case 4: return out(o->drun.code.p, o->drun.code.n);
    case 5: return out(o->prun.run_ptr.p, o->prun.run_ptr.n);
    case 6: return out(o->prun.tile_run.p, o->prun.tile_run.n);
    case 7: return out(o->drun.run_ptr.p, o->drun.run_ptr.n);
    case 8: return out(o->drun.tile_run.p, o->drun.tile_run.n);
    case 9: return out(o->L.big_vox_ptr.data(), o->L.big_vox_ptr.size());
    case 10: return out(o->L.big_pair_ptr.data(), o->L.big_pair_ptr.size());
    case 11: return out(o->L.big_pose.data(), o->L.big_pose.size());
    case 12: return out(o->H.dst.p, (size_t)o->H.n_rec);
    case 13: return out(o->H.by_dst.code.p, (size_t)o->H.n_rec);
    case 14: return out(o->H.by_dst.run_ptr.p, (size_t)o->H.by_dst.n_runs + 1);
    case 15: return out(o->g.dst.p, (size_t)o->g.n_rec);
    case 16: return out(o->g.by_dst.code.p, (size_t)o->g.n_rec);
    case 17: return out(o->g.by_dst.run_ptr.p, (size_t)o->g.by_dst.n_runs + 1);
    case 18: return out(o->row_of.data(), o->row_of.size());
    case 19: return out(o->first.data(), o->first.size());
    case 20: return out(o->row_start.data(), o->row_start.size());
  }
  return -1;
}

// One build of H [nblocks][36] and g [n_rows][6] over the rows from the tiles' run sums given by the caller (tile_H: [pair runs +
// pose runs][36], tile_g: [pose runs][6]) and the big voxels' passes at `poses`; *residual = sum of the big voxels' lambda_0.
// det = 1: records + GatherF, as lidar_build_hg in deterministic mode; det = 0: the run sums and the big voxels' contributions
// added one by one in the order the host policy visits the items, as the REDs of the default mode.
extern "C" void emu_fp_run(void* h, const double* tile_H, const double* tile_g, const double* poses, int det, double* H, double* g,
                           double* residual) {
  FpOut* o = static_cast<FpOut*>(h);
  HostExec ex;
  const big::View bv = o->view();
  const int64_t npr = o->prun.n_runs, ndr = o->drun.n_runs;
  const int64_t nb = bv.n_vox, nbs = (int64_t)o->L.big_pose.size(), nbp = o->L.big_pair_ptr.back();
  std::vector<double> params((size_t)nb * big::kParams), res((size_t)nb), feat((size_t)nbs * big::kFeat);
  std::memset(H, 0, (size_t)o->nblocks * 36 * sizeof(double));
  std::memset(g, 0, (size_t)o->n_rows * 6 * sizeof(double));
  ex.for_each(nb, big::ParamsF{bv, poses, params.data(), res.data()});
  *residual = 0.0;
  for (double r : res) *residual += r;
  if (det) {
    std::memcpy(o->H.rec.p, tile_H, (size_t)(npr + ndr) * 36 * sizeof(double));
    std::memcpy(o->g.rec.p, tile_g, (size_t)ndr * 6 * sizeof(double));
    ex.for_each(nbs, big::SlotsDetF{bv, poses, params.data(), feat.data(), o->H.rec.p + 36 * (npr + ndr), o->g.rec.p + 6 * ndr});
    ex.for_each(nbp, big::PairsDetF{bv, params.data(), feat.data(), o->H.rec.p + 36 * (npr + ndr + nbs)});
    ex.for_each(o->H.by_dst.n_runs * 36, tiles::gather_of(o->H, H));
    ex.for_each(o->g.by_dst.n_runs * 6, tiles::gather_of(o->g, g));
    return;
  }
  const tiles::FixedSum<HostExec>& fH = o->H;
  const tiles::FixedSum<HostExec>& fg = o->g;
  ex.for_each(npr + ndr, [&](int64_t r) { for (int e = 0; e < 36; ++e) H[fH.dst.p[r] * 36 + e] += tile_H[36 * r + e]; });
  ex.for_each(ndr, [&](int64_t r) { for (int e = 0; e < 6; ++e) g[fg.dst.p[r] * 6 + e] += tile_g[6 * r + e]; });
  ex.for_each(nbs, big::SlotsF{bv, poses, params.data(), feat.data(), H, g});
  ex.for_each(nbp, big::PairsF{bv, params.data(), feat.data(), H});
}

extern "C" int emu_fp_rows(void* h) { return static_cast<FpOut*>(h)->n_rows; }
extern "C" long long emu_fp_nblocks(void* h) { return static_cast<FpOut*>(h)->nblocks; }
extern "C" void emu_fp_free(void* h) { delete static_cast<FpOut*>(h); }
