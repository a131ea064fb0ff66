// det_emu.cpp — TEST INFRASTRUCTURE: the fixed-order sums of the deterministic LiDAR build (lidar_tiles.h FixedSum / GatherF,
// the record passes of lidar_big.h) run through the host policy, so that tests/test_deterministic_emu.py can check them without a
// GPU.  It calls the library's own set-up (global-lvba_b200/csrc/lidar_plan.h: lidar_layout, lidar_tables, lidar_det_index) and
// does only the per-slot gathers of poses and cluster records itself, which the library does on the device: voxels with more than
// kSlots slots go to the big-voxel passes, the others into tiles; records of H = [pair runs][pose runs][big slots][big pairs],
// of g = [pose runs][big slots].  Never part of the product.  emu_vdet_step does the same for the big-landmark passes of the
// visual build (visual_plan.h visual_det_index, visual_big.h).
#include <cmath>
#include <cstring>
#include <vector>

#include "../../global-lvba_b200/csrc/lidar_plan.h"
#include "../../global-lvba_b200/csrc/visual_plan.h"
#include "host_exec.h"

using namespace lvba;

struct DetOut {
  int W = 0;
  long long nblocks = 0;
  const int* first = nullptr;
  const long long* row_start = nullptr;
  LidarLayout L;
  std::vector<int> pidx;                 // pose of every local slot of the tiles
  std::vector<double> big_cl;            // AoS records of the big voxels' slots
  tiles::Runs<HostExec> prun, drun;
  tiles::FixedSum<HostExec> H, g;
  big::View view() const {
    return big::View{(int64_t)L.big_vox.size(), L.big_vox_ptr.data(), L.big_pose.data(), big_cl.data(), L.big_pair_ptr.data(), first, row_start};
  }
};

extern "C" void* emu_det_build(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const double* clusters,
                               const int* first, const long long* row_start, long long nblocks) {
  DetOut* o = new DetOut;
  o->W = W; o->nblocks = nblocks; o->first = first; o->row_start = row_start;
  LidarLayout& L = o->L;
  lidar_layout(W, V, vox_ptr, pose_idx, nullptr, 0, nullptr, L);
  for (size_t i = 0; i + 1 < L.l_vox_ptr.size(); ++i)
    for (int q = 0; q < L.l_vox_ptr[i + 1] - L.l_vox_ptr[i]; ++q) o->pidx.push_back(pose_idx[L.slot0[i] + q]);
  for (int q : L.big_src) o->big_cl.insert(o->big_cl.end(), clusters + 10 * (int64_t)q, clusters + 10 * (int64_t)q + 10);
  HostExec ex;
  const tiles::TableIn in{(int64_t)L.tile_vox.size() - 1, W, nblocks, L.tile_vox.data(), L.l_vox_ptr.data(), o->pidx.data(), nullptr,
                          first, row_start};
  if (lidar_tables(ex, in, (int64_t)L.slot0.size(), L.n_pairs, L.nnz, o->prun, o->drun) ||
      lidar_det_index(ex, in, o->prun, o->drun, o->view(), (int64_t)L.big_src.size(), L.big_pair_ptr.back(), o->H, o->g)) {
    delete o;
    return nullptr;
  }
  return o;
}

// which: 0 local vox_ptr, 1 local pidx, 2 tile_vox (int32); 3 pair codes, 4 slot codes (uint32); 5 pair run_ptr, 6 pair tile_run,
// 7 slot run_ptr, 8 slot tile_run (int64); 9 big_vox_ptr, 10 big_pair_ptr (int64), 11 big_pose (int32); H records: 12 dst (int64),
// 13 code (uint32), 14 run_ptr (int64); g records: 15 dst, 16 code, 17 run_ptr
extern "C" int64_t emu_det_get(void* h, int which, void* dst) {
  DetOut* o = static_cast<DetOut*>(h);
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
  }
  return -1;
}

// One build of H [nblocks][36] and g [W][6] from the tiles' run sums given by the caller (tile_H: [pair runs + pose runs][36],
// tile_g: [pose runs][6]) and the big voxels' passes at `poses`.  det = 1: records + GatherF, as lidar_build_hg in deterministic
// mode; det = 0: every run sum and every big-voxel contribution added into H and g one by one in the order the host policy visits
// the items, as the REDs of the default mode.
extern "C" void emu_det_run(void* h, const double* tile_H, const double* tile_g, const double* poses, int det, double* H, double* g) {
  DetOut* o = static_cast<DetOut*>(h);
  HostExec ex;
  const big::View bv = o->view();
  const int64_t npr = o->prun.n_runs, ndr = o->drun.n_runs;
  const int64_t nb = bv.n_vox, nbs = (int64_t)o->L.big_pose.size(), nbp = o->L.big_pair_ptr.back();
  std::vector<double> params((size_t)nb * big::kParams), res((size_t)nb), feat((size_t)nbs * big::kFeat);
  std::memset(H, 0, (size_t)o->nblocks * 36 * sizeof(double));
  std::memset(g, 0, (size_t)o->W * 6 * sizeof(double));
  ex.for_each(nb, big::ParamsF{bv, poses, params.data(), res.data()});
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

extern "C" void emu_det_free(void* h) { delete static_cast<DetOut*>(h); }

// The column-norm pass and the build of every landmark of a visual problem through the big-landmark passes (all landmarks "big",
// as tests/emu/visual_big_emu.cpp), at the state (q, t, X): cam_colsq0 [n_rows*6], pt_colsq0 [Tv*3], S [nblocks*36], rhs /
// cam_colsq / cam_grad [n_rows*6].  det = 1: records + GatherF in observation / pair order, as visual_compute_scale and
// visual_linearize_solve in deterministic mode; det = 0: the atomics of the default mode, in the order the host policy visits the
// items.
extern "C" void emu_vdet_step(int n_rows, int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row,
                              const float* obs_uv, const double* plane, const double* intr, double sigma_px, double sigma_pl,
                              const int* first, const long long* row_start, const double* q, const double* t, const double* X, int det,
                              double* cam_colsq0, double* pt_colsq0, double* S, double* rhs, double* cam_colsq, double* cam_grad) {
  VisualView vv{};
  vv.trk_ptr = trk_ptr; vv.trk_id = trk_id; vv.obs_cam = obs_cam; vv.obs_row = obs_row;
  vv.obs_uv = reinterpret_cast<const float2*>(obs_uv); vv.plane = plane;
  for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
  vv.inv_sigma_px = 1.0 / sigma_px;
  vv.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);
  std::vector<int64_t> pair_ptr((size_t)Tv + 1, 0);
  for (int64_t k = 0; k < Tv; ++k) { const int64_t K = trk_ptr[k + 1] - trk_ptr[k]; pair_ptr[k + 1] = pair_ptr[k] + K * (K - 1); }
  const vbig::View bv{Tv, 0, pair_ptr.data(), first, row_start};
  const long long nblocks = row_start[n_rows];
  const VisualState st{q, t, X};
  const int64_t nnz = trk_ptr[Tv], np = pair_ptr[(size_t)Tv];
  HostExec ex;
  HostExec::Buf<double> obs, params, cost, gmax, C;
  obs.alloc((size_t)nnz * vbig::kObs); params.alloc((size_t)Tv * kTrkParams); cost.alloc((size_t)Tv); gmax.alloc((size_t)Tv);
  tiles::FixedSum<HostExec> fS, fG;
  if (det) {                                                   // visual_det_setup without tiles
    const tiles::VisTableIn no_tiles{0, n_rows, nblocks, nullptr, trk_ptr, obs_row, nullptr, first, row_start};
    const tiles::Runs<HostExec> no_runs;
    visual_det_index(ex, no_tiles, no_runs, no_runs, vv, bv, nnz, np, fS, fG);
    C.alloc((size_t)std::max<int64_t>(nnz, 1) * 6);
  }
  for (double* a : {cam_colsq0, rhs, cam_colsq, cam_grad}) std::memset(a, 0, (size_t)n_rows * 6 * sizeof(double));
  std::memset(S, 0, (size_t)nblocks * 36 * sizeof(double));
  if (det) ex.for_each(nnz, vbig::ColObsDetF{vv, bv, st, obs.p, C.p});
  else ex.for_each(nnz, vbig::ColObsF{vv, bv, st, obs.p, cam_colsq0});
  ex.for_each(Tv, vbig::ColTrackF{vv, bv, st, obs.p, pt_colsq0});
  if (det) ex.for_each(fG.by_dst.n_runs * 6, tiles::gather_part(fG, C.p, 6, 0, 6, cam_colsq0));
  std::vector<double> s_cam((size_t)n_rows * 6), s_pt((size_t)Tv * 3);
  for (size_t i = 0; i < s_cam.size(); ++i) s_cam[i] = 1.0 / (1.0 + std::sqrt(cam_colsq0[i]));
  for (size_t i = 0; i < s_pt.size(); ++i) s_pt[i] = 1.0 / (1.0 + std::sqrt(pt_colsq0[i]));
  const VisualLM lm{1e4, 1e-6, 1e32, s_cam.data(), s_pt.data()};
  ex.for_each(nnz, vbig::ObsF{vv, bv, st, lm, obs.p});
  ex.for_each(Tv, vbig::TrackF{vv, bv, st, lm, obs.p, params.p, cost.p, gmax.p});
  if (!det) {
    ex.for_each(nnz, vbig::SlotsF{vv, bv, params.p, obs.p, S, rhs, cam_colsq, cam_grad});
    ex.for_each(np, vbig::PairsF{vv, bv, obs.p, S});
    return;
  }
  ex.for_each(nnz, vbig::SlotsDetF{vv, bv, params.p, obs.p, fS.rec.p, fG.rec.p, nullptr, nullptr});
  ex.for_each(np, vbig::PairsDetF{vv, bv, obs.p, fS.rec.p + 36 * nnz});
  ex.for_each(fS.by_dst.n_runs * 36, tiles::gather_of(fS, S));
  ex.for_each(fG.by_dst.n_runs * 6, tiles::gather_part(fG, fG.rec.p, 18, 0, 6, rhs));
  ex.for_each(fG.by_dst.n_runs * 6, tiles::gather_part(fG, fG.rec.p, 18, 6, 6, cam_colsq));
  ex.for_each(fG.by_dst.n_runs * 6, tiles::gather_part(fG, fG.rec.p, 18, 12, 6, cam_grad));
}
