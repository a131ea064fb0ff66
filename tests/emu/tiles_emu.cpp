// tiles_emu.cpp — TEST INFRASTRUCTURE: the set-up of the LiDAR Hessian build's tiles and destination table
// (global-lvba_b200/csrc/lidar_tiles.h) run through the host policy, so that tests/test_lidar_tiles_emu.py can check the table
// without a GPU.  The same steps as lidar_create_impl: voxel order, local CSR, tiles, the two runs tables.  Never part of the
// product.
#include <vector>

#include "../../global-lvba_b200/csrc/lidar_tiles.h"
#include "host_exec.h"

struct TilesOut {
  std::vector<int64_t> order;
  std::vector<int> vox_ptr, pidx, tile_vox;
  lvba::tiles::Runs<HostExec> prun, drun;
};

extern "C" int emu_tile_slots() { return lvba::tiles::kTileSlots; }
extern "C" int emu_max_vox_per_tile() { return lvba::tiles::kMaxVoxPerTile; }

// grp: window of every pose (null: one window).  first / row_start: the envelope of the pose system.  max_slots <= 0: the
// library's tile size.
extern "C" void* emu_tiles_build(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const int32_t* grp,
                                 const int* first, const long long* row_start, long long nblocks, int max_slots, int max_vox) {
  using namespace lvba::tiles;
  if (max_slots <= 0) { max_slots = kTileSlots; max_vox = kMaxVoxPerTile; }
  TilesOut* o = new TilesOut;
  std::vector<int> slot0;
  order_by_lowest_pose(W, nullptr, V, vox_ptr, pose_idx, slot0, o->vox_ptr);
  std::vector<int> vgrp((size_t)V, 0);
  for (int64_t i = 0; i < V; ++i) {
    for (int q = slot0[(size_t)i]; q < slot0[(size_t)i] + o->vox_ptr[(size_t)i + 1] - o->vox_ptr[(size_t)i]; ++q) o->pidx.push_back(pose_idx[q]);
    if (grp) vgrp[(size_t)i] = grp[pose_idx[slot0[(size_t)i]]];
    o->order.push_back(std::lower_bound(vox_ptr, vox_ptr + V, (int64_t)slot0[(size_t)i]) - vox_ptr);   // caller voxel of local voxel i
  }
  o->tile_vox = cut_ranges(V, o->vox_ptr.data(), grp ? vgrp.data() : nullptr, max_slots, max_vox);
  HostExec ex;
  std::vector<long long> cnt((size_t)V + 1), vox_pair((size_t)V + 1);
  ex.for_each(V + 1, PairCountF{o->vox_ptr.data(), V, cnt.data()});
  ex.exclusive_scan(cnt.data(), vox_pair.data(), V + 1);
  const TableIn in{(int64_t)o->tile_vox.size() - 1, W, nblocks, o->tile_vox.data(), o->vox_ptr.data(), o->pidx.data(),
                   vox_pair.data(), first, row_start};
  if (build_runs(ex, in, false, vox_pair[(size_t)V], o->prun) || build_runs(ex, in, true, o->vox_ptr[(size_t)V], o->drun)) {
    delete o;
    return nullptr;
  }
  return o;
}

// which: 0 order, 1 vox_ptr, 2 pidx, 3 tile_vox (int32 / int64 as listed in tests/test_lidar_tiles_emu.py), 4 pair codes,
// 5 pair run_ptr, 6 pair tile_run, 7 slot codes, 8 slot run_ptr, 9 slot tile_run
extern "C" int64_t emu_tiles_get(void* h, int which, void* dst) {
  TilesOut* o = static_cast<TilesOut*>(h);
  auto out = [&](const auto* p, size_t n) {
    if (dst) std::memcpy(dst, p, n * sizeof(*p));
    return (int64_t)n;
  };
  switch (which) {
    case 0: return out(o->order.data(), o->order.size());
    case 1: return out(o->vox_ptr.data(), o->vox_ptr.size());
    case 2: return out(o->pidx.data(), o->pidx.size());
    case 3: return out(o->tile_vox.data(), o->tile_vox.size());
    case 4: return out(o->prun.code.p, o->prun.code.n);
    case 5: return out(o->prun.run_ptr.p, o->prun.run_ptr.n);
    case 6: return out(o->prun.tile_run.p, o->prun.tile_run.n);
    case 7: return out(o->drun.code.p, o->drun.code.n);
    case 8: return out(o->drun.run_ptr.p, o->drun.run_ptr.n);
    case 9: return out(o->drun.tile_run.p, o->drun.tile_run.n);
  }
  return -1;
}

extern "C" void emu_tiles_free(void* h) { delete static_cast<TilesOut*>(h); }
