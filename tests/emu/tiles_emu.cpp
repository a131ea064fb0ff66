// tiles_emu.cpp — TEST INFRASTRUCTURE: the set-up of the LiDAR Hessian build's tiles and destination table run through the host
// policy, so that tests/test_lidar_tiles_emu.py can check the table without a GPU.  It calls the library's own set-up
// (global-lvba_b200/csrc/lidar_plan.h: lidar_layout, lidar_tables) and does only the per-slot pose gather itself, which the
// library does on the device.  Never part of the product.
#include <vector>

#include "../../global-lvba_b200/csrc/lidar_plan.h"
#include "host_exec.h"

struct TilesOut {
  std::vector<int64_t> order;
  std::vector<int> pidx;
  lvba::LidarLayout L;
  lvba::tiles::Runs<HostExec> prun, drun;
};

extern "C" int emu_tile_slots() { return lvba::tiles::kTileSlots; }
extern "C" int emu_max_vox_per_tile() { return lvba::tiles::kMaxVoxPerTile; }

// n_groups > 0: the poses fall into windows grp_ptr[0..n_groups].  first / row_start: the envelope of the pose system.
// max_slots <= 0: the library's tile size.
extern "C" void* emu_tiles_build(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, int n_groups, const int32_t* grp_ptr,
                                 const int* first, const long long* row_start, long long nblocks, int max_slots, int max_vox) {
  using namespace lvba;
  if (max_slots <= 0) { max_slots = tiles::kTileSlots; max_vox = tiles::kMaxVoxPerTile; }
  TilesOut* o = new TilesOut;
  LidarLayout& L = o->L;
  if (lidar_layout(W, V, vox_ptr, pose_idx, nullptr, n_groups, grp_ptr, L, max_slots, max_vox) != kLayoutOk) { delete o; return nullptr; }
  for (size_t i = 0; i + 1 < L.l_vox_ptr.size(); ++i) {
    for (int q = L.slot0[i]; q < L.slot0[i] + L.l_vox_ptr[i + 1] - L.l_vox_ptr[i]; ++q) o->pidx.push_back(pose_idx[q]);
    o->order.push_back(std::lower_bound(vox_ptr, vox_ptr + V, (int64_t)L.slot0[i]) - vox_ptr);   // caller voxel of local voxel i
  }
  HostExec ex;
  const tiles::TableIn in{(int64_t)L.tile_vox.size() - 1, W, nblocks, L.tile_vox.data(), L.l_vox_ptr.data(), o->pidx.data(), nullptr,
                          first, row_start};
  if (lidar_tables(ex, in, (int64_t)L.slot0.size(), L.n_pairs, L.nnz, o->prun, o->drun)) { delete o; return nullptr; }
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
    case 1: return out(o->L.l_vox_ptr.data(), o->L.l_vox_ptr.size());
    case 2: return out(o->pidx.data(), o->pidx.size());
    case 3: return out(o->L.tile_vox.data(), o->L.tile_vox.size());
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
