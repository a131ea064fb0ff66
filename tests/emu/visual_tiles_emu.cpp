// visual_tiles_emu.cpp — TEST INFRASTRUCTURE: the set-up of the reduced camera system build's tiles and destination table run
// through the host policy, so that tests/test_visual_tiles_emu.py can check the table without a GPU.  It calls the library's own
// set-up (global-lvba_b200/csrc/visual_plan.h: visual_first_rows, visual_layout, visual_tables) with every landmark valid, and
// does only the per-observation row gather itself, which the library does on the device.  Never part of the product.
#include <numeric>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_plan.h"
#include "host_exec.h"

struct VisTilesOut {
  std::vector<int64_t> order;
  std::vector<int> row;
  lvba::VisualLayout L;
  lvba::tiles::Runs<HostExec> prun, drun;
};

extern "C" int emu_vis_tile_slots() { return lvba::tiles::kVisTileSlots; }
extern "C" int emu_vis_max_trk_per_tile() { return lvba::tiles::kMaxTrkPerTile; }

// row_of_cam: system row of every camera, -1 for a constant one.  first / row_start: the envelope of the reduced camera system.
// max_slots <= 0: the library's tile size.
extern "C" void* emu_vis_tiles_build(int n_rows, int64_t T, const int64_t* obs_ptr, const int32_t* obs_cam, const int32_t* row_of_cam,
                                     const int* first, const long long* row_start, long long nblocks, int max_slots, int max_trk) {
  using namespace lvba;
  if (max_slots <= 0) { max_slots = tiles::kVisTileSlots; max_trk = tiles::kMaxTrkPerTile; }
  VisTilesOut* o = new VisTilesOut;
  VisualLayout& L = o->L;
  std::vector<int64_t> valid((size_t)T);
  std::iota(valid.begin(), valid.end(), (int64_t)0);
  std::vector<int> min_cam, min_row;
  visual_first_rows(n_rows, valid.data(), T, obs_ptr, obs_cam, row_of_cam, min_cam, min_row);
  visual_layout(n_rows, valid.data(), T, nullptr, min_row.data(), obs_ptr, obs_cam, row_of_cam, L, max_slots, max_trk);
  for (int64_t k = 0; k < L.Tv; ++k) {
    o->order.push_back(L.trk_id[k]);
    for (int64_t q = obs_ptr[L.trk_id[k]]; q < obs_ptr[L.trk_id[k] + 1]; ++q) o->row.push_back(row_of_cam[obs_cam[q]]);
  }
  HostExec ex;
  const tiles::VisTableIn in{(int64_t)L.tile_trk.size() - 1, n_rows, nblocks, L.tile_trk.data(), L.trk_ptr.data(), o->row.data(), nullptr,
                             first, row_start};
  int64_t n_pairs = 0;
  if (visual_tables(ex, in, L.Tv_small, L.n_ordered, L.nnz, o->prun, o->drun, &n_pairs)) { delete o; return nullptr; }
  return o;
}

// which: 0 order, 1 trk_ptr, 2 row, 3 tile_trk (int32 / int64 as listed in tests/test_visual_tiles_emu.py), 4 pair codes,
// 5 pair run_ptr, 6 pair tile_run, 7 observation codes, 8 observation run_ptr, 9 observation tile_run
extern "C" int64_t emu_vis_tiles_get(void* h, int which, void* dst) {
  VisTilesOut* o = static_cast<VisTilesOut*>(h);
  auto out = [&](const auto* p, size_t n) {
    if (dst) std::memcpy(dst, p, n * sizeof(*p));
    return (int64_t)n;
  };
  switch (which) {
    case 0: return out(o->order.data(), o->order.size());
    case 1: return out(o->L.trk_ptr.data(), o->L.trk_ptr.size());
    case 2: return out(o->row.data(), o->row.size());
    case 3: return out(o->L.tile_trk.data(), o->L.tile_trk.size());
    case 4: return out(o->prun.code.p, o->prun.code.n);
    case 5: return out(o->prun.run_ptr.p, o->prun.run_ptr.n);
    case 6: return out(o->prun.tile_run.p, o->prun.tile_run.n);
    case 7: return out(o->drun.code.p, o->drun.code.n);
    case 8: return out(o->drun.run_ptr.p, o->drun.run_ptr.n);
    case 9: return out(o->drun.tile_run.p, o->drun.tile_run.n);
  }
  return -1;
}

extern "C" void emu_vis_tiles_free(void* h) { delete static_cast<VisTilesOut*>(h); }
