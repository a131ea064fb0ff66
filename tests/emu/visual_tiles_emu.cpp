// visual_tiles_emu.cpp — TEST INFRASTRUCTURE: the set-up of the reduced camera system build's tiles and destination table
// (global-lvba_b200/csrc/visual_tiles.h) run through the host policy, so that tests/test_visual_tiles_emu.py can check the
// table without a GPU.  The same steps as visual_create_impl: landmark order, local CSR, tiles, the two runs tables.  Never
// part of the product.
#include <vector>

#include "../../global-lvba_b200/csrc/visual_tiles.h"
#include "host_exec.h"

struct VisTilesOut {
  std::vector<int64_t> order;
  std::vector<int> trk_ptr, row, tile_trk;
  lvba::tiles::Runs<HostExec> prun, drun;
};

extern "C" int emu_vis_tile_slots() { return lvba::tiles::kVisTileSlots; }
extern "C" int emu_vis_max_trk_per_tile() { return lvba::tiles::kMaxTrkPerTile; }

// obs_row: system row of every observation in the caller's order, -1 for a constant camera.  first / row_start: the envelope
// of the reduced camera system.  max_slots <= 0: the library's tile size.
extern "C" void* emu_vis_tiles_build(int n_rows, int64_t T, const int64_t* obs_ptr, const int32_t* obs_row, const int* first,
                                     const long long* row_start, long long nblocks, int max_slots, int max_trk) {
  using namespace lvba::tiles;
  if (max_slots <= 0) { max_slots = kVisTileSlots; max_trk = kMaxTrkPerTile; }
  VisTilesOut* o = new VisTilesOut;
  std::vector<int> key((size_t)T);
  for (int64_t i = 0; i < T; ++i) {
    int m = INT32_MAX;
    for (int64_t q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q) if (obs_row[q] >= 0) m = std::min(m, (int)obs_row[q]);
    key[(size_t)i] = m == INT32_MAX ? 0 : m;
  }
  o->order = order_by_key(std::max(n_rows, 1), key.data(), T);
  o->trk_ptr.push_back(0);
  for (int64_t a : o->order) {
    for (int64_t q = obs_ptr[a]; q < obs_ptr[a + 1]; ++q) o->row.push_back(obs_row[q]);
    o->trk_ptr.push_back((int)o->row.size());
  }
  o->tile_trk = cut_ranges(T, o->trk_ptr.data(), nullptr, max_slots, max_trk);
  HostExec ex;
  std::vector<long long> cnt((size_t)T + 1), trk_pair((size_t)T + 1);
  ex.for_each(T + 1, VisPairCountF{o->trk_ptr.data(), T, cnt.data()});
  ex.exclusive_scan(cnt.data(), trk_pair.data(), T + 1);
  const VisTableIn in{(int64_t)o->tile_trk.size() - 1, n_rows, nblocks, o->tile_trk.data(), o->trk_ptr.data(), o->row.data(),
                      trk_pair.data(), first, row_start};
  if (sort_runs(ex, trk_pair[(size_t)T], in.n_tiles, (uint64_t)nblocks, VisPairKeyF{in}, o->prun) ||
      sort_runs(ex, (int64_t)o->row.size(), in.n_tiles, (uint64_t)n_rows, ObsKeyF{in}, o->drun)) {
    delete o;
    return nullptr;
  }
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
    case 1: return out(o->trk_ptr.data(), o->trk_ptr.size());
    case 2: return out(o->row.data(), o->row.size());
    case 3: return out(o->tile_trk.data(), o->tile_trk.size());
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
