// visual_tiles.h — landmark order, tiles and destination table of the reduced camera system build (visual_build_kernel,
// visual.cuh).
//
// The build sums every distinct S block, diagonal block, rhs, column-norm and gradient row of a tile on chip and writes it
// with one RED per element, so the RED count falls with the number of landmarks of a tile that share cameras:
//   * order_by_key: the landmarks a rank owns, stably ordered by the lowest system row of their clique (counting sort,
//     O(Tv + n_rows)).  Neighbouring landmarks then share cameras.
//   * tiles::cut_ranges (lidar_tiles.h): consecutive landmarks into tiles of <= kVisTileSlots observations.
//   * tiles::sort_runs over VisPairKeyF / ObsKeyF: per tile, the camera-pair contributions grouped by destination S block,
//     and the observations grouped by system row.  The same functor passes as the LiDAR table, run by CudaExec (exec.cuh)
//     in the library and by the host policy of tests/emu in the CPU tests.
#pragma once
#include "lidar_tiles.h"

namespace lvba {
namespace tiles {

constexpr int kVisTileSlots = 256;             // observations (threads) per tile CTA of the reduced camera system build
constexpr int kMaxTrkPerTile = 128;            // landmarks per tile
constexpr int kMaxTrkPerBatch = 128;           // landmarks per batch CTA (<= kSlots observations) of back-substitution and cost

// 0..n-1 stably ordered by key[] in [0, n_keys)
inline std::vector<int64_t> order_by_key(int n_keys, const int* key, int64_t n) {
  std::vector<int64_t> at((size_t)n_keys + 1, 0), out((size_t)n);
  for (int64_t j = 0; j < n; ++j) ++at[(size_t)key[j] + 1];
  for (int r = 0; r < n_keys; ++r) at[(size_t)r + 1] += at[(size_t)r];
  for (int64_t j = 0; j < n; ++j) out[(size_t)at[(size_t)key[j]]++] = j;
  return out;
}

struct VisTableIn {
  int64_t n_tiles;
  int n_rows;                   // rows of the reduced camera system
  long long nblocks;            // blocks of its envelope
  const int* tile_trk;          // [n_tiles + 1] landmark range of every tile
  const int* trk_ptr;           // [Tv + 1] observation offsets (the tiles' landmark order)
  const int* obs_row;           // [nnz] system row of every observation, -1 for a constant camera
  const long long* trk_pair;    // [Tv + 1] prefix sums of K (K - 1)
  const int* first;             // envelope first[] per row
  const long long* row_start;   // envelope row_start[] per row
};

// items 0..Tv: cnt[i] = ordered observation pairs (x != y) of local landmark i (0 for i = Tv); its exclusive scan is
// VisTableIn::trk_pair
struct VisPairCountF {
  const int* trk_ptr; int64_t Tv; long long* cnt;
  LVBA_THD void operator()(int64_t i) const {
    const long long K = i < Tv ? trk_ptr[i + 1] - trk_ptr[i] : 0;
    cnt[i] = K * (K - 1);
  }
};

// One item per ordered observation pair (x, y), x != y, of a landmark.  It contributes -Y_x E_y^T to the lower-envelope block
// (row_x, row_y) when both rows are >= 0 and row_x >= row_y: every unordered pair once, a camera observed twice in both
// orders.  key = (tile, block), code = x | y << 16 (observations local to the tile); the other items have no destination.
struct VisPairKeyF {
  VisTableIn in; uint64_t* key = nullptr; uint32_t* code = nullptr;
  LVBA_THD void operator()(int64_t p) const {
    const VisTableIn& q = in;
    int64_t t = 0, hi = q.n_tiles;                            // tile: the last one starting at or before p
    while (hi - t > 1) { const int64_t m = (t + hi) >> 1; if (q.trk_pair[q.tile_trk[m]] <= p) t = m; else hi = m; }
    int64_t a = q.tile_trk[t];                                // landmark: the last one of the tile starting at or before p
    hi = q.tile_trk[t + 1];
    while (hi - a > 1) { const int64_t m = (a + hi) >> 1; if (q.trk_pair[m] <= p) a = m; else hi = m; }
    const int64_t r = p - q.trk_pair[a], K1 = q.trk_ptr[a + 1] - q.trk_ptr[a] - 1;
    const int64_t x = r / K1, y0 = r - x * K1, y = y0 + (y0 >= x);
    const int sx = q.trk_ptr[a] + (int)x, sy = q.trk_ptr[a] + (int)y;
    const int rx = q.obs_row[sx], ry = q.obs_row[sy];
    const int s0 = q.trk_ptr[q.tile_trk[t]];
    key[p] = (ry >= 0 && rx >= ry) ? (uint64_t)t * (uint64_t)q.nblocks + (uint64_t)(q.row_start[rx] + (ry - q.first[rx]))
                                   : (uint64_t)q.n_tiles * (uint64_t)q.nblocks;
    code[p] = (uint32_t)(sx - s0) | ((uint32_t)(sy - s0) << 16);
  }
};

// one item per observation: key = (tile, row), code = observation local to the tile; a constant camera has no destination
struct ObsKeyF {
  VisTableIn in; uint64_t* key = nullptr; uint32_t* code = nullptr;
  LVBA_THD void operator()(int64_t s) const {
    const VisTableIn& q = in;
    int64_t t = 0, hi = q.n_tiles;
    while (hi - t > 1) { const int64_t m = (t + hi) >> 1; if (q.trk_ptr[q.tile_trk[m]] <= s) t = m; else hi = m; }
    const int r = q.obs_row[s];
    key[s] = (uint64_t)(r >= 0 ? t * q.n_rows + r : q.n_tiles * q.n_rows);
    code[s] = (uint32_t)(s - q.trk_ptr[q.tile_trk[t]]);
  }
};

// Destinations of the records of the deterministic visual build (visual_build_kernel<true>, visual_colnorm_kernel<true>), in
// the units of FixedSum (lidar_tiles.h): one item per pair run (its lower S block), one per row run (the row's diagonal S block
// and its rhs / column-norm / gradient row).  tile_run / run_ptr / code: a Runs.
struct VisPairRunDstF {
  VisTableIn in; const int64_t* tile_run; const int64_t* run_ptr; const uint32_t* code; int64_t* dst_S;
  LVBA_THD void operator()(int64_t r) const {
    const int s0 = in.trk_ptr[in.tile_trk[tile_of_run(tile_run, in.n_tiles, r)]];
    const uint32_t c = code[run_ptr[r]];
    const int rx = in.obs_row[s0 + (int)(c & 0xffff)], ry = in.obs_row[s0 + (int)(c >> 16)];
    dst_S[r] = in.row_start[rx] + (ry - in.first[rx]);
  }
};
struct ObsRunDstF {
  VisTableIn in; const int64_t* tile_run; const int64_t* run_ptr; const uint32_t* code; int64_t* dst_S; int64_t* dst_row;
  LVBA_THD void operator()(int64_t r) const {
    const int s0 = in.trk_ptr[in.tile_trk[tile_of_run(tile_run, in.n_tiles, r)]];
    const int row = in.obs_row[s0 + (int)code[run_ptr[r]]];
    dst_S[r] = in.row_start[row] + (row - in.first[row]);
    dst_row[r] = row;
  }
};

}  // namespace tiles
}  // namespace lvba
