// lidar_tiles.h — voxel order, tiles and destination table of the LiDAR Hessian build (lidar_build_kernel, lidar.cuh).
//
// The build sums every distinct H block and gradient row of a tile on chip and writes it with one RED per element, so the
// RED count falls with the number of voxels of a tile that share a pose pair.  Three pieces set that up once per structure:
//   * order_by_lowest_pose: the voxels in the order of their lowest pose (stable counting sort, O(V + W)).  Neighbouring
//     voxels then share poses, and windows of the batched window BA (consecutive pose ranges) come out contiguous.
//   * cut_ranges: consecutive voxels into tiles of <= max_slots slots and <= max_vox voxels, never across a window.
//   * build_runs: per tile, the (slot i, slot j) pose pairs grouped by destination H block, and the slots grouped by pose
//     (diagonal blocks and gradient rows).  Functors over items run by an execution policy: CudaExec (exec.cuh) in the
//     library, the host policy of tests/emu in the CPU tests.  Its radix sort and run passes (sort_runs) also build the
//     table of the reduced camera system build (visual_tiles.h).
#pragma once
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define LVBA_THD __host__ __device__ __forceinline__
#else
#define LVBA_THD inline
#endif

namespace lvba {
namespace tiles {

constexpr int kTileSlots = 256;              // slots (threads) per tile CTA of the Hessian build (faster than 512 on the H100)
constexpr int kMaxVoxPerTile = kTileSlots / 2;
constexpr int kSlots = 128;                  // slots (threads) per batch CTA of the residual pass and of the visual kernels; the most
                                             // poses a voxel of the tiles may have (more: lidar_big.h)

// The voxels `in[0..n)` (all voxels 0..n-1 when `in` is null), stably ordered by their lowest pose index (pose_idx is ascending
// inside a voxel), as a local CSR: slot0[i] = first slot of local voxel i in the caller's arrays, l_vox_ptr[i] = its first local
// slot (l_vox_ptr has n + 1 entries).  Returns the number of slots.  Two sequential passes over the caller's CSR.
inline int64_t order_by_lowest_pose(int W, const int64_t* in, int64_t n, const int64_t* vox_ptr, const int32_t* pose_idx,
                                    std::vector<int>& slot0, std::vector<int>& l_vox_ptr) {
  std::vector<int64_t> at((size_t)W + 1, 0);
  for (int64_t j = 0; j < n; ++j) ++at[(size_t)pose_idx[vox_ptr[in ? in[j] : j]] + 1];
  for (int r = 0; r < W; ++r) at[(size_t)r + 1] += at[(size_t)r];
  slot0.resize((size_t)n); l_vox_ptr.assign((size_t)n + 1, 0);
  for (int64_t j = 0; j < n; ++j) {
    const int64_t a = in ? in[j] : j;
    const size_t i = (size_t)at[(size_t)pose_idx[vox_ptr[a]]]++;
    slot0[i] = (int)vox_ptr[a]; l_vox_ptr[i + 1] = (int)(vox_ptr[a + 1] - vox_ptr[a]);
  }
  for (int64_t i = 0; i < n; ++i) l_vox_ptr[(size_t)i + 1] += l_vox_ptr[(size_t)i];
  return l_vox_ptr[(size_t)n];
}

// voxel ranges [r[k], r[k+1]) of consecutive voxels with <= max_slots slots and <= max_vox voxels each; with `grp` (window
// of every voxel) a range never holds two windows.  A voxel has <= max_slots slots.
inline std::vector<int> cut_ranges(int64_t V, const int* vox_ptr, const int* grp, int max_slots, int max_vox) {
  std::vector<int> r{0};
  int ns = 0, nv = 0;
  for (int64_t i = 0; i < V; ++i) {
    const int K = vox_ptr[i + 1] - vox_ptr[i];
    const bool new_grp = grp && i > 0 && grp[i] != grp[i - 1];
    if (nv > 0 && (ns + K > max_slots || nv + 1 > max_vox || new_grp)) { r.push_back((int)i); ns = 0; nv = 0; }
    ns += K; ++nv;
  }
  if (V > 0) r.push_back((int)V);
  return r;
}

struct TableIn {
  int64_t n_tiles;
  int W;
  long long nblocks;            // blocks of the envelope
  const int* tile_vox;          // [n_tiles + 1] voxel range of every tile
  const int* vox_ptr;           // [V + 1] slot offsets (the tiles' voxel order)
  const int* pidx;              // [nnz] pose of every slot
  const long long* vox_pair;    // [V + 1] prefix sums of K (K - 1) / 2
  const int* first;             // envelope first[] per row
  const long long* row_start;   // envelope row_start[] per row
  // constant poses (lvba_lidar_opts::pose_fixed): row_of[pose] = its row of the pose system, -1 for a constant pose; null: every
  // pose is its own row.  A pair or slot of a constant pose has no destination.
  const int* row_of = nullptr;
};

LVBA_THD int row_of_pose(const TableIn& q, int pose) { return q.row_of ? q.row_of[pose] : pose; }

// items 0..V: cnt[i] = pose pairs of local voxel i (0 for i = V); its exclusive scan is TableIn::vox_pair
struct PairCountF {
  const int* vox_ptr; int64_t V; long long* cnt;
  LVBA_THD void operator()(int64_t i) const {
    const long long K = i < V ? vox_ptr[i + 1] - vox_ptr[i] : 0;
    cnt[i] = K * (K - 1) / 2;
  }
};

// one item per pose pair (i < j) of a voxel: key = (tile, lower-envelope block (pose_j, pose_i)), code = li | lj << 16 (slots
// local to the tile).  key / code are set by sort_runs.
struct PairKeyF {
  TableIn in; uint64_t* key = nullptr; uint32_t* code = nullptr;
  LVBA_THD void operator()(int64_t p) const {
    const TableIn& q = in;
    int64_t t = 0, hi = q.n_tiles;                            // tile: the last one starting at or before p
    while (hi - t > 1) { const int64_t m = (t + hi) >> 1; if (q.vox_pair[q.tile_vox[m]] <= p) t = m; else hi = m; }
    int64_t a = q.tile_vox[t];                                // voxel: the last one of the tile starting at or before p
    hi = q.tile_vox[t + 1];
    while (hi - a > 1) { const int64_t m = (a + hi) >> 1; if (q.vox_pair[m] <= p) a = m; else hi = m; }
    const int64_t r = p - q.vox_pair[a];                      // strict lower-triangular index: r = j (j - 1) / 2 + i, j > i
    int64_t j = (int64_t)((sqrt(8.0 * (double)r + 1.0) + 1.0) * 0.5);
    while (j * (j - 1) / 2 > r) --j;
    while ((j + 1) * j / 2 <= r) ++j;
    const int64_t i = r - j * (j - 1) / 2;
    const int s0 = q.vox_ptr[q.tile_vox[t]];
    const int si = q.vox_ptr[a] + (int)i, sj = q.vox_ptr[a] + (int)j;
    const int pi = row_of_pose(q, q.pidx[si]), pj = row_of_pose(q, q.pidx[sj]);   // ascending inside a voxel: pi < pj
    key[p] = (pi < 0 || pj < 0) ? (uint64_t)q.n_tiles * (uint64_t)q.nblocks
                                : (uint64_t)t * (uint64_t)q.nblocks + (uint64_t)(q.row_start[pj] + (pi - q.first[pj]));
    code[p] = (uint32_t)(si - s0) | ((uint32_t)(sj - s0) << 16);
  }
};

// one item per slot: key = (tile, pose), code = slot local to the tile (a slot of a constant pose: no destination)
struct SlotKeyF {
  TableIn in; uint64_t* key = nullptr; uint32_t* code = nullptr;
  LVBA_THD void operator()(int64_t s) const {
    const TableIn& q = in;
    int64_t t = 0, hi = q.n_tiles;
    while (hi - t > 1) { const int64_t m = (t + hi) >> 1; if (q.vox_ptr[q.tile_vox[m]] <= s) t = m; else hi = m; }
    key[s] = row_of_pose(q, q.pidx[s]) < 0 ? (uint64_t)q.n_tiles * (uint64_t)q.W : (uint64_t)t * (uint64_t)q.W + (uint64_t)q.pidx[s];
    code[s] = (uint32_t)(s - q.vox_ptr[q.tile_vox[t]]);
  }
};

// The sorted keys are tile * tile_keys + destination, followed by the items that have no destination (key = end, the number of
// tiles times tile_keys).  items 0..n: flag[p] = 1 where a run of equal keys starts (flag[n] = 0)
struct RunFlagF {
  const uint64_t* key; int64_t n; uint64_t end; int64_t* flag;
  LVBA_THD void operator()(int64_t p) const { flag[p] = (p < n && key[p] < end && (p == 0 || key[p] != key[p - 1])) ? 1 : 0; }
};
// items 0..n: run_ptr[r] = first item of run r, run_ptr[R] = the first item without a destination (n when there is none)
struct RunStartF {
  const uint64_t* key; const int64_t* flag; const int64_t* pos; int64_t n; uint64_t end; int64_t* run_ptr;
  LVBA_THD void operator()(int64_t p) const {
    if (p == n || key[p] >= end) { if (p == 0 || key[p - 1] < end) run_ptr[pos[p]] = p; }
    else if (flag[p]) run_ptr[pos[p]] = p;
  }
};
// items 0..n_tiles: tile_run[t] = first run of tile t, the run of the first sorted key >= t * tile_keys
struct TileRunF {
  const uint64_t* key; int64_t n; uint64_t tile_keys; const int64_t* pos; int64_t* tile_run;
  LVBA_THD void operator()(int64_t t) const {
    const uint64_t k = (uint64_t)t * tile_keys;
    int64_t lo = 0, hi = n;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (key[m] < k) lo = m + 1; else hi = m; }
    tile_run[t] = pos[lo];
  }
};

// items grouped by destination: run r of tile t (tile_run[t] <= r < tile_run[t + 1]) is code[run_ptr[r] .. run_ptr[r + 1])
template <class Ex>
struct Runs {
  typename Ex::template Buf<uint32_t> code;
  typename Ex::template Buf<int64_t> run_ptr;    // [n_runs + 1]
  typename Ex::template Buf<int64_t> tile_run;   // [n_tiles + 1]
  int64_t n_runs = 0;
};

// The n items of KeyF (a functor over items with members key and code: key = tile * tile_keys + destination < tile_keys, or
// n_tiles * tile_keys for an item without a destination) grouped by destination.  Inside a run the items keep their enumeration
// order (stable sort).
template <class Ex, class KeyF>
int sort_runs(Ex& ex, int64_t n, int64_t n_tiles, uint64_t tile_keys, KeyF kf, Runs<Ex>& out) {
#define LVBA_TILES_TRY(call) do { int rc__ = (call); if (rc__ != 0) return rc__; } while (0)
  typename Ex::template Buf<uint64_t> key, key_s;
  typename Ex::template Buf<uint32_t> code;
  typename Ex::template Buf<int64_t> flag, pos;
  LVBA_TILES_TRY(key.alloc((size_t)n)); LVBA_TILES_TRY(key_s.alloc((size_t)n));
  LVBA_TILES_TRY(code.alloc((size_t)n)); LVBA_TILES_TRY(out.code.alloc((size_t)n));
  kf.key = key.p; kf.code = code.p;
  LVBA_TILES_TRY(ex.for_each(n, kf));
  const uint64_t end = (uint64_t)n_tiles * tile_keys;
  int bits = 1;
  while (bits < 64 && (end >> bits) != 0) ++bits;
  LVBA_TILES_TRY(ex.sort_pairs(key.p, key_s.p, code.p, out.code.p, n, bits));
  LVBA_TILES_TRY(flag.alloc((size_t)n + 1)); LVBA_TILES_TRY(pos.alloc((size_t)n + 1));
  LVBA_TILES_TRY(ex.for_each(n + 1, RunFlagF{key_s.p, n, end, flag.p}));
  LVBA_TILES_TRY(ex.exclusive_scan(flag.p, pos.p, n + 1));
  LVBA_TILES_TRY(ex.fetch(&out.n_runs, pos.p + n, 1));
  LVBA_TILES_TRY(out.run_ptr.alloc((size_t)out.n_runs + 1));
  LVBA_TILES_TRY(ex.for_each(n + 1, RunStartF{key_s.p, flag.p, pos.p, n, end, out.run_ptr.p}));
  LVBA_TILES_TRY(out.tile_run.alloc((size_t)n_tiles + 1));
  LVBA_TILES_TRY(ex.for_each(n_tiles + 1, TileRunF{key_s.p, n, tile_keys, pos.p, out.tile_run.p}));
  return ex.sync();                                          // the scratch buffers are released on return
#undef LVBA_TILES_TRY
}

// by_slot = false: the pose pairs of every voxel (n = vox_pair[V]) grouped by H block; true: the slots (n = vox_ptr[V])
// grouped by pose.
template <class Ex>
int build_runs(Ex& ex, const TableIn& in, bool by_slot, int64_t n, Runs<Ex>& out) {
  if (by_slot) return sort_runs(ex, n, in.n_tiles, (uint64_t)in.W, SlotKeyF{in}, out);
  return sort_runs(ex, n, in.n_tiles, (uint64_t)in.nblocks, PairKeyF{in}, out);
}

// ---- fixed-order sums (deterministic mode).  Where the default build adds a run's sum into its destination by RED, the
// deterministic build stores it into a record of its own: the records of the tiles' runs in (tile, run) order, then those of
// the items of lidar_big.h in item order.  FixedSum lists per destination its records in ascending order (a stable sort of the
// records by destination), and GatherF adds them up in that order, so that every run gives the same bits.
template <class Ex>
struct FixedSum {
  typename Ex::template Buf<double> rec;     // [n_rec][width] one record per contribution
  typename Ex::template Buf<int64_t> dst;    // [n_rec] destination of every record, in units of width elements
  Runs<Ex> by_dst;                           // run r = the records of one destination, ascending
  int64_t n_rec = 0;
  int width = 0;
  int64_t bytes() const {
    return n_rec * (int64_t)(width * sizeof(double) + sizeof(int64_t) + sizeof(uint32_t)) + (by_dst.n_runs + 3) * (int64_t)sizeof(int64_t);
  }
};

template <class Ex>
int fixed_sum_alloc(FixedSum<Ex>& f, int64_t n_rec, int width) {
  f.n_rec = n_rec; f.width = width;
  const int rc = f.rec.alloc((size_t)std::max<int64_t>(n_rec, 1) * (size_t)width);
  return rc != 0 ? rc : f.dst.alloc((size_t)std::max<int64_t>(n_rec, 1));
}

// the memory of f (device policy: a set-up that failed part-way leaves nothing on its handle)
template <class Ex>
void fixed_sum_release(FixedSum<Ex>& f) {
  f.rec.release(); f.dst.release(); f.by_dst.code.release(); f.by_dst.run_ptr.release(); f.by_dst.tile_run.release();
  f.by_dst.n_runs = 0; f.n_rec = 0;
}

// items 0..n_rec: key = destination, code = record.  A record whose destination is n_dest has none (fixed_sum_index leaves it
// out of the runs).
struct RecKeyF {
  const int64_t* dst; uint64_t* key = nullptr; uint32_t* code = nullptr;
  LVBA_THD void operator()(int64_t p) const { key[p] = (uint64_t)dst[p]; code[p] = (uint32_t)p; }
};

// after f.dst is filled: the records grouped by destination (< n_dest); the records keep their order inside a group
template <class Ex>
int fixed_sum_index(Ex& ex, FixedSum<Ex>& f, int64_t n_dest) {
  return sort_runs(ex, f.n_rec, 1, (uint64_t)n_dest, RecKeyF{f.dst.p}, f.by_dst);
}

// items 0..n_runs * n_el: element el0 + e of destination run r = the sum of its records in ascending order, written to
// out[destination * n_el + e].  Records are `width` doubles apart.  Destinations without a record are not written.
struct GatherF {
  const int64_t* run_ptr; const uint32_t* code; const int64_t* dst; const double* rec; int width, el0, n_el; double* out;
  LVBA_THD void operator()(int64_t i) const {
    const int64_t r = i / n_el;
    const int e = (int)(i - r * n_el);
    const int64_t qa = run_ptr[r], qb = run_ptr[r + 1];
    double v = 0.0;
    for (int64_t q = qa; q < qb; ++q) v += rec[(int64_t)code[q] * width + el0 + e];
    out[dst[code[qa]] * n_el + e] = v;
  }
};
// the whole record of f's own records
template <class Ex>
GatherF gather_of(const FixedSum<Ex>& f, double* out) {
  return GatherF{f.by_dst.run_ptr.p, f.by_dst.code.p, f.dst.p, f.rec.p, f.width, 0, f.width, out};
}
// elements el0 .. el0 + n_el of other records `rec` (width doubles each) with the destinations and order of f
template <class Ex>
GatherF gather_part(const FixedSum<Ex>& f, const double* rec, int width, int el0, int n_el, double* out) {
  return GatherF{f.by_dst.run_ptr.p, f.by_dst.code.p, f.dst.p, rec, width, el0, n_el, out};
}

// Destinations of the records of the LiDAR build (lidar_build_kernel<true, *>): one item per pair run (the lower H block of its
// pose pair), one per pose run (the diagonal H block and the gradient row of its pose), addressed by row.  The runs hold only
// pairs and slots with rows.  tile_run / run_ptr / code: a Runs.
LVBA_THD int64_t tile_of_run(const int64_t* tile_run, int64_t n_tiles, int64_t r) {
  int64_t t = 0, hi = n_tiles;                                 // the last tile whose runs start at or before r
  while (hi - t > 1) { const int64_t m = (t + hi) >> 1; if (tile_run[m] <= r) t = m; else hi = m; }
  return t;
}
struct PairRunDstF {
  TableIn in; const int64_t* tile_run; const int64_t* run_ptr; const uint32_t* code; int64_t* dst_H;
  LVBA_THD void operator()(int64_t r) const {
    const int s0 = in.vox_ptr[in.tile_vox[tile_of_run(tile_run, in.n_tiles, r)]];
    const uint32_t c = code[run_ptr[r]];
    const int pi = row_of_pose(in, in.pidx[s0 + (int)(c & 0xffff)]), pj = row_of_pose(in, in.pidx[s0 + (int)(c >> 16)]);
    dst_H[r] = in.row_start[pj] + (pi - in.first[pj]);
  }
};
struct SlotRunDstF {
  TableIn in; const int64_t* tile_run; const int64_t* run_ptr; const uint32_t* code; int64_t* dst_H; int64_t* dst_g;
  LVBA_THD void operator()(int64_t r) const {
    const int s0 = in.vox_ptr[in.tile_vox[tile_of_run(tile_run, in.n_tiles, r)]];
    const int row = row_of_pose(in, in.pidx[s0 + (int)code[run_ptr[r]]]);
    dst_H[r] = in.row_start[row] + (row - in.first[row]);
    dst_g[r] = row;
  }
};

}  // namespace tiles
}  // namespace lvba
