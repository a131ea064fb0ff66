// nd_kernels.cuh — device kernels of the substructured block LDL^T (nd_plan.h / nd_passes.h): the multi-right-hand-side
// forward substitution ("spike") through a finished block factor and the symmetric rank update it feeds.
//
// Both serve the solve the reference gets from Eigen::SimplicialLDLT (include/BALM/bavoxel.hpp:695-710) / Ceres
// DENSE_SCHUR (src/lvba_system.cpp:1573-1575).  Neither is on the pivot chain of a factorisation: they only read
// finished columns of L, so they run on SMs the factorising CTAs leave idle (one CTA per group of right-hand sides / per
// tile of the update), FP64 FMA + shared memory, no HBM traffic to speak of (everything is L2 resident).
#pragma once
#include "envelope.cuh"
#include "factor_la.cuh"
#include "nd_passes.h"

namespace lvba {

// grid-stride item pass (functors of nd_passes.h)
template <class F>
__global__ void __launch_bounds__(256) nd_pass_kernel(long long n, F f) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) f(i);
}

// ---------------------------------------------------------------------------------------------------------------
// Spike: Z = L^-1 E for KS right-hand sides (SpikeJob, nd_passes.h).  blockIdx.x = group of kSpikeCols right-hand sides,
// blockIdx.y = job.
//
// Row k of the recurrence is  z_k = e_k - sum_j L_kj z_j  over the <= 30 blocks of row k of L.  A warp owns kSpikeC
// right-hand sides for the whole job and its LANE owns one block: lane s multiplies L_{k, first+s} — fetched ONCE, 18
// LDS.128 — with the kSpikeC columns of z_{first+s} (36 DFMA per column), then a reduce-scatter over the 32 lanes (xor 16,
// 8, 4 halve the 6 x kSpikeC partial sums, xor 2, 1 finish them: 27 shuffles for 24 values) leaves every output with one
// lane of eight.  Letting every lane fetch whole blocks for ONE right-hand side instead moves 43 kB per warp and row
// through the shared-memory return path (128 B/clk per SM); here it is 15 kB.
// The last 32 block rows of Z of the warp's columns live in shared memory private to the warp (column height <= 30), so the
// only block-wide hand-shake per row is the one that publishes the next row of L: its blocks are contiguous in the envelope
// and are staged by cp.async two rows ahead, into slots of 38 doubles (consecutive lanes 48 bytes apart modulo 128:
// conflict-free LDS.128).  Row labels (first / row_start) and the entering rows of E are fetched four / one rows ahead: no
// global-memory latency sits on the row-to-row chain.  (Labels in a shared-memory ring + E rows by cp.async
// do not help: the loop is bound by the number of instructions a warp issues per row, not by a load latency.)
constexpr int kSpikeC = 4;                       // right-hand sides per warp
constexpr int kSpikeWarps = 4;
constexpr int kSpikeCols = kSpikeC * kSpikeWarps;   // right-hand sides per CTA
constexpr int kSpikeThreads = 32 * kSpikeWarps;
constexpr int kSpikeZStride = 26;                // doubles per block row of a warp's Z window: [6][4] + 2 (lanes 80 bytes apart modulo 128)
constexpr int kSpikeBS = 38;                     // doubles per staged block of L
constexpr int kSpikeBufs = 3;                    // rows of L in flight (cp.async, two rows ahead)
constexpr size_t kSpikeSmem = sizeof(double) * (kSpikeBufs * 32 * kSpikeBS + kSpikeWarps * 33 * kSpikeZStride);
constexpr int kSpikePublish = 4;                 // rows of Z between two publications of SpikeJob::zprog
static_assert(kSpikeC == 4, "the reduce-scatter below is written for 24 values per lane");

__global__ void __launch_bounds__(kSpikeThreads)
nd_spike_kernel(const nd::SpikeJob* __restrict__ jobs) {
  pdl_launch_dependents();                                     // the SYRK that follows this spike's rows (nd_syrk_kernel)
  extern __shared__ __align__(16) double smem_spike[];
  double* sRow = smem_spike;                                   // [kSpikeBufs][32][kSpikeBS] blocks of rows k, k+1, k+2
  const nd::SpikeJob J = jobs[blockIdx.y];
  const EnvView e = J.e;
  const int c0 = blockIdx.x * kSpikeCols;
  if (c0 >= J.KS) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cw = c0 + warp * kSpikeC;                          // first right-hand side of this warp
  double* sZw = smem_spike + kSpikeBufs * 32 * kSpikeBS + warp * 33 * kSpikeZStride;   // [32 rows + 1 zero row][6][4]
  const int n = e.n, n_stop = J.n_stop, KS = J.KS;
  if (lane < kSpikeZStride) sZw[32 * kSpikeZStride + lane] = 0.0;        // row 32: zeros (operand of the lanes without a block)
  for (int o = tid; o < kSpikeBufs * 32 * kSpikeBS; o += kSpikeThreads) sRow[o] = 0.0;   // L slots never hold non-finite garbage
  const int sb0 = tid / 18, sh = tid - sb0 * 18;
  // after the reduce-scatter lane l (l & 3 == 0) holds the outputs o = 3 (l >> 2) + {0, 1, 2} of the 24 (o = x * 4 + column)
  const int og = (lane >> 2) * 3;
  const bool owner = (lane & 3) == 0;
  int ox[3], oc[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) { ox[q] = (og + q) >> 2; oc[q] = (og + q) & 3; }
  __syncthreads();
  auto stage_row = [&](int k, int f, long long rs) {           // blocks (k, f .. min(k, n_stop)-1) -> sRow[k % 3]
    if (k >= n) return;
    const int jend = k < n_stop ? k : n_stop;
    const int nb = jend > f ? jend - f : 0;
    const double* src = J.L + rs * 36;
    double* dst = sRow + (k % kSpikeBufs) * (32 * kSpikeBS);
    if (tid < 126)                                             // thread -> (block, 16-byte piece): 7 blocks per sweep
      for (int b = sb0; b < nb; b += 7) cp_async16_zfill(dst + b * kSpikeBS + 2 * sh, src + b * 36 + 2 * sh, true);
  };
  // labels: row k (f0), rows k+1 .. k+3 (f1..f3, rs2, rs3): fetched four rows ahead of their use in the chain
  int f0 = e.first[0];
  int f1 = n > 1 ? e.first[1] : 0; long long rs1 = n > 1 ? e.row_start[1] : 0;
  int f2 = n > 2 ? e.first[2] : 0; long long rs2 = n > 2 ? e.row_start[2] : 0;
  int f3 = n > 3 ? e.first[3] : 0; long long rs3 = n > 3 ? e.row_start[3] : 0;
  double en[3];                                                // E of the next row: this lane's three outputs
#pragma unroll
  for (int q = 0; q < 3; ++q) en[q] = (owner && cw + oc[q] < KS && 0 < J.nE) ? J.E[((long long)ox[q]) * KS + cw + oc[q]] : 0.0;
  // side by side with the factorisation (J.progress): row r of L is final once min(r, n_stop) columns are; one thread polls, the
  // block barrier hands the acquired view to the others (the rows are fetched by cp.async.cg: L2, never a stale L1 line)
  int seen = J.progress ? 0 : 0x7fffffff;
  auto wait_row = [&](int r) {
    const int need = r < n_stop ? r : n_stop;
    if (tid == 0) while (seen < need) { seen = progress_read(J.progress); if (seen < need) __nanosleep(100); }
  };
  wait_row(1);
  __syncthreads();
  stage_row(0, f0, e.row_start[0]);
  asm volatile("cp.async.commit_group;" ::: "memory");
  stage_row(1, f1, rs1);
  asm volatile("cp.async.commit_group;" ::: "memory");
  for (int k = 0; k < n; ++k) {
    asm volatile("cp.async.wait_group 1;" ::: "memory");       // everything but the newest group (row k+1): row k has landed
    if (k + 2 < n) wait_row(k + 2);
    __syncthreads();                                           // row k of L staged by everybody; everybody is done with row k-1
    stage_row(k + 2, f2, rs2);                                 // into the buffer row k-1 used
    asm volatile("cp.async.commit_group;" ::: "memory");
    const int f4 = (k + 4 < n) ? e.first[k + 4] : 0;
    const long long rs4 = (k + 4 < n) ? e.row_start[k + 4] : 0;
    double ecur[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) ecur[q] = en[q];
#pragma unroll
    for (int q = 0; q < 3; ++q)
      en[q] = (owner && cw + oc[q] < KS && k + 1 < J.nE) ? J.E[((long long)(k + 1) * 6 + ox[q]) * KS + cw + oc[q]] : 0.0;
    const int jend = k < n_stop ? k : n_stop;
    // ---- this lane's block L_{k, f0 + lane} times the four columns of z_{f0 + lane}
    double v[24];
    {
      const int j = f0 + lane;
      const int zr = (j < jend) ? (j & 31) : 32;               // no block: the zero row (the L slot holds finite stale data)
      const double2* b2 = reinterpret_cast<const double2*>(sRow + (k % kSpikeBufs) * (32 * kSpikeBS) + lane * kSpikeBS);
      const double2* z2 = reinterpret_cast<const double2*>(sZw + zr * kSpikeZStride);
      double z[24];                                            // z[y * 4 + c]
#pragma unroll
      for (int h = 0; h < 12; ++h) { const double2 t = z2[h]; z[2 * h] = t.x; z[2 * h + 1] = t.y; }
#pragma unroll
      for (int x = 0; x < 6; ++x) {
        const double2 p0 = b2[3 * x], p1 = b2[3 * x + 1], p2 = b2[3 * x + 2];
        const double l[6] = {p0.x, p0.y, p1.x, p1.y, p2.x, p2.y};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          double a = l[0] * z[c];
#pragma unroll
          for (int y = 1; y < 6; ++y) a = fma(l[y], z[y * 4 + c], a);
          v[x * 4 + c] = a;
        }
      }
    }
    // ---- reduce-scatter over the 32 lanes: 24 -> 12 -> 6 -> 3 values per lane, then two plain butterflies
    const bool b16 = lane & 16, b8 = lane & 8, b4 = lane & 4;
    double w12[12], w6[6], w3[3];
#pragma unroll
    for (int o = 0; o < 12; ++o) {
      const double send = b16 ? v[o] : v[o + 12];
      const double keep = b16 ? v[o + 12] : v[o];
      w12[o] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int o = 0; o < 6; ++o) {
      const double send = b8 ? w12[o] : w12[o + 6];
      const double keep = b8 ? w12[o + 6] : w12[o];
      w6[o] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const double send = b4 ? w6[o] : w6[o + 3];
      const double keep = b4 ? w6[o + 3] : w6[o];
      w3[o] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      w3[o] += __shfl_xor_sync(0xffffffffu, w3[o], 2);
      w3[o] += __shfl_xor_sync(0xffffffffu, w3[o], 1);
    }
    // lane l now holds the outputs 12 (l >> 4 & 1) + 6 (l >> 3 & 1) + 3 (l >> 2 & 1) + {0,1,2} = 3 (l >> 2) + {0,1,2}
    __syncwarp();                                              // every lane has read the window entries it needs of row k-32
    // rows 0..k-1 of Z (stored by all four warps before this row's block barrier) -> the SYRK, once per chunk of its rows: here,
    // where the publishing lane's own stores of row k-1 have long landed, the release costs the row chain little
    if (J.zprog && tid == 32 && k > 0 && k % kSpikePublish == 0) progress_publish(J.zprog + blockIdx.x, k);
    if (owner) {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const double r = ecur[q] - w3[q];
        sZw[(k & 31) * kSpikeZStride + ox[q] * 4 + oc[q]] = r;       // row k-32 is no longer needed (column height <= 30)
        if (cw + oc[q] < KS) J.Z[((long long)k * 6 + ox[q]) * KS + cw + oc[q]] = r;
      }
    }
    __syncwarp();
    f0 = f1; f1 = f2; f2 = f3; rs2 = rs3; f3 = f4; rs3 = rs4;
  }
  if (J.zprog) {
    // the final value waits for the factorisation's last write as well: once every counter of a node reads e.n, spike and
    // factorisation are both done with it (the SYRK's last CTAs wait for exactly that)
    wait_row(n);
    __syncthreads();
    if (tid == 0) progress_publish(J.zprog + blockIdx.x, n);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// SYRK: U -= sum_k Z_k^T K_k Z_k, u -= sum_k Z_k^T K_k w_k over the pivot rows of a node (SyrkSeg, nd_passes.h): the
// product (KS x R)(R x KS), R = 6 rows, of Z^T with Y = K Z.  grid = (tiles of 64 x 64 scalars of the lower triangle,
// groups of kSyrkSplit block rows, segments); a CTA walks its rows in chunks of 4 block rows: Z for the tile's row side is
// brought to shared memory by cp.async one chunk ahead, for the column side (one buffer: 55 kB of shared memory in all, so that
// a SYRK CTA fits on an SM beside three spike CTAs) as soon as Y = K Z of the previous chunk is formed; each thread accumulates a
// 8 x 8 register tile (64 threads per 64 x 64 tile: 16 operand doubles from shared memory per 64 FMAs — a 4 x 4 tile loads 8 per 16
// and is bound by the 128 B/clk shared-memory return path, at half the FP64 rate).  A thread's rows / columns are four PAIRS 16 apart
// (2 t + 16 m + {0,1}), so that the LDS.128 of a warp cover 128 contiguous bytes.  Partial sums of the row groups meet in U by
// RED.ADD.F64.  grid = (tiles, segments, groups of kSyrkSplit block rows): the first rows of every segment are placed first.
//
// Beside the spike (SyrkSeg::zprog): a chunk of rows [kc, kc + 4) needs rows < kc + 4 of Z from the spike CTAs that own the
// tile's two column ranges, and of K and w from the factorisation; nine threads poll those counters before the chunk is staged
// (cp.async.cg reads L2, never a stale L1 line), the block barrier hands the acquired view to the others.  Nothing starves:
// the factorisation, the spike and the SYRK are launched in this order on one stream, the spike and the SYRK with
// programmatic stream serialisation, and both the factorisation and the spike execute griddepcontrol.launch_dependents first
// thing — so no CTA of the spike is placed before every CTA of the factorisation runs, and no CTA of the SYRK before every CTA
// of the spike runs.  A consumer only ever waits for producers that are already running and wait for nobody downstream.  This
// holds for eager launches (the multi-GPU solve) and for the programmatic edges a stream capture turns them into.
constexpr int kSyrkTile = 64;            // scalar columns per tile side
constexpr int kSyrkThreads = 64;         // 8 x 8 threads, 8 x 8 outputs each
constexpr int kSyrkChunk = 4;            // block rows per shared-memory chunk (24 scalar rows)
constexpr int kSyrkSplit = 8;            // block rows per CTA: two chunks
constexpr int kSyrkLd = kSyrkTile + 4;   // leading dimension of the shared tiles
constexpr int kSyrkTileDoubles = kSyrkChunk * 6 * kSyrkLd;
constexpr size_t kSyrkSmem = sizeof(double) * (4 * kSyrkTileDoubles + 2 * kSyrkChunk * 36 + 2 * kSyrkChunk * 6 + kSyrkChunk * 6);
constexpr int kSyrkTileGroups = kSyrkTile / kSpikeCols;      // spike CTAs per tile side
static_assert(kSyrkTile % kSpikeCols == 0 && kSyrkChunk % kSpikePublish == 0 && kSyrkSplit % kSyrkChunk == 0,
              "a chunk of the SYRK must end where the spike publishes");
static_assert(2 * kSyrkTileGroups + 1 <= kSyrkThreads, "one polling thread per counter");

__global__ void __launch_bounds__(kSyrkThreads)
nd_syrk_kernel(const nd::SyrkSeg* __restrict__ segs, int split) {
  constexpr int TS = kSyrkTile, RC = kSyrkChunk * 6, LD = kSyrkLd;
  extern __shared__ __align__(16) double smem_syrk[];
  double* sA = smem_syrk;                             // [2][RC][LD] Z[r][tile row side]
  double* sB = sA + 2 * kSyrkTileDoubles;             // [RC][LD]    Z[r][tile column side]
  double* sY = sB + kSyrkTileDoubles;                 // [RC][LD]    (K Z)[r][tile column side]
  double* sK = sY + kSyrkTileDoubles;                 // [2][chunk][36]
  double* sW = sK + 2 * kSyrkChunk * 36;              // [2][RC] w
  double* sKw = sW + 2 * RC;                          // [RC]
  const nd::SyrkSeg G = segs[blockIdx.y];
  int ti = 0, tj = 0;                                 // tile (ti, tj), tj <= ti, from the linear index
  { int t = blockIdx.x; while ((ti + 1) * (ti + 2) / 2 <= t) ++ti; tj = t - ti * (ti + 1) / 2; }
  if (ti * TS >= G.KS) return;
  const int k0 = blockIdx.z * split;
  if (k0 >= G.rows) return;
  const int k1 = min(G.rows, k0 + split);
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  const int KS = G.KS;
  // threads 0 .. 2 kSyrkTileGroups - 1: the spike counters of the row and the column tile; the next one: the factorisation's
  const int* poll = nullptr;
  if (G.zprog) {
    if (tid < 2 * kSyrkTileGroups) {
      const int g = (tid < kSyrkTileGroups ? ti : tj) * kSyrkTileGroups + tid % kSyrkTileGroups;
      if (g * kSpikeCols < KS) poll = G.zprog + g;
    } else if (tid == 2 * kSyrkTileGroups) {
      poll = G.fprog;
    }
  }
  // rows < r of Z, K and w final: Z once the spike counters read r, K and w once the factorisation's reads r + 1 (its counter
  // covers D^-1 and z one row behind L) or its final value.  The caller's block barrier follows.
  auto need = [&](int r) { return poll == G.fprog ? min(r + 1, G.rows) : r; };
  auto wait_rows = [&](int r) {
    if (poll) { const int v = need(r); while (progress_read(poll) < v) __nanosleep(64); }
  };
  auto rows_ready = [&](int r) { return !poll || progress_read(poll) >= need(r); };
  auto wait_spike_done = [&]() {                      // spike (and with it the factorisation) finished with this node
    if (poll && tid < 2 * kSyrkTileGroups) while (progress_read(poll) < G.zdone) __nanosleep(64);
  };
  // chunk kc -> buffer par: 16-byte pieces (KS is even, the tiles start at even columns); rows / columns beyond the data are zero-filled
  auto prefetch = [&](int kc, int par) {              // row side, K, w
    const int nr = min(kSyrkChunk, k1 - kc) * 6;
    double* dA = sA + par * kSyrkTileDoubles;
    for (int o = tid; o < RC * (TS / 2); o += kSyrkThreads) {
      const int r = o / (TS / 2), a2 = (o - r * (TS / 2)) * 2;
      const bool va = r < nr && ti * TS + a2 < KS;
      cp_async16_zfill(dA + r * LD + a2, va ? G.Z + ((long long)kc * 6 + r) * KS + ti * TS + a2 : G.Z, va);
    }
    for (int o = tid; o < kSyrkChunk * 18; o += kSyrkThreads) {
      const int bk = o / 18;
      const bool v = kc + bk < k1;
      cp_async16_zfill(sK + par * kSyrkChunk * 36 + 2 * o, v ? G.K + (long long)kc * 36 + 2 * o : G.K, v);
    }
    for (int o = tid; o < kSyrkChunk * 3; o += kSyrkThreads) {
      const int bk = o / 3;
      const bool v = kc + bk < k1;
      cp_async16_zfill(sW + par * RC + 2 * o, v ? G.w + (long long)kc * 6 + 2 * o : G.w, v);
    }
  };
  auto prefetch_col = [&](int kc) {                   // column side
    const int nr = min(kSyrkChunk, k1 - kc) * 6;
    for (int o = tid; o < RC * (TS / 2); o += kSyrkThreads) {
      const int r = o / (TS / 2), a2 = (o - r * (TS / 2)) * 2;
      const bool vb = r < nr && tj * TS + a2 < KS;
      cp_async16_zfill(sB + r * LD + a2, vb ? G.Z + ((long long)kc * 6 + r) * KS + tj * TS + a2 : G.Z, vb);
    }
  };
  double acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
  double racc = 0.0;
  wait_rows(min(k0 + kSyrkChunk, k1));
  __syncthreads();
  prefetch(k0, 0);
  prefetch_col(k0);
  asm volatile("cp.async.commit_group;" ::: "memory");
  int par = 0;
  for (int kc = k0; kc < k1; kc += kSyrkChunk, par ^= 1) {
    const int nr = min(kSyrkChunk, k1 - kc) * 6, next_r = min(kc + 2 * kSyrkChunk, k1);
    const bool more = kc + kSyrkChunk < k1;                              // (uniform over the CTA)
    // the next chunk comes in while this one is computed if its rows are final already; otherwise this chunk is computed
    // first and the next one waited for afterwards (chasing the spike, the chunk at hand is not held up by the next)
    const bool early = more && __syncthreads_and(rows_ready(next_r));
    if (early) prefetch(kc + kSyrkChunk, par ^ 1);                       // its buffer was consumed before the last barrier of the previous chunk
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");               // everything but the row side of chunk kc+1
    __syncthreads();                                                     // chunk kc landed
    const double* cA = sA + par * kSyrkTileDoubles;
    const double* cB = sB;
    const double* cK = sK + par * kSyrkChunk * 36;
    for (int o = tid; o < nr * TS; o += kSyrkThreads) {                  // Y = K Z on the column side (rows beyond nr: zero)
      const int r = o / TS, b = o - r * TS, bk = r / 6, x = r - bk * 6;
      const double* Kx = cK + bk * 36 + x * 6;
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) s += Kx[q] * cB[(bk * 6 + q) * LD + b];
      sY[r * LD + b] = s;
    }
    if (tj == 0 && tid < nr) {                                           // (K w)[r]
      const int bk = tid / 6, x = tid - bk * 6;
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < 6; ++q) s += cK[bk * 36 + x * 6 + q] * sW[par * RC + bk * 6 + q];
      sKw[tid] = s;
    }
    __syncthreads();                                                     // sB consumed: the column side of the next chunk may come in
    if (early) prefetch_col(kc + kSyrkChunk);
    asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll 2
    for (int r = 0; r < nr; ++r) {
      double av[8], bv[8];
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const double2 a = *reinterpret_cast<const double2*>(cA + r * LD + 2 * ty + 16 * m);
        const double2 b = *reinterpret_cast<const double2*>(sY + r * LD + 2 * tx + 16 * m);
        av[2 * m] = a.x; av[2 * m + 1] = a.y; bv[2 * m] = b.x; bv[2 * m + 1] = b.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
    }
    if (tj == 0 && tid < TS) {
      double s = 0.0;
      for (int r = 0; r < nr; ++r) s += cA[r * LD + tid] * sKw[r];
      racc += s;
    }
    if (more && !early) wait_rows(next_r);
    __syncthreads();                                                     // sY, sKw and this chunk's buffers are free again
    if (more && !early) {
      prefetch(kc + kSyrkChunk, par ^ 1);
      prefetch_col(kc + kSyrkChunk);
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  }
  if (k1 == G.rows) wait_spike_done();               // the last rows: this grid ends after the spike and the factorisation
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ga = ti * TS + 2 * ty + 16 * (i >> 1) + (i & 1), gb = tj * TS + 2 * tx + 16 * (j >> 1) + (j & 1);   // scalar row / column inside the boundary
      const int bi = ga / 6, bj = gb / 6;
      if (bj <= bi && ga < KS && gb < KS) atomicAdd(&G.U[((long long)bi * (bi + 1) / 2 + bj) * 36 + (ga - 6 * bi) * 6 + (gb - 6 * bj)], -acc[i][j]);
    }
  if (tj == 0 && tid < TS && ti * TS + tid < KS) atomicAdd(&G.u[ti * TS + tid], -racc);
}

// ---------------------------------------------------------------------------------------------------------------
// Downwards: x_K = D^-1 (w_K - Z x_boundary) for the pivot rows of the nodes of one level (CorrectApplyF of nd_passes.h
// with a CTA per block row: warp q forms the dot product of row (k, q) of Z with the boundary solution, coalesced).
__global__ void __launch_bounds__(192)
nd_correct_apply_kernel(nd::Tables t, const int* __restrict__ ids, int stride) {
  __shared__ double sc[6];
  const nd::NodeDev v = t.nodes[ids[blockIdx.x / stride]];
  const int k = blockIdx.x % stride;
  if (k >= v.npiv) return;
  const int tid = threadIdx.x, lane = tid & 31, q = tid >> 5;
  const double* wv = (v.kind == 0 ? t.z : t.zs) + 6 * (long long)(v.r0 + k);
  const double* zr = t.Z + v.offZ + ((long long)k * 6 + q) * v.ks;
  const int na = 6 * v.wa;
  const double* xa = t.x + 6 * (long long)v.sa;
  const double* xc = t.x + 6 * (long long)v.sc;
  double s = 0.0;
  for (int col = lane; col < v.ks; col += 32) s += zr[col] * (col < na ? xa[col] : xc[col - na]);
  s = warp_sum(s);
  if (lane == 0) sc[q] = wv[q] - s;
  __syncthreads();
  if (tid < 6) {
    const double* K = t.dinv + (long long)(v.r0 + k) * 36 + tid * 6;
    double o = 0.0;
#pragma unroll
    for (int qq = 0; qq < 6; ++qq) o += K[qq] * sc[qq];
    t.x[6 * (long long)(v.r0 + k) + tid] = o;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Dense block LDL^T of a separator (<= 30 x 30 blocks, every block inside the envelope): FactorJob semantics for a complete
// factorisation (n_stop == n, no dump) of a matrix in the dense lower layout (block (i,j) at (i(i+1)/2 + j)*36).
//
// The register-window kernel of factor_la.cuh slides a 31-row window along a band and pays the same per pivot column
// whatever the column holds; a separator is dense and SHRINKS (the trailing matrix of pivot k has (29-k)(30-k)/2 blocks),
// and its 30 pivots sit on the critical path of every tree level.  Every block of the lower triangle lives in the registers
// of one PAIR thread for the whole factorisation (thread <-> (i, j)); a COLUMN GROUP of six warps owns the pivot column and
// runs ONE PIVOT AHEAD of the pair threads (look-ahead), thread <-> (block row i, row r of the 6 x 6 block):
//   iteration s, column group:  column s arrives as the pair threads left it (updated through pivot s-2); apply pivot s-1 to
//                               it (36 DFMA per thread); the diagonal block goes to warp 0, which inverts it (two
//                               reciprocals on the dependent chain, factor_la.cuh); every thread scales its row:
//                               L_is = T_is D_s^-1 -> shared + global memory, z_i -= L_is z_s;
//   iteration s, pair threads:  G -= L_{i,s-1} T_{j,s-1}^T for their blocks of columns j >= s+1 (216 DFMA; the thread map
//                               groups 8 x 4 patches of blocks into a warp: <= 8 + 4 distinct operand blocks per warp);
//                               column s+1 is then handed to the column group through shared memory.
// One block barrier per pivot; the column group's chain (update 36 + inverse ~300 + scale ~90 instructions per warp) and the
// pair threads' update overlap (without the look-ahead one warp inverting and scaling, 216 DFMA per lane, and the
// FP64-bound trailing update run one after the other).
// One CTA per separator; grid = separators of the tree level.
constexpr int kDenseMax = 30;
constexpr int kDensePairThreads = 480;       // 465 blocks of the 30 x 30 lower triangle
constexpr int kDenseInvWarp = 480;           // threads 480..511: the warp that inverts the pivot block (pair-side register budget)
constexpr int kDenseColBase = 512;           // threads 512..703: 6 warps, warp = row of the 6 x 6 block, lane = block row
constexpr int kDenseColThreads = 192;
constexpr int kDenseThreads = 768;           // 4 + 2 warpgroups (704..767 idle): the register re-allocation works on warpgroups
constexpr int kDensePairRegs = 96, kDenseColRegs = 48;       // 512 * 96 + 256 * 48 == 768 * 80 = 61440, the pool the CTA is launched with: setmaxnreg.inc waits for ever if the budgets exceed it
static_assert((kDenseColBase) * kDensePairRegs + (kDenseThreads - kDenseColBase) * kDenseColRegs <= kDenseThreads * 80, "register budgets exceed the launch pool");
constexpr int kDenseS = 38;                  // doubles per operand block in shared memory (bank spread, 16 B aligned)
constexpr size_t kDenseSmem = sizeof(double) * (6 * kDenseMax * kDenseS + 36 + 72 + kDenseMax * 6 + 8 + 48);

__global__ void __launch_bounds__(kDenseThreads, 1)
nd_dense_factor_kernel(const FactorJob* __restrict__ jobs, const unsigned short* __restrict__ tmap) {
  extern __shared__ __align__(16) double smem_dense[];
  double* sL = smem_dense;                                 // [2][30][S] L_{i,s}^T ([q * 6 + x] = L[x][q])   parity s & 1
  double* sT = sL + 2 * kDenseMax * kDenseS;               // [2][30][S] T_{i,s}^T   parity s & 1
  double* sC = sT + 2 * kDenseMax * kDenseS;               // [2][30][S] column c as the pair threads left it, parity c & 1
  double* sD = sC + 2 * kDenseMax * kDenseS;               // [36] pivot block (rows written by the six threads of block row s)
  double* sK = sD + 36;                                    // [2][36] its inverse, parity s & 1 (an idle warp copies it to global memory one step later)
  double* sZ = sK + 72;                                    // [30][6]
  double* sInv = sZ + kDenseMax * 6 + 8;                   // [48] scratch of sym6_block_inverse_warp
  const FactorJob J = jobs[blockIdx.x];
  const int n = J.e.n;
  const int tid = threadIdx.x;
  pdl_launch_dependents();
  for (int o = tid; o < n * 6; o += kDenseThreads) sZ[o] = J.z[o];
  // register re-allocation: one setmaxnreg site per warpgroup-uniform branch (warpgroups 0-3: pair threads + inverting warp)
  if (tid >= kDenseColBase) reg_dealloc<kDenseColRegs>(); else reg_alloc<kDensePairRegs>();
  if (tid >= kDenseColBase) {
    // ================================================= column group (+ two idle warps that only keep the block barriers company)
    const int ct = tid - kDenseColBase;
    const bool idle = ct >= kDenseColThreads;
    const int r = idle ? 0 : (ct >> 5), i = idle ? 31 : (ct & 31); // row r of block row i
    const bool mine = !idle && i < n;
    double lrow[6] = {0, 0, 0, 0, 0, 0};                           // row r of L_{i,s-1}
    __syncthreads();                                               // (P) columns 0 and 1 published by the pair threads
    for (int s = 0; s < n; ++s) {
      const int par = s & 1;
      // ---- (1) column s as of pivot s-1: row r of block (i, s), i >= s
      double t[6] = {0, 0, 0, 0, 0, 0};
      if (mine && i >= s) {
        const double2* c2 = reinterpret_cast<const double2*>(sC + (par * kDenseMax + i) * kDenseS + r * 6);
        const double2 q0 = c2[0], q1 = c2[1], q2 = c2[2];
        t[0] = q0.x; t[1] = q0.y; t[2] = q1.x; t[3] = q1.y; t[4] = q2.x; t[5] = q2.y;
        if (s > 0) {                                               // -= L_{i,s-1}[r][.] T_{s,s-1}^T   (sT holds T^T: [q][y])
          const double2* ts = reinterpret_cast<const double2*>(sT + ((par ^ 1) * kDenseMax + s) * kDenseS);
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const double2 u0 = ts[3 * q], u1 = ts[3 * q + 1], u2 = ts[3 * q + 2];
            const double l = -lrow[q];
            t[0] = fma(l, u0.x, t[0]); t[1] = fma(l, u0.y, t[1]); t[2] = fma(l, u1.x, t[2]);
            t[3] = fma(l, u1.y, t[3]); t[4] = fma(l, u2.x, t[4]); t[5] = fma(l, u2.y, t[5]);
          }
        }
        if (i == s) {
          double2* d2 = reinterpret_cast<double2*>(sD + r * 6);
          d2[0] = make_double2(t[0], t[1]); d2[1] = make_double2(t[2], t[3]); d2[2] = make_double2(t[4], t[5]);
        }
      }
      if (!idle) {
        named_bar_sync(2, kDenseColThreads + 32);                  // pivot block complete -> the inverting warp
        named_bar_sync(3, kDenseColThreads + 32);                  // D_s^-1 visible
      }
      // ---- (2) scale: row r of L_is = T_is D_s^-1, publish T and L, forward substitution
      if (mine && i > s) {
        double lr[6] = {0, 0, 0, 0, 0, 0};
        const double2* k2 = reinterpret_cast<const double2*>(sK + par * 36);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const double2 k0 = k2[3 * q], k1 = k2[3 * q + 1], kk2 = k2[3 * q + 2];
          lr[0] = fma(t[q], k0.x, lr[0]); lr[1] = fma(t[q], k0.y, lr[1]); lr[2] = fma(t[q], k1.x, lr[2]);
          lr[3] = fma(t[q], k1.y, lr[3]); lr[4] = fma(t[q], kk2.x, lr[4]); lr[5] = fma(t[q], kk2.y, lr[5]);
        }
        double* tt = sT + (par * kDenseMax + i) * kDenseS + r;       // transposed operand blocks: [q * 6 + row]
        double* lt = sL + (par * kDenseMax + i) * kDenseS + r;
        double2* g2 = reinterpret_cast<double2*>(J.L + ((long long)i * (i + 1) / 2 + s) * 36 + r * 6);
#pragma unroll
        for (int q = 0; q < 6; ++q) { tt[q * 6] = t[q]; lt[q * 6] = lr[q]; }
#pragma unroll
        for (int h = 0; h < 3; ++h) g2[h] = make_double2(lr[2 * h], lr[2 * h + 1]);
        double zs = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) { zs = fma(lr[q], sZ[s * 6 + q], zs); lrow[q] = lr[q]; }
        sZ[i * 6 + r] -= zs;
      }
      __syncthreads();                                             // (s) L_s, T_s published; column s+2 handed over by the pair threads
      // the two idle warps of this group: D_s^-1 to global memory (the inverting warp left it in sK[par]; it writes that buffer again
      // two pivots from now) with the final z_s (no pivot after s-1 touches row s), and word to the spike and the SYRK running beside
      // this CTA that columns 0..s of L — and with them D^-1 and z of rows 0..s-1, stored one barrier ago — are in global memory
      // (the warp that publishes has no stores of its own in flight: the release does not wait for them)
      if (idle) {
        const int l = ct - kDenseColThreads;
        if (l < 18)
          reinterpret_cast<double2*>(J.dinv + (long long)s * 36)[l] = reinterpret_cast<const double2*>(sK + par * 36)[l];
        else if (l < 24)
          J.z[s * 6 + l - 18] = sZ[s * 6 + l - 18];
        // (never the final value n: that one comes after the last barrier, when D^-1 and z of the last row are out too)
        if (J.progress && l == 32 && (s & 3) == 3 && s + 1 < n) progress_publish(J.progress, s + 1);
      }
    }
  } else if (tid >= kDenseInvWarp) {
    // ================================================= the inverting warp
    const int lane = tid - kDenseInvWarp;
    int bad = 0;
    __syncthreads();                                               // (P)
    for (int s = 0; s < n; ++s) {
      named_bar_sync(2, kDenseColThreads + 32);
      double* Kp = sK + (s & 1) * 36;                              // D_s^-1 (full symmetric) for the column group, and for the idle warp that copies it out
      sym6_block_inverse_warp(sD, Kp, sInv, lane);
      __syncwarp();
      if (!isfinite((Kp[0] + Kp[35]) + (Kp[18] + Kp[13]))) bad = 1;
      named_bar_sync(3, kDenseColThreads + 32);
      __syncthreads();                                             // (s)
    }
    if (bad && lane == 0) J.status[0] = 1;
  } else {
    // ================================================= pair threads
    const unsigned short tm = tmap[tid];
    const int i = tm & 0xff, j = tm >> 8;                          // block (i, j), j <= i ; 0xffff: idle thread
    const bool live = tm != 0xffff && i < n;
    double G[36];
    if (live) {
      const double2* src = reinterpret_cast<const double2*>(J.L + ((long long)i * (i + 1) / 2 + j) * 36);
#pragma unroll
      for (int q = 0; q < 18; ++q) { const double2 v = src[q]; G[2 * q] = v.x; G[2 * q + 1] = v.y; }
    } else {
#pragma unroll
      for (int q = 0; q < 36; ++q) G[q] = 0.0;
    }
    // hand column c (this thread's block (i, c)) to the column group
    auto publish = [&](int c) {
      double2* d2 = reinterpret_cast<double2*>(sC + ((c & 1) * kDenseMax + i) * kDenseS);
#pragma unroll
      for (int q = 0; q < 18; ++q) d2[q] = make_double2(G[2 * q], G[2 * q + 1]);
    };
    if (live && j <= 1) publish(j);                                // columns 0 and 1 as they are
    __syncthreads();                                               // (P)
    for (int s = 0; s < n; ++s) {
      // the trailing update of pivot s-1 for the columns the pair threads still own (j >= s+1)
      if (s >= 1 && live && j >= s + 1) {
        const int par = (s - 1) & 1;
        // rank-1 steps over the contraction index q: column q of T_j (six values) and two entries of column q of L_i at a time are
        // live beside the 36 accumulators — 16 operand registers, which is what fits the 96-register budget without spilling G
        const double2* l2 = reinterpret_cast<const double2*>(sL + (par * kDenseMax + i) * kDenseS);     // L_i^T: [q][x]
        const double2* t2 = reinterpret_cast<const double2*>(sT + (par * kDenseMax + j) * kDenseS);     // T_j^T: [q][y]
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const double2 t0 = t2[3 * q], t1 = t2[3 * q + 1], t2v = t2[3 * q + 2];
#pragma unroll
          for (int xp = 0; xp < 3; ++xp) {
            const double2 lv = l2[3 * q + xp];
            const double l0 = -lv.x, l1 = -lv.y;
            double* g0 = G + (2 * xp) * 6;
            double* g1 = G + (2 * xp + 1) * 6;
            g0[0] = fma(l0, t0.x, g0[0]); g0[1] = fma(l0, t0.y, g0[1]); g0[2] = fma(l0, t1.x, g0[2]);
            g0[3] = fma(l0, t1.y, g0[3]); g0[4] = fma(l0, t2v.x, g0[4]); g0[5] = fma(l0, t2v.y, g0[5]);
            g1[0] = fma(l1, t0.x, g1[0]); g1[1] = fma(l1, t0.y, g1[1]); g1[2] = fma(l1, t1.x, g1[2]);
            g1[3] = fma(l1, t1.y, g1[3]); g1[4] = fma(l1, t2v.x, g1[4]); g1[5] = fma(l1, t2v.y, g1[5]);
          }
        }
        if (j == s + 1) publish(s + 1);                            // column s+1 (updated through pivot s-1) -> column group, iteration s+1
      }
      __syncthreads();                                             // (s)
    }
  }
  __syncthreads();                                                 // (z went out row by row, with D^-1)
  if (J.progress && tid == 0) progress_publish(J.progress, n);     // the last global write of the CTA
}

// thread -> block map of nd_dense_factor_kernel: blocks of the 30 x 30 lower triangle grouped by 8 x 4 patches
inline std::vector<unsigned short> dense_thread_map() {
  struct B { int i, j; };
  std::vector<B> v;
  for (int i = 0; i < kDenseMax; ++i) for (int j = 0; j <= i; ++j) v.push_back(B{i, j});
  std::stable_sort(v.begin(), v.end(), [](const B& a, const B& b) {
    const int ka[4] = {a.i / 8, a.j / 4, a.i, a.j}, kb[4] = {b.i / 8, b.j / 4, b.i, b.j};
    for (int q = 0; q < 4; ++q) if (ka[q] != kb[q]) return ka[q] < kb[q];
    return false;
  });
  std::vector<unsigned short> m((size_t)kDensePairThreads, (unsigned short)0xffff);
  for (size_t t = 0; t < v.size(); ++t) m[t] = (unsigned short)(v[t].i | (v[t].j << 8));
  return m;
}

}  // namespace lvba
