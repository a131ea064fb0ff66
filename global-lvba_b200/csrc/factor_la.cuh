// factor_la.cuh — register-window block LDL^T with a panel look-ahead group, and the single-warp backward
// substitution that follows it.
//
// Same job as SimplicialLDLT in BALM2::damping_iter (reference include/BALM/bavoxel.hpp:695-710, lower
// triangle, no pivoting — SURVEY.md Q4/Q5) and as the DENSE_SCHUR Cholesky of the reduced camera system
// inside ceres::Solve (src/lvba_system.cpp:1574,1643), for a block envelope whose column height is < P.
//
// One CTA walks the pivot columns.  Every live 6x6 block of the trailing window (rows/cols k..k+P-1) lives in
// the registers of one PAIR thread for its whole life (thread <-> unordered slot pair {a,b}, slot = row mod P).
//   * symmetric update form.  The stored block G always has its rows on slot a and its columns on slot b,
//     whichever of the two is the lower row: A_ab -= L_a D L_b^T = L_a T_b^T holds for both orientations, so a
//     thread reads the SAME two shared-memory operands (L of slot a, T of slot b) at every step;
//   * the look-ahead group owns the NEXT pivot column.  During step k it applies column k to column k+1 itself
//     (30 block updates), inverts D_{k+1} (two 3x3 adjugates + Schur complement: two reciprocals on the dependent
//     chain instead of the six of a scalar LDL^T), scales the column and publishes L_{.,k+1} / T_{.,k+1} for step
//     k+1, all overlapped with the pair threads' trailing update of step k: ONE block barrier per pivot column;
//   * the entering row is streamed global -> shared with cp.async in its natural (contiguous) order.
// The step is bound by shared-memory wavefronts (operand fetch of the pair threads, ~3 wavefronts per LDS.128) and by
// the latency of the look-ahead chain, not by HBM.
#pragma once
#include "envelope.cuh"

namespace lvba {

// kTile2: a pair thread owns TWO blocks that share their row slot ({a,b1} and {a,b2}): the L operand of slot a is
// fetched once for both updates (three operand blocks per two updates instead of four), and half as many pair
// warps contend with the look-ahead warps for the issue slots and the shared-memory pipe.
// Two blocks per thread pay off for the widest windows (P > 24: the look-ahead chain gains most, since half as many
// pair warps compete with it and it keeps 96 registers); for P <= 24 the pair warps that remain do not spread evenly
// over the four SMSPs and the 144 accumulator registers cost more than the saved operand fetches.
constexpr bool la_tile2(int P) { return P > 24; }
constexpr int la_tile2_threads(int P) { int s = 0; for (int m = 1; m <= P; ++m) s += (m + 1) / 2; return s; }
template <int P, bool kTile2>
struct LaCfg {
  static constexpr int kPairs = P * (P + 1) / 2;
  static constexpr int kOwners = kTile2 ? la_tile2_threads(P) : kPairs;          // threads that own blocks
  // the register re-allocation (setmaxnreg) works on warpgroups of 4 warps: P = 31 keeps whole warpgroups
  static constexpr bool kRealloc = P > 24;
  static constexpr int kPairThreads = kRealloc ? ((kOwners + 127) / 128) * 128 : ((kOwners + 31) / 32) * 32;
  static constexpr int kLaThreads = 128;                         // one look-ahead warpgroup
  static constexpr int kThreads = kPairThreads + kLaThreads;
  static constexpr int kItemThreads = 96;                        // look-ahead warps 1..3
  static constexpr int kItems = (P - 1) * 6;                     // (row of the next column, block row x)
  static constexpr int kRounds = (kItems + kItemThreads - 1) / kItemThreads;
  static constexpr int S = 38;                                   // doubles per transposed block (16 B aligned, conflict-free over 8 slots)
  // P = 31: one block per thread: 640 threads launch at 96 registers, 512*104 + 128*64 == 640*96
  //         two blocks per thread: 384 threads launch at 168, 256*200 + 128*96 <= 384*168
  static constexpr int kPairRegs = kTile2 ? 200 : 104, kLaRegs = kTile2 ? 96 : 64;
  static constexpr int kDoubles = 6 * P * S + 2 * P * 36 + 2 * 36 + 36 + 2 * 36 + P * 6 + 48 + 40 + 48;    // ... + scratch of the warp-cooperative 6x6 inverse
  static constexpr size_t kSmem = sizeof(double) * (size_t)kDoubles + sizeof(long long) * 64 + sizeof(int) * 64 + 32;
};

LVBA_DEV void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz));
}
LVBA_DEV void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
LVBA_DEV void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// progress counters between a factorisation and the spike kernel that consumes its columns while it runs (FactorJob::progress)
LVBA_DEV void progress_publish(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
LVBA_DEV int progress_read(const int* p) { int v; asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
// programmatic dependent launch: the next kernel of the stream, if it was launched with programmatic stream serialisation, may
// start once every CTA of this grid has executed this — i.e. IS RUNNING, which is what a consumer that spins on progress counters
// needs to be free of deadlock; without such a dependent this is a no-op
LVBA_DEV void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Inverse of a symmetric 6x6 block from its lower triangle x[i(i+1)/2 + j] (i >= j), no pivoting:
// D = [A B^T; B C] (3x3 blocks): A^-1 by the adjugate, W = B A^-1, S = C - W B^T, S^-1 by the adjugate,
// K22 = S^-1, K21 = -S^-1 W, K11 = A^-1 - W^T K21.  Two reciprocals on the dependent chain.
// K is returned as the packed lower triangle.  Needs det(A) != 0 and det(S) != 0 (a scalar LDL^T needs all six
// leading minors non-zero).
LVBA_DEV void sym3_adj_inverse(double a00, double a10, double a11, double a20, double a21, double a22, double (&o)[6]) {
  const double c00 = a11 * a22 - a21 * a21;
  const double c10 = a20 * a21 - a10 * a22;
  const double c20 = a10 * a21 - a20 * a11;
  const double c11 = a00 * a22 - a20 * a20;
  const double c21 = a10 * a20 - a00 * a21;
  const double c22 = a00 * a11 - a10 * a10;
  const double det = a00 * c00 + a10 * c10 + a20 * c20;
  const double r = __drcp_rn(det);
  o[0] = c00 * r; o[1] = c10 * r; o[2] = c11 * r; o[3] = c20 * r; o[4] = c21 * r; o[5] = c22 * r;   // (0,0) (1,0) (1,1) (2,0) (2,1) (2,2)
}
LVBA_DEV void sym6_block_inverse(const double (&x)[21], double (&K)[21]) {
  double Ai[6];
  sym3_adj_inverse(x[LVBA_T(0, 0)], x[LVBA_T(1, 0)], x[LVBA_T(1, 1)], x[LVBA_T(2, 0)], x[LVBA_T(2, 1)], x[LVBA_T(2, 2)], Ai);
  auto ai = [&](int i, int j) -> double { return i >= j ? Ai[i * (i + 1) / 2 + j] : Ai[j * (j + 1) / 2 + i]; };
  double W[3][3];                                   // W = B A^-1, B[i][m] = x(3+i, m)
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      W[i][j] = x[LVBA_T(3 + i, 0)] * ai(0, j) + x[LVBA_T(3 + i, 1)] * ai(1, j) + x[LVBA_T(3 + i, 2)] * ai(2, j);
  double Sm[6];                                     // S = C - W B^T (lower triangle)
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j)
      Sm[i * (i + 1) / 2 + j] = x[LVBA_T(3 + i, 3 + j)] - (W[i][0] * x[LVBA_T(3 + j, 0)] + W[i][1] * x[LVBA_T(3 + j, 1)] + W[i][2] * x[LVBA_T(3 + j, 2)]);
  double Si[6];
  sym3_adj_inverse(Sm[0], Sm[1], Sm[2], Sm[3], Sm[4], Sm[5], Si);
  auto si = [&](int i, int j) -> double { return i >= j ? Si[i * (i + 1) / 2 + j] : Si[j * (j + 1) / 2 + i]; };
  double K21[3][3];                                 // K21 = -S^-1 W
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      K21[i][j] = -(si(i, 0) * W[0][j] + si(i, 1) * W[1][j] + si(i, 2) * W[2][j]);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      K[LVBA_T(i, j)] = ai(i, j) - (W[0][i] * K21[0][j] + W[1][i] * K21[1][j] + W[2][i] * K21[2][j]);
      K[LVBA_T(3 + i, 3 + j)] = si(i, j);
    }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) K[LVBA_T(3 + i, j)] = K21[i][j];
}

// The same inverse computed by a WARP: lanes 0..8 <-> entry (i, j) of the 3 x 3 blocks, stages handed over through 45 doubles of
// shared memory private to the warp; a lane issues ~120 instructions where one thread working through sym6_block_inverse issues
// ~280, and 84 registers of the calling warp become free.  It is not faster than
// the one-thread inverse (in-kernel clocks of the separator kernel, taken with a development build no longer in the tree): the
// segment is bound by the latency of the two reciprocals and of the hand-overs, not by the instruction count.  Kept for the
// registers it frees.  D: 36 doubles row-major, LOWER triangle read.  K: 36 doubles, full, exactly
// symmetric (the mirror entries are copies).  All 32 lanes must call; `scr` holds >= 48 doubles.
LVBA_DEV void sym6_block_inverse_warp(const double* __restrict__ D, double* __restrict__ K, double* __restrict__ scr, int lane) {
  const unsigned full = 0xffffffffu;
  const bool on = lane < 9;
  const int l = on ? lane : 0;
  const int i = l / 3, j = l - 3 * i;
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  double* Ai = scr; double* W = scr + 9; double* S = scr + 18; double* Si = scr + 27; double* K21 = scr + 36;
  auto d6 = [](int p, int q) { return p >= q ? p * 6 + q : q * 6 + p; };     // lower-triangle offsets of a 6 x 6 / 3 x 3 row-major block
  auto d3 = [](int p, int q) { return p >= q ? p * 3 + q : q * 3 + p; };
  {                                                                         // A^-1 = cofactors / det (A symmetric)
    const double c = D[d6(i1, j1)] * D[d6(i2, j2)] - D[d6(i1, j2)] * D[d6(i2, j1)];
    const double c0 = __shfl_sync(full, c, 0), c1 = __shfl_sync(full, c, 1), c2 = __shfl_sync(full, c, 2);
    const double det = D[0] * c0 + D[6] * c1 + D[12] * c2;
    const double r = __drcp_rn(det);
    if (on) Ai[l] = c * r;
  }
  __syncwarp();
  {                                                                         // W = B A^-1, B[i][m] = D(3+i, m)
    const double* b = D + (3 + i) * 6;
    const double w = b[0] * Ai[j] + b[1] * Ai[3 + j] + b[2] * Ai[6 + j];
    if (on) W[l] = w;
  }
  __syncwarp();
  {                                                                         // S = C - W B^T
    const double* b = D + (3 + j) * 6;
    const double v = D[d6(3 + i, 3 + j)] - (W[3 * i] * b[0] + W[3 * i + 1] * b[1] + W[3 * i + 2] * b[2]);
    if (on) S[l] = v;
  }
  __syncwarp();
  {                                                                         // S^-1 (lower triangle of S read)
    const double c = S[d3(i1, j1)] * S[d3(i2, j2)] - S[d3(i1, j2)] * S[d3(i2, j1)];
    const double c0 = __shfl_sync(full, c, 0), c1 = __shfl_sync(full, c, 1), c2 = __shfl_sync(full, c, 2);
    const double det = S[0] * c0 + S[3] * c1 + S[6] * c2;
    const double r = __drcp_rn(det);
    if (on) Si[l] = c * r;
  }
  __syncwarp();
  {                                                                         // K21 = -S^-1 W
    const double v = -(Si[d3(i, 0)] * W[j] + Si[d3(i, 1)] * W[3 + j] + Si[d3(i, 2)] * W[6 + j]);
    if (on) K21[l] = v;
  }
  __syncwarp();
  if (on) {                                                                 // K11 = A^-1 - W^T K21 ; assemble K (lanes i >= j write the symmetric pairs)
    const double k21 = K21[l];
    K[(3 + i) * 6 + j] = k21; K[j * 6 + 3 + i] = k21;
    if (i >= j) {
      const double k11 = Ai[d3(i, j)] - (W[i] * K21[j] + W[3 + i] * K21[3 + j] + W[6 + i] * K21[6 + j]);
      const double k22 = Si[d3(i, j)];
      K[i * 6 + j] = k11; K[j * 6 + i] = k11;
      K[(3 + i) * 6 + 3 + j] = k22; K[(3 + j) * 6 + 3 + i] = k22;
    }
  }
  __syncwarp();
}

template <int P, bool kTile2>
__global__ void __launch_bounds__(LaCfg<P, kTile2>::kThreads, 1)
env_factor_la_kernel(const FactorJob* __restrict__ jobs, const unsigned* __restrict__ pair_map) {
  using Cfg = LaCfg<P, kTile2>;
  constexpr int S = Cfg::S;
  constexpr int PS = P * S;                       // one parity of sL / sT / sA
  const FactorJob J = jobs[blockIdx.x];
  const EnvView e = J.e;
  double* __restrict__ L = J.L;
  double* __restrict__ dinv = J.dinv;
  double* __restrict__ z = J.z;
  const int n_stop = J.n_stop;
  pdl_launch_dependents();

  extern __shared__ __align__(16) double smem_la[];
  double* sL = smem_la;                          // [2][P][S] L_ik transposed ([q*6+x] = L[x][q]); parity = pivot column & 1
  double* sT = sL + 2 * PS;                      // [2][P][S] T_ik = A_ik (updated, unscaled), same layout
  double* sA = sT + 2 * PS;                      // [2][P][S] next-next column handed to the look-ahead group, same layout
  double* sEnter = sA + 2 * PS;                  // [2][P][36] entering row r: block (r, r-P+1+d) at index d (d = P-1: diagonal), row-major
  double* sDg = sEnter + 2 * P * 36;             // [2][36]   diagonal block of the next pivot (before column k's update)
  double* sDu = sDg + 72;                        // [36]      updated diagonal block of the next pivot (kept for the window dump)
  double* sK = sDu + 36;                         // [2][36]   D^-1 of the pivot block (full symmetric, row-major)
  double* sZ = sK + 72;                          // [P][6]
  double* sZin = sZ + P * 6;                     // [8][6]   rhs entries of the rows about to enter (ring by row & 7)
  double* sZero = sZin + 48;                     // [S]      zero operand (a block that must not change this step)
  double* sInv = sZero + 40;                     // [48]     scratch of sym6_block_inverse_warp
  long long* sLabRS = reinterpret_cast<long long*>(sInv + 48);    // [64] row_start of row r at r & 63 (ring, filled by cp.async)
  int* sLabF = reinterpret_cast<int*>(sLabRS + 64);              // [64] first column of row r at r & 63
  const int tid = threadIdx.x, lane = tid & 31;
  const int n = e.n;
  const bool is_la = tid >= Cfg::kPairThreads;                 // warp-uniform

  // ---------------- prologue: labels and rhs of the first P rows
  for (int r = tid; r < 64; r += Cfg::kThreads) {
    sLabF[r] = (r < n) ? e.first[r] : 0; sLabRS[r] = (r < n) ? e.row_start[r] : 0;
  }
  for (int o = tid; o < (P + 4) * 6; o += Cfg::kThreads) {             // rhs of rows 0..P-1 (window) and P..P+3 (entering ring)
    const int r = o / 6, q = o - r * 6;
    const double v = (r < n) ? z[6 * (long long)r + q] : 0.0;
    if (r < P) sZ[o] = v; else sZin[(r & 7) * 6 + q] = v;
  }
  for (int o = tid; o < 6 * PS; o += Cfg::kThreads) sL[o] = 0.0;         // sL, sT, sA (padding included)
  if (tid < 40) sZero[tid] = 0.0;
  __syncthreads();

  if (!is_la && kTile2) {
    // =================================================== pair threads, two live 6x6 blocks each: {a,b0} and {a,b1}
    if (Cfg::kRealloc) reg_alloc<Cfg::kPairRegs>();
    const unsigned pm = pair_map[tid];
    const bool is_pair = pm != 0xffffffffu;
    const int a = pm & 0xff, b0 = (pm >> 8) & 0xff, b1r = (pm >> 16) & 0xff;     // a >= b0, b1 ; b1r == 0xff: no second block
    const bool has1 = b1r != 0xff;
    const int b1 = has1 ? b1r : b0;
    double G0[36], G1[36];                                     // rows <-> slot a, columns <-> slot b0 / b1
    auto publish_T = [&](const double (&G)[36], double* dst) {  // dst[q*6+x] = G[x][q]
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        double2* d2 = reinterpret_cast<double2*>(dst + q * 6);
        d2[0] = make_double2(G[q], G[6 + q]);
        d2[1] = make_double2(G[12 + q], G[18 + q]);
        d2[2] = make_double2(G[24 + q], G[30 + q]);
      }
    };
    auto publish_N = [&](const double (&G)[36], double* dst) {  // dst[q*6+x] = G[q][x]
      double2* d2 = reinterpret_cast<double2*>(dst);
#pragma unroll
      for (int q = 0; q < 18; ++q) d2[q] = make_double2(G[2 * q], G[2 * q + 1]);
    };
    auto load_N = [&](double (&G)[36], const double2* src) {    // G = E
#pragma unroll
      for (int q = 0; q < 18; ++q) { const double2 v = src[q]; G[2 * q] = v.x; G[2 * q + 1] = v.y; }
    };
    auto load_T = [&](double (&G)[36], const double2* src) {    // G = E^T
#pragma unroll
      for (int x = 0; x < 6; ++x)
#pragma unroll
        for (int y2 = 0; y2 < 3; ++y2) { const double2 v = src[x * 3 + y2]; G[(2 * y2) * 6 + x] = v.x; G[(2 * y2 + 1) * 6 + x] = v.y; }
    };
    auto init_block = [&](double (&G)[36], int b, bool on) {
      if (on && a < n && b >= sLabF[a]) load_N(G, reinterpret_cast<const double2*>(L + (sLabRS[a] + (b - sLabF[a])) * 36));
      else {
#pragma unroll
        for (int q = 0; q < 36; ++q) G[q] = 0.0;
      }
      if (!on) return;
      if (b == 0 && a >= 1) publish_T(G, sT + a * S);                    // column 0 -> sT[0]
      if (a == 0 && b == 0) publish_N(G, sDg + 36);                      // pivot 0 (scratch: sDg[1])
      if (P > 1 && b == 1 % P && a >= 2) publish_T(G, sA + a * S);       // column 1 -> sA[0]
      if (a == 1 % P && b == 1 % P) publish_N(G, sDg);                   // block (1,1) -> sDg[0]
    };
    init_block(G0, b0, is_pair);
    init_block(G1, b1, is_pair && has1);
    __syncthreads();     // (A) columns 0, 1 published
    __syncthreads();     // (B) look-ahead group: K_0, L_{.,0}, entering row P
    const double2* lp0 = reinterpret_cast<const double2*>(sL + a * S);
    const double2* tq0 = reinterpret_cast<const double2*>(sT + b0 * S);
    const double2* tq1 = reinterpret_cast<const double2*>(sT + b1 * S);
    const double2* zero2 = reinterpret_cast<const double2*>(sZero);
    int da = a, db0 = b0, db1 = b1;                            // (slot - c) mod P ; c = k mod P
    // after its update (if any) a block either takes the entering block, or hands column k+2 over, or rests
    auto settle = [&](double (&G)[36], int b, int db, int cur) {
      const int lo = da < db ? da : db, hi = da < db ? db : da;
      if (lo == 0) {
        const int eidx = (hi == 0) ? P - 1 : hi - 1;           // block (k+P, k+hi) ; hi == 0: the diagonal (k+P,k+P)
        const double2* src = reinterpret_cast<const double2*>(sEnter + (cur * P + eidx) * 36);
        if (da == 0) load_N(G, src); else load_T(G, src);      // slot a / slot b is the entering row
      }
      if (lo != 1 && P > 2 && (da == 2 || db == 2)) {          // column k+2 goes to the look-ahead group of the next step
        double* nA = sA + (cur ^ 1) * PS;
        if (da == 2 && db == 2) publish_N(G, sDg + (cur ^ 1) * 36);
        else if (db == 2) publish_T(G, nA + a * S);            // slot a is the row
        else publish_N(G, nA + b * S);                         // slot b is the row: G = A^T
      }
    };
    for (int k = 0; k < n_stop; ++k) {
      const int cur = k & 1;
      if (is_pair) {
        if (da >= 2) {
          // both blocks in one sweep over L_a; a block that must not change (dead, resting or absent) multiplies by zero
          const double2* lp = lp0 + cur * (PS / 2);
          const double2* t0p = (db0 >= 2) ? tq0 + cur * (PS / 2) : zero2;
          const double2* t1p = (has1 && db1 >= 2) ? tq1 + cur * (PS / 2) : zero2;
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const double2 u0 = t0p[3 * q], u1 = t0p[3 * q + 1], u2 = t0p[3 * q + 2];
            const double2 w0 = t1p[3 * q], w1 = t1p[3 * q + 1], w2 = t1p[3 * q + 2];
#pragma unroll
            for (int xx = 0; xx < 3; ++xx) {
              const double2 l = lp[3 * q + xx];
              double* c0 = G0 + (2 * xx) * 6;
              double* c1 = G0 + (2 * xx + 1) * 6;
              c0[0] -= l.x * u0.x; c0[1] -= l.x * u0.y; c0[2] -= l.x * u1.x; c0[3] -= l.x * u1.y; c0[4] -= l.x * u2.x; c0[5] -= l.x * u2.y;
              c1[0] -= l.y * u0.x; c1[1] -= l.y * u0.y; c1[2] -= l.y * u1.x; c1[3] -= l.y * u1.y; c1[4] -= l.y * u2.x; c1[5] -= l.y * u2.y;
              double* e0 = G1 + (2 * xx) * 6;
              double* e1 = G1 + (2 * xx + 1) * 6;
              e0[0] -= l.x * w0.x; e0[1] -= l.x * w0.y; e0[2] -= l.x * w1.x; e0[3] -= l.x * w1.y; e0[4] -= l.x * w2.x; e0[5] -= l.x * w2.y;
              e1[0] -= l.y * w0.x; e1[1] -= l.y * w0.y; e1[2] -= l.y * w1.x; e1[3] -= l.y * w1.y; e1[4] -= l.y * w2.x; e1[5] -= l.y * w2.y;
            }
          }
        }
        settle(G0, b0, db0, cur);
        if (has1) settle(G1, b1, db1, cur);
      }
      __syncthreads();
      da =(da == 0) ? P - 1 : da - 1;
      db0 = (db0 == 0) ? P - 1 : db0 - 1;
      db1 = (db1 == 0) ? P - 1 : db1 - 1;
    }
    // partial factorisation: hand the Schur-updated trailing window (rows/cols n_stop..n-1) to the separator solve
    if (n_stop < n && J.wdump && is_pair) {
      const int bs = n - n_stop, fin = n_stop & 1;
      auto dump = [&](const double (&G)[36], int b, int db) {
        const int lo = da < db ? da : db, hi = da < db ? db : da;
        if (hi >= bs) return;
        double* dst = J.wdump + ((long long)hi * bs + lo) * 36;      // block (n_stop+hi, n_stop+lo), rows on the hi row
        if (lo == 0 && hi == 0) {
          for (int q = 0; q < 36; ++q) { const int i = q / 6, j = q % 6; dst[q] = (i >= j) ? sDu[i * 6 + j] : sDu[j * 6 + i]; }
        } else if (lo == 0) {
          const int row_slot = (da == 0) ? b : a;                    // column n_stop was the look-ahead group's
          const double* t = sT + fin * PS + row_slot * S;
          for (int q = 0; q < 36; ++q) { const int x = q / 6, y = q % 6; dst[q] = t[y * 6 + x]; }
        } else if (da >= db) {
#pragma unroll
          for (int q = 0; q < 36; ++q) dst[q] = G[q];
        } else {
#pragma unroll
          for (int x = 0; x < 6; ++x)
#pragma unroll
            for (int y = 0; y < 6; ++y) dst[x * 6 + y] = G[y * 6 + x];
        }
      };
      dump(G0, b0, db0);
      if (has1) dump(G1, b1, db1);
    }
  } else if (!is_la) {
    // =================================================== pair threads: one live 6x6 block in registers
    if (Cfg::kRealloc) reg_alloc<Cfg::kPairRegs>();
    const unsigned pm = pair_map[tid];
    const bool is_pair = pm != 0xffffffffu;
    const int a = pm & 0xff, b = (pm >> 8) & 0xff;             // a >= b
    double G[36];                                              // rows <-> slot a, columns <-> slot b
    auto publish_T = [&](double* dst) {                        // dst[q*6+x] = G[x][q]
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        double2* d2 = reinterpret_cast<double2*>(dst + q * 6);
        d2[0] = make_double2(G[q], G[6 + q]);
        d2[1] = make_double2(G[12 + q], G[18 + q]);
        d2[2] = make_double2(G[24 + q], G[30 + q]);
      }
    };
    auto publish_N = [&](double* dst) {                        // dst[q*6+x] = G[q][x]
      double2* d2 = reinterpret_cast<double2*>(dst);
#pragma unroll
      for (int q = 0; q < 18; ++q) d2[q] = make_double2(G[2 * q], G[2 * q + 1]);
    };
    if (is_pair) {
      if (a < n && b >= sLabF[a]) {
        const double2* src = reinterpret_cast<const double2*>(L + (sLabRS[a] + (b - sLabF[a])) * 36);
#pragma unroll
        for (int q = 0; q < 18; ++q) { const double2 v = src[q]; G[2 * q] = v.x; G[2 * q + 1] = v.y; }
      } else {
#pragma unroll
        for (int q = 0; q < 36; ++q) G[q] = 0.0;
      }
      if (b == 0 && a >= 1) publish_T(sT + a * S);                       // column 0 -> sT[0]
      if (a == 0 && b == 0) publish_N(sDg + 36);                         // pivot 0 (scratch: sDg[1])
      if (P > 1 && b == 1 % P && a >= 2) publish_T(sA + a * S);          // column 1 -> sA[0]
      if (a == 1 % P && b == 1 % P) publish_N(sDg);                      // block (1,1) -> sDg[0]
    }
    __syncthreads();     // (A) columns 0, 1 published
    __syncthreads();     // (B) look-ahead group: K_0, L_{.,0}, entering row P
    // per-thread constants of the loop: operand addresses (parity 0) and the distances of the two slots from the pivot
    const double2* lp0 = reinterpret_cast<const double2*>(sL + a * S);
    const double2* tp0 = reinterpret_cast<const double2*>(sT + b * S);
    int da = a, db = b;                                        // (slot - c) mod P ; c = k mod P
    for (int k = 0; k < n_stop; ++k) {
      const int cur = k & 1;
      if (is_pair) {
        const int lo = da < db ? da : db, hi = da < db ? db : da;
        if (lo == 0) {
          // the column-k block is dead: take the entering block (k+P, k+hi) (hi == 0: the diagonal (k+P,k+P))
          const int eidx = (hi == 0) ? P - 1 : hi - 1;
          const double2* src = reinterpret_cast<const double2*>(sEnter + (cur * P + eidx) * 36);
          if (da == 0) {                          // slot a is the entering row: G = E
#pragma unroll
            for (int q = 0; q < 18; ++q) { const double2 v = src[q]; G[2 * q] = v.x; G[2 * q + 1] = v.y; }
          } else {                                // slot b is the entering row: G = E^T
#pragma unroll
            for (int x = 0; x < 6; ++x)
#pragma unroll
              for (int y2 = 0; y2 < 3; ++y2) { const double2 v = src[x * 3 + y2]; G[(2 * y2) * 6 + x] = v.x; G[(2 * y2 + 1) * 6 + x] = v.y; }
          }
        } else if (lo >= 2) {
          const double2* lp = lp0 + cur * (PS / 2);
          const double2* tp = tp0 + cur * (PS / 2);
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const double2 t0 = tp[3 * q], t1 = tp[3 * q + 1], t2 = tp[3 * q + 2];
#pragma unroll
            for (int xx = 0; xx < 3; ++xx) {
              const double2 l = lp[3 * q + xx];
              double* c0 = G + (2 * xx) * 6;
              double* c1 = G + (2 * xx + 1) * 6;
              c0[0] -= l.x * t0.x; c0[1] -= l.x * t0.y; c0[2] -= l.x * t1.x; c0[3] -= l.x * t1.y; c0[4] -= l.x * t2.x; c0[5] -= l.x * t2.y;
              c1[0] -= l.y * t0.x; c1[1] -= l.y * t0.y; c1[2] -= l.y * t1.x; c1[3] -= l.y * t1.y; c1[4] -= l.y * t2.x; c1[5] -= l.y * t2.y;
            }
          }
        }
        // hand column k+2 (the look-ahead group's column of the NEXT step) over: blocks (k+hi, k+2)
        if (lo != 1 && P > 2 && (da == 2 || db == 2)) {
          double* nA = sA + (cur ^ 1) * PS;
          if (da == 2 && db == 2) publish_N(sDg + (cur ^ 1) * 36);
          else if (db == 2) publish_T(nA + a * S);           // slot a is the row
          else publish_N(nA + b * S);                        // slot b is the row: G = A^T
        }
      }
      __syncthreads();
      da = (da == 0) ? P - 1 : da - 1;
      db = (db == 0) ? P - 1 : db - 1;
    }
    // partial factorisation: hand the Schur-updated trailing window (rows/cols n_stop..n-1) to the separator solve
    if (n_stop < n && J.wdump && is_pair) {
      const int lo = da < db ? da : db, hi = da < db ? db : da;
      const int bs = n - n_stop;
      if (hi < bs) {
        double* dst = J.wdump + ((long long)hi * bs + lo) * 36;      // block (n_stop+hi, n_stop+lo), rows on the hi row
        const int fin = n_stop & 1;
        if (lo == 0 && hi == 0) {
          for (int q = 0; q < 36; ++q) { const int i = q / 6, j = q % 6; dst[q] = (i >= j) ? sDu[i * 6 + j] : sDu[j * 6 + i]; }
        } else if (lo == 0) {
          // column n_stop was the look-ahead group's: T_{i,n_stop} sits in sT[fin][slot of the hi row], [q*6+x] = T[x][q]
          const int row_slot = (da == 0) ? b : a;
          const double* t = sT + fin * PS + row_slot * S;
          for (int q = 0; q < 36; ++q) { const int x = q / 6, y = q % 6; dst[q] = t[y * 6 + x]; }
        } else if (da >= db) {
#pragma unroll
          for (int q = 0; q < 36; ++q) dst[q] = G[q];
        } else {
#pragma unroll
          for (int x = 0; x < 6; ++x)
#pragma unroll
            for (int y = 0; y < 6; ++y) dst[x * 6 + y] = G[y * 6 + x];
        }
      }
    }
  } else {
    // =================================================== look-ahead warpgroup (4 warps, one per SMSP)
    if (Cfg::kRealloc) reg_dealloc<Cfg::kLaRegs>();
    const int lt = tid - Cfg::kPairThreads;                     // 0..127
    const int aw = lt >> 5;                                     // 0: pivot chain + forward substitution + labels; 1..3: column items + row stream
    const int it = lt - 32;                                     // item thread id (0..95), negative on warp 0
    int bad = 0;
    // row labels and entering rhs entries reach shared memory by cp.async (rings above): no global-load result is
    // ever held in a look-ahead register (a spilled in-flight load would stall the chain for a full memory latency)
    auto lab_first = [&](int r) -> int { return r < n ? sLabF[r & 63] : 0x7fffffff; };
    auto lab_rs = [&](int r) -> long long { return sLabRS[r & 63]; };

    // row kc+P -> sEnter[kc & 1] in natural order: 16-byte chunk o of the row's envelope part lands at chunk
    // o_lo + o, o_lo = 18 (first - kc - 1); everything else is zero-filled (cp.async src-size 0)
    auto stream_row = [&](int kc) {
      double* dstb = sEnter + ((kc & 1) * P) * 36;
      const int o_lo = (kc + P < n) ? (lab_first(kc + P) - kc - 1) * 18 : 0x40000000;
      const double* rowp = L + lab_rs(kc + P) * 36;
#pragma unroll 2
      for (int o = it; o < P * 18; o += Cfg::kItemThreads) {
        const bool valid = o >= o_lo;
        cp_async16_zfill(dstb + 2 * o, valid ? rowp + 2 * (o - o_lo) : L, valid);
      }
    };
    // warp 0: K = D^-1.  src: 36 row-major, lower triangle read.  dst: 36 row-major, full symmetric.
    auto invert_pivot = [&](const double* src, double* dst, int kc) {
      sym6_block_inverse_warp(src, dst, sInv, lane);
      // every entry of K carries one of the two reciprocals: four entries are enough to catch a singular pivot
      if (!isfinite((dst[0] + dst[35]) + (dst[18] + dst[13]))) bad = 1;
      if (lane < 18 && kc < n_stop) reinterpret_cast<double2*>(dinv + (long long)kc * 36)[lane] = reinterpret_cast<const double2*>(dst)[lane];
    };
    // column item: row slot `slot`, block row x.  t = T_{i,col}[x][.] (already updated); writes L_{i,col}[x][.] = t K
    auto scale_item = [&](const double* Kp, const double (&t)[6], int slot, int x, int row, int col, int par) {
      const double2* k2 = reinterpret_cast<const double2*>(Kp);
      double v0[6], v1[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) { v0[c] = 0.0; v1[c] = 0.0; }
#pragma unroll
      for (int q = 0; q < 6; q += 2) {
        const double2 a0 = k2[3 * q], a1 = k2[3 * q + 1], a2 = k2[3 * q + 2];
        const double2 b0 = k2[3 * q + 3], b1 = k2[3 * q + 4], b2 = k2[3 * q + 5];
        v0[0] += t[q] * a0.x; v0[1] += t[q] * a0.y; v0[2] += t[q] * a1.x; v0[3] += t[q] * a1.y; v0[4] += t[q] * a2.x; v0[5] += t[q] * a2.y;
        v1[0] += t[q + 1] * b0.x; v1[1] += t[q + 1] * b0.y; v1[2] += t[q + 1] * b1.x; v1[3] += t[q + 1] * b1.y; v1[4] += t[q + 1] * b2.x; v1[5] += t[q + 1] * b2.y;
      }
      double* lt_ = sL + par * PS + slot * S;
#pragma unroll
      for (int c = 0; c < 6; ++c) { v0[c] += v1[c]; lt_[c * 6 + x] = v0[c]; }
      const int rf = lab_first(row);
      if (col >= rf && col < n_stop) {      // a partial factorisation leaves column n_stop (the separator's first) untouched in memory
        double2* g = reinterpret_cast<double2*>(L + (lab_rs(row) + (col - rf)) * 36 + x * 6);
        g[0] = make_double2(v0[0], v0[1]); g[1] = make_double2(v0[2], v0[3]); g[2] = make_double2(v0[4], v0[5]);
      }
    };

    __syncthreads();     // (A)
    // ---- column 0: K_0, L_{.,0}; entering row P; labels
    if (aw == 0) invert_pivot(sDg + 36, sK, 0);
    else stream_row(0);
    named_bar_sync(1, Cfg::kLaThreads);
    if (aw != 0) {
      for (int o = it; o < Cfg::kItems; o += Cfg::kItemThreads) {
        const int h = 1 + o / 6, x = o - (h - 1) * 6;              // row h of column 0, slot h
        double t[6];
#pragma unroll
        for (int q = 0; q < 6; ++q) t[q] = sT[h * S + q * 6 + x];
        scale_item(sK, t, h, x, h, 0, 0);
      }
      cp_async_wait_all();
    }
    __syncthreads();     // (B)

    // per-thread item constants: item o -> row k+h (h = 2..P), block row x ; slot = (c + h) mod P advances with c
    int slot_[Cfg::kRounds], x_[Cfg::kRounds], h_[Cfg::kRounds];
    bool act_[Cfg::kRounds], ent_[Cfg::kRounds];
#pragma unroll
    for (int rd = 0; rd < Cfg::kRounds; ++rd) {
      const int o = it + rd * Cfg::kItemThreads;
      const int oo = (o >= 0 && o < Cfg::kItems) ? o : 0;
      const int h = 2 + oo / 6;
      x_[rd] = oo - (h - 2) * 6;
      h_[rd] = h;
      slot_[rd] = h % P;                                            // c = 0
      act_[rd] = o >= 0 && o < Cfg::kItems;
      ent_[rd] = h == P;                                            // the entering row k+P
    }
    int c = 0;
    for (int k = 0; k < n_stop; ++k) {
      const int cur = k & 1, nxt = cur ^ 1;
      int s1 = c + 1; if (s1 >= P) s1 -= P;
      const double* Lc = sL + cur * PS;
      const double* T1 = sT + cur * PS + s1 * S;                    // T_{k+1,k}: [r*6+q] = T[q][r]
      if (aw == 0) {
        // ---- pivot chain: D_{k+1} = A_{k+1,k+1} - L_{k+1,k} T_{k+1,k}^T (lane <-> lower-triangle element), inverse
        if (k + 1 < n) {
          const double* dg = sDg + cur * 36;
          const double* l1 = Lc + s1 * S;
          const int l21 = lane < 21 ? lane : 0;
          const int i = (l21 >= 15) ? 5 : (l21 >= 10) ? 4 : (l21 >= 6) ? 3 : (l21 >= 3) ? 2 : (l21 >= 1) ? 1 : 0;
          const int j = l21 - i * (i + 1) / 2;
          double v = dg[i * 6 + j];
          double w = 0.0;
#pragma unroll
          for (int q = 0; q < 6; q += 2) { v -= l1[q * 6 + i] * T1[q * 6 + j]; w += l1[(q + 1) * 6 + i] * T1[(q + 1) * 6 + j]; }
          v -= w;
          if (lane < 21) sDu[i * 6 + j] = v;
          __syncwarp();
          invert_pivot(sDu, sK + nxt * 36, k + 1);
        }
        named_bar_sync(1, Cfg::kLaThreads);                         // K_{k+1} visible to the item warps
        // ---- forward substitution with the final z_k : lane <-> row k+1+lane
        double zk[6];
#pragma unroll
        for (int q = 0; q < 6; ++q) zk[q] = sZ[c * 6 + q];
        if (lane < 6) z[6 * (long long)k + lane] = sZ[c * 6 + lane];
        __syncwarp();
        if (lane + 1 < P) {
          int slot = c + 1 + lane; if (slot >= P) slot -= P;
          const double2* lt2 = reinterpret_cast<const double2*>(Lc + slot * S);
          double acc[6];
#pragma unroll
          for (int x = 0; x < 6; ++x) acc[x] = sZ[slot * 6 + x];
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const double2 l0 = lt2[3 * q], l1 = lt2[3 * q + 1], l2 = lt2[3 * q + 2];
            acc[0] -= l0.x * zk[q]; acc[1] -= l0.y * zk[q]; acc[2] -= l1.x * zk[q]; acc[3] -= l1.y * zk[q]; acc[4] -= l2.x * zk[q]; acc[5] -= l2.y * zk[q];
          }
#pragma unroll
          for (int x = 0; x < 6; ++x) sZ[slot * 6 + x] = acc[x];
        }
        __syncwarp();
        if (lane < 6) sZ[c * 6 + lane] = (k + P < n) ? sZin[((k + P) & 7) * 6 + lane] : 0.0;   // row k+P takes slot c
        // columns 0..k of L were complete in global memory before the block barrier this warp passed at the top of the step
        // (never the final value n_stop: that one comes after the last barrier, when the dumps and the status are out too)
        if (J.progress && lane == 0 && (k & 3) == 3 && k + 1 < n_stop) progress_publish(J.progress, k + 1);
      } else {
        // ---- column items: T_{i,k+1} = A_{i,k+1} - L_{i,k} T_{k+1,k}^T for rows i = k+2 .. k+P, then L = T D_{k+1}^-1
        stream_row(k + 1);                                          // row k+1+P -> sEnter[nxt]
        if (it < 5) {                                               // ring refills: labels of row k+40, rhs of row k+P+4
          const int rl = k + 40, rz = k + P + 4;
          if (it == 0 && rl < n) {
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(sLabF + (rl & 63))), "l"(e.first + rl));
          } else if (it == 1 && rl < n) {
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(sLabRS + (rl & 63))), "l"(e.row_start + rl));
          } else if (it >= 2 && rz < n) {
            cp_async16_zfill(sZin + (rz & 7) * 6 + 2 * (it - 2), z + 6 * (long long)rz + 2 * (it - 2), true);
          }
        }
        double t[Cfg::kRounds][6];
#pragma unroll
        for (int rd = 0; rd < Cfg::kRounds; ++rd) {
          const int slot = slot_[rd], x = x_[rd];
          if (ent_[rd]) {
            const double* en = sEnter + (cur * P) * 36 + x * 6;     // block (k+P, k+1): index 0, row-major
#pragma unroll
            for (int q = 0; q < 6; ++q) t[rd][q] = en[q];
          } else {
            const double* as = sA + cur * PS + slot * S;
#pragma unroll
            for (int q = 0; q < 6; ++q) t[rd][q] = as[q * 6 + x];
            const double* lr = Lc + slot * S;
#pragma unroll
            for (int r = 0; r < 6; ++r) {
              const double lv = lr[r * 6 + x];
              const double2 u0 = reinterpret_cast<const double2*>(T1 + r * 6)[0];
              const double2 u1 = reinterpret_cast<const double2*>(T1 + r * 6)[1];
              const double2 u2 = reinterpret_cast<const double2*>(T1 + r * 6)[2];
              t[rd][0] -= lv * u0.x; t[rd][1] -= lv * u0.y; t[rd][2] -= lv * u1.x; t[rd][3] -= lv * u1.y; t[rd][4] -= lv * u2.x; t[rd][5] -= lv * u2.y;
            }
          }
          if (act_[rd]) {
            double* tn = sT + nxt * PS + slot * S;
#pragma unroll
            for (int q = 0; q < 6; ++q) tn[q * 6 + x] = t[rd][q];
          }
        }
        named_bar_sync(1, Cfg::kLaThreads);                         // K_{k+1} ready
        const double* Kp = sK + nxt * 36;
#pragma unroll
        for (int rd = 0; rd < Cfg::kRounds; ++rd) {
          if (act_[rd]) scale_item(Kp, t[rd], slot_[rd], x_[rd], k + h_[rd], k + 1, nxt);
          if (++slot_[rd] == P) slot_[rd] = 0;
        }
        cp_async_wait_all();
      }
      __syncthreads();
      if (++c == P) c = 0;
    }
    if (n_stop < n && J.zdump && aw == 0) {                         // forward-substituted rhs of the separator rows
      for (int o = lane; o < (n - n_stop) * 6; o += 32) {
        const int i = n_stop + o / 6;
        J.zdump[o] = sZ[(i % P) * 6 + o % 6];
      }
    }
    if (bad) J.status[0] = 1;
  }
  if (J.progress) {                                               // the last global write of the CTA (env_types.h)
    __syncthreads();
    if (tid == 0) progress_publish(J.progress, n_stop);
  }
}

// =====================================================================================================
// Backward substitution  x <- L^-T x  on ONE consumer warp, no block barriers.
//
// Row-oriented: when x_i is final, every block L_ij of row i (columns first[i]..i-1, contiguous in memory) sends
// x_j -= L_ij^T x_i.  Lane s of the consumer warp OWNS x_j for the row j == s (mod 32) of the live 32-row window and
// keeps it in registers; x_i reaches the other lanes by shuffles, so the dependent chain per row is one shuffle +
// a short FMA tree instead of two block barriers.  A producer warp streams L through a ring of shared-memory stages
// guarded by full/empty mbarriers: rows are contiguous in memory, so ONE cp.async.bulk brings a group of kBsGroup
// consecutive rows; it also leaves each row's first column and offset in the stage header.  The x entries that
// enter the window are fetched kBsXDist rows ahead, and the next row's block is loaded from shared memory while the
// current row is applied (software pipeline).
constexpr int kBsStages = 6;
constexpr int kBsGroup = 4;                                  // rows per stage (divides 32)
constexpr int kBsRowsDoubles = kBsGroup * 31 * 36;           // L blocks of the staged rows
constexpr int kBsStageDoubles = kBsRowsDoubles + kBsGroup * 6;   // + the x entries that enter the window with these rows
constexpr size_t kBsSmem = sizeof(double) * (size_t)kBsStages * kBsStageDoubles + 2 * kBsStages * sizeof(unsigned long long) +
                           kBsStages * kBsGroup * 3 * sizeof(int) + 64;

LVBA_DEV unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
LVBA_DEV void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
LVBA_DEV void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LVBA_DEV void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
LVBA_DEV void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
LVBA_DEV void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__global__ void __launch_bounds__(64, 1)
env_backsolve_warp_kernel(const BacksolveJob* __restrict__ jobs) {
  constexpr int NS = kBsStages, R = kBsGroup;
  extern __shared__ __align__(128) double smem_bs[];
  double* ring = smem_bs;                                                       // [NS][kBsStageDoubles]
  unsigned long long* full = reinterpret_cast<unsigned long long*>(ring + NS * kBsStageDoubles);   // [NS]
  unsigned long long* empty = full + NS;                                        // [NS]
  int* sRowF = reinterpret_cast<int*>(empty + NS);                              // [NS][R] first column of each staged row
  int* sRowOff = sRowF + NS * R;                                                // [NS][R] offset (doubles) of each staged row inside the stage
  int* sRowX = sRowOff + NS * R;                                                // [NS][R] offset (doubles) of the x entry that replaces the row, or -1
  const BacksolveJob J = jobs[blockIdx.x];
  const EnvView e = J.e;
  const double* __restrict__ L = J.L;
  double* __restrict__ x = J.x;
  const int n_given = J.n_given, n = e.n;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) {
    for (int d = 0; d < NS; ++d) { mbar_init(full + d, 1); mbar_init(empty + d, 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (n <= 0) return;
  const int n_groups = (n + R - 1) / R;
  if (tid >= 32) {
    // ------------------------------------------------ producer warp: two bulk copies per group of R rows (L rows, x entries)
    int lab_f = 0; long long lab_rs = 0;
    for (int g = 0; g < n_groups; ++g) {
      const int itn = g * R;                         // rows i_hi = n-1-itn down to i_lo
      const int i_hi = n - 1 - itn;
      const int i_lo = (i_hi - R + 1 > 0) ? i_hi - R + 1 : 0;
      if ((itn & 31) == 0) {                         // labels of rows i_hi, i_hi-1, .., i_hi-31 : lane l holds row i_hi-l
        const int r = i_hi - lane;
        lab_f = (r >= 0) ? e.first[r] : 0;
        lab_rs = (r >= 0) ? e.row_start[r] : 0;
      }
      const int base_l = itn & 31;
      const int f_hi = __shfl_sync(0xffffffffu, lab_f, base_l);
      const long long rs_hi = __shfl_sync(0xffffffffu, lab_rs, base_l);
      const long long rs_lo = __shfl_sync(0xffffffffu, lab_rs, base_l + (i_hi - i_lo));
      // this lane's row of the group (lanes 0..R-1): first column and offset from the group's base
      const int my_f = __shfl_sync(0xffffffffu, lab_f, base_l + (lane < R ? lane : 0));
      const long long my_rs = __shfl_sync(0xffffffffu, lab_rs, base_l + (lane < R ? lane : 0));
      const int st = g % NS;
      const unsigned ph = (unsigned)((g / NS) & 1);
      if (lane == 0) mbar_wait(empty + st, ph ^ 1u);
      __syncwarp();
      const int xr_hi = i_hi - 32;                   // x entries of rows i_lo-32 .. i_hi-32 (those >= 0), ascending in memory
      const int xr_lo = (i_lo - 32 > 0) ? i_lo - 32 : 0;
      if (lane < R && i_hi - lane >= 0) {
        const int i = i_hi - lane;
        sRowF[st * R + lane] = my_f;
        sRowOff[st * R + lane] = (int)((my_rs - rs_lo) * 36);
        sRowX[st * R + lane] = (i - 32 >= 0) ? kBsRowsDoubles + (i - 32 - xr_lo) * 6 : -1;
      }
      __syncwarp();
      if (lane == 0) {
        const long long nblk = rs_hi + (i_hi - f_hi + 1) - rs_lo;      // blocks of rows i_lo..i_hi, diagonal blocks included
        const unsigned xbytes = (xr_hi >= xr_lo) ? (unsigned)((xr_hi - xr_lo + 1) * 48) : 0u;
        double* dst = ring + st * kBsStageDoubles;
        mbar_arrive_expect_tx(full + st, (unsigned)(nblk * 288) + xbytes);
        bulk_g2s(dst, L + rs_lo * 36, (unsigned)(nblk * 288), full + st);
        if (xbytes) bulk_g2s(dst + kBsRowsDoubles, x + 6 * (long long)xr_lo, xbytes, full + st);
      }
    }
  } else {
    // ------------------------------------------------ consumer warp: three-stage software pipeline over the rows
    //   M: row metadata (first column, offsets) two rows ahead ; B: block + x entry one row ahead ; C: apply
    double xs[6];
    {
      const int r = (n - 1) - (((n - 1) - lane) % 32 + 32) % 32;   // the row == lane (mod 32) inside [n-32, n-1]
#pragma unroll
      for (int q = 0; q < 6; ++q) xs[q] = (r >= 0) ? x[6 * (long long)r + q] : 0.0;
    }
    double2 blk0[18], blk1[18];
    double2 xe0[3], xe1[3];
    bool on0 = false, on1 = false, xon0 = false, xon1 = false;
    int mF = 0, mOff = 0, mX = -1;                     // metadata of the row whose block is loaded next
    auto meta = [&](int itn) {                         // stage M for the row of iteration itn
      const int g = itn / R, st = g % NS, rr = itn % R;
      if (rr == 0) { mbar_wait(full + st, (unsigned)((g / NS) & 1)); __syncwarp(); }
      mF = sRowF[st * R + rr]; mOff = sRowOff[st * R + rr]; mX = sRowX[st * R + rr];
    };
    // stage B for row i, using the metadata in mF/mOff/mX.  The loaded values are used unconditionally; the flags
    // decide at the END of the apply stage whether they count (no select sits between the loads and their use)
    auto fetch = [&](int i, int itn, double2 (&blk)[18], double2 (&xe)[3], bool& on, bool& xon) {
      const double* stg = ring + ((itn / R) % NS) * kBsStageDoubles;
      const int upto = i < n_given ? i : n_given;      // given rows only act on the pivots' columns
      const int cnt = upto > mF ? upto - mF : 0;
      const int jo = (lane - mF) & 31;                 // column mF + jo is the one congruent to this lane
      on = jo < cnt;
      xon = mX >= 0;
      const double2* b2 = reinterpret_cast<const double2*>(stg + mOff + (on ? jo : 0) * 36);
#pragma unroll
      for (int t = 0; t < 18; ++t) blk[t] = b2[t];
      const double2* x2 = reinterpret_cast<const double2*>(stg + (xon ? mX : 0));
#pragma unroll
      for (int t = 0; t < 3; ++t) xe[t] = x2[t];
    };
    auto apply = [&](int i, int itn, const double2 (&blk)[18], const double2 (&xe)[3], bool on, bool xon) {   // stage C for row i
      const int owner = i & 31;
      const bool mine = lane == owner;
      double xi[6];
#pragma unroll
      for (int q = 0; q < 6; ++q) xi[q] = __shfl_sync(0xffffffffu, xs[q], owner);
      if (mine) {
        double2* xo = reinterpret_cast<double2*>(x + 6 * (long long)i);
        xo[0] = make_double2(xs[0], xs[1]); xo[1] = make_double2(xs[2], xs[3]); xo[2] = make_double2(xs[4], xs[5]);
      }
      double v0[6], v1[6];
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) { v0[cc] = 0.0; v1[cc] = 0.0; }
#pragma unroll
      for (int q = 0; q < 6; q += 2) {
        const double2 a0 = blk[3 * q], a1 = blk[3 * q + 1], a2 = blk[3 * q + 2];
        const double2 c0 = blk[3 * q + 3], c1 = blk[3 * q + 4], c2 = blk[3 * q + 5];
        v0[0] += a0.x * xi[q]; v0[1] += a0.y * xi[q]; v0[2] += a1.x * xi[q]; v0[3] += a1.y * xi[q]; v0[4] += a2.x * xi[q]; v0[5] += a2.y * xi[q];
        v1[0] += c0.x * xi[q + 1]; v1[1] += c0.y * xi[q + 1]; v1[2] += c1.x * xi[q + 1]; v1[3] += c1.y * xi[q + 1]; v1[4] += c2.x * xi[q + 1]; v1[5] += c2.y * xi[q + 1];
      }
      const double xen[6] = {xe[0].x, xe[0].y, xe[1].x, xe[1].y, xe[2].x, xe[2].y};
#pragma unroll
      for (int cc = 0; cc < 6; ++cc) {
        const double upd = xs[cc] - (v0[cc] + v1[cc]);
        // row i leaves the window and row i-32 takes its lane; lanes without a block in row i keep their value
        xs[cc] = mine ? (xon ? xen[cc] : 0.0) : (on ? upd : xs[cc]);
      }
      if ((itn % R) == R - 1 || i == 0) {              // every row of this group has been applied: the stage is free
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + ((itn / R) % NS));
      }
    };
    meta(0);
    fetch(n - 1, 0, blk0, xe0, on0, xon0);
    if (n > 1) meta(1);
    for (int i = n - 1; i >= 0; i -= 2) {
      const int itn = n - 1 - i;
      if (i >= 1) fetch(i - 1, itn + 1, blk1, xe1, on1, xon1);
      if (i >= 2) meta(itn + 2);
      apply(i, itn, blk0, xe0, on0, xon0);
      if (i >= 1) {
        if (i >= 2) fetch(i - 2, itn + 2, blk0, xe0, on0, xon0);
        if (i >= 3) meta(itn + 3);
        apply(i - 1, itn + 1, blk1, xe1, on1, xon1);
      }
    }
  }
}

}  // namespace lvba
