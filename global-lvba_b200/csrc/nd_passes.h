// nd_passes.h — the passes of the substructured block LDL^T (plan: nd_plan.h) and the order they run in.
//
// Replaces the single sequential elimination the reference gets from Eigen::SimplicialLDLT
// (include/BALM/bavoxel.hpp:695-710) / Ceres DENSE_SCHUR (src/lvba_system.cpp:1573-1575); SURVEY.md section 8(e).
//
// Every data-layout pass is a functor over an index range (as envelope_wide.h / voxel_pipeline.h): the device runs it as
// a grid-stride kernel (nd_solver.cuh), the CPU check as a plain loop (tests/emu/nd_emu.cpp) — the same code.  The four
// heavy steps (banded / dense factorisation, spike forward substitution, SYRK, backward substitution) are kernels on the
// device (factor_la.cuh, nd_kernels.cuh) and reference loops in the CPU check; `run()` below is the one place that says
// in which order everything happens, for both.
#pragma once
#include <math.h>
#include <stdint.h>

#include "env_types.h"
#include "nd_plan.h"

#if defined(__CUDACC__)
#define LVBA_NHD __host__ __device__ __forceinline__
#else
#define LVBA_NHD inline
#endif

namespace lvba {
namespace nd {

// device copy of a plan node
struct NodeDev {
  int kind, r0, npiv, ntrail, sa, wa, sc, wc, left, right, ks, nE, nb, zrows;
  long long offU, offu, offZ, offE, offT, offW, offw;
};
inline NodeDev to_dev(const Node& v) {
  return NodeDev{v.kind, v.r0, v.npiv, v.ntrail, v.sa, v.wa, v.sc, v.wc, v.left, v.right, v.ks, v.nE, v.nb, v.zrows,
                 v.offU, v.offu, v.offZ, v.offE, v.offT, v.offW, v.offw};
}

// Forward substitution of KS right-hand sides through the unit-lower block factor of one factorisation instance:
//   rows k < n_stop (pivots):      Z_k = E_k - sum_{j<k} L_kj Z_j
//   rows k >= n_stop (trailing):   Z_k =     - sum_{j<n_stop} L_kj Z_j      (what the right boundary inherits)
// E has nE block rows ([nE][6][KS], zero beyond); Z is [e.n][6][KS].
struct SpikeJob {
  EnvView e;
  const double* L;
  int n_stop;
  const double* E;
  int nE;
  double* Z;
  int KS;
  const int* progress = nullptr;   // FactorJob::progress of the factorisation that produces L, when the two run side by side
  // per group of right-hand sides (one spike CTA): the number of leading block rows of Z that are final in global memory,
  // published with release semantics every few rows and, once the factorisation has finished too, with the value e.n; for
  // the SYRK that runs beside the spike.  nullptr: nothing is published.
  int* zprog = nullptr;
};
// U -= sum_k Z_k^T K_k Z_k  and  u -= sum_k Z_k^T K_k w_k  over the pivot rows of one node (K_k = D_k^-1).
// U: dense lower block triangle over KS/6 block rows, block (i,j), j <= i, at (i(i+1)/2 + j)*36 (leading part of the node's U).
struct SyrkSeg {
  const double* Z;     // [rows][6][KS]
  const double* K;     // [rows][36]
  const double* w;     // [rows][6]
  int rows;
  int KS;
  double* U;
  double* u;
  // running beside the spike that produces Z and the factorisation that produces K and w: the SYRK stages rows below r once
  // the zprog counters (SpikeJob::zprog) of its two column tiles have reached r and fprog (FactorJob::progress, which covers
  // D^-1 and z one row behind L) r + 1 or its final value; the CTAs of the last rows also wait for zdone (the spike's final
  // value), so that the SYRK finishes after both.  nullptr: no waiting.
  const int* fprog = nullptr;
  const int* zprog = nullptr;
  int zdone = 0;
};

// everything the passes touch
struct Tables {
  int n;
  const int* first;               // global envelope
  const long long* row_start;
  const NodeDev* nodes;
  const double* H;                // input matrix (envelope layout), lower triangle of the diagonal blocks valid
  const double* dadd;             // [6n] added to the scalar diagonal
  double* L;                      // working copy of H + dadd; the leaves factorise in place
  double* z;                      // [6n] in: right-hand side; interiors: forward-substituted in place
  double* zs;                     // [6n] separator rows: assembled right-hand side, forward-substituted in place
  double* dinv;                   // [n][36]
  double* x;                      // [6n] solution
  double* U; double* u; double* Z; double* E; double* T; double* W; double* w;     // pools (offsets in NodeDev); u == U (one pool)
  // multi-GPU only: writable views of H / dadd (the rows of the other ranks' rank separators arrive through the exchange region)
  double* Hw; double* daddw;
  int* prog = nullptr;            // [nodes] progress counters (FactorJob::progress), then [nodes][zstride] those of the spike CTAs
                                  // (SpikeJob::zprog), or null: factorisation, spike and SYRK run one after the other
  int zstride = 0;                // spike counters per node (groups of right-hand sides of the widest node)
};

LVBA_NHD void tri_dec(long long t, int& a, int& b) {
  long long i = (long long)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
  while ((i + 1) * (i + 2) / 2 <= t) ++i;
  while (i * (i + 1) / 2 > t) --i;
  a = (int)i;
  b = (int)(t - i * (i + 1) / 2);
}
LVBA_NHD long long tri_off(int i, int j) { return ((long long)i * (i + 1) / 2 + j) * 36; }
// element [x][y] of block (r, c), c <= r, of the input matrix with the damping on its scalar diagonal; 0 outside the envelope.
// Diagonal blocks are read through their lower triangle only (SURVEY.md Q4).
LVBA_NHD double mat_elem(const Tables& t, int r, int c, int x, int y) {
  if (c < t.first[r]) return 0.0;
  const double* b = t.H + (t.row_start[r] + (c - t.first[r])) * 36;
  if (r == c) {
    const double v = (x >= y) ? b[x * 6 + y] : b[y * 6 + x];
    return (x == y) ? v + t.dadd[6 * r + x] : v;
  }
  return b[x * 6 + y];
}
// element [x][y] of block (i, j) of a child's update matrix (any i, j: the lower triangle is stored)
LVBA_NHD double upd_elem(const double* U, int i, int j, int x, int y) {
  return (i >= j) ? U[tri_off(i, j) + x * 6 + y] : U[tri_off(j, i) + y * 6 + x];
}

// ---- L = H + diag(dadd): a plain copy, then items = 6 n
struct AddDiagF {
  Tables t;
  LVBA_NHD void operator()(int64_t i) const {
    const int r = (int)(i / 6), a = (int)(i % 6);
    t.L[(t.row_start[r] + (r - t.first[r])) * 36 + a * 7] += t.dadd[i];
  }
};

// ---- right-hand sides of the leaves' spikes: E[k][x][6 si + y] = A(r0 + k, sa + si)[x][y].  items = ids x stride
struct LeafEF {
  Tables t; const int* ids; long long stride;
  LVBA_NHD void operator()(int64_t it) const {
    const NodeDev& v = t.nodes[ids[it / stride]];
    const long long e = it % stride;
    if (e >= (long long)v.nE * 6 * v.ks) return;
    const int k = (int)(e / (6 * v.ks)), rem = (int)(e % (6 * v.ks)), x = rem / v.ks, col = rem % v.ks, si = col / 6, y = col % 6;
    const int r = v.r0 + k, c = v.sa + si;
    double val = 0.0;
    if (c >= t.first[r]) val = t.H[(t.row_start[r] + (c - t.first[r])) * 36 + x * 6 + y];
    t.E[v.offE + e] = val;
  }
};
inline long long leaf_e_stride(const Plan& P) {
  long long s = 1;
  for (int c = 0; c < P.p; ++c) s = std::max<long long>(s, (long long)P.nodes[c].nE * 6 * P.nodes[c].ks);
  return s;
}

// ---- update matrix of a leaf beyond what the SYRK accumulates: [c,a] = trailing rows of the spike, [c,c] = the factor
//      kernel's trailing window minus the original entries, u[c] = forward-substituted minus original right-hand side
struct LeafFinalF {
  Tables t; const int* ids; long long stride;
  LVBA_NHD void operator()(int64_t it) const {
    const NodeDev& v = t.nodes[ids[it / stride]];
    const long long e = it % stride;
    const long long nU = (long long)v.nb * (v.nb + 1) / 2 * 36;
    if (e < nU) {
      int bi, bj;
      tri_dec(e / 36, bi, bj);
      const int el = (int)(e % 36), x = el / 6, y = el % 6;
      if (bi < v.wa) return;                                        // [a,a]: zeroed, then accumulated by the SYRK
      const int ci = bi - v.wa;
      if (bj < v.wa) {                                              // [c,a]
        t.U[v.offU + e] = t.Z[v.offZ + ((long long)(v.npiv + ci) * 6 + x) * v.ks + 6 * bj + y];
      } else {                                                      // [c,c]
        const int cj = bj - v.wa;
        int xx = x, yy = y;
        if (ci == cj && x < y) { xx = y; yy = x; }                  // diagonal blocks: lower triangle only
        const double wd = t.W[v.offW + ((long long)ci * v.wc + cj) * 36 + xx * 6 + yy];
        t.U[v.offU + e] = wd - mat_elem(t, v.sc + ci, v.sc + cj, xx, yy);
      }
    } else if (e < nU + (long long)v.nb * 6) {
      const int o = (int)(e - nU), bi = o / 6, q = o % 6;
      if (bi < v.wa) return;
      const int ci = bi - v.wa;
      t.u[v.offu + o] = t.w[v.offw + ci * 6 + q] - t.z[6 * (long long)(v.sc + ci) + q];
    }
  }
};
inline long long leaf_final_stride(const Plan& P) {
  long long s = 1;
  for (int c = 0; c < P.p; ++c) s = std::max<long long>(s, (long long)P.nodes[c].nb * (P.nodes[c].nb + 1) / 2 * 36 + P.nodes[c].nb * 6);
  return s;
}

// ---- front of a separator node: pivot block T, right-hand side, boundary columns E, initial update matrix
//      (extend-add of the two children; original entries enter where the first of the two rows is eliminated)
struct SepAssembleF {
  Tables t; const int* ids; long long stride;
  LVBA_NHD void operator()(int64_t it) const {
    const NodeDev& v = t.nodes[ids[it / stride]];
    long long e = it % stride;
    const NodeDev& lc = t.nodes[v.left];           // boundary (a, v): a-part v.wa rows, c-part = this separator
    const NodeDev& rc = t.nodes[v.right];          // boundary (v, c): a-part = this separator, c-part v.wc rows
    const double* UL = t.U + lc.offU;
    const double* UR = t.U + rc.offU;
    const long long nT = (long long)v.npiv * (v.npiv + 1) / 2 * 36;
    if (e < nT) {
      int bi, bj;
      tri_dec(e / 36, bi, bj);
      const int el = (int)(e % 36), x = el / 6, y = el % 6;
      double val;
      if (bi == bj && x < y) val = 0.0;                            // never read (lower triangle of the pivot blocks)
      else val = mat_elem(t, v.r0 + bi, v.r0 + bj, x, y) + upd_elem(UL, v.wa + bi, v.wa + bj, x, y) + upd_elem(UR, bi, bj, x, y);
      t.T[v.offT + e] = val;
      return;
    }
    e -= nT;
    const long long nEe = (long long)v.npiv * 6 * v.ks;
    if (e < nEe) {
      const int k = (int)(e / (6 * v.ks)), rem = (int)(e % (6 * v.ks)), x = rem / v.ks, col = rem % v.ks;
      double val;
      if (col < 6 * v.wa) {                                         // A(S_v row k, S_a row aj)[x][y]
        const int aj = col / 6, y = col % 6;
        val = mat_elem(t, v.r0 + k, v.sa + aj, x, y) + upd_elem(UL, v.wa + k, aj, x, y);
      } else {                                                      // A(S_c row cj, S_v row k)[y][x]
        const int cc = col - 6 * v.wa, cj = cc / 6, y = cc % 6;
        val = mat_elem(t, v.sc + cj, v.r0 + k, y, x) + upd_elem(UR, v.npiv + cj, k, y, x);
      }
      t.E[v.offE + e] = val;
      return;
    }
    e -= nEe;
    const long long nU = (long long)v.nb * (v.nb + 1) / 2 * 36;
    if (e < nU) {
      int bi, bj;
      tri_dec(e / 36, bi, bj);
      const int el = (int)(e % 36), x = el / 6, y = el % 6;
      double val = 0.0;
      if (bi < v.wa) val = upd_elem(UL, bi, bj, x, y);                                   // [a,a]
      else if (bj >= v.wa) val = upd_elem(UR, v.npiv + (bi - v.wa), v.npiv + (bj - v.wa), x, y);   // [c,c]
      t.U[v.offU + e] = val;                                                             // [c,a]: filled by the SYRK alone
      return;
    }
    e -= nU;
    if (e < (long long)v.npiv * 6) {
      const int k = (int)(e / 6), q = (int)(e % 6);
      t.zs[6 * (long long)(v.r0 + k) + q] = t.z[6 * (long long)(v.r0 + k) + q] + t.u[lc.offu + (v.wa + k) * 6 + q] + t.u[rc.offu + k * 6 + q];
      return;
    }
    e -= (long long)v.npiv * 6;
    if (e < (long long)v.nb * 6) {
      const int bi = (int)(e / 6), q = (int)(e % 6);
      t.u[v.offu + e] = (bi < v.wa) ? t.u[lc.offu + bi * 6 + q] : t.u[rc.offu + (v.npiv + (bi - v.wa)) * 6 + q];
    }
  }
};
inline long long sep_items(const Node& v) {
  return (long long)v.npiv * (v.npiv + 1) / 2 * 36 + (long long)v.npiv * 6 * v.ks + (long long)v.nb * (v.nb + 1) / 2 * 36 + (long long)v.npiv * 6 + (long long)v.nb * 6;
}

// ---- downwards: x_K = D^-1 (w_K - Z x_boundary) for the pivot rows (the backward substitution with L^T follows).
//      items = ids x stride rows
struct CorrectApplyF {
  Tables t; const int* ids; long long stride;
  LVBA_NHD void operator()(int64_t it) const {
    const NodeDev& v = t.nodes[ids[it / stride]];
    const int k = (int)(it % stride);
    if (k >= v.npiv) return;
    const double* wv = (v.kind == 0 ? t.z : t.zs) + 6 * (long long)(v.r0 + k);
    double c[6];
    for (int q = 0; q < 6; ++q) {
      const double* zr = t.Z + v.offZ + ((long long)k * 6 + q) * v.ks;
      double s0 = 0.0, s1 = 0.0;
      const int na = 6 * v.wa;
      const double* xa = t.x + 6 * (long long)v.sa;
      const double* xc = t.x + 6 * (long long)v.sc;
      int col = 0;
      for (; col + 1 < v.ks; col += 2) {
        s0 += zr[col] * (col < na ? xa[col] : xc[col - na]);
        s1 += zr[col + 1] * (col + 1 < na ? xa[col + 1] : xc[col + 1 - na]);
      }
      if (col < v.ks) s0 += zr[col] * (col < na ? xa[col] : xc[col - na]);
      c[q] = wv[q] - (s0 + s1);
    }
    const double* K = t.dinv + (long long)(v.r0 + k) * 36;
    for (int xr = 0; xr < 6; ++xr) {
      double s = 0.0;
      for (int q = 0; q < 6; ++q) s += K[xr * 6 + q] * c[q];
      t.x[6 * (long long)(v.r0 + k) + xr] = s;
    }
  }
};

// ---- multi-GPU exchange (nd_plan.h): every rank owns one slot of the region [U root][u root][rows of its rank separator][dadd]
struct RegionDev {
  int n_ranks, my_rank, slot_rows, max_col;
  long long region0, slot, slotU, slotu, slotH;
  const int* sep_row0;          // [n_ranks] first row of the rank separator owned by rank r (right of its range), -1: none
  const int* sep_rows;          // [n_ranks] its width
};
// own rank separator -> own slot.  items = slotH + slot_rows * 6
struct PackF {
  Tables t; RegionDev g;
  LVBA_NHD void operator()(int64_t e) const {
    const int s0 = g.sep_row0[g.my_rank];
    if (s0 < 0) return;
    double* slot = t.U + g.region0 + (long long)g.my_rank * g.slot + g.slotU + g.slotu;
    if (e < g.slotH) {
      const int per_row = (g.max_col + 1) * 36;
      const int ri = (int)(e / per_row), rem = (int)(e % per_row), b = rem / 36, el = rem % 36;
      double v = 0.0;
      if (ri < g.sep_rows[g.my_rank]) {
        const int r = s0 + ri;
        if (b <= r - t.first[r]) v = t.H[(t.row_start[r] + b) * 36 + el];
      }
      slot[e] = v;
    } else {
      const int o = (int)(e - g.slotH);
      slot[e] = (o < g.sep_rows[g.my_rank] * 6) ? t.dadd[6 * (long long)s0 + o] : 0.0;
    }
  }
};
// the other ranks' rank separators: slot -> H, dadd.  items = n_ranks x (slotH + slot_rows * 6)
struct UnpackF {
  Tables t; RegionDev g;
  LVBA_NHD void operator()(int64_t it) const {
    const long long per = g.slotH + (long long)g.slot_rows * 6;
    const int r_src = (int)(it / per);
    const long long e = it % per;
    if (r_src == g.my_rank) return;
    const int s0 = g.sep_row0[r_src];
    if (s0 < 0) return;
    const double* slot = t.U + g.region0 + (long long)r_src * g.slot + g.slotU + g.slotu;
    if (e < g.slotH) {
      const int per_row = (g.max_col + 1) * 36;
      const int ri = (int)(e / per_row), rem = (int)(e % per_row), b = rem / 36, el = rem % 36;
      if (ri >= g.sep_rows[r_src]) return;
      const int r = s0 + ri;
      if (b <= r - t.first[r]) t.Hw[(t.row_start[r] + b) * 36 + el] = slot[e];
    } else {
      const int o = (int)(e - g.slotH);
      if (o < g.sep_rows[r_src] * 6) t.daddw[6 * (long long)s0 + o] = slot[e];
    }
  }
};
// x := 0 outside the rows this rank owns (the all-reduce that follows then assembles the solution).  items = 6 n
struct ZeroForeignF {
  double* x; int row_begin, row_end;
  LVBA_NHD void operator()(int64_t i) const {
    const int r = (int)(i / 6);
    if (r < row_begin || r >= row_end) x[i] = 0.0;
  }
};

struct ZeroProgF {
  int* prog;
  LVBA_NHD void operator()(long long i) const { prog[i] = 0; }
};

// ---------------------------------------------------------------------------------------------------------------
// Per-level job tables (host side; uploaded once per structure).  Dense views of the separator nodes share three small
// arrays: first = 0, row_start[i] = i(i+1)/2, last = w - 1.
struct LevelJobs {
  std::vector<int> ids;
  std::vector<FactorJob> factor;
  std::vector<SpikeJob> spike;
  std::vector<SyrkSeg> syrk;
  std::vector<BacksolveJob> back;
  long long asm_stride = 0;       // separator levels: items per node of SepAssembleF
  int corr_stride = 0;            // rows per node of CorrectApplyF
  int max_ks = 0, max_rows = 0, max_col = 0;
};

// pointers of the small shared arrays of the dense views
struct DenseViewArrays {
  const int* zeros;               // [32]
  const long long* tri;           // [33]
  const int* last_by_w;           // [32][32]: last_by_w[w*32 + i] = w - 1
};

inline void build_level_jobs(const Plan& P, const Tables& t, const int* first_rel, const long long* rs_adj, const int* last_rel,
                             long long nblocks, const DenseViewArrays& dv, int* status, std::vector<LevelJobs>& out, int my_rank = 0) {
  out.assign(P.levels.size(), LevelJobs());
  for (size_t lv = 0; lv < P.levels.size(); ++lv) {
    LevelJobs& J = out[lv];
    for (int id : P.levels[lv])
      if (P.nodes[id].owner < 0 || P.nodes[id].owner == my_rank) J.ids.push_back(id);   // own nodes + the replicated top tree
    for (int id : J.ids) {
      const Node& v = P.nodes[id];
      EnvView e;
      double* Lp;
      double* zp;
      if (v.kind == 0) {
        e = EnvView{v.npiv + v.ntrail, first_rel + v.r0, rs_adj + v.r0, last_rel + v.r0, nblocks};
        Lp = t.L; zp = t.z + 6 * (long long)v.r0;
        for (int r = v.r0; r < v.r0 + v.npiv + v.ntrail; ++r) J.max_col = std::max(J.max_col, r - v.r0 - P.first_rel[r]);
      } else {
        e = EnvView{v.npiv, dv.zeros, dv.tri, dv.last_by_w + v.npiv * 32, (long long)v.npiv * (v.npiv + 1) / 2};
        Lp = t.T + v.offT; zp = t.zs + 6 * (long long)v.r0;
        J.max_col = std::max(J.max_col, v.npiv - 1);
      }
      J.factor.push_back(FactorJob{e, Lp, t.dinv + 36 * (long long)v.r0, zp, v.npiv,
                                   v.ntrail ? t.W + v.offW : nullptr, v.ntrail ? t.w + v.offw : nullptr, status + id,
                                   (t.prog && v.ks > 0) ? t.prog + id : nullptr});
      J.back.push_back(BacksolveJob{e, Lp, t.x + 6 * (long long)v.r0, v.npiv});
      if (v.ks > 0) {
        int* zprog = t.prog ? t.prog + (long long)P.nodes.size() + (long long)id * t.zstride : nullptr;
        J.spike.push_back(SpikeJob{e, Lp, v.npiv, t.E + v.offE, v.kind == 0 ? v.nE : v.npiv, t.Z + v.offZ, v.ks, t.prog ? t.prog + id : nullptr,
                                   zprog});
        J.syrk.push_back(SyrkSeg{t.Z + v.offZ, t.dinv + 36 * (long long)v.r0, zp, v.npiv, v.ks, t.U + v.offU, t.u + v.offu,
                                 t.prog ? t.prog + id : nullptr, zprog, e.n});
        J.max_ks = std::max(J.max_ks, v.ks);
      }
      J.max_rows = std::max(J.max_rows, v.npiv);
      J.corr_stride = std::max(J.corr_stride, v.npiv);
      if (v.kind == 1) J.asm_stride = std::max(J.asm_stride, sep_items(v));
    }
  }
}

// device-resident copies of the per-level tables (the executor owns the memory)
struct LevelDev {
  const int* ids; int n_ids;
  const FactorJob* factor; int n_factor;
  const SpikeJob* spike; int n_spike;
  const SyrkSeg* syrk; int n_syrk;
  const BacksolveJob* back; int n_back;
  long long asm_stride; int corr_stride; int max_ks, max_rows, max_col;
};

// The whole solve.  Exec provides:
//   pass(n_items, functor)                         item-parallel pass
//   zero(ptr, count)                               fill doubles with 0
//   copy(dst, src, count)                          copy doubles
//   factor(jobs, n, max_col)                       block LDL^T instances (FactorJob semantics, env_types.h)
//   factor_dense(jobs, n, max_col)                 the same for complete factorisations of dense lower matrices (separators)
//   spike(jobs, n, max_ks, max_rows)               SpikeJob semantics
//   syrk(segs, n, max_ks, max_rows)                SyrkSeg semantics
//   backsolve(jobs, n)                             BacksolveJob semantics
//   correct_apply(tables, ids, n_ids, stride)      CorrectApplyF over n_ids x stride rows
// upwards through the levels this rank owns (single GPU: all of them); multi-GPU: ends with the rank's slot of the exchange
// region filled (the SYRK / LeafFinal of the subtree root wrote U, u into it; PackF adds the rank separator's rows)
template <class Exec>
inline void run_up_local(Exec& ex, const Plan& P, const Tables& t, const LevelDev* lv, int n_levels, long long nblocks,
                         long long leaf_e, long long leaf_fin, const RegionDev* reg) {
  ex.copy(t.L, t.H, nblocks * 36);
  if (t.prog) ex.pass((long long)P.nodes.size() * (1 + t.zstride), ZeroProgF{t.prog});
  ex.pass((long long)6 * t.n, AddDiagF{t});
  ex.zero(t.U, P.sizeU);
  // ---- leaves
  const LevelDev& L0 = lv[0];
  if (L0.n_spike) ex.pass((long long)L0.n_ids * leaf_e, LeafEF{t, L0.ids, leaf_e});
  ex.factor(L0.factor, L0.n_factor, L0.max_col);
  if (L0.n_spike) {
    ex.spike(L0.spike, L0.n_spike, L0.max_ks, P.max_zrows_leaf);
    ex.syrk(L0.syrk, L0.n_syrk, L0.max_ks, L0.max_rows);
  }
  ex.pass((long long)L0.n_ids * leaf_fin, LeafFinalF{t, L0.ids, leaf_fin});
  // ---- separator levels of the own subtree
  const int n_local = P.n_ranks > 1 ? P.local_levels : n_levels;
  for (int l = 1; l < n_local; ++l) {
    const LevelDev& J = lv[l];
    if (J.n_ids == 0) continue;
    ex.pass((long long)J.n_ids * J.asm_stride, SepAssembleF{t, J.ids, J.asm_stride});
    ex.factor_dense(J.factor, J.n_factor, J.max_col);
    if (J.n_spike) {
      ex.spike(J.spike, J.n_spike, J.max_ks, J.max_rows);
      ex.syrk(J.syrk, J.n_syrk, J.max_ks, J.max_rows);
    }
  }
  if (P.n_ranks > 1 && reg) ex.pass(reg->slotH + (long long)reg->slot_rows * 6, PackF{t, *reg});
}

// multi-GPU: after the all-gather of the exchange region — the top tree upwards (every rank the same), then everything
// downwards; single GPU: just the downward sweep
template <class Exec>
inline void run_top_down(Exec& ex, const Plan& P, const Tables& t, const LevelDev* lv, int n_levels, const RegionDev* reg) {
  if (P.n_ranks > 1 && reg) {
    ex.pass((long long)reg->n_ranks * (reg->slotH + (long long)reg->slot_rows * 6), UnpackF{t, *reg});
    for (int l = P.local_levels; l < n_levels; ++l) {
      const LevelDev& J = lv[l];
      if (J.n_ids == 0) continue;
      ex.pass((long long)J.n_ids * J.asm_stride, SepAssembleF{t, J.ids, J.asm_stride});
      ex.factor_dense(J.factor, J.n_factor, J.max_col);
      if (J.n_spike) {
        ex.spike(J.spike, J.n_spike, J.max_ks, J.max_rows);
        ex.syrk(J.syrk, J.n_syrk, J.max_ks, J.max_rows);
      }
    }
  }
  for (int l = n_levels - 1; l >= 0; --l) {
    const LevelDev& J = lv[l];
    if (J.n_ids == 0) continue;
    ex.correct_apply(t, J.ids, J.n_ids, J.corr_stride);
    ex.backsolve(J.back, J.n_back);
  }
}

template <class Exec>
inline void run(Exec& ex, const Plan& P, const Tables& t, const LevelDev* lv, int n_levels, long long nblocks,
                long long leaf_e, long long leaf_fin) {
  run_up_local(ex, P, t, lv, n_levels, nblocks, leaf_e, leaf_fin, nullptr);
  run_top_down(ex, P, t, lv, n_levels, nullptr);
}

}  // namespace nd
}  // namespace lvba
