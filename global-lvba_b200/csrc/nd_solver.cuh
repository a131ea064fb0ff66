// nd_solver.cuh — device side of the substructured block LDL^T: buffers, job tables and the CUDA executor of nd::run
// (nd_passes.h).  The banded / dense factorisations and the backward substitutions are the register-window kernels of
// factor_la.cuh (one CTA per chunk interior / separator: grid = number of nodes of a tree level), launched through the
// callbacks EnvSolver passes in; the whole solve (~10 launches per tree level) is captured once per structure into a CUDA
// graph and replayed per LM pass.
//
// Replaces Eigen::SimplicialLDLT in BALM2::damping_iter (reference include/BALM/bavoxel.hpp:695-710) and the DENSE_SCHUR
// Cholesky of ceres::Solve (src/lvba_system.cpp:1573-1575, 1643) for systems long enough to be cut (SURVEY.md 8(e)).
#pragma once
#include <functional>

#include "nd_kernels.cuh"

namespace lvba {

struct NdDevice {
  nd::Plan plan;
  bool ready = false;
  int chunks = 0;
  // structure
  DevBuf<int> d_first_rel, d_last_rel, d_zeros, d_last_by_w, d_ids;
  DevBuf<long long> d_rs_adj, d_tri;
  DevBuf<nd::NodeDev> d_nodes;
  DevBuf<int> d_sep_row0, d_sep_rows;      // multi-GPU: rank separators (nd::RegionDev)
  nd::RegionDev reg{};
  int n_ranks = 1, my_rank = 0;
  DevBuf<double> xchg;                     // multi-GPU: rows received from the left neighbour (exchange_rows)
  DevBuf<unsigned short> d_dense_map;      // thread -> block of nd_dense_factor_kernel
  // the spike kernels start while the factorisation they read from is still running and follow its progress counters, and
  // the SYRK starts while the spike is running and follows the counters of the spike CTAs (programmatic dependent launch)
  DevBuf<int> d_prog;                      // [nodes] factorisations, then [nodes][zstride] spike CTAs (nd::Tables::prog)
  int zstride = 0;
  // numeric pools
  DevBuf<double> zs, U, u, Z, E, T, W, w;
  // job tables (rebuilt when the caller's pointers change)
  DevBuf<FactorJob> d_factor;
  DevBuf<nd::SpikeJob> d_spike;
  DevBuf<nd::SyrkSeg> d_syrk;
  DevBuf<BacksolveJob> d_back;
  std::vector<nd::LevelDev> lv;
  nd::Tables tab{};
  long long leaf_e = 1, leaf_fin = 1;
  const double* key_H = nullptr; const double* key_dadd = nullptr; const double* key_x = nullptr; const double* key_z = nullptr;
  // CUDA graph of one solve
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  bool use_graph = true;
  int64_t launches_per_solve = 0;

  ~NdDevice() { drop_graph(); }
  void drop_graph() {
    if (graph_exec) { cudaGraphExecDestroy(graph_exec); graph_exec = nullptr; }
    if (graph) { cudaGraphDestroy(graph); graph = nullptr; }
  }

  // number of chunks for a system of n block rows with columns of at most max_col blocks: the chain is
  // (interior) + (tree depth) x (separator width) pivot columns; more chunks shorten the first term and lengthen the second
  static int default_chunks(int n, int max_col) {
    // a leaf costs a fixed time per row (factor + spike + substitutions), a tree level a time that grows with the separator
    // width w; the twisted pair a (smaller) time per row of the whole system.  More chunks also mean more leaf factorisations
    // and spikes at once, which crowd the SMs, so the best p grows more slowly than n: the largest power of two up to
    // 16 sqrt(n) / w.  tools/solver_bench.py on an H100 80GB HBM3 at a 400 W power limit, with the SYRK beside the spike
    // (ms per solve, p = 16 / 24 / 32 / 64): 2000x30 0.852 / 0.866 / 0.901 / 1.144 -> 16; 2000x20 0.595 / 0.588 / 0.573 / 0.701
    // -> 32; 5000x30 1.477 / 1.306 / 1.316 / 1.559 -> 32; 5000x20 1.033 / 0.895 / 0.816 / 0.937 -> 32.  (The former rule,
    // n / (3 w + 30), took 16 at 2000x20 and would take 64 from ~4600 rows at w = 20.)  Below ~800 rows the two-CTA twisted
    // solve wins.
    if (n < 768) return 0;
    const double want = 16.0 * sqrt((double)n) / max_col;
    int best = 0;
    for (int p = 4; p <= 256 && p <= want; p *= 2) best = p;
    return best;
  }

  // n_ranks_ > 1: the plan is cut so that rank r owns p / n_ranks consecutive chunks (nd_plan.h); p_want is rounded up to a
  // multiple of n_ranks
  int prepare(int n, const std::vector<int>& first, const std::vector<int>& last, const std::vector<long long>& row_start, int max_col,
              int p_want, cudaStream_t s, int n_ranks_ = 1, int my_rank_ = 0) {
    ready = false; chunks = 0;
    drop_graph();
    key_H = key_dadd = key_x = key_z = nullptr;
    n_ranks = n_ranks_; my_rank = my_rank_;
    if (n_ranks > 1) p_want = std::max(n_ranks, ((p_want + n_ranks - 1) / n_ranks) * n_ranks);
    if (p_want < 2) return LVBA_OK;
    const int p = nd::choose_chunks(n, first.data(), last.data(), row_start.data(), max_col, p_want, plan, n_ranks);
    if (p < 2) return LVBA_OK;                               // structure cannot be cut: the caller keeps its other paths
    if (n_ranks > 1) {
      for (int r = 0; r < n_ranks; ++r)                        // the overflow of a rank's Hessian rows must stay inside the next rank
        if (plan.rank_row_end[r] - plan.rank_row_begin[r] < max_col + 1) return LVBA_OK;
    }
    {
      // LVBA_ND_GRAPH=0 runs nd::run eagerly on every solve.  That code is needed anyway (the fall-back when stream capture
      // fails, and how the multi-GPU solve runs); this switch is the only way a one-GPU test reaches it.
      const char* g = getenv("LVBA_ND_GRAPH");
      use_graph = !(g && g[0] == '0');
    }
    int64_t dummy = 0;
    LVBA_TRY(d_first_rel.upload(plan.first_rel, s, &dummy));
    LVBA_TRY(d_last_rel.upload(plan.last_rel, s, &dummy));
    LVBA_TRY(d_rs_adj.upload(plan.rs_adj, s, &dummy));
    std::vector<int> zeros(32, 0), last_by_w(32 * 32, 0);
    std::vector<long long> tri(33, 0);
    for (int i = 0; i < 33; ++i) tri[i] = (long long)i * (i + 1) / 2;
    for (int w_ = 0; w_ < 32; ++w_) for (int i = 0; i < 32; ++i) last_by_w[w_ * 32 + i] = w_ - 1;
    LVBA_TRY(d_zeros.upload(zeros, s, &dummy));
    LVBA_TRY(d_last_by_w.upload(last_by_w, s, &dummy));
    LVBA_TRY(d_tri.upload(tri, s, &dummy));
    std::vector<nd::NodeDev> nodes;
    for (const nd::Node& v : plan.nodes) nodes.push_back(nd::to_dev(v));
    LVBA_TRY(d_nodes.upload(nodes, s, &dummy));
    const std::vector<unsigned short> dmap = dense_thread_map();
    LVBA_TRY(d_dense_map.upload(dmap, s, &dummy));
    LVBA_TRY(zs.alloc((size_t)n * 6));
    LVBA_TRY(U.alloc((size_t)std::max<long long>(plan.sizeU, 1))); LVBA_TRY(u.alloc((size_t)std::max<long long>(plan.sizeu, 1)));
    LVBA_TRY(Z.alloc((size_t)std::max<long long>(plan.sizeZ, 1))); LVBA_TRY(E.alloc((size_t)std::max<long long>(plan.sizeE, 1)));
    LVBA_TRY(T.alloc((size_t)std::max<long long>(plan.sizeT, 1))); LVBA_TRY(W.alloc((size_t)std::max<long long>(plan.sizeW, 1)));
    LVBA_TRY(w.alloc((size_t)std::max<long long>(plan.sizew, 1)));
    if (n_ranks > 1) {
      std::vector<int> s0((size_t)n_ranks, -1), sr((size_t)n_ranks, 0);
      for (int r = 0; r + 1 < n_ranks; ++r) { s0[r] = plan.sep_start[(r + 1) * plan.q]; sr[r] = plan.sep_width[(r + 1) * plan.q]; }
      LVBA_TRY(d_sep_row0.upload(s0, s, &dummy)); LVBA_TRY(d_sep_rows.upload(sr, s, &dummy));
      reg = nd::RegionDev{n_ranks, my_rank, plan.slot_rows, plan.max_col, plan.region0, plan.slot, plan.slotU, plan.slotu, plan.slotH,
                          d_sep_row0.p, d_sep_rows.p};
      long long mx = 0;
      for (int r = 0; r < n_ranks; ++r) {
        const int b = plan.rank_row_begin[r], e2 = std::min(n, b + max_col);
        mx = std::max(mx, (row_start[e2] - row_start[b]) * 36);
      }
      LVBA_TRY(xchg.alloc((size_t)std::max<long long>(mx, 1)));
    }
    zstride = 0;
    for (const nd::Node& v : plan.nodes) zstride = std::max(zstride, (v.ks + kSpikeCols - 1) / kSpikeCols);
    LVBA_TRY(d_prog.alloc(plan.nodes.size() * (size_t)(1 + zstride)));
    LVBA_CUDA(cudaFuncSetAttribute(nd_spike_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSpikeSmem));
    LVBA_CUDA(cudaFuncSetAttribute(nd_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
    LVBA_CUDA(cudaFuncSetAttribute(nd_dense_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmem));
    LVBA_CUDA(cudaStreamSynchronize(s));                     // local vectors
    leaf_e = nd::leaf_e_stride(plan); leaf_fin = nd::leaf_final_stride(plan);
    chunks = p; ready = true;
    return LVBA_OK;
  }

  // job tables for the caller's buffers: L (working copy, envelope layout), dinv [n][36], z [6n] (rhs in / scratch), status
  // [1 + nodes], H, dadd, x
  int build_tables(const EnvView& genv, const double* H, const double* dadd, double* L, double* dinv, double* z, double* x,
                   int* status, cudaStream_t s) {
    if (key_H == H && key_dadd == dadd && key_x == x && key_z == z && !lv.empty()) return LVBA_OK;
    drop_graph();
    tab = nd::Tables{};
    tab.n = plan.n; tab.first = genv.first; tab.row_start = genv.row_start; tab.nodes = d_nodes.p;
    tab.H = H; tab.dadd = dadd; tab.L = L; tab.z = z; tab.zs = zs.p; tab.dinv = dinv; tab.x = x;
    tab.U = U.p; tab.u = U.p; tab.Z = Z.p; tab.E = E.p; tab.T = T.p; tab.W = W.p; tab.w = w.p;
    tab.Hw = n_ranks > 1 ? const_cast<double*>(H) : nullptr;       // multi-GPU: the other ranks' rank-separator rows are written into
    tab.daddw = n_ranks > 1 ? const_cast<double*>(dadd) : nullptr; // the caller's H / dadd (documented at EnvSolver::solve)
    tab.prog = d_prog.p; tab.zstride = zstride;
    std::vector<nd::LevelJobs> jobs;
    nd::DenseViewArrays dv{d_zeros.p, d_tri.p, d_last_by_w.p};
    nd::build_level_jobs(plan, tab, d_first_rel.p, d_rs_adj.p, d_last_rel.p, genv.nblocks, dv, status + 1, jobs, my_rank);
    std::vector<int> ids; std::vector<FactorJob> fj; std::vector<nd::SpikeJob> sj; std::vector<nd::SyrkSeg> yj; std::vector<BacksolveJob> bj;
    struct Off { size_t ids, f, s, y, b; };
    std::vector<Off> off;
    for (auto& J : jobs) {
      off.push_back(Off{ids.size(), fj.size(), sj.size(), yj.size(), bj.size()});
      ids.insert(ids.end(), J.ids.begin(), J.ids.end());
      fj.insert(fj.end(), J.factor.begin(), J.factor.end());
      sj.insert(sj.end(), J.spike.begin(), J.spike.end());
      yj.insert(yj.end(), J.syrk.begin(), J.syrk.end());
      bj.insert(bj.end(), J.back.begin(), J.back.end());
    }
    LVBA_TRY(d_ids.upload(ids, s)); LVBA_TRY(d_factor.upload(fj, s)); LVBA_TRY(d_back.upload(bj, s));
    if (!sj.empty()) { LVBA_TRY(d_spike.upload(sj, s)); LVBA_TRY(d_syrk.upload(yj, s)); }
    LVBA_CUDA(cudaStreamSynchronize(s));                     // local vectors
    lv.clear();
    for (size_t l = 0; l < jobs.size(); ++l) {
      const auto& J = jobs[l];
      lv.push_back(nd::LevelDev{d_ids.p + off[l].ids, (int)J.ids.size(), d_factor.p + off[l].f, (int)J.factor.size(),
                                d_spike.p + off[l].s, (int)J.spike.size(), d_syrk.p + off[l].y, (int)J.syrk.size(),
                                d_back.p + off[l].b, (int)J.back.size(), J.asm_stride, J.corr_stride, J.max_ks, J.max_rows, J.max_col});
    }
    key_H = H; key_dadd = dadd; key_x = x; key_z = z;
    return LVBA_OK;
  }
};

// CUDA executor of nd::run
struct NdCudaExec {
  cudaStream_t s;
  std::function<int(int, int, const FactorJob*)> factor_fn;        // (max_col, n_jobs, jobs)
  std::function<void(int, const BacksolveJob*)> back_fn;           // (n_jobs, jobs)
  const unsigned short* dense_map = nullptr;                       // thread -> block of nd_dense_factor_kernel (NdDevice::d_dense_map)
  int64_t launches = 0;
  int rc = LVBA_OK;
  template <class F> void pass(long long n, const F& f) {
    if (n <= 0) return;
    const int grid = (int)std::min<long long>((n + 255) / 256, kNumSMs * 8);
    nd_pass_kernel<<<grid, 256, 0, s>>>(n, f);
    ++launches;
  }
  void copy(double* dst, const double* src, long long n) { cudaMemcpyAsync(dst, src, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s); }
  void zero(double* p, long long n) { if (n > 0) cudaMemsetAsync(p, 0, (size_t)n * sizeof(double), s); }
  void factor(const FactorJob* jobs, int n, int max_col) {
    if (n <= 0) return;
    const int r = factor_fn(max_col, n, jobs);
    if (r != LVBA_OK) rc = r;
  }
  void factor_dense(const FactorJob* jobs, int n, int max_col) {
    if (n <= 0) return;
    nd_dense_factor_kernel<<<n, kDenseThreads, kDenseSmem, s>>>(jobs, dense_map);
    ++launches;
  }
  void spike(const nd::SpikeJob* jobs, int n, int max_ks, int) {
    if (n <= 0 || max_ks <= 0) return;
    // the kernel launched just before this one is the factorisation whose L these jobs read: start as soon as all of ITS CTAs run
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((max_ks + kSpikeCols - 1) / kSpikeCols, n); cfg.blockDim = dim3(kSpikeThreads); cfg.dynamicSmemBytes = kSpikeSmem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, nd_spike_kernel, jobs);
    if (e != cudaSuccess) rc = fail(LVBA_ERR_CUDA, "cudaLaunchKernelEx(nd_spike_kernel): %s", cudaGetErrorString(e));
    ++launches;
  }
  void syrk(const nd::SyrkSeg* segs, int n, int max_ks, int max_rows) {
    if (n <= 0 || max_ks <= 0) return;
    // the kernel launched just before this one is the spike whose Z these segments read: start as soon as all of ITS CTAs run
    // (nd_syrk_kernel says why nothing can starve).  Row groups are the slowest grid dimension, so that the CTAs of the first
    // rows of every segment are placed first.
    const int nt1 = (max_ks + kSyrkTile - 1) / kSyrkTile, nt = nt1 * (nt1 + 1) / 2;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nt, n, (max_rows + kSyrkSplit - 1) / kSyrkSplit); cfg.blockDim = dim3(kSyrkThreads); cfg.dynamicSmemBytes = kSyrkSmem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, nd_syrk_kernel, segs, kSyrkSplit);
    if (e != cudaSuccess) rc = fail(LVBA_ERR_CUDA, "cudaLaunchKernelEx(nd_syrk_kernel): %s", cudaGetErrorString(e));
    ++launches;
  }
  void correct_apply(const nd::Tables& t, const int* ids, int n_ids, int stride) {
    if (n_ids <= 0 || stride <= 0) return;
    nd_correct_apply_kernel<<<n_ids * stride, 192, 0, s>>>(t, ids, stride);
    ++launches;
  }
  void backsolve(const BacksolveJob* jobs, int n) {
    if (n <= 0) return;
    back_fn(n, jobs);
    ++launches;
  }
};

}  // namespace lvba
