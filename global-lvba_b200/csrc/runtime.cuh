// runtime.cuh — host-side plumbing shared by both paths: error reporting, device buffers,
// CUDA-event phase timers, the block-envelope structure builder and the LDL^T solve driver.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/lvba_b200.h"
#include "setup_pool.h"
#include "envelope.cuh"
#include "envelope_wide.h"
#include "factor_la.cuh"

namespace lvba {

// one pass of the any-width factorisation (envelope_wide.h): grid-stride over its items
template <class F>
__global__ void __launch_bounds__(128) env_wide_pass_kernel(int64_t n, F f) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) f(i);
}
// one such pass over `items` items on `s`, counted in *launches (nothing to launch for no items)
template <class F>
inline void wide_pass(cudaStream_t s, int64_t items, const F& f, int64_t* launches) {
  if (items <= 0) return;
  const int grid = (int)std::min<int64_t>((items + 127) / 128, kNumSMs * 16);
  env_wide_pass_kernel<<<grid, 128, 0, s>>>(items, f);
  ++*launches;
}

// ---------------------------------------------------------------- errors
inline std::string& last_error_ref() {
  static thread_local std::string s;
  return s;
}
inline int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  last_error_ref() = buf;
  return code;
}
#define LVBA_CUDA(call)                                                                        \
  do {                                                                                         \
    cudaError_t err__ = (call);                                                                \
    if (err__ != cudaSuccess)                                                                  \
      return ::lvba::fail(LVBA_ERR_CUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,  \
                          cudaGetErrorString(err__));                                          \
  } while (0)
// Every extern "C" entry point is a function-try-block: no C++ exception (std::bad_alloc / std::length_error from the host
// containers of the set-up passes) crosses the C ABI — the caller gets a status code and lvba_last_error().
#define LVBA_ABI_BEGIN try
#define LVBA_ABI_END(name)                                                                                          \
  catch (const std::bad_alloc&) { return ::lvba::fail(LVBA_ERR_NOMEM, name ": host allocation failed"); }            \
  catch (const std::exception& e) { return ::lvba::fail(LVBA_ERR_NOMEM, name ": exception: %s", e.what()); }         \
  catch (...) { return ::lvba::fail(LVBA_ERR_INVALID_ARG, name ": unexpected exception"); }
#define LVBA_TRY(call)             \
  do {                             \
    int rc__ = (call);             \
    if (rc__ != LVBA_OK) return rc__; \
  } while (0)

inline int device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}
inline int select_device(int device) {
  const int n = device_count();
  if (n <= 0) return fail(LVBA_ERR_NO_DEVICE, "no CUDA device available: the LVBA hot path has no CPU fallback");
  if (device >= n) return fail(LVBA_ERR_INVALID_ARG, "device %d out of range (have %d)", device, n);
  if (device >= 0) LVBA_CUDA(cudaSetDevice(device));
  return LVBA_OK;
}

// ---------------------------------------------------------------- host parallel loop (symbolic set-up)
constexpr int kMaxSetupThreads = 8;

// ---------------------------------------------------------------- device memory pool
// cudaMalloc / cudaFree cost milliseconds each (cudaFree also synchronises the device); the one-shot ABI calls
// create and destroy ~40 buffers per call.  Freed buffers are therefore parked in a per-device, size-bucketed
// pool and reused by later calls of the same process (identical problem sizes hit exactly).  The pool is
// capped; lvba_release_cached_memory() (include/lvba_b200.h) empties it.
struct DevicePool {
  std::mutex mu;
  std::multimap<std::pair<int, size_t>, void*> free_list;     // (device, bytes) -> pointer
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCached = 8ull << 30;          // a tenth of an H100's 80 GB
  static size_t bucket(size_t bytes) { return (bytes + 511) & ~size_t(511); }
  void* take(int dev, size_t bytes) {
    std::lock_guard<std::mutex> g(mu);
    auto it = free_list.find({dev, bytes});
    if (it == free_list.end()) return nullptr;
    void* p = it->second;
    free_list.erase(it);
    cached_bytes -= bytes;
    return p;
  }
  void give(int dev, size_t bytes, void* p) {
    std::lock_guard<std::mutex> g(mu);
    if (cached_bytes + bytes > kMaxCached) { cudaFree(p); return; }
    free_list.insert({{dev, bytes}, p});
    cached_bytes += bytes;
  }
  void clear() {
    std::lock_guard<std::mutex> g(mu);
    for (auto& kv : free_list) cudaFree(kv.second);
    free_list.clear();
    cached_bytes = 0;
  }
};
inline DevicePool& device_pool() {
  static DevicePool* p = new DevicePool();     // intentionally leaked: no CUDA calls in static destructors
  return *p;
}

// Pinned host scratch (the few doubles every LM pass reads back): cudaMallocHost / cudaFreeHost page-lock and unlock memory
// through the driver on every one-shot call; the blocks are parked like the device buffers above.
struct PinnedPool {
  std::mutex mu;
  std::multimap<size_t, void*> free_list;
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCached = 64ull << 20;
  static size_t bucket(size_t bytes) { return (std::max<size_t>(bytes, 1) + 4095) & ~size_t(4095); }
  int take(size_t bytes, void** out) {
    const size_t b = bucket(bytes);
    {
      std::lock_guard<std::mutex> g(mu);
      auto it = free_list.find(b);
      if (it != free_list.end()) { *out = it->second; free_list.erase(it); cached_bytes -= b; return LVBA_OK; }
    }
    LVBA_CUDA(cudaMallocHost(out, b));
    return LVBA_OK;
  }
  void give(void* p, size_t bytes) {
    if (!p) return;
    const size_t b = bucket(bytes);
    std::lock_guard<std::mutex> g(mu);
    if (cached_bytes + b > kMaxCached) { cudaFreeHost(p); return; }
    free_list.insert({b, p});
    cached_bytes += b;
  }
  void clear() {
    std::lock_guard<std::mutex> g(mu);
    for (auto& kv : free_list) cudaFreeHost(kv.second);
    free_list.clear();
    cached_bytes = 0;
  }
};
inline PinnedPool& pinned_pool() {
  static PinnedPool* p = new PinnedPool();     // intentionally leaked: no CUDA calls in static destructors
  return *p;
}

// ---------------------------------------------------------------- device buffer
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  size_t bytes_ = 0;
  int dev_ = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) device_pool().give(dev_, bytes_, p);
    p = nullptr; n = 0; bytes_ = 0;
  }
  void swap(DevBuf& o) { std::swap(p, o.p); std::swap(n, o.n); std::swap(bytes_, o.bytes_); std::swap(dev_, o.dev_); }
  int alloc(size_t count) {
    release();
    n = count;
    if (count == 0) return LVBA_OK;
    bytes_ = DevicePool::bucket(count * sizeof(T));
    cudaGetDevice(&dev_);
    p = (T*)device_pool().take(dev_, bytes_);
    if (p) return LVBA_OK;
    cudaError_t e = cudaMalloc((void**)&p, bytes_);
    if (e != cudaSuccess) {
      cudaGetLastError();
      device_pool().clear();                                   // give cached memory back and retry once
      e = cudaMalloc((void**)&p, bytes_);
    }
    if (e != cudaSuccess) { p = nullptr; n = 0; bytes_ = 0; return fail(LVBA_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", count * sizeof(T), cudaGetErrorString(e)); }
    return LVBA_OK;
  }
  int upload(const T* h, size_t count, cudaStream_t s, int64_t* bytes = nullptr) {
    if (count > n) LVBA_TRY(alloc(count));
    if (count) LVBA_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
    if (bytes) *bytes += (int64_t)(count * sizeof(T));
    return LVBA_OK;
  }
  int upload(const std::vector<T>& h, cudaStream_t s, int64_t* bytes = nullptr) { return upload(h.data(), h.size(), s, bytes); }
  int zero(cudaStream_t s) {
    if (n) LVBA_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s));
    return LVBA_OK;
  }
};

// ---------------------------------------------------------------- phase timers (CUDA events on the launch stream)
enum Phase { PH_BUILD = 0, PH_SOLVE = 1, PH_RESID = 2, PH_COUNT = 3 };
struct PhaseTimers {
  struct Span { cudaEvent_t a, b; int ph; };
  std::vector<Span> spans;
  std::vector<cudaEvent_t> pool;
  cudaStream_t stream = nullptr;
  cudaEvent_t get() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }
  void begin(int ph) { Span s{get(), get(), ph}; cudaEventRecord(s.a, stream); spans.push_back(s); }
  void end() { cudaEventRecord(spans.back().b, stream); }
  // must be called after a stream synchronize
  void collect(double ms[PH_COUNT]) {
    for (auto& s : spans) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, s.a, s.b) == cudaSuccess) ms[s.ph] += t;
      pool.push_back(s.a); pool.push_back(s.b);
    }
    spans.clear();
  }
  ~PhaseTimers() {
    for (auto& s : spans) { cudaEventDestroy(s.a); cudaEventDestroy(s.b); }
    for (auto e : pool) cudaEventDestroy(e);
  }
};
// two CUDA events that cannot leak on an early return (LVBA_TRY / LVBA_CUDA inside a timed section)
struct EventPair {
  cudaEvent_t a = nullptr, b = nullptr;
  EventPair() = default;
  EventPair(const EventPair&) = delete;
  EventPair& operator=(const EventPair&) = delete;
  int create() {
    LVBA_CUDA(cudaEventCreate(&a));
    LVBA_CUDA(cudaEventCreate(&b));
    return LVBA_OK;
  }
  ~EventPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
};
// Device buffers go back to the pool when they leave scope, and the pool hands them to whatever stream asks next; work
// queued on `stream` may still be using them (an error exit between an upload and its consumer, a handle destroyed right
// after an asynchronous call).  Declared AFTER the buffers of a scope — destruction runs in reverse order of declaration —
// this waits for the stream first, so every buffer of the scope is idle when it is parked (ADVICE r1).
struct StreamDrain {
  cudaStream_t s;
  explicit StreamDrain(cudaStream_t s_) : s(s_) {}
  ~StreamDrain() { cudaStreamSynchronize(s); }
};
inline double wall_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------- LM summaries and the one-shot calls
// *s from the LM counts, costs and damping of a call; with `ms` (collected PhaseTimers) also its phase times, wall time
// and the launches and bytes it moved
inline void write_summary(lvba_summary* s, int iters, int accepted, int builds, int term, double cost_first, double cost_last,
                          double damping, const double* ms = nullptr, double ms_total = 0.0, int64_t launches = 0, int64_t h2d = 0,
                          int64_t d2h = 0) {
  memset(s, 0, sizeof *s);
  s->iterations = iters; s->accepted = accepted; s->hessian_builds = builds; s->termination = term;
  s->cost_first = cost_first; s->cost_last = cost_last; s->damping_last = damping;
  if (ms) { s->ms_build = ms[PH_BUILD]; s->ms_solve = ms[PH_SOLVE]; s->ms_residual = ms[PH_RESID]; }
  s->ms_total = ms_total;
  s->kernel_launches = launches; s->h2d_bytes = h2d; s->d2h_bytes = d2h;
}

// the summary of a one-shot call: the handle's set-up time and everything it launched and moved, the call's wall time from t0
template <class Problem>
inline void one_shot_totals(lvba_summary* s, const Problem* p, double t0) {
  s->ms_setup = p->ms_setup;
  s->kernel_launches = p->launches; s->h2d_bytes = p->h2d; s->d2h_bytes = p->d2h;
  s->ms_total = wall_ms() - t0;
}

// A one-shot call once it has created its handle p: reset the LM to `o`, run o.max_iter passes if `solve`, write the result
// back (write_back()) and fill *summary only while every step succeeds, and destroy the handle in every case.
template <class Problem, class Opts, class WriteBack>
inline int lm_one_shot(Problem* p, const Opts& o, bool solve, int (*reset_lm)(Problem*, const Opts*),
                       int (*iterate)(Problem*, int32_t, lvba_summary*), int (*destroy)(Problem*), const WriteBack& write_back,
                       double t0, lvba_summary* summary) {
  lvba_summary s;
  memset(&s, 0, sizeof s);
  int rc = reset_lm(p, &o);
  if (rc == LVBA_OK && solve) rc = iterate(p, o.max_iter, &s);
  if (rc == LVBA_OK) rc = write_back();
  if (rc == LVBA_OK && summary) {
    *summary = s;
    one_shot_totals(summary, p, t0);
  }
  destroy(p);
  return rc;
}

// ---------------------------------------------------------------- block envelope (host build + device copy)
struct Envelope {
  int n = 0;
  std::vector<int> first, last;
  std::vector<long long> row_start;
  long long nblocks = 0;
  int max_col = 0;
  DevBuf<int> d_first, d_last;
  DevBuf<long long> d_row_start;

  // first_raw[r] = smallest column coupled to row r (<= r).  Made monotone so that the rows below a
  // pivot column form a contiguous range (see envelope.cuh header).
  int build(const std::vector<int>& first_raw, cudaStream_t s, int64_t* bytes) {
    n = (int)first_raw.size();
    first = first_raw;
    for (int r = 0; r < n; ++r) first[r] = std::min(first[r], r);
    for (int r = n - 2; r >= 0; --r) first[r] = std::min(first[r], first[r + 1]);
    row_start.assign(n + 1, 0);
    for (int r = 0; r < n; ++r) row_start[r + 1] = row_start[r] + (r - first[r] + 1);
    nblocks = row_start[n];
    last.assign(n, 0);
    // last[k] = max i with first[i] <= k ; first monotone => two-pointer sweep
    int i = 0;
    max_col = 0;
    for (int k = 0; k < n; ++k) {
      if (i < k) i = k;
      while (i + 1 < n && first[i + 1] <= k) ++i;
      last[k] = i;
      max_col = std::max(max_col, i - k);
    }
    LVBA_TRY(d_first.upload(first, s, bytes));
    LVBA_TRY(d_last.upload(last, s, bytes));
    LVBA_TRY(d_row_start.upload(row_start, s, bytes));
    return LVBA_OK;
  }
  EnvView view() const { return EnvView{n, d_first.p, d_row_start.p, d_last.p, nblocks}; }
};

// Thread -> slot-pair map of the register-window kernel.  Pairs {a,b}, a >= b, are grouped by 8x8 super
// blocks of the slot triangle so that the 32 lanes of a warp touch <= 8 distinct slots per operand: the
// shared-memory operand loads of a warp then need 1-2 wavefronts instead of 4-5.
inline std::vector<unsigned short> build_pair_map(int P, int n_threads) {
  std::vector<std::vector<unsigned short>> chunks;          // full 32-lane chunks first, leftovers after
  std::vector<std::vector<unsigned short>> left;
  const int nb = (P + 7) / 8;
  for (int A = 0; A < nb; ++A)
    for (int B = 0; B <= A; ++B) {
      std::vector<unsigned short> cur;
      for (int a = 8 * A; a < std::min(P, 8 * A + 8); ++a)
        for (int b = 8 * B; b < std::min(P, 8 * B + 8) && b <= a; ++b) {
          cur.push_back((unsigned short)(a | (b << 8)));
          if ((int)cur.size() == 32) { chunks.push_back(cur); cur.clear(); }
        }
      if (!cur.empty()) left.push_back(cur);
    }
  std::sort(left.begin(), left.end(), [](const auto& x, const auto& y) { return x.size() > y.size(); });
  const int n_warps = n_threads / 32;
  std::vector<std::vector<unsigned short>> warps = chunks;
  for (auto& l : left) {                                     // first-fit into a warp with room, else a new warp, else split
    bool placed = false;
    for (size_t w = chunks.size(); w < warps.size() && !placed; ++w)
      if (warps[w].size() + l.size() <= 32) { warps[w].insert(warps[w].end(), l.begin(), l.end()); placed = true; }
    if (!placed && (int)warps.size() < n_warps) { warps.push_back(l); placed = true; }
    if (!placed) {
      for (auto& w : warps)
        while (w.size() < 32 && !l.empty()) { w.push_back(l.back()); l.pop_back(); }
    }
  }
  std::vector<unsigned short> map((size_t)n_threads, (unsigned short)0xffff);
  for (size_t w = 0; w < warps.size() && (int)w < n_warps; ++w)
    for (size_t i = 0; i < warps[w].size(); ++i) map[w * 32 + i] = warps[w][i];
  return map;
}

// Thread -> blocks map of the register-window kernel, one 32-bit word per pair thread: a | b0 << 8 | b1 << 16
// (b1 = 0xff: no second block; 0xffffffff: idle thread).  kTile2 = false: one block {a,b0} per thread, grouped as
// build_pair_map does.  kTile2 = true: the blocks {a,b}, b <= a, of one row slot are paired (b = 2m, 2m+1) and the
// threads are ordered by 8x8 super block so that the lanes of a warp share few distinct operand slots.
inline std::vector<unsigned> build_pair_map32(int P, bool tile2, int n_threads) {
  std::vector<unsigned> map((size_t)n_threads, 0xffffffffu);
  if (!tile2) {
    const std::vector<unsigned short> m16 = build_pair_map(P, n_threads);
    for (int t = 0; t < n_threads; ++t)
      if (m16[t] != 0xffff) map[t] = (unsigned)(m16[t] & 0xff) | ((unsigned)(m16[t] >> 8) << 8) | (0xffu << 16);
    return map;
  }
  struct Tri { int a, b0, b1; };
  std::vector<Tri> tris;
  for (int a = 0; a < P; ++a)
    for (int b = 0; b <= a; b += 2) tris.push_back(Tri{a, b, (b + 1 <= a) ? b + 1 : 0xff});
  std::stable_sort(tris.begin(), tris.end(), [](const Tri& x, const Tri& y) {
    const int kx[4] = {x.a / 8, x.b0 / 8, x.a, x.b0}, ky[4] = {y.a / 8, y.b0 / 8, y.a, y.b0};
    for (int i = 0; i < 4; ++i) if (kx[i] != ky[i]) return kx[i] < ky[i];
    return false;
  });
  for (size_t t = 0; t < tris.size() && (int)t < n_threads; ++t)
    map[t] = (unsigned)tris[t].a | ((unsigned)tris[t].b0 << 8) | ((unsigned)tris[t].b1 << 16);
  return map;
}

}  // namespace lvba
#define LVBA_RUNTIME_PRELUDE 1
#include "comm.cuh"
#include "nd_solver.cuh"
namespace lvba {

// ---------------------------------------------------------------- LDL^T solve driver
// The path is chosen once, by prepare(), from the structure of the system, and solve() follows it.
constexpr int kSolveBatch = -1;       // EnvSolver::path of a block-diagonal window batch (not an lvba_env_solve path)
struct EnvSolver {
  DevBuf<double> L, dinv, z;
  DevBuf<int> status;
  // LVBA_SOLVE_* (include/lvba_b200.h) or kSolveBatch; LVBA_SOLVE_AUTO until prepare() has run
  int path = LVBA_SOLVE_AUTO;
  // device job tables of the register-window path (built at the first solve, when the solution buffer is known)
  DevBuf<FactorJob> d_fjobs;
  DevBuf<BacksolveJob> d_bjobs;
  const double* jobs_x = nullptr;
  // ---- batched mode (window BA): the system is block diagonal; every group is factorised by its own CTA
  int n_groups = 0;
  std::vector<int> grp_ptr;     // [n_groups+1] row offsets
  DevBuf<int> first_rel;        // first[r] relative to the first row of r's group
  // window sizes P the register-window kernel is built for (P - 1 = widest column it holds): the work per pivot column
  // grows with P^2, so a system is factorised with the smallest P that fits its envelope
  static constexpr int kNumP = 6;
  DevBuf<unsigned> pair_map[kNumP];     // thread -> blocks of the register-window kernel, per P
  bool have_map[kNumP] = {false, false, false, false, false, false};
  bool configured = false;
  // ---- any-width path (envelope_wide.h): columns taller than kEnvMaxCol blocks (loop closures)
  DevBuf<double> colT;          // [max_col * 36] unscaled copy of the current pivot column
  // ---- twisted (two-ended) factorisation: top half in natural order on one SM, bottom half reversed on another,
  //      joined at a separator of `tw_bs` rows (see envelope.cuh, FactorJob)
  // ---- substructured solve (nd_solver.cuh): p chunk interiors + a tree of separators, one CTA per node; chosen for
  //      systems long enough that  interior + depth x separator  pivot columns beat the two halves of the twisted solve
  NdDevice nd;
  // deterministic mode: the separator SYRK runs without split-K (one CTA per tile covers all rows of its node, so every element
  // of U and u gets exactly one add); the graph of the other mode is dropped and the solve captured again
  bool det = false;
  void set_deterministic(bool d) {
    if (d != det) nd.drop_graph();
    det = d;
  }
  // multi-GPU, row-owned system: rank r owns the rows dist_begin() .. dist_end()-1 of H / S (its chunks, inner separators and
  // its right rank separator); voxels / tracks are assigned to the owner of their lowest row, so a rank's contributions reach
  // at most max_col rows into the next rank's range: exchange_rows() ships exactly those rows
  bool dist() const { return path == LVBA_SOLVE_CHUNKED && nd.n_ranks > 1; }
  int dist_begin() const { return nd.plan.rank_row_begin[nd.my_rank]; }
  int dist_end() const { return nd.plan.rank_row_end[nd.my_rank]; }
  int dist_owner(int row) const {
    const auto& e = nd.plan.rank_row_end;
    return (int)(std::upper_bound(e.begin(), e.end(), row) - e.begin());
  }
  // adds the left neighbour's contributions to this rank's first rows and ships this rank's contributions to the right
  // neighbour's first rows (block rows of M in envelope storage are contiguous: one send, one receive, one add kernel)
  int exchange_rows(const Envelope& env, double* M, cudaStream_t s, int64_t* launches) {
    if (!dist()) return LVBA_OK;
    Comm& cm = comm();
    const int n = env.n, ov = env.max_col;
    const int sb = dist_end(), se = std::min(n, sb + ov);                  // rows I contributed to but do not own
    const int rb = dist_begin(), re = std::min(n, rb + ov);                // my rows the left neighbour contributed to
    const size_t n_send = (nd.my_rank + 1 < nd.n_ranks) ? (size_t)(env.row_start[se] - env.row_start[sb]) * 36 : 0;
    const size_t n_recv = (nd.my_rank > 0) ? (size_t)(env.row_start[re] - env.row_start[rb]) * 36 : 0;
    LVBA_TRY(cm.shift_right(M + env.row_start[sb] * 36, n_send, nd.xchg.p, n_recv, s));
    if (n_recv > 0) {
      env_axpy_kernel<<<(unsigned)((n_recv + 255) / 256), 256, 0, s>>>((long long)n_recv, nd.xchg.p, M + env.row_start[rb] * 36);
      ++*launches;
    }
    return LVBA_OK;
  }
  int tw_m = 0, tw_send = 0, tw_bs = 0, tw_nb = 0, tw_nbstop = 0;
  Envelope env_bot, env_sep;
  DevBuf<double> Lbot, dinv_bot, zbot, xbot, wtop, wbot, ztopd, zbotd, Lsep, dinv_sep, zsep, xsep;

  static int pid(int mc) { return mc <= 7 ? 0 : mc <= 11 ? 1 : mc <= 15 ? 2 : mc <= 20 ? 3 : mc <= 23 ? 4 : 5; }
  static int pval(int id) { return id == 0 ? 8 : id == 1 ? 12 : id == 2 ? 16 : id == 3 ? 21 : id == 4 ? 24 : 31; }

  // Chooses the path and allocates what it needs.  want = LVBA_SOLVE_AUTO picks by structure (what lvba_lidar_lm /
  // lvba_visual_lm run); any other LVBA_SOLVE_* value pins that path and fails with LVBA_ERR_UNSUPPORTED if the structure
  // does not allow it.  chunks: for LVBA_SOLVE_CHUNKED (< 2: default_chunks).  groups (window BA): row offsets
  // [n_groups + 1] of a block-diagonal system, every group factorised by its own CTA; want must then be LVBA_SOLVE_AUTO.
  int prepare(const Envelope& env, cudaStream_t s, int want = LVBA_SOLVE_AUTO, int chunks = 0, const std::vector<int>& groups = {}) {
    path = LVBA_SOLVE_AUTO;
    LVBA_TRY(L.alloc((size_t)env.nblocks * 36));
    LVBA_TRY(dinv.alloc((size_t)env.n * 36));
    LVBA_TRY(z.alloc((size_t)env.n * 6));
    LVBA_TRY(status.alloc(4));
    jobs_x = nullptr;
    if (!configured) {
      LVBA_CUDA(cudaFuncSetAttribute(env_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)factor_smem()));
#define LVBA_SET_SMEM(PP) LVBA_CUDA(cudaFuncSetAttribute(env_factor_la_kernel<PP, la_tile2(PP)>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LaCfg<PP, la_tile2(PP)>::kSmem))
      LVBA_SET_SMEM(8); LVBA_SET_SMEM(12); LVBA_SET_SMEM(16); LVBA_SET_SMEM(21); LVBA_SET_SMEM(24); LVBA_SET_SMEM(31);
#undef LVBA_SET_SMEM
      LVBA_CUDA(cudaFuncSetAttribute(env_backsolve_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBsSmem));
      configured = true;
    }
    if (!groups.empty()) {
      // windows are <= 31 poses: always the register-window kernel, one CTA per window
      n_groups = (int)groups.size() - 1;
      grp_ptr = groups;
      std::vector<int> fr((size_t)env.n);
      for (int g = 0; g < n_groups; ++g) {
        if (groups[g + 1] - groups[g] > 31)
          return fail(LVBA_ERR_UNSUPPORTED, "window %d has %d poses; the batched solve handles <= 31 per window", g, groups[g + 1] - groups[g]);
        for (int r = groups[g]; r < groups[g + 1]; ++r) {
          if (env.first[r] < groups[g]) return fail(LVBA_ERR_INVALID_ARG, "row %d couples to a pose outside its window", r);
          fr[r] = env.first[r] - groups[g];
        }
      }
      LVBA_TRY(first_rel.upload(fr, s));
      LVBA_TRY(status.alloc((size_t)std::max(n_groups, 4)));
      LVBA_CUDA(cudaStreamSynchronize(s));
      path = kSolveBatch;
      return LVBA_OK;
    }
    // the register-window kernel holds columns of <= 30 blocks; the shared-memory window those of <= kEnvMaxCol
    const bool reg_ok = env.max_col <= 30 && env.n >= 3;
    if (want == LVBA_SOLVE_ANY_WIDTH || env.max_col > kEnvMaxCol) {
      LVBA_TRY(colT.alloc((size_t)std::max(env.max_col, 1) * 36));
      path = LVBA_SOLVE_ANY_WIDTH;
    } else if (want != LVBA_SOLVE_SHARED_WINDOW && reg_ok) {
      if (want == LVBA_SOLVE_AUTO || want == LVBA_SOLVE_CHUNKED) LVBA_TRY(prepare_chunked(env, s, want == LVBA_SOLVE_CHUNKED ? chunks : 0));
      if (path == LVBA_SOLVE_AUTO && (want == LVBA_SOLVE_AUTO ? env.n >= 256 : want == LVBA_SOLVE_TWISTED)) LVBA_TRY(prepare_twisted(env, s));
      if (path == LVBA_SOLVE_AUTO) path = LVBA_SOLVE_ONE_CTA;
    }
    if (path == LVBA_SOLVE_AUTO) path = LVBA_SOLVE_SHARED_WINDOW;
    if (want != LVBA_SOLVE_AUTO && path != want)
      return fail(LVBA_ERR_UNSUPPORTED, "path %d is not available for this structure (n = %d, tallest column %d blocks): would take path %d", want, env.n, env.max_col, path);
    return LVBA_OK;
  }
  // substructured split: p chunks (chunks < 2: default_chunks); sets path = LVBA_SOLVE_CHUNKED if the structure can be cut
  int prepare_chunked(const Envelope& env, cudaStream_t s, int chunks) {
    const int pw1 = chunks >= 2 ? chunks : NdDevice::default_chunks(env.n, std::max(env.max_col, 1));
    Comm& cm = comm();
    const int nr = cm.active() ? cm.n_ranks : 1;                   // the chunks are the multi-GPU unit (SURVEY.md 8(e))
    const int pw = (nr > 1 && pw1 < nr) ? nr : pw1;                // one chunk per rank at least
    if (pw < 2) return LVBA_OK;
    LVBA_TRY(nd.prepare(env.n, env.first, env.last, env.row_start, env.max_col, pw, s, nr, nr > 1 ? cm.rank : 0));
    if (nr > 1 && !nd.ready && pw1 >= 2) LVBA_TRY(nd.prepare(env.n, env.first, env.last, env.row_start, env.max_col, pw1, s, 1, 0));   // not cuttable per rank
    if (!nd.ready) return LVBA_OK;
    LVBA_TRY(status.alloc((size_t)std::max<size_t>(4, nd.plan.nodes.size() + 1)));
    path = LVBA_SOLVE_CHUNKED;
    return LVBA_OK;
  }
  // twisted split: top half in natural order, bottom half reversed, joined at a separator of tw_bs rows; worthwhile when each
  // half is many pivots long.  Sets path = LVBA_SOLVE_TWISTED if the split fits the register window
  int prepare_twisted(const Envelope& env, cudaStream_t s) {
    const int n = env.n;
    if (n < 8) return LVBA_OK;
    const int m = n / 2;
    const int send = env.last[m - 1] + 1;            // rows >= send do not couple to rows < m
    const int bs = send - m;
    if (bs < 3 || bs > 30 || send >= n - 32) return LVBA_OK;
    tw_m = m; tw_send = send; tw_bs = bs; tw_nb = n - m; tw_nbstop = n - send;
    std::vector<int> fb((size_t)tw_nb);
    for (int rp = 0; rp < tw_nb; ++rp) fb[rp] = n - 1 - env.last[n - 1 - rp];     // reversed row couples up to the original column's last row
    int64_t dummy = 0;
    LVBA_TRY(env_bot.build(fb, s, &dummy));
    std::vector<int> fs((size_t)bs, 0);
    LVBA_TRY(env_sep.build(fs, s, &dummy));
    if (env_bot.max_col > 30) return LVBA_OK;
    LVBA_TRY(Lbot.alloc((size_t)env_bot.nblocks * 36)); LVBA_TRY(dinv_bot.alloc((size_t)tw_nb * 36));
    LVBA_TRY(zbot.alloc((size_t)tw_nb * 6)); LVBA_TRY(xbot.alloc((size_t)tw_nb * 6));
    LVBA_TRY(wtop.alloc((size_t)bs * bs * 36)); LVBA_TRY(wbot.alloc((size_t)bs * bs * 36));
    LVBA_TRY(ztopd.alloc((size_t)bs * 6)); LVBA_TRY(zbotd.alloc((size_t)bs * 6));
    LVBA_TRY(Lsep.alloc((size_t)env_sep.nblocks * 36)); LVBA_TRY(dinv_sep.alloc((size_t)bs * 36));
    LVBA_TRY(zsep.alloc((size_t)bs * 6)); LVBA_TRY(xsep.alloc((size_t)bs * 6));
    LVBA_TRY(wtop.zero(s)); LVBA_TRY(wbot.zero(s));
    path = LVBA_SOLVE_TWISTED;
    return LVBA_OK;
  }
  static size_t factor_smem() { return sizeof(double) * (2 * kEnvMaxCol * 36 + 36 + 8); }

  int ensure_map(int id, cudaStream_t s) {
    if (have_map[id]) return LVBA_OK;
    const int P = pval(id);
    const int nthr = id == 0 ? LaCfg<8, la_tile2(8)>::kPairThreads : id == 1 ? LaCfg<12, la_tile2(12)>::kPairThreads
                   : id == 2 ? LaCfg<16, la_tile2(16)>::kPairThreads : id == 3 ? LaCfg<21, la_tile2(21)>::kPairThreads
                   : id == 4 ? LaCfg<24, la_tile2(24)>::kPairThreads : LaCfg<31, la_tile2(31)>::kPairThreads;
    const bool tile2 = la_tile2(P);
    std::vector<unsigned> m = build_pair_map32(P, tile2, nthr);
    size_t cnt = 0;
    for (auto v2 : m) if (v2 != 0xffffffffu) cnt += ((v2 >> 16) & 0xff) != 0xff ? 2 : 1;
    if ((int)cnt != P * (P + 1) / 2) return fail(LVBA_ERR_UNSUPPORTED, "pair map for P=%d covers %zu of %d pairs", P, cnt, P * (P + 1) / 2);
    LVBA_TRY(pair_map[id].upload(m, s));
    LVBA_CUDA(cudaStreamSynchronize(s));               // `m` is a local vector
    have_map[id] = true;
    return LVBA_OK;
  }
  int launch_factor(int id, int grid, const FactorJob* jobs, cudaStream_t s, int64_t* launches) {
    LVBA_TRY(ensure_map(id, s));
    const unsigned* pm = pair_map[id].p;
#define LVBA_LAUNCH_LA(PP) env_factor_la_kernel<PP, la_tile2(PP)><<<grid, LaCfg<PP, la_tile2(PP)>::kThreads, LaCfg<PP, la_tile2(PP)>::kSmem, s>>>(jobs, pm)
    switch (id) {
      case 0: LVBA_LAUNCH_LA(8); break;
      case 1: LVBA_LAUNCH_LA(12); break;
      case 2: LVBA_LAUNCH_LA(16); break;
      case 3: LVBA_LAUNCH_LA(21); break;
      case 4: LVBA_LAUNCH_LA(24); break;
      default: LVBA_LAUNCH_LA(31);
    }
#undef LVBA_LAUNCH_LA
    ++*launches;
    return LVBA_OK;
  }
  // x = D^-1 z for the pivots
  void launch_apply(int nrows, const double* dinv_p, const double* z_p, double* x_p, cudaStream_t s) {
    if (nrows > 0) env_dinv_apply_kernel<<<(6 * nrows + 127) / 128, 128, 0, s>>>(nrows, dinv_p, z_p, x_p);
  }
  void launch_backsolve(int grid, const BacksolveJob* bj, cudaStream_t s) { env_backsolve_warp_kernel<<<grid, 64, kBsSmem, s>>>(bj); }

  int build_jobs(const Envelope& env, double* x, cudaStream_t s) {
    if (jobs_x == x && d_fjobs.p) return LVBA_OK;
    const EnvView v = env.view();
    std::vector<FactorJob> fj;
    std::vector<BacksolveJob> bj;
    if (path == kSolveBatch) {
      for (int g = 0; g < n_groups; ++g) {
        const int r0 = grp_ptr[g], ng = grp_ptr[g + 1] - r0;
        EnvView vg{ng, first_rel.p + r0, env.d_row_start.p + r0, env.d_last.p + r0, env.nblocks};
        fj.push_back(FactorJob{vg, L.p, dinv.p + 36 * (size_t)r0, z.p + 6 * (size_t)r0, ng, nullptr, nullptr, status.p + g});
        bj.push_back(BacksolveJob{vg, L.p, x + 6 * (size_t)r0, ng});
      }
    } else if (path == LVBA_SOLVE_TWISTED) {
      EnvView vt = v; vt.n = tw_send;                               // the top instance is a prefix of the matrix
      const EnvView vb = env_bot.view(), vs = env_sep.view();
      fj.push_back(FactorJob{vt, L.p, dinv.p, z.p, tw_m, wtop.p, ztopd.p, status.p});
      fj.push_back(FactorJob{vb, Lbot.p, dinv_bot.p, zbot.p, tw_nbstop, wbot.p, zbotd.p, status.p + 1});
      fj.push_back(FactorJob{vs, Lsep.p, dinv_sep.p, zsep.p, tw_bs, nullptr, nullptr, status.p + 2});
      bj.push_back(BacksolveJob{vs, Lsep.p, xsep.p, tw_bs});
      bj.push_back(BacksolveJob{vt, L.p, x, tw_m});
      bj.push_back(BacksolveJob{vb, Lbot.p, xbot.p, tw_nbstop});
    } else {
      fj.push_back(FactorJob{v, L.p, dinv.p, z.p, env.n, nullptr, nullptr, status.p});
      bj.push_back(BacksolveJob{v, L.p, x, env.n});
    }
    LVBA_TRY(d_fjobs.upload(fj, s));
    LVBA_TRY(d_bjobs.upload(bj, s));
    LVBA_CUDA(cudaStreamSynchronize(s));               // local vectors
    jobs_x = x;
    return LVBA_OK;
  }

  // Substructured solve: nd::run (nd_passes.h) through the CUDA executor, captured into a graph at its first use
  int solve_nd(const Envelope& env, const double* H, const double* dadd, double* x, cudaStream_t s, int64_t* launches) {
    const EnvView v = env.view();
    LVBA_TRY(nd.build_tables(v, H, dadd, L.p, dinv.p, z.p, x, status.p, s));
    for (const auto& J : nd.lv) LVBA_TRY(ensure_map(pid(J.max_col), s));           // uploads + syncs: not inside a capture
    auto record = [&](int64_t* n_launch) -> int {
      NdCudaExec ex;
      ex.s = s;
      ex.det = det;
      ex.dense_map = nd.d_dense_map.p;
      ex.factor_fn = [&](int max_col, int nj, const FactorJob* jobs) { return launch_factor(pid(max_col), nj, jobs, s, &ex.launches); };
      ex.back_fn = [&](int nj, const BacksolveJob* jobs) { launch_backsolve(nj, jobs, s); };
      cudaMemsetAsync(status.p, 0, status.n * sizeof(int), s);
      nd::run(ex, nd.plan, nd.tab, nd.lv.data(), (int)nd.lv.size(), env.nblocks, nd.leaf_e, nd.leaf_fin);
      env_status_or_kernel<<<1, 32, 0, s>>>(status.p, (int)nd.plan.nodes.size() + 1);
      *n_launch = ex.launches + 1;
      return ex.rc;
    };
    if (dist()) {
      // ---- multi-GPU: own subtree, ONE all-gather of the fixed-size slots, top tree (replicated), downwards, x assembled
      Comm& cm = comm();
      NdCudaExec ex;
      ex.s = s;
      ex.dense_map = nd.d_dense_map.p;
      ex.factor_fn = [&](int max_col, int nj, const FactorJob* jobs) { return launch_factor(pid(max_col), nj, jobs, s, &ex.launches); };
      ex.back_fn = [&](int nj, const BacksolveJob* jobs) { launch_backsolve(nj, jobs, s); };
      cudaMemsetAsync(status.p, 0, status.n * sizeof(int), s);
      nd::run_up_local(ex, nd.plan, nd.tab, nd.lv.data(), (int)nd.lv.size(), env.nblocks, nd.leaf_e, nd.leaf_fin, &nd.reg);
      LVBA_TRY(cm.allgather_inplace(nd.U.p + nd.plan.region0, (size_t)nd.plan.slot, s));
      nd::run_top_down(ex, nd.plan, nd.tab, nd.lv.data(), (int)nd.lv.size(), &nd.reg);
      ex.pass((long long)6 * env.n, nd::ZeroForeignF{x, dist_begin(), dist_end()});
      LVBA_TRY(cm.allreduce_sum(x, (size_t)6 * env.n, s));
      env_status_or_kernel<<<1, 32, 0, s>>>(status.p, (int)nd.plan.nodes.size() + 1);
      LVBA_TRY(cm.allreduce_max_int(status.p, 1, s));
      *launches += ex.launches + 1;
      if (ex.rc != LVBA_OK) return ex.rc;
      LVBA_CUDA(cudaGetLastError());
      return LVBA_OK;
    }
    if (nd.use_graph && !nd.graph_exec) {
      if (cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
        const int rc = record(&nd.launches_per_solve);
        cudaGraph_t g = nullptr;
        const cudaError_t e1 = cudaStreamEndCapture(s, &g);
        if (rc == LVBA_OK && e1 == cudaSuccess && g && cudaGraphInstantiate(&nd.graph_exec, g, 0) == cudaSuccess) nd.graph = g;
        else {
          if (g) cudaGraphDestroy(g);
          nd.graph_exec = nullptr; nd.use_graph = false;
          cudaGetLastError();
        }
      } else { nd.use_graph = false; cudaGetLastError(); }
    }
    if (nd.use_graph && nd.graph_exec) {
      LVBA_CUDA(cudaGraphLaunch(nd.graph_exec, s));
      *launches += nd.launches_per_solve;
    } else {
      int64_t nl = 0;
      LVBA_TRY(record(&nl));
      *launches += nl;
    }
    LVBA_CUDA(cudaGetLastError());
    return LVBA_OK;
  }

  // Solves (H + diag(dadd)) x = z_in where z already holds the right-hand side.  Multi-GPU (dist()): H and dadd need to be valid
  // on the rows this rank owns only (exchange_rows() done); the rows of the other ranks' rank separators are WRITTEN into H and
  // dadd (const is cast away for that), z must be valid everywhere, x comes back complete on every rank.  status[0] != 0 afterwards flags a
  // singular pivot (batched mode: status[g] per group).
  int solve(const Envelope& env, const double* H, const double* dadd, double* x, cudaStream_t s, int64_t* launches) {
    if (path == LVBA_SOLVE_CHUNKED) return solve_nd(env, H, dadd, x, s, launches);
    const EnvView v = env.view();
    LVBA_CUDA(cudaMemcpyAsync(L.p, H, (size_t)env.nblocks * 36 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    LVBA_CUDA(cudaMemsetAsync(status.p, 0, status.n * sizeof(int), s));
    const int n6 = 6 * env.n;
    env_add_diag_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(v, dadd, L.p);
    ++*launches;
    const int mc = env.max_col;
    if (path == LVBA_SOLVE_ANY_WIDTH) {
      // ---------------- any width: every column step spread over the device (envelope_wide.h); 4 launches per block row
      const wide::View wv{env.n, env.d_first.p, env.d_row_start.p};                                       // z holds the right-hand side (written by the caller)
      auto launch = [&](int64_t items, const auto& f) { wide_pass(s, items, f, launches); };
      wide::factor_and_solve(launch, wv, env.first.data(), env.last.data(), L.p, dinv.p, z.p, colT.p, x, status.p);
      LVBA_CUDA(cudaGetLastError());
      return LVBA_OK;
    }
    if (path != LVBA_SOLVE_SHARED_WINDOW) LVBA_TRY(build_jobs(env, x, s));
    if (path == kSolveBatch) {
      LVBA_TRY(launch_factor(pid(mc), n_groups, d_fjobs.p, s, launches));
      launch_apply(env.n, dinv.p, z.p, x, s);
      launch_backsolve(n_groups, d_bjobs.p, s);
      *launches += 2;
    } else if (path == LVBA_SOLVE_TWISTED) {
      // ---------------- twisted: two half factorisations on two SMs, joined at the separator
      const int n = env.n, m = tw_m, bs = tw_bs;
      const EnvView vb = env_bot.view();
      env_reverse_gather_kernel<<<std::min(tw_nb, 2048), 128, 0, s>>>(v, vb, L.p, Lbot.p, z.p, zbot.p);
      ++*launches;
      LVBA_TRY(launch_factor(pid(std::max(mc, env_bot.max_col)), 2, d_fjobs.p, s, launches));
      env_twist_combine_kernel<<<1, 1024, 0, s>>>(v, m, bs, L.p, z.p, wtop.p, wbot.p, ztopd.p, zbotd.p, Lsep.p, zsep.p);
      ++*launches;
      LVBA_TRY(launch_factor(pid(env_sep.max_col), 1, d_fjobs.p + 2, s, launches));
      launch_apply(bs, dinv_sep.p, zsep.p, xsep.p, s);
      launch_backsolve(1, d_bjobs.p, s);
      launch_apply(m, dinv.p, z.p, x, s);
      launch_apply(tw_nbstop, dinv_bot.p, zbot.p, xbot.p, s);
      env_twist_place_sep_kernel<<<(bs * 6 + 127) / 128, 128, 0, s>>>(m, bs, tw_nbstop, xsep.p, x, xbot.p);
      launch_backsolve(2, d_bjobs.p + 1, s);
      env_twist_scatter_kernel<<<(tw_nbstop * 6 + 255) / 256, 256, 0, s>>>(n, tw_nbstop, xbot.p, x);
      env_status_or_kernel<<<1, 32, 0, s>>>(status.p, 3);
      *launches += 8;
    } else if (path == LVBA_SOLVE_ONE_CTA) {
      LVBA_TRY(launch_factor(pid(mc), 1, d_fjobs.p, s, launches));
      launch_apply(env.n, dinv.p, z.p, x, s);
      launch_backsolve(1, d_bjobs.p, s);
      *launches += 2;
    } else {
      env_factor_kernel<<<1, kFactorThreads, factor_smem(), s>>>(v, L.p, dinv.p, z.p, status.p);
      env_backsolve_kernel<<<1, 32, 0, s>>>(v, L.p, dinv.p, z.p, x);
      *launches += 2;
    }
    LVBA_CUDA(cudaGetLastError());
    return LVBA_OK;
  }
};

}  // namespace lvba
