// lvba_b200.cu — the single translation unit of liblvba_b200.so (sm_90a).
// Kernels live in the .cuh files next to this one; this file adds the path-independent entry points.
#include <memory>

#include "lidar_api.cuh"
#include "visual_api.cuh"
#include "voxel_api.cuh"
#include "depth_api.cuh"
#include "track_api.cuh"
#include "anchor_api.cuh"
#include "fuse_api.cuh"
#include "color_api.cuh"

extern "C" {

int lvba_version(void) { return LVBA_B200_VERSION; }
int lvba_device_count(void) { return lvba::device_count(); }
const char* lvba_last_error(void) { return lvba::last_error_ref().c_str(); }
int lvba_release_cached_memory(void) { lvba::device_pool().clear(); lvba::pinned_pool().clear(); return LVBA_OK; }
const char* lvba_status_string(int status) {
  switch (status) {
    case LVBA_OK: return "ok";
    case LVBA_ERR_INVALID_ARG: return "invalid argument";
    case LVBA_ERR_NO_DEVICE: return "no CUDA device (no CPU fallback)";
    case LVBA_ERR_CUDA: return "CUDA runtime error";
    case LVBA_ERR_UNSUPPORTED: return "unsupported problem shape";
    case LVBA_ERR_NUMERIC: return "numerical failure";
    case LVBA_ERR_COMM: return "communication (NCCL) error";
    case LVBA_ERR_NOMEM: return "out of memory";
    default: return "unknown status";
  }
}

// ---------------------------------------------------------------- the block LDL^T on its own (diagnostics / tests)
int lvba_env_solve(int32_t n, const int32_t* first, const double* blocks, const double* dadd, const double* rhs,
                   double* x, int32_t path, int32_t chunks, int32_t reps, int32_t device, double* ms, int32_t* info) LVBA_ABI_BEGIN {
  using namespace lvba;
  if (n <= 0 || !first || !blocks || !dadd || !rhs || !x) return fail(LVBA_ERR_INVALID_ARG, "null argument or n <= 0");
  if (path < LVBA_SOLVE_AUTO || path > LVBA_SOLVE_ANY_WIDTH) return fail(LVBA_ERR_INVALID_ARG, "unknown path %d", path);
  for (int r = 0; r < n; ++r) {
    if (first[r] < 0 || first[r] > r) return fail(LVBA_ERR_INVALID_ARG, "first[%d] = %d outside [0, %d]", r, first[r], r);
    if (r > 0 && first[r] < first[r - 1]) return fail(LVBA_ERR_INVALID_ARG, "first[] must be non-decreasing (row %d)", r);
  }
  LVBA_TRY(select_device(device));
  cudaStream_t s = nullptr;
  LVBA_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamSynchronize(s); cudaStreamDestroy(s); } } guard{s};
  int rc = LVBA_OK;
  {
    Envelope env;
    int64_t bytes = 0;
    std::vector<int> fr(first, first + n);
    LVBA_TRY(env.build(fr, s, &bytes));
    EnvSolver sol;
    LVBA_TRY(sol.prepare(env, s, path, chunks));
    const bool chunked = sol.path == LVBA_SOLVE_CHUNKED;
    DevBuf<double> dH, dD, dR, dX;
    LVBA_TRY(dH.upload(blocks, (size_t)env.nblocks * 36, s)); LVBA_TRY(dD.upload(dadd, (size_t)n * 6, s));
    LVBA_TRY(dR.upload(rhs, (size_t)n * 6, s)); LVBA_TRY(dX.alloc((size_t)n * 6));
    cudaEvent_t e0, e1;
    LVBA_CUDA(cudaEventCreate(&e0)); LVBA_CUDA(cudaEventCreate(&e1));
    float best = 1e30f;
    int64_t launches = 0, per = 0;
    for (int rep = 0; rep < std::max(reps, 1) && rc == LVBA_OK; ++rep) {
      cudaMemcpyAsync(sol.z.p, dR.p, (size_t)n * 6 * sizeof(double), cudaMemcpyDeviceToDevice, s);
      cudaMemsetAsync(dX.p, 0, (size_t)n * 6 * sizeof(double), s);
      const int64_t l0 = launches;
      cudaEventRecord(e0, s);
      rc = sol.solve(env, dH.p, dD.p, dX.p, s, &launches);
      cudaEventRecord(e1, s);
      per = launches - l0;
      if (rc == LVBA_OK && cudaStreamSynchronize(s) != cudaSuccess) rc = fail(LVBA_ERR_CUDA, "solve: %s", cudaGetErrorString(cudaGetLastError()));
      float t = 0.f;
      if (rc == LVBA_OK && cudaEventElapsedTime(&t, e0, e1) == cudaSuccess) best = std::min(best, t);
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (rc == LVBA_OK) {
      int st = 0;
      LVBA_CUDA(cudaMemcpy(&st, sol.status.p, sizeof(int), cudaMemcpyDeviceToHost));
      LVBA_CUDA(cudaMemcpy(x, dX.p, (size_t)n * 6 * sizeof(double), cudaMemcpyDeviceToHost));
      if (st) rc = fail(LVBA_ERR_NUMERIC, "singular / non-finite pivot block");
    }
    if (ms) *ms = best;
    if (info) { info[0] = sol.path; info[1] = chunked ? sol.nd.chunks : 0; info[2] = chunked ? (int)sol.nd.plan.levels.size() : 0; info[3] = (int)per; }
    cudaStreamSynchronize(s);       // nothing of `sol` / the buffers may be in flight when they go back to the pool
  }
  return rc;
} LVBA_ABI_END("lvba_env_solve")

// ---------------------------------------------------------------- multi-GPU
int lvba_comm_unique_id(void* id_out) LVBA_ABI_BEGIN {
  if (!id_out) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  lvba::Comm& c = lvba::comm();
  LVBA_TRY(c.load());
  ncclUniqueId id;
  static_assert(sizeof(ncclUniqueId) == LVBA_NCCL_ID_BYTES, "ncclUniqueId size");
  ncclResult_t r = c.GetUniqueId(&id);
  if (r != ncclSuccess) return lvba::fail(LVBA_ERR_COMM, "ncclGetUniqueId: %s", c.GetErrorString(r));
  memcpy(id_out, &id, sizeof id);
  return LVBA_OK;
} LVBA_ABI_END("lvba_comm_unique_id")

int lvba_comm_init(int32_t n_ranks, int32_t rank, const void* id, int32_t device) LVBA_ABI_BEGIN {
  if (n_ranks < 1 || rank < 0 || rank >= n_ranks) return lvba::fail(LVBA_ERR_INVALID_ARG, "bad rank %d / %d", rank, n_ranks);
  lvba::Comm& c = lvba::comm();
  if (c.comm) return lvba::fail(LVBA_ERR_INVALID_ARG, "communicator already initialised");
  c.n_ranks = n_ranks; c.rank = rank;
  if (n_ranks == 1) return LVBA_OK;
  if (!id) return lvba::fail(LVBA_ERR_INVALID_ARG, "null unique id");
  LVBA_TRY(lvba::select_device(device));
  LVBA_TRY(c.load());
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof uid);
  ncclResult_t r = c.CommInitRank(&c.comm, n_ranks, uid, rank);
  if (r != ncclSuccess) { c.comm = nullptr; c.n_ranks = 1; c.rank = 0; return lvba::fail(LVBA_ERR_COMM, "ncclCommInitRank: %s", c.GetErrorString(r)); }
  return LVBA_OK;
} LVBA_ABI_END("lvba_comm_init")

int lvba_comm_destroy(void) LVBA_ABI_BEGIN {
  lvba::Comm& c = lvba::comm();
  if (c.comm) { c.CommDestroy(c.comm); c.comm = nullptr; }
  c.n_ranks = 1; c.rank = 0;
  return LVBA_OK;
} LVBA_ABI_END("lvba_comm_destroy")

int lvba_comm_info(int32_t* n_ranks, int32_t* rank) LVBA_ABI_BEGIN {
  lvba::Comm& c = lvba::comm();
  if (n_ranks) *n_ranks = c.n_ranks;
  if (rank) *rank = c.rank;
  return LVBA_OK;
} LVBA_ABI_END("lvba_comm_info")

int64_t lvba_comm_bytes_sent(void) {
  lvba::Comm& c = lvba::comm();
  const int64_t b = c.bytes_sent;
  c.bytes_sent = 0;
  return b;
}
int lvba_lidar_owned_rows(lvba_lidar_problem* p, int32_t* row_begin, int32_t* row_end, int32_t* sharded) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null problem");
  const bool d = p->solver.dist();
  if (row_begin) *row_begin = d ? p->solver.dist_begin() : 0;
  if (row_end) *row_end = d ? p->solver.dist_end() : p->W;
  if (sharded) *sharded = d ? 1 : 0;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_owned_rows")
int lvba_visual_owned_rows(lvba_visual_problem* p, int32_t* row_begin, int32_t* row_end, int32_t* sharded) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null problem");
  const bool d = p->n_rows > 0 && p->solver.dist();
  if (row_begin) *row_begin = d ? p->solver.dist_begin() : 0;
  if (row_end) *row_end = d ? p->solver.dist_end() : p->n_rows;
  if (sharded) *sharded = d ? 1 : 0;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_owned_rows")

int32_t lvba_shard_owner(int32_t min_pose, int32_t n_rows, int32_t n_ranks) { return lvba::shard_owner(min_pose, n_rows, n_ranks); }

}  // extern "C"
