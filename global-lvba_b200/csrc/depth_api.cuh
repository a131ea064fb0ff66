// depth_api.cuh — boundary B4 (SURVEY.md §8f N3, first half): depth images rendered from the world point grid on the device.
// Passes: depth_pipeline.h; execution policy: CudaExec (exec.cuh).  No host path.
#pragma once
#include "depth_pipeline.h"
#include "voxel_api.cuh"

struct lvba_depth_grid {
  lvba::depth::DepthGrid<lvba::CudaExec> grid;
  int device = 0;
  lvba_depth_summary sum{};
  ~lvba_depth_grid() { cudaStreamSynchronize(grid.ex.stream); }     // members are parked in the pool after this body: they must be idle
};

extern "C" {

int lvba_depth_grid_create(int32_t n_frames, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats,
                           const double* poses, const double* frame_ts, double voxel_size, int32_t device,
                           lvba_depth_grid** out, lvba_depth_summary* summary) LVBA_ABI_BEGIN {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  if (!out) return lvba::fail(LVBA_ERR_INVALID_ARG, "null output handle");
  *out = nullptr;
  if (n_frames < 0 || !scan_ptr || (n_frames > 0 && (!poses || !frame_ts))) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative frame count");
  if (xyz_stride_floats < 3) return lvba::fail(LVBA_ERR_INVALID_ARG, "xyz_stride %d < 3 floats", xyz_stride_floats);
  if (!(voxel_size > 0.0) || !std::isfinite(voxel_size)) return lvba::fail(LVBA_ERR_INVALID_ARG, "voxel_size must be positive and finite");
  if (scan_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "scan_ptr[0] != 0");
  for (int32_t j = 0; j < n_frames; ++j) {
    if (scan_ptr[j + 1] < scan_ptr[j]) return lvba::fail(LVBA_ERR_INVALID_ARG, "scan_ptr not monotone at frame %d", j);
    if (!std::isfinite(frame_ts[j]) || (j > 0 && frame_ts[j] < frame_ts[j - 1]))
      return lvba::fail(LVBA_ERR_INVALID_ARG, "frame_ts must be finite and ascending (frame %d)", j);   // the window search is a lower/upper_bound
  }
  const int64_t N = scan_ptr[n_frames];
  if (N >= (int64_t)0xfffffff0ll) return lvba::fail(LVBA_ERR_UNSUPPORTED, "%lld points: more than 2^32 per grid", (long long)N);
  if (N > 0 && !xyz) return lvba::fail(LVBA_ERR_INVALID_ARG, "null xyz");
  for (int64_t k = 0; k < (int64_t)n_frames * 12; ++k)
    if (!std::isfinite(poses[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite pose entry %lld", (long long)k);
  LVBA_TRY(lvba::select_device(device));
  std::unique_ptr<lvba_depth_grid> h(new lvba_depth_grid());
  cudaGetDevice(&h->device);
  lvba::CudaExec& ex = h->grid.ex;
  lvba::DevBuf<float> d_xyz;
  lvba::DevBuf<int64_t> d_scan;
  lvba::DevBuf<double> d_poses, d_ts;
  lvba::StreamDrain drain(nullptr);      // every path of this handle runs on the NULL stream
  int64_t h2d = 0;
  std::vector<float> packed;
  const float* src = xyz;
  if (xyz_stride_floats != 3 && N > 0) {
    packed.resize((size_t)N * 3);
    float* dst = packed.data();
    const int stride = xyz_stride_floats;
    lvba::parallel_chunks(N, 1 << 16, [=](int64_t a, int64_t b, int) {
      for (int64_t i = a; i < b; ++i) { dst[3 * i] = xyz[i * stride]; dst[3 * i + 1] = xyz[i * stride + 1]; dst[3 * i + 2] = xyz[i * stride + 2]; }
    });
    src = packed.data();
  }
  LVBA_TRY(d_xyz.upload(src, (size_t)N * 3, ex.stream, &h2d));
  LVBA_TRY(d_scan.upload(scan_ptr, (size_t)n_frames + 1, ex.stream, &h2d));
  LVBA_TRY(d_poses.upload(poses, (size_t)n_frames * 12, ex.stream, &h2d));
  LVBA_TRY(d_ts.upload(frame_ts, (size_t)n_frames, ex.stream, &h2d));
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  const cudaEvent_t e0 = ev.a, e1 = ev.b;
  LVBA_CUDA(cudaEventRecord(e0, ex.stream));
  const auto t1 = clk::now();
  const int rc = h->grid.build(d_xyz.p, d_scan.p, d_poses.p, d_ts.p, n_frames, N, voxel_size);
  if (rc != LVBA_OK) {
    if (h->grid.error[0]) return lvba::fail(rc, "%s", h->grid.error);
    return rc;
  }
  LVBA_CUDA(cudaEventRecord(e1, ex.stream));
  LVBA_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  LVBA_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  ex.temp.release();
  lvba_depth_summary& s = h->sum;
  s.n_points = N; s.n_voxels = h->grid.n_voxels; s.n_pairs = h->grid.n_pairs;
  s.ms_device = ms;
  s.ms_upload = std::chrono::duration<double, std::milli>(t1 - t0).count();
  s.ms_total = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
  s.kernel_launches = ex.launches; s.h2d_bytes = h2d;
  if (summary) *summary = s;
  *out = h.release();
  return LVBA_OK;
} LVBA_ABI_END("lvba_depth_grid_create")

int lvba_depth_render(lvba_depth_grid* g, int32_t n_images, const double* cams, const double* image_ts, double half_window,
                      const double intr[8], int32_t width, int32_t height, float* depth, lvba_depth_summary* summary) LVBA_ABI_BEGIN {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  if (!g || n_images < 0 || (n_images > 0 && (!cams || !image_ts || !depth)) || !intr) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative image count");
  if (width <= 0 || height <= 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "image size %d x %d", width, height);
  if (!(half_window >= 0.0)) return lvba::fail(LVBA_ERR_INVALID_ARG, "half_window must be >= 0");
  for (int64_t k = 0; k < (int64_t)n_images * 12; ++k)
    if (!std::isfinite(cams[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite camera entry %lld", (long long)k);
  for (int k = 0; k < 8; ++k)
    if (!std::isfinite(intr[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite intrinsic %d", k);
  LVBA_CUDA(cudaSetDevice(g->device));
  auto& G = g->grid;
  lvba::CudaExec& ex = G.ex;
  const int64_t launches0 = ex.launches;
  const int64_t pix = (int64_t)width * height;
  const int64_t batch = std::max<int64_t>(1, ((int64_t)1 << 28) / pix);          // <= 2^28 pixels (1 GiB of floats) per pass
  lvba::DevBuf<double> d_cams, d_ts;
  lvba::DevBuf<float> d_depth;
  lvba::StreamDrain drain(nullptr);
  int64_t h2d = 0, d2h = 0, pairs = 0, chunks = 0;
  float ms_dev = 0.f;
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  const cudaEvent_t e0 = ev.a, e1 = ev.b;
  for (int64_t k0 = 0; k0 < n_images; k0 += batch) {
    const int64_t nb = std::min<int64_t>(batch, n_images - k0);
    LVBA_TRY(d_cams.upload(cams + 12 * k0, (size_t)nb * 12, ex.stream, &h2d));
    LVBA_TRY(d_ts.upload(image_ts + k0, (size_t)nb, ex.stream, &h2d));
    if (d_depth.n < (size_t)(nb * pix)) LVBA_TRY(d_depth.alloc((size_t)(nb * pix)));
    LVBA_CUDA(cudaEventRecord(e0, ex.stream));
    const int rc = G.render(nb, d_cams.p, d_ts.p, half_window, intr, width, height, d_depth.p);
    if (rc != LVBA_OK) return rc;
    LVBA_CUDA(cudaEventRecord(e1, ex.stream));
    LVBA_CUDA(cudaMemcpyAsync(depth + k0 * pix, d_depth.p, (size_t)(nb * pix) * sizeof(float), cudaMemcpyDeviceToHost, ex.stream));
    LVBA_CUDA(cudaStreamSynchronize(ex.stream));
    float ms = 0.f;
    LVBA_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    ms_dev += ms; d2h += nb * pix * 4; pairs += G.last_pairs; chunks += G.last_chunks;
  }
  ex.temp.release();
  if (summary) {
    *summary = g->sum;
    summary->ms_device = ms_dev; summary->ms_upload = 0.0;
    summary->ms_total = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
    summary->kernel_launches = ex.launches - launches0; summary->h2d_bytes = h2d; summary->d2h_bytes = d2h;
    summary->work_pairs = pairs; summary->work_chunks = chunks;
  }
  return LVBA_OK;
} LVBA_ABI_END("lvba_depth_render")

// The depth-candidate loop of BuildTracksAndFuse3D (src/lvba_system.cpp:1020-1038) for every keypoint of every image: the
// images are rendered batch by batch and sampled where they are; they never leave the device.
int lvba_depth_backproject(lvba_depth_grid* g, int32_t n_images, const double* cams, const double* image_ts, double half_window,
                           const double intr[8], int32_t width, int32_t height, const int64_t* kp_ptr, const float* kp_uv,
                           double* Xw, uint8_t* valid, lvba_depth_summary* summary) LVBA_ABI_BEGIN {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  if (!g || n_images < 0 || !intr || !kp_ptr || (n_images > 0 && (!cams || !image_ts))) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative image count");
  if (width <= 1 || height <= 1) return lvba::fail(LVBA_ERR_INVALID_ARG, "image size %d x %d", width, height);
  if (!(half_window >= 0.0)) return lvba::fail(LVBA_ERR_INVALID_ARG, "half_window must be >= 0");
  if (kp_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "kp_ptr[0] != 0");
  for (int32_t k = 0; k < n_images; ++k)
    if (kp_ptr[k + 1] < kp_ptr[k]) return lvba::fail(LVBA_ERR_INVALID_ARG, "kp_ptr not monotone at image %d", k);
  const int64_t n_kp = kp_ptr[n_images];
  if (n_kp > 0 && (!kp_uv || !Xw || !valid)) return lvba::fail(LVBA_ERR_INVALID_ARG, "null keypoint / output array");
  for (int64_t k = 0; k < (int64_t)n_images * 12; ++k)
    if (!std::isfinite(cams[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite camera entry %lld", (long long)k);
  for (int k = 0; k < 8; ++k)
    if (!std::isfinite(intr[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite intrinsic %d", k);
  LVBA_CUDA(cudaSetDevice(g->device));
  auto& G = g->grid;
  lvba::CudaExec& ex = G.ex;
  const int64_t launches0 = ex.launches;
  const int64_t pix = (int64_t)width * height;
  const int64_t batch = std::max<int64_t>(1, ((int64_t)1 << 28) / pix);
  lvba::DevBuf<double> d_cams, d_ts, d_Xw;
  lvba::DevBuf<float> d_depth, d_uv;
  lvba::DevBuf<int64_t> d_kp;
  lvba::DevBuf<uint8_t> d_valid;
  lvba::StreamDrain drain(nullptr);
  int64_t h2d = 0, d2h = 0, pairs = 0, chunks = 0;
  float ms_dev = 0.f;
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  const cudaEvent_t e0 = ev.a, e1 = ev.b;
  int rc = LVBA_OK;
  for (int64_t k0 = 0; k0 < n_images && rc == LVBA_OK; k0 += batch) {
    const int64_t nb = std::min<int64_t>(batch, n_images - k0);
    const int64_t q0 = kp_ptr[k0], nq = kp_ptr[k0 + nb] - q0;
    LVBA_TRY(d_cams.upload(cams + 12 * k0, (size_t)nb * 12, ex.stream, &h2d));
    LVBA_TRY(d_ts.upload(image_ts + k0, (size_t)nb, ex.stream, &h2d));
    LVBA_TRY(d_kp.upload(kp_ptr + k0, (size_t)nb + 1, ex.stream, &h2d));
    if (nq > 0) LVBA_TRY(d_uv.upload(kp_uv + 2 * q0, (size_t)nq * 2, ex.stream, &h2d));
    if (d_depth.n < (size_t)(nb * pix)) LVBA_TRY(d_depth.alloc((size_t)(nb * pix)));
    if (d_Xw.n < (size_t)nq * 3) LVBA_TRY(d_Xw.alloc((size_t)nq * 3));
    if (d_valid.n < (size_t)nq) LVBA_TRY(d_valid.alloc((size_t)nq));
    LVBA_CUDA(cudaEventRecord(e0, ex.stream));
    rc = G.render(nb, d_cams.p, d_ts.p, half_window, intr, width, height, d_depth.p);
    if (rc == LVBA_OK && nq > 0) rc = G.backproject(nb, d_depth.p, d_cams.p, intr, width, height, d_kp.p, nq, d_uv.p, d_Xw.p, d_valid.p);
    if (rc != LVBA_OK) break;
    LVBA_CUDA(cudaEventRecord(e1, ex.stream));
    if (nq > 0) {
      LVBA_CUDA(cudaMemcpyAsync(Xw + 3 * q0, d_Xw.p, (size_t)nq * 3 * sizeof(double), cudaMemcpyDeviceToHost, ex.stream));
      LVBA_CUDA(cudaMemcpyAsync(valid + q0, d_valid.p, (size_t)nq, cudaMemcpyDeviceToHost, ex.stream));
    }
    LVBA_CUDA(cudaStreamSynchronize(ex.stream));
    float ms = 0.f;
    LVBA_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    ms_dev += ms; d2h += nq * 25; pairs += G.last_pairs; chunks += G.last_chunks;
  }
  ex.temp.release();
  if (rc != LVBA_OK) return rc;
  if (summary) {
    *summary = g->sum;
    summary->ms_device = ms_dev; summary->ms_upload = 0.0;
    summary->ms_total = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
    summary->kernel_launches = ex.launches - launches0; summary->h2d_bytes = h2d; summary->d2h_bytes = d2h;
    summary->work_pairs = pairs; summary->work_chunks = chunks;
  }
  return LVBA_OK;
} LVBA_ABI_END("lvba_depth_backproject")

int lvba_depth_grid_destroy(lvba_depth_grid* g) LVBA_ABI_BEGIN {
  if (!g) return LVBA_OK;
  cudaSetDevice(g->device);
  delete g;
  return LVBA_OK;
} LVBA_ABI_END("lvba_depth_grid_destroy")

}  // extern "C"
