// color_api.cuh — boundary B8: the coloured LiDAR map of VisualizeOptComparison (src/lvba_system.cpp:1932-2143) on the device.
// Passes: color_pipeline.h; execution policy: CudaExec (exec.cuh).  No host path.
#pragma once
#include "color_pipeline.h"
#include "voxel_api.cuh"

struct lvba_colorizer {
  lvba::color::Colorizer<lvba::CudaExec> cz;
  int device = 0;
  std::vector<int64_t> scan_ptr;     // host copies: the batches are cut on the host
  std::vector<double> frame_ts;
  lvba::DevBuf<float> d_xyz;
  lvba::DevBuf<int64_t> d_scan;
  lvba::DevBuf<double> d_ts, d_poses;
  int state = 0;                     // 0 created / finished, 1 inside begin .. finish, 2 finished (export allowed)
  lvba_colorize_summary sum{};
  std::chrono::steady_clock::time_point t_begin;
  int64_t launches0 = 0;
  ~lvba_colorizer() { cudaStreamSynchronize(cz.ex.stream); }     // members are parked in the pool after this body: they must be idle
};

namespace lvba {
constexpr int64_t kColorBatchItems = (int64_t)1 << 26;      // (image, window point) items per device batch: ~2 GB of scratch
constexpr int64_t kColorBatchRgb = (int64_t)1 << 28;        // image bytes per device batch
}  // namespace lvba

extern "C" {

int lvba_colorizer_create(int32_t n_frames, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats,
                          const double* frame_ts, int32_t device, lvba_colorizer** out) LVBA_ABI_BEGIN {
  if (!out) return lvba::fail(LVBA_ERR_INVALID_ARG, "null output handle");
  *out = nullptr;
  if (n_frames < 0 || !scan_ptr || (n_frames > 0 && !frame_ts)) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative frame count");
  if (xyz_stride_floats < 3) return lvba::fail(LVBA_ERR_INVALID_ARG, "xyz_stride %d < 3 floats", xyz_stride_floats);
  if (scan_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "scan_ptr[0] != 0");
  for (int32_t j = 0; j < n_frames; ++j)
    if (scan_ptr[j + 1] < scan_ptr[j]) return lvba::fail(LVBA_ERR_INVALID_ARG, "scan_ptr not monotone at frame %d", j);
  const int64_t N = scan_ptr[n_frames];
  if (N >= (int64_t)0xfffffff0ll) return lvba::fail(LVBA_ERR_UNSUPPORTED, "%lld points: more than 2^32", (long long)N);
  if (N > 0 && !xyz) return lvba::fail(LVBA_ERR_INVALID_ARG, "null xyz");
  LVBA_TRY(lvba::select_device(device));
  std::unique_ptr<lvba_colorizer> h(new lvba_colorizer());
  cudaGetDevice(&h->device);
  lvba::CudaExec& ex = h->cz.ex;
  lvba::StreamDrain drain(nullptr);      // every path of this handle runs on the NULL stream
  h->scan_ptr.assign(scan_ptr, scan_ptr + n_frames + 1);
  h->frame_ts.assign(frame_ts, frame_ts + n_frames);
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
  int64_t h2d = 0;
  LVBA_TRY(h->d_xyz.upload(src, (size_t)N * 3, ex.stream, &h2d));
  LVBA_TRY(h->d_scan.upload(scan_ptr, (size_t)n_frames + 1, ex.stream, &h2d));
  LVBA_TRY(h->d_ts.upload(frame_ts, (size_t)n_frames, ex.stream, &h2d));
  LVBA_CUDA(cudaStreamSynchronize(ex.stream));
  h->cz.setup(h->d_xyz.p, h->d_scan.p, h->d_ts.p, n_frames, N);
  h->sum.n_points = N;
  h->sum.h2d_bytes = h2d;
  *out = h.release();
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_create")

int lvba_colorizer_begin(lvba_colorizer* c, const double* frame_poses, double half_window, double leaf) LVBA_ABI_BEGIN {
  if (!c) return lvba::fail(LVBA_ERR_INVALID_ARG, "null handle");
  const int F = c->cz.F;
  if (F > 0 && !frame_poses) return lvba::fail(LVBA_ERR_INVALID_ARG, "null frame_poses");
  if (!(half_window >= 0.0) || !std::isfinite(half_window)) return lvba::fail(LVBA_ERR_INVALID_ARG, "half_window must be finite and >= 0");
  if (!(leaf >= 0.0) || !std::isfinite(leaf)) return lvba::fail(LVBA_ERR_INVALID_ARG, "leaf must be finite and >= 0");
  for (int64_t k = 0; k < (int64_t)F * 12; ++k)
    if (!std::isfinite(frame_poses[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite pose entry %lld", (long long)k);
  LVBA_CUDA(cudaSetDevice(c->device));
  lvba::CudaExec& ex = c->cz.ex;
  lvba::StreamDrain drain(nullptr);
  c->state = 0;
  c->t_begin = std::chrono::steady_clock::now();
  c->launches0 = ex.launches;
  const int64_t n_points = c->sum.n_points;
  c->sum = lvba_colorize_summary{};
  c->sum.n_points = n_points;
  LVBA_TRY(c->d_poses.upload(frame_poses, (size_t)F * 12, ex.stream, &c->sum.h2d_bytes));
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  LVBA_CUDA(cudaEventRecord(ev.a, ex.stream));
  const int rc = c->cz.begin(c->d_poses.p, half_window, leaf);
  if (rc != LVBA_OK) return c->cz.error[0] ? lvba::fail(rc, "%s", c->cz.error) : rc;
  LVBA_CUDA(cudaEventRecord(ev.b, ex.stream));
  LVBA_CUDA(cudaEventSynchronize(ev.b));
  float ms = 0.f;
  LVBA_CUDA(cudaEventElapsedTime(&ms, ev.a, ev.b));
  c->sum.ms_device += ms;
  ex.temp.release();
  c->state = 1;
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_begin")

int lvba_colorizer_add_images(lvba_colorizer* c, int32_t n_images, const double* image_ts, const double* cams, const double intr[8],
                              int32_t width, int32_t height, const uint8_t* rgb, uint8_t* listed) LVBA_ABI_BEGIN {
  if (!c) return lvba::fail(LVBA_ERR_INVALID_ARG, "null handle");
  if (c->state != 1) return lvba::fail(LVBA_ERR_INVALID_ARG, "add_images outside begin .. finish");
  if (n_images < 0 || !intr || (n_images > 0 && (!image_ts || !cams || !listed))) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative image count");
  if (width <= 0 || height <= 0 || (int64_t)width * height >= ((int64_t)1 << 31)) return lvba::fail(LVBA_ERR_INVALID_ARG, "image size %d x %d", width, height);
  for (int64_t k = 0; k < (int64_t)n_images * 12; ++k)
    if (!std::isfinite(cams[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite camera entry %lld", (long long)k);
  for (int k = 0; k < 8; ++k)
    if (!std::isfinite(intr[k])) return lvba::fail(LVBA_ERR_INVALID_ARG, "non-finite intrinsic %d", k);
  LVBA_CUDA(cudaSetDevice(c->device));
  auto& Z = c->cz;
  lvba::CudaExec& ex = Z.ex;
  lvba::StreamDrain drain(nullptr);
  const int F = Z.F;
  const int64_t n_pix = (int64_t)width * height, img_bytes = rgb ? n_pix * 3 : 0;
  std::vector<int64_t> items((size_t)n_images, 0);      // window points of every image (the rule of WindowCountF)
  for (int32_t k = 0; k < n_images; ++k)
    for (int f = 0; f < F; ++f)
      if (!(std::fabs(c->frame_ts[(size_t)f] - image_ts[k]) > Z.half_window)) items[(size_t)k] += c->scan_ptr[(size_t)f + 1] - c->scan_ptr[(size_t)f];
  lvba::DevBuf<double> d_cams, d_its;
  lvba::DevBuf<uint8_t> d_rgb, d_listed;
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  int32_t k0 = 0;
  while (k0 < n_images) {
    int32_t nb = 1;
    int64_t T = items[(size_t)k0];
    while (k0 + nb < n_images && T + items[(size_t)(k0 + nb)] <= lvba::kColorBatchItems && (int64_t)(nb + 1) * img_bytes <= lvba::kColorBatchRgb) {
      T += items[(size_t)(k0 + nb)]; ++nb;
    }
    LVBA_TRY(d_cams.upload(cams + 12 * (int64_t)k0, (size_t)nb * 12, ex.stream, &c->sum.h2d_bytes));
    LVBA_TRY(d_its.upload(image_ts + k0, (size_t)nb, ex.stream, &c->sum.h2d_bytes));
    if (rgb) LVBA_TRY(d_rgb.upload(rgb + (int64_t)k0 * img_bytes, (size_t)(nb * img_bytes), ex.stream, &c->sum.h2d_bytes));
    if (d_listed.n < (size_t)nb) LVBA_TRY(d_listed.alloc((size_t)nb));
    LVBA_CUDA(cudaEventRecord(ev.a, ex.stream));
    const int rc = Z.add_images(nb, d_its.p, d_cams.p, intr, width, height, rgb ? d_rgb.p : nullptr, d_listed.p);
    if (rc != LVBA_OK) { c->state = 0; return Z.error[0] ? lvba::fail(rc, "%s", Z.error) : rc; }
    LVBA_CUDA(cudaEventRecord(ev.b, ex.stream));
    LVBA_CUDA(cudaMemcpyAsync(listed + k0, d_listed.p, (size_t)nb, cudaMemcpyDeviceToHost, ex.stream));
    LVBA_CUDA(cudaStreamSynchronize(ex.stream));
    float ms = 0.f;
    LVBA_CUDA(cudaEventElapsedTime(&ms, ev.a, ev.b));
    c->sum.ms_device += ms;
    c->sum.d2h_bytes += nb;
    for (int32_t k = 0; k < nb; ++k) c->sum.n_listed += listed[k0 + k];
    const int64_t batch_bytes = (int64_t)(d_cams.n * 8 + d_its.n * 8 + d_rgb.n + d_listed.n);
    if (Z.peak_bytes + batch_bytes > c->sum.peak_device_bytes) c->sum.peak_device_bytes = Z.peak_bytes + batch_bytes;
    k0 += nb;
  }
  ex.temp.release();
  c->sum.n_images += n_images;
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_add_images")

int lvba_colorizer_finish(lvba_colorizer* c, int64_t* n_out, lvba_colorize_summary* summary) LVBA_ABI_BEGIN {
  if (!c) return lvba::fail(LVBA_ERR_INVALID_ARG, "null handle");
  if (c->state != 1) return lvba::fail(LVBA_ERR_INVALID_ARG, "finish without begin");
  LVBA_CUDA(cudaSetDevice(c->device));
  auto& Z = c->cz;
  lvba::CudaExec& ex = Z.ex;
  lvba::StreamDrain drain(nullptr);
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  LVBA_CUDA(cudaEventRecord(ev.a, ex.stream));
  const int rc = Z.finish();
  if (rc != LVBA_OK) { c->state = 0; return Z.error[0] ? lvba::fail(rc, "%s", Z.error) : rc; }
  LVBA_CUDA(cudaEventRecord(ev.b, ex.stream));
  LVBA_CUDA(cudaEventSynchronize(ev.b));
  float ms = 0.f;
  LVBA_CUDA(cudaEventElapsedTime(&ms, ev.a, ev.b));
  ex.temp.release();
  lvba_colorize_summary& s = c->sum;
  s.ms_device += ms;
  s.n_projections = Z.n_projections; s.n_landed = Z.n_landed; s.n_survivors = Z.n_merged; s.n_out = Z.n_out;
  s.kernel_launches = ex.launches - c->launches0;
  if (Z.peak_bytes > s.peak_device_bytes) s.peak_device_bytes = Z.peak_bytes;
  s.ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - c->t_begin).count();
  c->state = 2;
  if (n_out) *n_out = Z.n_out;
  if (summary) *summary = s;
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_finish")

int lvba_colorizer_export(lvba_colorizer* c, float* xyz, uint8_t* rgb) LVBA_ABI_BEGIN {
  if (!c) return lvba::fail(LVBA_ERR_INVALID_ARG, "null handle");
  if (c->state != 2) return lvba::fail(LVBA_ERR_INVALID_ARG, "export before finish");
  LVBA_CUDA(cudaSetDevice(c->device));
  auto& Z = c->cz;
  cudaStream_t s = Z.ex.stream;
  if (xyz && Z.n_out) LVBA_CUDA(cudaMemcpyAsync(xyz, Z.out_xyz(), (size_t)Z.n_out * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (rgb && Z.n_out) LVBA_CUDA(cudaMemcpyAsync(rgb, Z.out_rgb.p, (size_t)Z.n_out * 3, cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaStreamSynchronize(s));
  c->sum.d2h_bytes += (xyz ? Z.n_out * 12 : 0) + (rgb ? Z.n_out * 3 : 0);
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_export")

int lvba_colorizer_destroy(lvba_colorizer* c) LVBA_ABI_BEGIN {
  if (!c) return LVBA_OK;
  cudaSetDevice(c->device);
  delete c;
  return LVBA_OK;
} LVBA_ABI_END("lvba_colorizer_destroy")

}  // extern "C"
