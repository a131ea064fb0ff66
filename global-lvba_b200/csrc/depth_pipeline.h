// depth_pipeline.h — depth rendering from the world point grid (SURVEY.md §8f N3, first half; boundary B4):
//   buildGridMapFromOptimized   src/lvba_system.cpp:1266-1338
//   generateDepthWithVoxel      src/lvba_system.cpp:835-919      (projectCameraToPixel / distortNormalized, include/utils.hpp:169-197)
//
// The reference keeps an unordered_map<VOXEL_LOC, vector<Vector3d>> of ALL world points in 0.5 m voxels plus one
// std::set of voxels per LiDAR frame; an image renders every point of every voxel touched by a frame within +-0.5 s of
// its timestamp, through a per-pixel `if (d == 0 || Z < d) d = (float)Z`.  That z-buffer is float(min Z) whatever the
// order, so on the device it is an atomicMin on the float's bit pattern and the images are reproducible bit for bit.
//
//   grid    G1  world point + voxel key per point                  G2  radix sort by packed key -> points grouped by voxel
//           G3  voxel table (run heads), points gathered in order  G4  unique (voxel, frame) pairs with the PREVIOUS frame
//           touching the same voxel (so that a voxel seen by several frames of a window is rendered once), regrouped by frame
//   render  R1  frame window of every image -> a contiguous pair range        R2  64-point chunks of the pairs that are
//           first in their window (two-level load-balanced expansion)          R3  splat: project, truncate, atomicMin
//           R4  finalize: untouched pixels -> 0
//
// Written against the same Exec policy as voxel_pipeline.h: CUDA in depth_api.cuh, a sequential host policy in
// tests/emu/ for the no-GPU suite.  All arithmetic that decides a pixel goes through mul_/add_ (never an FMA).
#pragma once
#include <stdint.h>
#include <string.h>

#include "voxel_pipeline.h"

namespace lvba {
namespace depth {

using vox::add_;
using vox::mul_;
using vox::KeyPacking;

constexpr int kChunk = 64;                      // points per splat work item
constexpr uint32_t kEmpty = 0x7f800000u;        // +inf: larger than any depth

LVBA_HD uint32_t float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
LVBA_HD float bits_float(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  float f; memcpy(&f, &u, 4); return f;
#endif
}
LVBA_HD void atomic_min_u32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
  atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}
LVBA_HD bool finite_(double x) { return fabs(x) <= 1.79769313486231570e308; }

// y = A x + b with A row-major 3x3 in m[0..8], b in m[9..11]; each coefficient (a0 x0 + a1 x1) + a2 x2, then + b
LVBA_HD void affine3(const double* m, const double* x, double* y) {
  for (int k = 0; k < 3; ++k)
    y[k] = add_(add_(add_(mul_(m[3 * k], x[0]), mul_(m[3 * k + 1], x[1])), mul_(m[3 * k + 2], x[2])), m[9 + k]);
}

// projectCameraToPixel / projectWorldToPixel (include/utils.hpp:169-205) for one world point: false when the point is not in
// front of the camera or an intermediate is non-finite, else the distorted pixel (uu, vv) and the camera depth Z.  Shared by the
// depth z-buffer (B4) and the colour z-buffer (B8, color_pipeline.h), which differ only in the gate on Z and the pixel rounding.
LVBA_HD bool project_uv(const double* cam, const double* intr, const double* pw, double* u_out, double* v_out, double* Z_out) {
  double pc[3];
  affine3(cam, pw, pc);
  const double Z = pc[2];
  if (!(finite_(pc[0]) && finite_(pc[1]) && finite_(pc[2])) || !(Z > 1e-12)) return false;   // utils.hpp:186-188
  const double x = pc[0] / Z, y = pc[1] / Z;
  if (!(finite_(x) && finite_(y))) return false;
  const double fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3], k1 = intr[4], k2 = intr[5], p1 = intr[6], p2 = intr[7];
  const double r2 = add_(mul_(x, x), mul_(y, y));                             // utils.hpp:173-179
  const double r4 = mul_(r2, r2);
  const double radial = add_(add_(1.0, mul_(k1, r2)), mul_(k2, r4));
  const double x_tan = add_(mul_(mul_(mul_(2.0, p1), x), y), mul_(p2, add_(r2, mul_(mul_(2.0, x), x))));
  const double y_tan = add_(mul_(p1, add_(r2, mul_(mul_(2.0, y), y))), mul_(mul_(mul_(2.0, p2), x), y));
  const double xd = add_(mul_(x, radial), x_tan), yd = add_(mul_(y, radial), y_tan);
  if (!(finite_(xd) && finite_(yd))) return false;
  const double uu = add_(mul_(fx, xd), cx), vv = add_(mul_(fy, yd), cy);      // utils.hpp:193-194
  if (!(finite_(uu) && finite_(vv))) return false;
  *u_out = uu; *v_out = vv; *Z_out = Z;
  return true;
}

// generateDepthWithVoxel's inner loop (:885-901) for one world point: returns the pixel index or -1, and (float)Z.
LVBA_HD int64_t project_pixel(const double* cam, const double* intr, int width, int height, const double* pw, float* zf) {
  double uu, vv, Z;
  if (!project_uv(cam, intr, pw, &uu, &vv, &Z) || Z < 1e-3) return -1;      // :889 (a pure rejection, so its place is free)
  if (!(fabs(uu) < 2147483648.0 && fabs(vv) < 2147483648.0)) return -1;       // the (int) cast below is only defined in range
  const int u = (int)uu, v = (int)vv;                                          // :894-895 truncation toward zero
  if (u < 0 || u >= width || v < 0 || v >= height) return -1;
  *zf = (float)Z;
  return (int64_t)v * width + u;
}

// upper_bound / lower_bound over ascending doubles
LVBA_HD int lower_bound_f64(const double* a, int n, double x) { int lo = 0, hi = n; while (lo < hi) { const int m = (lo + hi) >> 1; if (a[m] < x) lo = m + 1; else hi = m; } return lo; }
LVBA_HD int upper_bound_f64(const double* a, int n, double x) { int lo = 0, hi = n; while (lo < hi) { const int m = (lo + hi) >> 1; if (a[m] <= x) lo = m + 1; else hi = m; } return lo; }
// last index i in [0, n) with off[i] <= x (off ascending, off[0] <= x)
LVBA_HD int64_t owner_i64(const int64_t* off, int64_t n, int64_t x) { int64_t lo = 0, hi = n; while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (off[m] <= x) lo = m; else hi = m; } return lo; }

// ================================================================ grid passes
struct GridPointF {          // G1
  const float* xyz; const int64_t* scan_ptr; const double* poses; int F; double voxel_size;
  int32_t* frame_of; double* pw; int32_t* kx; int32_t* ky; int32_t* kz; int32_t* bad;
  LVBA_HD void operator()(int64_t i) const {
    int lo = 0, hi = F;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (scan_ptr[mid] <= i) lo = mid; else hi = mid; }
    frame_of[i] = lo;
    double w[3];
    vox::world_point(poses + 12 * (int64_t)lo, xyz + 3 * i, w);               // :1284-1286
    int64_t k[3] = {0, 0, 0};
    bool ok = true;
    for (int a = 0; a < 3; ++a) { pw[3 * i + a] = w[a]; ok = vox::root_key_axis(w[a], voxel_size, &k[a]) && ok; }   // :1287-1291
    if (!ok) { *bad = 1; k[0] = k[1] = k[2] = 0; }
    kx[i] = (int32_t)k[0]; ky[i] = (int32_t)k[1]; kz[i] = (int32_t)k[2];
  }
};
struct GridKeyF {            // G2
  const int32_t* kx; const int32_t* ky; const int32_t* kz; KeyPacking pk; uint64_t* key; uint32_t* idx;
  LVBA_HD void operator()(int64_t i) const { const int64_t k[3] = {kx[i], ky[i], kz[i]}; key[i] = pk.pack(k); idx[i] = (uint32_t)i; }
};
struct HeadF {               // run heads over [0, n] (terminator 0)
  const uint64_t* key; int64_t n; uint32_t* flag;
  LVBA_HD void operator()(int64_t r) const { flag[r] = (r < n && (r == 0 || key[r] != key[r - 1])) ? 1u : 0u; }
};
struct GridGatherF {         // G3, over [0, N]
  const uint32_t* idx; const uint32_t* flag; const uint32_t* pos; const double* pw_in; const int32_t* frame_of; int64_t N; int F;
  uint32_t* vox_start; double* pw; uint64_t* pair_key; uint32_t* pair_idx;
  LVBA_HD void operator()(int64_t r) const {
    if (r == N) { vox_start[pos[N]] = (uint32_t)N; return; }
    const uint32_t rank = pos[r] + flag[r] - 1u;
    if (flag[r]) vox_start[rank] = (uint32_t)r;
    const int64_t i = idx[r];
    for (int a = 0; a < 3; ++a) pw[3 * r + a] = pw_in[3 * i + a];
    pair_key[r] = (uint64_t)rank * (uint64_t)F + (uint64_t)frame_of[i];
    pair_idx[r] = (uint32_t)r;
  }
};
struct PairScatterF {        // G4a, over the sorted (voxel, frame) keys: unique pairs, with the previous frame of the same voxel
  const uint64_t* key; const uint32_t* flag; const uint32_t* pos; int64_t n; int F;
  uint64_t* frame_key; uint32_t* order; uint32_t* vox_of; int32_t* prev_of;
  LVBA_HD void operator()(int64_t r) const {
    if (!flag[r]) return;
    const uint32_t j = pos[r];
    const uint64_t v = key[r] / (uint64_t)F, f = key[r] % (uint64_t)F;
    int32_t prev = -1;
    if (r > 0) { const uint64_t pv = key[r - 1] / (uint64_t)F; if (pv == v) prev = (int32_t)(key[r - 1] % (uint64_t)F); }
    frame_key[j] = f; order[j] = j; vox_of[j] = (uint32_t)v; prev_of[j] = prev;
  }
};
struct PairRegroupF {        // G4b: pairs in (frame, voxel) order
  const uint32_t* order; const uint32_t* vox_of; const int32_t* prev_of; uint32_t* pair_vox; int32_t* pair_prev;
  LVBA_HD void operator()(int64_t j) const { pair_vox[j] = vox_of[order[j]]; pair_prev[j] = prev_of[order[j]]; }
};
struct FramePairF {          // G4c, over [0, F]: first pair of every frame
  const uint64_t* frame_key_sorted; int64_t np; uint32_t* frame_pair;
  LVBA_HD void operator()(int64_t f) const { frame_pair[f] = (uint32_t)vox::lower_bound_u64(frame_key_sorted, np, (uint64_t)f); }
};

// ================================================================ render passes
struct ImageRangeF {         // R1, over [0, n_img] (terminator 0)
  const double* image_ts; const double* frame_ts; int F; double half_window; const uint32_t* frame_pair; int64_t n_img;
  int32_t* f_lo; int64_t* pair_lo; int64_t* count;
  LVBA_HD void operator()(int64_t k) const {
    if (k == n_img) { count[k] = 0; return; }
    const double t = image_ts[k];
    int fl = 0, fr = 0;
    if (finite_(t)) { fl = lower_bound_f64(frame_ts, F, t - half_window); fr = upper_bound_f64(frame_ts, F, t + half_window); }   // :1316-1319
    if (fr < fl) fr = fl;
    f_lo[k] = fl; pair_lo[k] = frame_pair[fl]; count[k] = (int64_t)frame_pair[fr] - (int64_t)frame_pair[fl];
  }
};
struct PairChunksF {         // R2, over [0, T1] (terminator 0)
  const int64_t* off1; int64_t n_img; int64_t T1; const int32_t* f_lo; const int64_t* pair_lo;
  const int32_t* pair_prev; const uint32_t* pair_vox; const uint32_t* vox_start; int64_t* chunks;
  LVBA_HD void operator()(int64_t t) const {
    if (t == T1) { chunks[t] = 0; return; }
    const int64_t k = owner_i64(off1, n_img + 1, t);
    const int64_t j = pair_lo[k] + (t - off1[k]);
    int64_t c = 0;
    if (pair_prev[j] < f_lo[k]) {                          // no earlier frame of this window touches the voxel: render it here
      const uint32_t v = pair_vox[j];
      c = ((int64_t)(vox_start[v + 1] - vox_start[v]) + kChunk - 1) / kChunk;
    }
    chunks[t] = c;
  }
};
struct CopyF64F { const double* src; double* dst; LVBA_HD void operator()(int64_t i) const { dst[i] = src[i]; } };
struct FillU32F { uint32_t* p; uint32_t v; LVBA_HD void operator()(int64_t i) const { p[i] = v; } };
struct SplatF {              // R3, over the T2 chunks
  const int64_t* off2; int64_t T1; const int64_t* off1; int64_t n_img; const int64_t* pair_lo; const uint32_t* pair_vox;
  const uint32_t* vox_start; const double* pw; const double* cams; double intr[8]; int width; int height; uint32_t* depth_bits;
  LVBA_HD void operator()(int64_t c) const {
    const int64_t t = owner_i64(off2, T1 + 1, c);
    const int64_t k = owner_i64(off1, n_img + 1, t);
    const uint32_t v = pair_vox[pair_lo[k] + (t - off1[k])];
    const int64_t first = (int64_t)vox_start[v] + (c - off2[t]) * kChunk;
    int64_t last = first + kChunk;
    if (last > (int64_t)vox_start[v + 1]) last = vox_start[v + 1];
    const double* cam = cams + 12 * k;
    uint32_t* img = depth_bits + k * (int64_t)width * height;
    for (int64_t r = first; r < last; ++r) {
      float zf;
      const int64_t pix = project_pixel(cam, intr, width, height, pw + 3 * r, &zf);
      if (pix >= 0) atomic_min_u32(img + pix, float_bits(zf));               // `if (d == 0 || Z < d) d = (float)Z`  :898-899
    }
  }
};
struct FinalizeF {           // R4 (bits and depth are the same words)
  const uint32_t* bits; float* depth;
  LVBA_HD void operator()(int64_t i) const { const uint32_t b = bits[i]; depth[i] = b == kEmpty ? 0.0f : bits_float(b); }
};

// ---------------------------------------------------------------- depth-fused 3-D candidates of the track fusion
// BuildTracksAndFuse3D, src/lvba_system.cpp:1020-1038, for one keypoint of one image:
//   fetchDepthBilinear (include/utils.hpp:246-275, float arithmetic)  ->  backProjectPixelDepthDistorted (:235-243,
//   undistortPixelToNormalized :207-233: 8 fixed-point iterations)    ->  camToWorld (:277-283)
LVBA_HD bool fetch_depth_bilinear(const float* depth, int w, int h, float u, float v, float* d_out) {
  if (!(u >= 0.0f) || !(v >= 0.0f) || u >= (float)(w - 1) || v >= (float)(h - 1)) return false;     // (a NaN pixel is refused too)
  const int x = (int)floorf(u), y = (int)floorf(v);
  const float du = vox::fadd_(u, -(float)x), dv = vox::fadd_(v, -(float)y);
  const float d00 = depth[(int64_t)y * w + x], d10 = depth[(int64_t)y * w + x + 1];
  const float d01 = depth[(int64_t)(y + 1) * w + x], d11 = depth[(int64_t)(y + 1) * w + x + 1];
  if (d00 <= 0 || d10 <= 0 || d01 <= 0 || d11 <= 0) return false;
  const float omu = vox::fadd_(1.0f, -du), omv = vox::fadd_(1.0f, -dv);
  const float a = vox::fmul_(vox::fmul_(omu, omv), d00), b = vox::fmul_(vox::fmul_(du, omv), d10);
  const float c = vox::fmul_(vox::fmul_(omu, dv), d01), e = vox::fmul_(vox::fmul_(du, dv), d11);
  *d_out = vox::fadd_(vox::fadd_(vox::fadd_(a, b), c), e);
  return *d_out > 0.0f;
}
LVBA_HD bool undistort_pixel(const double* intr, double u, double v, double* x, double* y) {
  const double fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3], k1 = intr[4], k2 = intr[5], p1 = intr[6], p2 = intr[7];
  if (!finite_(u) || !finite_(v)) return false;
  if (fabs(fx) < 1e-12 || fabs(fy) < 1e-12) return false;
  const double xd = vox::sub_(u, cx) / fx, yd = vox::sub_(v, cy) / fy;
  double xu = xd, yu = yd;
  for (int it = 0; it < 8; ++it) {
    const double r2 = add_(mul_(xu, xu), mul_(yu, yu));
    const double r4 = mul_(r2, r2);
    const double radial = add_(add_(1.0, mul_(k1, r2)), mul_(k2, r4));
    if (fabs(radial) < 1e-12 || !finite_(radial)) return false;
    const double x_tan = add_(mul_(mul_(mul_(2.0, p1), xu), yu), mul_(p2, add_(r2, mul_(mul_(2.0, xu), xu))));
    const double y_tan = add_(mul_(p1, add_(r2, mul_(mul_(2.0, yu), yu))), mul_(mul_(mul_(2.0, p2), xu), yu));
    xu = vox::sub_(xd, x_tan) / radial;
    yu = vox::sub_(yd, y_tan) / radial;
    if (!finite_(xu) || !finite_(yu)) return false;
  }
  *x = xu; *y = yu;
  return true;
}
struct BackprojectF {        // over the keypoints of the images of one batch
  const float* depth; const double* cams; double intr[8]; int width; int height;
  const int64_t* kp_ptr; int64_t n_img; const float* kp_uv; double* Xw; uint8_t* valid;
  LVBA_HD void operator()(int64_t q) const {
    valid[q] = 0; Xw[3 * q] = 0.0; Xw[3 * q + 1] = 0.0; Xw[3 * q + 2] = 0.0;                  // points3d[t] = Zero, valid_mask[t] = 0
    const int64_t k = owner_i64(kp_ptr, n_img + 1, q + kp_ptr[0]);
    const float u = kp_uv[2 * q], v = kp_uv[2 * q + 1];
    float d;
    if (!fetch_depth_bilinear(depth + k * (int64_t)width * height, width, height, u, v, &d)) return;   // :1030
    if (d <= 0.0f) return;                                                                      // :1031
    const double dd = (double)d;
    double x, y;
    if (!(dd > 0.0) || !finite_(dd) || !undistort_pixel(intr, (double)u, (double)v, &x, &y)) return;
    const double Xc[3] = {mul_(x, dd), mul_(y, dd), dd};
    if (!(finite_(Xc[0]) && finite_(Xc[1]) && finite_(Xc[2]))) return;
    const double* R = cams + 12 * k;
    const double* t = R + 9;
    for (int i = 0; i < 3; ++i) {                                                               // camToWorld: Rwc = Rcw^T, twc = -(Rwc tcw)
      const double twc = -add_(add_(mul_(R[i], t[0]), mul_(R[3 + i], t[1])), mul_(R[6 + i], t[2]));
      Xw[3 * q + i] = add_(add_(add_(mul_(R[i], Xc[0]), mul_(R[3 + i], Xc[1])), mul_(R[6 + i], Xc[2])), twc);
    }
    valid[q] = 1;
  }
};

// ================================================================ the grid
template <class Exec>
struct DepthGrid {
  Exec ex;
  int F = 0;
  int64_t N = 0, n_voxels = 0, n_pairs = 0;
  double voxel_size = 0.5;
  KeyPacking pk{};
  typename Exec::template Buf<double> pw;            // [N*3] world points, grouped by voxel
  typename Exec::template Buf<uint32_t> vox_start;   // [n_voxels + 1]
  typename Exec::template Buf<uint32_t> pair_vox;    // [n_pairs] in (frame, voxel) order
  typename Exec::template Buf<int32_t> pair_prev;    // [n_pairs] previous frame touching the voxel, -1
  typename Exec::template Buf<uint32_t> frame_pair;  // [F + 1]
  typename Exec::template Buf<double> frame_ts;      // [F]
  int64_t last_pairs = 0, last_chunks = 0;           // work of the last render call
  const char* error = "";

  // xyz [N*3], scan_ptr [F+1], poses [F*12], ts [F] ascending: pointers the Exec's passes can dereference
  int build(const float* xyz, const int64_t* scan_ptr, const double* poses, const double* ts, int F_, int64_t N_, double voxel_size_) {
    F = F_; N = N_; voxel_size = voxel_size_;
    n_voxels = 0; n_pairs = 0;
    pk = KeyPacking{{0, 0, 0}, {0, 0, 0}, 0, 0};
    LVBA_VOX_TRY(frame_ts.alloc((size_t)F));
    LVBA_VOX_TRY(ex.for_each((int64_t)F, CopyF64F{ts, frame_ts.p}));
    LVBA_VOX_TRY(frame_pair.alloc((size_t)F + 1));
    LVBA_VOX_TRY(ex.fill_zero(frame_pair.p, (size_t)F + 1));
    LVBA_VOX_TRY(vox_start.alloc(1));
    LVBA_VOX_TRY(ex.fill_zero(vox_start.p, 1));
    if (N == 0) return ex.sync();
    typename Exec::template Buf<int32_t> frame_of, kx, ky, kz, bad;
    typename Exec::template Buf<double> pw_in;
    LVBA_VOX_TRY(frame_of.alloc((size_t)N)); LVBA_VOX_TRY(pw_in.alloc((size_t)N * 3));
    LVBA_VOX_TRY(kx.alloc((size_t)N)); LVBA_VOX_TRY(ky.alloc((size_t)N)); LVBA_VOX_TRY(kz.alloc((size_t)N));
    LVBA_VOX_TRY(bad.alloc(1));
    LVBA_VOX_TRY(ex.fill_zero(bad.p, 1));
    LVBA_VOX_TRY(ex.for_each(N, GridPointF{xyz, scan_ptr, poses, F, voxel_size, frame_of.p, pw_in.p, kx.p, ky.p, kz.p, bad.p}));
    int32_t h_bad = 0;
    LVBA_VOX_TRY(ex.fetch(&h_bad, bad.p, 1));
    if (h_bad) { error = "a point is non-finite or more than 2^30 grid voxels from the origin"; return vox::kErrInvalid; }
    const int32_t* axis[3] = {kx.p, ky.p, kz.p};
    for (int a = 0; a < 3; ++a) {
      int32_t mn = 0, mx = 0;
      LVBA_VOX_TRY(ex.min_max(axis[a], N, &mn, &mx));
      pk.mn[a] = mn;
      pk.bits[a] = vox::bit_length((uint64_t)((int64_t)mx - (int64_t)mn));
    }
    pk.root_bits = pk.bits[0] + pk.bits[1] + pk.bits[2];
    if (pk.root_bits > 62) { error = "grid voxel keys span more than 62 bits"; return vox::kErrUnsupported; }
    typename Exec::template Buf<uint64_t> key, key_s;
    typename Exec::template Buf<uint32_t> idx, idx_s, flag, pos;
    LVBA_VOX_TRY(key.alloc((size_t)N)); LVBA_VOX_TRY(key_s.alloc((size_t)N));
    LVBA_VOX_TRY(idx.alloc((size_t)N)); LVBA_VOX_TRY(idx_s.alloc((size_t)N));
    LVBA_VOX_TRY(ex.for_each(N, GridKeyF{kx.p, ky.p, kz.p, pk, key.p, idx.p}));
    LVBA_VOX_TRY(ex.sort_pairs(key.p, key_s.p, idx.p, idx_s.p, N, pk.root_bits > 0 ? pk.root_bits : 1));
    LVBA_VOX_TRY(flag.alloc((size_t)N + 1)); LVBA_VOX_TRY(pos.alloc((size_t)N + 1));
    LVBA_VOX_TRY(ex.for_each(N + 1, HeadF{key_s.p, N, flag.p}));
    LVBA_VOX_TRY(ex.exclusive_scan(flag.p, pos.p, N + 1));
    uint32_t nv = 0;
    LVBA_VOX_TRY(ex.fetch(&nv, pos.p + N, 1));
    n_voxels = nv;
    if ((uint64_t)nv * (uint64_t)F >= ((uint64_t)1 << 62)) { error = "voxel x frame table too large"; return vox::kErrUnsupported; }
    LVBA_VOX_TRY(vox_start.alloc((size_t)nv + 1));
    LVBA_VOX_TRY(pw.alloc((size_t)N * 3));
    // key / idx are reused for the (voxel, frame) pair keys
    LVBA_VOX_TRY(ex.for_each(N + 1, GridGatherF{idx_s.p, flag.p, pos.p, pw_in.p, frame_of.p, N, F, vox_start.p, pw.p, key.p, idx.p}));
    const int pair_bits = vox::bit_length((uint64_t)nv * (uint64_t)F);
    LVBA_VOX_TRY(ex.sort_pairs(key.p, key_s.p, idx.p, idx_s.p, N, pair_bits > 0 ? pair_bits : 1));
    LVBA_VOX_TRY(ex.for_each(N + 1, HeadF{key_s.p, N, flag.p}));
    LVBA_VOX_TRY(ex.exclusive_scan(flag.p, pos.p, N + 1));
    uint32_t np = 0;
    LVBA_VOX_TRY(ex.fetch(&np, pos.p + N, 1));
    n_pairs = np;
    typename Exec::template Buf<uint64_t> fkey, fkey_s;
    typename Exec::template Buf<uint32_t> order, order_s, vox_of;
    typename Exec::template Buf<int32_t> prev_of;
    LVBA_VOX_TRY(fkey.alloc(np)); LVBA_VOX_TRY(fkey_s.alloc(np)); LVBA_VOX_TRY(order.alloc(np)); LVBA_VOX_TRY(order_s.alloc(np));
    LVBA_VOX_TRY(vox_of.alloc(np)); LVBA_VOX_TRY(prev_of.alloc(np));
    LVBA_VOX_TRY(ex.for_each(N, PairScatterF{key_s.p, flag.p, pos.p, N, F, fkey.p, order.p, vox_of.p, prev_of.p}));
    const int fbits = vox::bit_length((uint64_t)(F > 0 ? F - 1 : 0));
    LVBA_VOX_TRY(ex.sort_pairs(fkey.p, fkey_s.p, order.p, order_s.p, np, fbits > 0 ? fbits : 1));
    LVBA_VOX_TRY(pair_vox.alloc(np)); LVBA_VOX_TRY(pair_prev.alloc(np));
    LVBA_VOX_TRY(ex.for_each(np, PairRegroupF{order_s.p, vox_of.p, prev_of.p, pair_vox.p, pair_prev.p}));
    LVBA_VOX_TRY(ex.for_each((int64_t)F + 1, FramePairF{fkey_s.p, np, frame_pair.p}));
    return ex.sync();
  }

  // cams [n_img*12] (Rcw row-major, tcw), image_ts [n_img], depth [n_img*height*width] floats: Exec-dereferenceable
  int render(int64_t n_img, const double* cams, const double* image_ts, double half_window, const double intr[8], int width,
             int height, float* depth) {
    last_pairs = 0; last_chunks = 0;
    if (n_img <= 0) return 0;
    const int64_t n_pix = n_img * (int64_t)width * height;
    uint32_t* const bits = reinterpret_cast<uint32_t*>(depth);      // the z-buffer of bit patterns lives in the output images
    LVBA_VOX_TRY(ex.for_each(n_pix, FillU32F{bits, kEmpty}));
    if (N > 0 && n_pairs > 0) {
      typename Exec::template Buf<int32_t> f_lo;
      typename Exec::template Buf<int64_t> pair_lo, count, off1;
      LVBA_VOX_TRY(f_lo.alloc((size_t)n_img)); LVBA_VOX_TRY(pair_lo.alloc((size_t)n_img));
      LVBA_VOX_TRY(count.alloc((size_t)n_img + 1)); LVBA_VOX_TRY(off1.alloc((size_t)n_img + 1));
      LVBA_VOX_TRY(ex.for_each(n_img + 1, ImageRangeF{image_ts, frame_ts.p, F, half_window, frame_pair.p, n_img, f_lo.p, pair_lo.p, count.p}));
      LVBA_VOX_TRY(ex.exclusive_scan(count.p, off1.p, n_img + 1));
      int64_t T1 = 0;
      LVBA_VOX_TRY(ex.fetch(&T1, off1.p + n_img, 1));
      last_pairs = T1;
      if (T1 > 0) {
        typename Exec::template Buf<int64_t> chunks, off2;
        LVBA_VOX_TRY(chunks.alloc((size_t)T1 + 1)); LVBA_VOX_TRY(off2.alloc((size_t)T1 + 1));
        LVBA_VOX_TRY(ex.for_each(T1 + 1, PairChunksF{off1.p, n_img, T1, f_lo.p, pair_lo.p, pair_prev.p, pair_vox.p, vox_start.p, chunks.p}));
        LVBA_VOX_TRY(ex.exclusive_scan(chunks.p, off2.p, T1 + 1));
        int64_t T2 = 0;
        LVBA_VOX_TRY(ex.fetch(&T2, off2.p + T1, 1));
        last_chunks = T2;
        SplatF sf{off2.p, T1, off1.p, n_img, pair_lo.p, pair_vox.p, vox_start.p, pw.p, cams, {}, width, height, bits};
        for (int q = 0; q < 8; ++q) sf.intr[q] = intr[q];
        LVBA_VOX_TRY(ex.for_each(T2, sf));
      }
    }
    LVBA_VOX_TRY(ex.for_each(n_pix, FinalizeF{bits, depth}));                // in place: every item reads and writes its own word
    return ex.sync();
  }

  // depth [n_img*height*width] as written by render(); kp_ptr [n_img+1] offsets into the caller's keypoint array (only
  // differences are used: kp_uv / Xw / valid point at the first keypoint of this batch); all Exec-dereferenceable
  int backproject(int64_t n_img, const float* depth, const double* cams, const double intr[8], int width, int height,
                  const int64_t* kp_ptr, int64_t n_kp, const float* kp_uv, double* Xw, uint8_t* valid) {
    BackprojectF f{depth, cams, {}, width, height, kp_ptr, n_img, kp_uv, Xw, valid};
    for (int q = 0; q < 8; ++q) f.intr[q] = intr[q];
    LVBA_VOX_TRY(ex.for_each(n_kp, f));
    return ex.sync();
  }
};

}  // namespace depth
}  // namespace lvba
