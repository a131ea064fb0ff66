// color_pipeline.h — the coloured LiDAR map of VisualizeOptComparison (boundary B8), src/lvba_system.cpp:1932-2143:
//   per image k: the scans idx with |x_buf[idx].t - id| <= 0.5 (a linear scan over all frames, :1973-1977), each point moved to
//   the world as (float)(R p + t) (:1983-1990); a z-buffer over the image in cloud order (scan order, then point order):
//     projectWorldToPixel (include/utils.hpp:183-205); uu = round(u), vv = round(v); bounds;
//     if (zc + 1e-6f < zbuf[idx]) { zbuf[idx] = (float)zc; pix[idx] = point with the colour img(vv, uu) }      (:2037-2060)
//   the survivors appended to `merged` in pixel order (:2062-2069); after all images down_sampling_voxel2(merged, leaf)
//   (include/BALM/tools.hpp:301-359): per voxel the original point nearest the centre, the first in merged order on ties.
//
// The z-buffer rule is order dependent (the eps is about one float ulp at 10 m and the stored depth is the float-rounded Z), so
// it is not a minimum and not an atomicMin.  Here, per batch of images:
//   C1  window      one item per (image, frame): the frame's point count if it is in the image's window, else 0; scan -> offsets.
//                   The concatenation over (image, frame, point) is every image's cloud in the reference's order.
//   C2  project     one item per (image, window point): key = (image in batch, pixel) for the points that land in the image
//   C3  compact     the landed items, keeping their order; STABLE radix sort by key on the used bits only
//   C4  resolve     one thread per (image, pixel) run applies the reference's rule sequentially in cloud order
//   C5  emit        the survivors in (image, pixel) order — the reference's append order — with their colour, voxel key and d2
// and across batches the thinning is folded into a running table sorted by packed voxel key: the per-voxel choice (least d2, the
// earliest merged ordinal on ties) is associative, so pending survivors are merged into the table (a stable sort of table then
// pending by key and an arg-min per run) whenever they outnumber it.  Device memory is bounded by the scans, the table and one
// batch, never by the number of images.  The output is ascending (kx, ky, kz), x-major and signed: the std::map order of the host
// restatement colmap_points_from_lidar (host/lvba_visual_offline.hpp).
//
// Same Exec-policy scheme as anchor_pipeline.h / depth_pipeline.h: CUDA in color_api.cuh, a sequential host policy in tests/emu/.
// Every product and sum that decides a pixel or a distance goes through mul_/add_ (never an FMA).
#pragma once
#include <stdint.h>

#include "depth_pipeline.h"

namespace lvba {
namespace color {

using vox::add_;
using vox::KeyPacking;
using vox::mul_;

constexpr uint32_t kGrey = 0x808080u;               // (128, 128, 128) when no images are given
constexpr float kEps = 1e-6f;                       // `zc + 1e-6f < zbuf[idx]`  (:2050)

// (float)(R p + t) per coordinate.  A finite world point more than 2^30 leaf voxels from the origin sets `bad` (the anchor
// stage's rule); a non-finite one never lands in an image and is left out of the key range: lo = key or INT32_MAX, hi = key or
// INT32_MIN, per axis.
struct WorldPointF {
  const float* xyz; const int64_t* scan_ptr; const double* poses; int F; double leaf; bool thin;
  float* pw; int32_t* lo; int32_t* hi; int32_t* bad; int64_t N;
  LVBA_HD void operator()(int64_t i) const {
    int a = 0, b = F;
    while (b - a > 1) { const int m = (a + b) >> 1; if (scan_ptr[m] <= i) a = m; else b = m; }
    double w[3];
    vox::world_point(poses + 12 * (int64_t)a, xyz + 3 * i, w);                // :1983-1990
    bool finite = true;
    for (int c = 0; c < 3; ++c) { pw[3 * i + c] = (float)w[c]; finite = finite && depth::finite_((double)(float)w[c]); }
    for (int c = 0; c < 3; ++c) {
      int64_t k = 0;
      bool ok = finite;
      if (thin && finite && !vox::root_key_axis((double)pw[3 * i + c], leaf, &k)) { *bad = 1; ok = false; }
      lo[c * N + i] = ok ? (int32_t)k : INT32_MAX;
      hi[c * N + i] = ok ? (int32_t)k : INT32_MIN;
    }
  }
};

// C1 over [0, nb*F]: point count of frame f in the window of image k (terminator 0).  `!(fabs(t - id) > hw)` as at :1975.
struct WindowCountF {
  const double* image_ts; const double* frame_ts; const int64_t* scan_ptr; int F; int64_t nb; double half_window; int64_t* count;
  LVBA_HD void operator()(int64_t q) const {
    if (q == nb * F) { count[q] = 0; return; }
    const int64_t k = q / F; const int f = (int)(q % F);
    count[q] = !(fabs(frame_ts[f] - image_ts[k]) > half_window) ? scan_ptr[f + 1] - scan_ptr[f] : 0;
  }
};
struct ListedF {             // over [0, nb]: the image has LiDAR in its window (:1993-1996)
  const int64_t* off; int F; uint8_t* listed;
  LVBA_HD void operator()(int64_t k) const { listed[k] = off[(k + 1) * F] > off[k * F] ? 1 : 0; }
};

// (image in batch, point index) of window item t
LVBA_HD void locate(const int64_t* off, int64_t nb, int F, const int64_t* scan_ptr, int64_t t, int64_t* k_out, int64_t* p_out) {
  const int64_t q = depth::owner_i64(off, nb * F + 1, t);    // last (image, frame) slot starting at or before t (empty slots skipped)
  const int64_t k = q / F; const int f = (int)(q % F);
  *k_out = k; *p_out = scan_ptr[f] + (t - off[q]);
}

// The reference's pixel of one world point: rounded projection (round half away from zero), bounds; -1 if none.
LVBA_HD int64_t project_round(const double* cam, const double* intr, int width, int height, const float* p, double* Z) {
  const double pw[3] = {(double)p[0], (double)p[1], (double)p[2]};
  double u, v;
  if (!depth::project_uv(cam, intr, pw, &u, &v, Z)) return -1;
  const double ur = round(u), vr = round(v);
  if (!(fabs(ur) < 2147483648.0 && fabs(vr) < 2147483648.0)) return -1;      // the (int) cast is only defined in range
  const int uu = (int)ur, vv = (int)vr;
  if (uu < 0 || uu >= width || vv < 0 || vv >= height) return -1;
  return (int64_t)vv * width + uu;
}

struct ProjectF {            // C2, over the T window items
  const int64_t* off; int64_t nb; int F; const int64_t* scan_ptr; const float* pw; const double* cams; double intr[8];
  int width; int height; int pix_bits; uint64_t* key; double* z; uint32_t* flag;
  LVBA_HD void operator()(int64_t t) const {
    int64_t k, p;
    locate(off, nb, F, scan_ptr, t, &k, &p);
    double Z = 0.0;
    const int64_t pix = project_round(cams + 12 * k, intr, width, height, pw + 3 * p, &Z);
    flag[t] = pix >= 0 ? 1u : 0u;
    key[t] = ((uint64_t)k << pix_bits) | (uint64_t)(pix >= 0 ? pix : 0);
    z[t] = Z;
  }
};
struct CompactF {            // C3, over the T items
  const uint32_t* flag; const uint32_t* pos; const uint64_t* key_in; uint64_t* key; uint32_t* val;
  LVBA_HD void operator()(int64_t t) const { if (flag[t]) { key[pos[t]] = key_in[t]; val[pos[t]] = (uint32_t)t; } }
};
struct HeadF {               // run heads over [0, n] (terminator 0)
  const uint64_t* key; int64_t n; uint32_t* flag;
  LVBA_HD void operator()(int64_t r) const { flag[r] = (r < n && (r == 0 || key[r] != key[r - 1])) ? 1u : 0u; }
};
struct RunStartF {           // over [0, n]
  const uint32_t* flag; const uint32_t* pos; int64_t n; uint32_t* start;
  LVBA_HD void operator()(int64_t r) const { if (r == n) start[pos[n]] = (uint32_t)n; else if (flag[r]) start[pos[r]] = (uint32_t)r; }
};
// C4, one item per (image, pixel) run: the z-buffer rule of :2050 in cloud order.  A pixel is kept when its final depth is
// finite (the host restatement's `std::isfinite(zbuf[i])`; only a Z beyond FLT_MAX can leave it infinite).
struct ResolveF {
  const uint32_t* start; const uint32_t* val; const double* z; uint32_t* best; uint32_t* keep;
  LVBA_HD void operator()(int64_t v) const {
    float zbuf = depth::bits_float(depth::kEmpty);            // +inf
    uint32_t b = val[start[v]];
    for (uint32_t r = start[v]; r < start[v + 1]; ++r) {
      const uint32_t t = val[r];
      if (add_(z[t], (double)kEps) < (double)zbuf) { zbuf = (float)z[t]; b = t; }
    }
    best[v] = b;
    keep[v] = depth::finite_((double)zbuf) ? 1u : 0u;
  }
};
// C5, over the runs: survivors in run order with colour; voxel key and distance to the voxel centre when thinning
struct EmitF {
  const uint32_t* keep; const uint32_t* spos; const uint32_t* best; const uint32_t* start; const uint64_t* key_s; int pix_bits;
  const int64_t* off; int64_t nb; int F; const int64_t* scan_ptr; const float* pw; const uint8_t* rgb; int64_t n_pix;
  bool thin; double leaf; KeyPacking pk; int64_t base;
  uint64_t* okey; double* od2; float* oxyz; uint32_t* orgb;
  LVBA_HD void operator()(int64_t v) const {
    if (!keep[v]) return;
    const int64_t o = base + spos[v];
    int64_t k, p;
    locate(off, nb, F, scan_ptr, best[v], &k, &p);
    const uint64_t pix = key_s[start[v]] & (((uint64_t)1 << pix_bits) - 1);
    uint32_t c = kGrey;
    if (rgb) { const uint8_t* px = rgb + 3 * (k * n_pix + (int64_t)pix); c = ((uint32_t)px[0] << 16) | ((uint32_t)px[1] << 8) | px[2]; }
    orgb[o] = c;
    int64_t kk[3] = {0, 0, 0};
    double dd = 0.0;
    for (int a = 0; a < 3; ++a) {
      const float x = pw[3 * p + a];
      oxyz[3 * o + a] = x;
      if (thin) {
        vox::root_key_axis((double)x, leaf, &kk[a]);                          // tools.hpp:317-327 (in range: checked in begin)
        const double cc = mul_(add_((double)kk[a], 0.5), leaf);                // :332-334
        const double d = vox::sub_((double)x, cc);
        dd = add_(dd, mul_(d, d));                                             // :339
      }
    }
    if (thin) { okey[o] = pk.pack(kk); od2[o] = dd; }
  }
};
struct ConcatF {             // fold input: table entries first, then the pending ones (both already in merged order)
  const uint64_t* tk; int64_t nt; const uint64_t* pk_; uint64_t* key; uint32_t* idx;
  LVBA_HD void operator()(int64_t i) const { key[i] = i < nt ? tk[i] : pk_[i - nt]; idx[i] = (uint32_t)i; }
};
// per voxel run of the fold: `if (d2 < best_d2)` in merged order (tools.hpp:341-346); gathers the winner into the new table
struct FoldBestF {
  const uint32_t* start; const uint32_t* idx; int64_t nt;
  const uint64_t* tk; const double* td; const float* tx; const uint32_t* tc;
  const uint64_t* pk_; const double* pd; const float* px; const uint32_t* pc;
  uint64_t* nk; double* nd; float* nx; uint32_t* nc;
  LVBA_HD void operator()(int64_t v) const {
    uint32_t b = idx[start[v]];
    double bd = b < nt ? td[b] : pd[b - nt];
    for (uint32_t r = start[v] + 1; r < start[v + 1]; ++r) {
      const uint32_t i = idx[r];
      const double d = i < nt ? td[i] : pd[i - nt];
      if (d < bd) { bd = d; b = i; }
    }
    const bool in_t = b < nt;
    const int64_t j = in_t ? (int64_t)b : (int64_t)b - nt;
    nk[v] = in_t ? tk[j] : pk_[j]; nd[v] = bd; nc[v] = in_t ? tc[j] : pc[j];
    for (int a = 0; a < 3; ++a) nx[3 * v + a] = in_t ? tx[3 * j + a] : px[3 * j + a];
  }
};
template <class T>
struct CopyF { const T* src; T* dst; LVBA_HD void operator()(int64_t i) const { dst[i] = src[i]; } };
struct UnpackRgbF {
  const uint32_t* c; uint8_t* rgb;
  LVBA_HD void operator()(int64_t i) const { rgb[3 * i] = (uint8_t)(c[i] >> 16); rgb[3 * i + 1] = (uint8_t)(c[i] >> 8); rgb[3 * i + 2] = (uint8_t)c[i]; }
};

// One set of scans on the device; begin() .. add_images() .. finish() once per pose set (after, then before the optimisation).
template <class Exec>
struct Colorizer {
  template <class T>
  using Buf = typename Exec::template Buf<T>;
  struct Points {            // survivors: table (one per voxel, key order) or pending (merged order)
    Buf<uint64_t> key; Buf<double> d2; Buf<float> xyz; Buf<uint32_t> rgb;
    int64_t n = 0, cap = 0;
    int64_t bytes() const { return cap * (int64_t)(sizeof(uint64_t) + sizeof(double) + 3 * sizeof(float) + sizeof(uint32_t)); }
  };
  Exec ex;
  int F = 0;
  int64_t N = 0;
  const float* xyz = nullptr; const int64_t* scan_ptr = nullptr; const double* frame_ts = nullptr;   // Exec-dereferenceable
  const double* poses = nullptr;
  double half_window = 0.5, leaf = 0.0;
  bool thin = false;
  KeyPacking pk{};
  Buf<float> pw;
  Points table, pending;
  Buf<uint8_t> out_rgb;      // after finish(): [n_out * 3]
  int64_t n_merged = 0, n_out = 0;
  int64_t n_projections = 0, n_landed = 0;          // window items and items that land in their image, since begin()
  int64_t peak_bytes = 0;                           // the stage's own device buffers at their largest (sort scratch aside)
  const char* error = "";

  int64_t resident_bytes() const { return (int64_t)pw.n * 4 + table.bytes() + pending.bytes() + (int64_t)out_rgb.n; }
  void note(int64_t transient) { const int64_t b = resident_bytes() + transient; if (b > peak_bytes) peak_bytes = b; }

  void setup(const float* xyz_, const int64_t* scan_ptr_, const double* frame_ts_, int F_, int64_t N_) {
    xyz = xyz_; scan_ptr = scan_ptr_; frame_ts = frame_ts_; F = F_; N = N_;
  }

  // poses [F*12] Exec-dereferenceable, alive until finish()
  int begin(const double* poses_, double half_window_, double leaf_) {
    poses = poses_; half_window = half_window_; leaf = leaf_; thin = !(leaf < 0.001);
    table.n = pending.n = 0; n_merged = n_out = n_projections = n_landed = 0; peak_bytes = 0;
    pk = KeyPacking{{0, 0, 0}, {0, 0, 0}, 0, 0};
    LVBA_VOX_TRY(pw.alloc((size_t)N * 3));
    if (N == 0) return ex.sync();
    Buf<int32_t> lo, hi, bad;
    LVBA_VOX_TRY(lo.alloc((size_t)N * 3)); LVBA_VOX_TRY(hi.alloc((size_t)N * 3)); LVBA_VOX_TRY(bad.alloc(1));
    LVBA_VOX_TRY(ex.fill_zero(bad.p, 1));
    note((int64_t)N * 24);
    LVBA_VOX_TRY(ex.for_each(N, WorldPointF{xyz, scan_ptr, poses, F, thin ? leaf : 1.0, thin, pw.p, lo.p, hi.p, bad.p, N}));
    if (!thin) return ex.sync();
    int32_t h_bad = 0;
    LVBA_VOX_TRY(ex.fetch(&h_bad, bad.p, 1));
    if (h_bad) { error = "a world point is more than 2^30 leaf voxels from the origin"; return vox::kErrInvalid; }
    for (int a = 0; a < 3; ++a) {
      int32_t mn = 0, mx = 0, unused = 0;
      LVBA_VOX_TRY(ex.min_max(lo.p + (int64_t)a * N, N, &mn, &unused));
      LVBA_VOX_TRY(ex.min_max(hi.p + (int64_t)a * N, N, &unused, &mx));
      if (mn > mx) mn = mx = 0;                     // no finite point: nothing will ever be kept
      pk.mn[a] = mn;
      pk.bits[a] = vox::bit_length((uint64_t)((int64_t)mx - (int64_t)mn));
    }
    pk.root_bits = pk.bits[0] + pk.bits[1] + pk.bits[2];
    if (pk.root_bits > 62) { error = "leaf voxel keys span more than 62 bits"; return vox::kErrUnsupported; }
    return ex.sync();
  }

  int reserve(Points& s, int64_t want) {             // grow keeping the first s.n entries
    if (want <= s.cap) return 0;
    const int64_t cap = want > 2 * s.cap ? want : 2 * s.cap;
    Points g;
    LVBA_VOX_TRY(g.key.alloc((size_t)cap)); LVBA_VOX_TRY(g.d2.alloc((size_t)cap)); LVBA_VOX_TRY(g.xyz.alloc((size_t)cap * 3)); LVBA_VOX_TRY(g.rgb.alloc((size_t)cap));
    note(g.bytes());
    if (s.n) {
      LVBA_VOX_TRY(ex.for_each(s.n, CopyF<uint64_t>{s.key.p, g.key.p})); LVBA_VOX_TRY(ex.for_each(s.n, CopyF<double>{s.d2.p, g.d2.p}));
      LVBA_VOX_TRY(ex.for_each(s.n * 3, CopyF<float>{s.xyz.p, g.xyz.p})); LVBA_VOX_TRY(ex.for_each(s.n, CopyF<uint32_t>{s.rgb.p, g.rgb.p}));
      LVBA_VOX_TRY(ex.sync());
    }
    s.key.swap(g.key); s.d2.swap(g.d2); s.xyz.swap(g.xyz); s.rgb.swap(g.rgb);
    s.cap = cap;
    return 0;
  }

  // pending -> table: stable sort of (table, pending) by voxel key, arg-min per run
  int fold() {
    if (pending.n == 0) return 0;
    const int64_t nt = table.n, n = table.n + pending.n;
    if (n >= (int64_t)0xfffffff0ll) { error = "more than 2^32 points in one fold"; return vox::kErrUnsupported; }
    Buf<uint64_t> key, key_s; Buf<uint32_t> idx, idx_s, flag, pos, start;
    LVBA_VOX_TRY(key.alloc((size_t)n)); LVBA_VOX_TRY(key_s.alloc((size_t)n)); LVBA_VOX_TRY(idx.alloc((size_t)n)); LVBA_VOX_TRY(idx_s.alloc((size_t)n));
    LVBA_VOX_TRY(flag.alloc((size_t)n + 1)); LVBA_VOX_TRY(pos.alloc((size_t)n + 1));
    LVBA_VOX_TRY(ex.for_each(n, ConcatF{table.key.p, nt, pending.key.p, key.p, idx.p}));
    LVBA_VOX_TRY(ex.sort_pairs(key.p, key_s.p, idx.p, idx_s.p, n, pk.root_bits > 0 ? pk.root_bits : 1));
    LVBA_VOX_TRY(ex.for_each(n + 1, HeadF{key_s.p, n, flag.p}));
    LVBA_VOX_TRY(ex.exclusive_scan(flag.p, pos.p, n + 1));
    uint32_t nv = 0;
    LVBA_VOX_TRY(ex.fetch(&nv, pos.p + n, 1));
    LVBA_VOX_TRY(start.alloc((size_t)nv + 1));
    LVBA_VOX_TRY(ex.for_each(n + 1, RunStartF{flag.p, pos.p, n, start.p}));
    Points t;
    t.cap = nv > 0 ? (int64_t)nv : 1;
    LVBA_VOX_TRY(t.key.alloc((size_t)t.cap)); LVBA_VOX_TRY(t.d2.alloc((size_t)t.cap)); LVBA_VOX_TRY(t.xyz.alloc((size_t)t.cap * 3)); LVBA_VOX_TRY(t.rgb.alloc((size_t)t.cap));
    note(t.bytes() + n * 24 + (int64_t)nv * 4);
    LVBA_VOX_TRY(ex.for_each((int64_t)nv, FoldBestF{start.p, idx_s.p, nt, table.key.p, table.d2.p, table.xyz.p, table.rgb.p,
                                                     pending.key.p, pending.d2.p, pending.xyz.p, pending.rgb.p, t.key.p, t.d2.p, t.xyz.p, t.rgb.p}));
    LVBA_VOX_TRY(ex.sync());
    t.n = nv;
    table.key.swap(t.key); table.d2.swap(t.d2); table.xyz.swap(t.xyz); table.rgb.swap(t.rgb);
    table.n = t.n; table.cap = t.cap;
    pending.n = 0;
    return 0;
  }

  // One batch of nb images: image_ts [nb], cams [nb*12] (Rcw row-major, tcw), rgb [nb*height*width*3] or null (grey),
  // listed [nb] out — all Exec-dereferenceable.  Survivors join the pending list (merged order) and are folded when they
  // outnumber the table.
  int add_images(int64_t nb, const double* image_ts, const double* cams, const double intr[8], int width, int height,
                 const uint8_t* rgb, uint8_t* listed) {
    if (nb <= 0) return 0;
    const int64_t n_pix = (int64_t)width * height;
    const int64_t slots = nb * F;
    Buf<int64_t> count, off;
    LVBA_VOX_TRY(count.alloc((size_t)slots + 1)); LVBA_VOX_TRY(off.alloc((size_t)slots + 1));
    LVBA_VOX_TRY(ex.for_each(slots + 1, WindowCountF{image_ts, frame_ts, scan_ptr, F, nb, half_window, count.p}));
    LVBA_VOX_TRY(ex.exclusive_scan(count.p, off.p, slots + 1));
    LVBA_VOX_TRY(ex.for_each(nb, ListedF{off.p, F, listed}));
    int64_t T = 0;
    LVBA_VOX_TRY(ex.fetch(&T, off.p + slots, 1));
    n_projections += T;
    if (T == 0) return ex.sync();
    if (T >= (int64_t)0xfffffff0ll) { error = "more than 2^32 window points in one batch"; return vox::kErrUnsupported; }
    const int pix_bits = vox::bit_length((uint64_t)(n_pix - 1));
    const int key_bits = pix_bits + vox::bit_length((uint64_t)(nb - 1));
    if (key_bits > 62) { error = "image and pixel index span more than 62 bits"; return vox::kErrUnsupported; }
    Buf<uint64_t> key_all, key, key_s; Buf<double> z; Buf<uint32_t> flag, pos, val, val_s;
    LVBA_VOX_TRY(key_all.alloc((size_t)T)); LVBA_VOX_TRY(z.alloc((size_t)T)); LVBA_VOX_TRY(flag.alloc((size_t)T + 1)); LVBA_VOX_TRY(pos.alloc((size_t)T + 1));
    ProjectF pf{off.p, nb, F, scan_ptr, pw.p, cams, {}, width, height, pix_bits, key_all.p, z.p, flag.p};
    for (int q = 0; q < 8; ++q) pf.intr[q] = intr[q];
    LVBA_VOX_TRY(ex.for_each(T, pf));
    LVBA_VOX_TRY(ex.fill_zero(flag.p + T, 1));
    LVBA_VOX_TRY(ex.exclusive_scan(flag.p, pos.p, T + 1));
    uint32_t nl = 0;
    LVBA_VOX_TRY(ex.fetch(&nl, pos.p + T, 1));
    n_landed += nl;
    if (nl == 0) return ex.sync();
    LVBA_VOX_TRY(key.alloc(nl)); LVBA_VOX_TRY(key_s.alloc(nl)); LVBA_VOX_TRY(val.alloc(nl)); LVBA_VOX_TRY(val_s.alloc(nl));
    LVBA_VOX_TRY(ex.for_each(T, CompactF{flag.p, pos.p, key_all.p, key.p, val.p}));
    LVBA_VOX_TRY(ex.sort_pairs(key.p, key_s.p, val.p, val_s.p, nl, key_bits > 0 ? key_bits : 1));
    const int64_t n = nl;
    Buf<uint32_t> rflag, rpos, start, best, keep, spos;
    LVBA_VOX_TRY(rflag.alloc((size_t)n + 1)); LVBA_VOX_TRY(rpos.alloc((size_t)n + 1));
    LVBA_VOX_TRY(ex.for_each(n + 1, HeadF{key_s.p, n, rflag.p}));
    LVBA_VOX_TRY(ex.exclusive_scan(rflag.p, rpos.p, n + 1));
    uint32_t nr = 0;
    LVBA_VOX_TRY(ex.fetch(&nr, rpos.p + n, 1));
    LVBA_VOX_TRY(start.alloc((size_t)nr + 1)); LVBA_VOX_TRY(best.alloc((size_t)nr)); LVBA_VOX_TRY(keep.alloc((size_t)nr + 1)); LVBA_VOX_TRY(spos.alloc((size_t)nr + 1));
    LVBA_VOX_TRY(ex.for_each(n + 1, RunStartF{rflag.p, rpos.p, n, start.p}));
    LVBA_VOX_TRY(ex.for_each((int64_t)nr, ResolveF{start.p, val_s.p, z.p, best.p, keep.p}));
    LVBA_VOX_TRY(ex.fill_zero(keep.p + nr, 1));
    LVBA_VOX_TRY(ex.exclusive_scan(keep.p, spos.p, (int64_t)nr + 1));
    uint32_t ns = 0;
    LVBA_VOX_TRY(ex.fetch(&ns, spos.p + nr, 1));
    note(T * 25 + 8 + n * 24 + 8 + (int64_t)nr * 16 + 12);
    if (ns == 0) return ex.sync();
    LVBA_VOX_TRY(reserve(pending, pending.n + ns));
    note(T * 25 + 8 + n * 24 + 8 + (int64_t)nr * 16 + 12);
    LVBA_VOX_TRY(ex.for_each((int64_t)nr, EmitF{keep.p, spos.p, best.p, start.p, key_s.p, pix_bits, off.p, nb, F, scan_ptr, pw.p, rgb, n_pix,
                                                 thin, thin ? leaf : 1.0, pk, pending.n, pending.key.p, pending.d2.p, pending.xyz.p, pending.rgb.p}));
    LVBA_VOX_TRY(ex.sync());
    pending.n += ns;
    n_merged += ns;
    if (thin && pending.n > table.n) LVBA_VOX_TRY(fold());
    return 0;
  }

  // The thinned cloud (or, with leaf < 0.001, every survivor in merged order): out_xyz() / out_rgb after this.
  int finish() {
    if (thin) LVBA_VOX_TRY(fold());
    const Points& s = thin ? table : pending;
    n_out = s.n;
    LVBA_VOX_TRY(out_rgb.alloc((size_t)n_out * 3));
    note(0);
    LVBA_VOX_TRY(ex.for_each(n_out, UnpackRgbF{s.rgb.p, out_rgb.p}));
    return ex.sync();
  }
  const float* out_xyz() const { return thin ? table.xyz.p : pending.xyz.p; }
};

}  // namespace color
}  // namespace lvba
