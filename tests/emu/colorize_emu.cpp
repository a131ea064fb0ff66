// colorize_emu.cpp — TEST INFRASTRUCTURE: the coloured-map pipeline of global-lvba_b200/csrc/color_pipeline.h run with the
// sequential host policy, compared with oracle/colorize_oracle.py by tests/test_colorize_emu.py.  Never part of the product.
#include "../../global-lvba_b200/csrc/color_pipeline.h"
#include "host_exec.h"

using Col = lvba::color::Colorizer<HostExec>;

extern "C" {

int emu_color_create(int32_t F, const int64_t* scan_ptr, const float* xyz, const double* frame_ts, void** out) {
  Col* c = new Col();
  c->setup(xyz, scan_ptr, frame_ts, F, scan_ptr[F]);
  *out = c;
  return 0;
}

int emu_color_begin(void* h, const double* poses, double half_window, double leaf) { return ((Col*)h)->begin(poses, half_window, leaf); }

int emu_color_add(void* h, int64_t nb, const double* image_ts, const double* cams, const double* intr, int32_t width, int32_t height,
                  const uint8_t* rgb, uint8_t* listed) {
  return ((Col*)h)->add_images(nb, image_ts, cams, intr, width, height, rgb, listed);
}

int emu_color_finish(void* h, int64_t* n_out, int64_t* stats) {
  Col* c = (Col*)h;
  const int rc = c->finish();
  *n_out = c->n_out;
  if (stats) { stats[0] = c->n_projections; stats[1] = c->n_landed; stats[2] = c->n_merged; stats[3] = c->peak_bytes; stats[4] = c->table.n; }
  return rc;
}

int emu_color_export(void* h, float* xyz, uint8_t* rgb) {
  Col* c = (Col*)h;
  if (c->n_out) { std::memcpy(xyz, c->out_xyz(), (size_t)c->n_out * 12); std::memcpy(rgb, c->out_rgb.p, (size_t)c->n_out * 3); }
  return 0;
}

int emu_color_destroy(void* h) { delete (Col*)h; return 0; }

}  // extern "C"
