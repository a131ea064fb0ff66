// A visual BA problem with one landmark seen 300 times through lvba_b200::solve_visual (global-lvba_b200/host/lvba_shim.hpp): the
// call `lvba_offline --visual` makes.  Pinhole cameras 0.5 m apart along x, all looking along +z; a facade point 30 m away is
// seen by cameras 0..299, short tracks of 4 observations fill the rest.  Prints "ok: ..." and exits 0 when the solve returns
// LVBA_OK and lowers the cost; prints the status and exits 1 otherwise.
#include <array>
#include <cmath>
#include <cstdio>

#include "../../global-lvba_b200/host/lvba_shim.hpp"

int main() {
  const int M = 320;
  const double fx = 400.0, fy = 400.0, cx = 320.0, cy = 256.0;
  std::vector<std::array<double, 4>> qs(M, {1.0, 0.0, 0.0, 0.0});
  std::vector<std::array<double, 3>> ts(M);
  for (int k = 0; k < M; ++k) ts[k] = {-0.5 * k, 0.01 * std::sin(k), 0.0};
  std::vector<std::array<double, 3>> Xs;
  std::vector<std::vector<lvba_b200::Observation>> obs;
  auto add = [&](double x, double y, double z, int c0, int K) {
    std::vector<lvba_b200::Observation> o;
    for (int j = 0; j < K; ++j) {
      const int c = c0 + j;
      const double xc = x - 0.5 * c, yc = y, zc = z;
      const double jitter = 0.3 * std::sin(0.7 * (c + 3 * Xs.size()));
      o.push_back({c, (float)(fx * xc / zc + cx + jitter), (float)(fy * yc / zc + cy - jitter)});
    }
    Xs.push_back({x + 0.05, y - 0.04, z + 0.1});       // start off the true position
    obs.push_back(o);
  };
  add(75.0, 1.0, 30.0, 0, 300);                        // the long track
  for (int i = 0; i < 150; ++i) add(0.5 * (2 * i + 2) + 1.0, -1.0 + 0.01 * i, 8.0 + (i % 7), 2 * i, 4);
  const int64_t T = (int64_t)Xs.size();
  std::vector<std::array<double, 3>> plane_n(T);
  std::vector<double> plane_d(T);
  for (int64_t i = 0; i < T; ++i) {
    plane_n[i] = {0.0, 0.0, 1.0};
    plane_d[i] = -(Xs[i][2] - 0.1);                    // the plane z = true depth
  }
  lvba_summary s{};
  const int rc = lvba_b200::solve_visual(qs, ts, Xs, plane_n, plane_d, obs, fx, fy, cx, cy, 0, 0, 0, 0, 0.5, 0.01, nullptr, &s);
  if (rc != LVBA_OK) {
    std::printf("solve_visual: %s (%s)\n", lvba_status_string(rc), lvba_last_error());
    return 1;
  }
  if (!(s.cost_last < s.cost_first)) {
    std::printf("solve_visual: cost %g -> %g\n", s.cost_first, s.cost_last);
    return 1;
  }
  std::printf("ok: %d iterations, cost %g -> %g\n", s.iterations, s.cost_first, s.cost_last);
  return 0;
}
