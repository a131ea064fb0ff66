// lvba_b200::solve_visual_remove_outliers (global-lvba_b200/host/lvba_shim.hpp): reads a visual problem in the layout of
// write_visual_problem (global-lvba_b200/host/lvba_visual_offline.hpp; the state after the solve is not read), runs solve ->
// remove_outliers(PX, N) -> solve on one handle in deterministic mode, and writes q [M*4], t [M*3], X [T*3], the removed mask
// [nnz] (uint8, per point in the order of its observation list), and of both summaries iterations, accepted, termination
// (int32 each) and cost_first, cost_last (double) to the output file.
//   visual_outliers_shim IN OUT PX N
#include <array>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

#include "../../global-lvba_b200/host/lvba_shim.hpp"

int main(int argc, char** argv) {
  if (argc != 5) { std::fprintf(stderr, "usage: visual_outliers_shim IN OUT PX N\n"); return 64; }
  std::ifstream f(argv[1], std::ios::binary);
  char magic[8];
  int64_t M, T, nnz;
  double intr[8], sig[2];
  auto get = [&](void* p, size_t n) { if (n) f.read(static_cast<char*>(p), (std::streamsize)n); };
  get(magic, 8); get(&M, 8); get(&T, 8); get(&nnz, 8); get(intr, 64); get(sig, 16);
  if (!f || std::string(magic, 8) != "LVBAVP01") { std::fprintf(stderr, "not a visual problem file\n"); return 1; }
  std::vector<std::array<double, 4>> qs((size_t)M);
  std::vector<std::array<double, 3>> ts((size_t)M), Xs((size_t)T), plane_n((size_t)T);
  std::vector<double> plane_nd((size_t)T * 4), plane_d((size_t)T);
  std::vector<int64_t> obs_ptr((size_t)T + 1);
  std::vector<int32_t> obs_cam((size_t)nnz);
  std::vector<float> obs_uv((size_t)nnz * 2);
  get(qs.data(), (size_t)M * 32); get(ts.data(), (size_t)M * 24); get(Xs.data(), (size_t)T * 24);
  get(plane_nd.data(), plane_nd.size() * 8); get(obs_ptr.data(), obs_ptr.size() * 8);
  get(obs_cam.data(), obs_cam.size() * 4); get(obs_uv.data(), obs_uv.size() * 4);
  if (!f) { std::fprintf(stderr, "truncated problem file\n"); return 1; }
  std::vector<std::vector<lvba_b200::Observation>> obs((size_t)T);
  for (int64_t i = 0; i < T; ++i) {
    plane_n[(size_t)i] = {plane_nd[4 * (size_t)i], plane_nd[4 * (size_t)i + 1], plane_nd[4 * (size_t)i + 2]};
    plane_d[(size_t)i] = plane_nd[4 * (size_t)i + 3];
    for (int64_t s = obs_ptr[(size_t)i]; s < obs_ptr[(size_t)i + 1]; ++s)
      obs[(size_t)i].push_back({obs_cam[(size_t)s], obs_uv[2 * (size_t)s], obs_uv[2 * (size_t)s + 1]});
  }
  lvba_visual_opts o;
  lvba_visual_default_opts(&o);
  o.deterministic = 1;
  lvba_summary s1{}, s2{};
  std::vector<std::vector<uint8_t>> removed;
  const int rc = lvba_b200::solve_visual_remove_outliers(qs, ts, Xs, plane_n, plane_d, obs, intr[0], intr[1], intr[2], intr[3], intr[4], intr[5],
                                                         intr[6], intr[7], sig[0], sig[1], &o, std::atof(argv[3]), std::atoi(argv[4]), &removed,
                                                         &s1, &s2);
  if (rc != LVBA_OK) { std::fprintf(stderr, "solve_visual_remove_outliers: %s (%s)\n", lvba_status_string(rc), lvba_last_error()); return 1; }
  std::ofstream g(argv[2], std::ios::binary);
  g.write(reinterpret_cast<const char*>(qs.data()), (std::streamsize)(M * 32));
  g.write(reinterpret_cast<const char*>(ts.data()), (std::streamsize)(M * 24));
  g.write(reinterpret_cast<const char*>(Xs.data()), (std::streamsize)(T * 24));
  for (const auto& r : removed) g.write(reinterpret_cast<const char*>(r.data()), (std::streamsize)r.size());
  for (const lvba_summary* s : {&s1, &s2}) {
    const int32_t ints[3] = {s->iterations, s->accepted, s->termination};
    const double costs[2] = {s->cost_first, s->cost_last};
    g.write(reinterpret_cast<const char*>(ints), 12);
    g.write(reinterpret_cast<const char*>(costs), 16);
  }
  return g ? 0 : 1;
}
