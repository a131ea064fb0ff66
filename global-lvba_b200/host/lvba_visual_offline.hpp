// lvba_visual_offline.hpp — the VISUAL half of the reference's pipeline without ROS, OpenCV, PCL or SiftGPU (SURVEY.md §8f N4):
//   Config                          the ROS parameters of DatasetIO::readParameters (src/dataset_io.cpp:27-62) and
//                                   LvbaSystem::LvbaSystem (src/lvba_system.cpp:124-131), read from the reference's own YAML
//   list_images                     DatasetIO::handleImages                  src/dataset_io.cpp:77-131
//   load_colmap_db                  LvbaSystem::loadFromColmapDB             src/lvba_system.cpp:510-685
//   update_camera_poses_from_lidar  LvbaSystem::updateCameraPosesFromLidar   src/lvba_system.cpp:412-446
//   run_visual_ba                   LvbaSystem::runVisualBAWithLidarAssist   src/lvba_system.cpp:144-154
//                                   (buildGridMapFromOptimized -> updateCameraPosesFromLidar -> generateDepthWithVoxel ->
//                                    [keypoints and matches from the COLMAP database] -> BuildTracksAndFuse3D -> optimizeCameraPoses)
//   write_images_txt / write_points3D_txt   the COLMAP text model the reference writes in pubRGBCloud's colouring pass
//                                   (src/lvba_system.cpp:1949-1952, :2018-2024, :2121-2137)
// Everything numeric runs in liblvba_b200.so through lvba_shim.hpp; this header is the host glue the reference keeps in
// LvbaSystem.  Feature extraction and matching (SiftGPU) are out of scope (SURVEY.md §8): the database must already hold them —
// the reference takes the same path whenever the database matches the image list (:693-700).
// SQLite is bound at run time (dlopen of libsqlite3.so.0; its C API is declared below because this image has no sqlite3.h).
#pragma once
#include <limits>
#include <dlfcn.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "lvba_dataset.hpp"
#include "lvba_shim.hpp"

namespace lvba_b200 {
namespace offline {

using dataset::Cloud;
using dataset::Pose;

// ------------------------------------------------------------------------------------------------ configuration
struct Config {
  std::string data_path = "dataset/cbd_new/", colmap_db_path;
  int image_stride = 10, width = 1280, height = 1024;
  double scale = 0.5, fx = 1293.56944, fy = 1293.3155, cx = 626.91359, cy = 522.799224;
  double d0 = -0.076160, d1 = 0.123001, d2 = -0.00113, d3 = 0.000251;
  std::vector<double> extrinT, extrinR, Pcl, Rcl;
  bool window_enable = true, window_rel = false, stage1_enable = true;
  int window_size = 10;
  double anchor_leaf = 0.1, stage1_voxel = 0.5, stage2_voxel = -1.0;       // stage 2 defaults to stage 1's size (:57)
  std::vector<float> eigen1{0.3f, 0.1f, 0.06f, 0.03f}, eigen2{0.3f, 0.1f, 0.06f, 0.03f};     // bavoxel.hpp:17
  bool enable_lidar_ba = true, enable_visual_ba = true, colmap_output = true;
  double min_view_angle = 8.0, reproj_mean_thr = 3.0, filter_size_points3D = 0.01;
  int fuse_map_order = LVBA_FUSE_ORDER_LIBSTDCXX;     // not a reference parameter: which unordered_map order the track fusion mimics (lvba_b200.h)
  bool scaled = false;
  // the tail of readParameters (:59-62): the image is used at `scale`
  void apply_scale() {
    if (scaled) return;
    width = (int)std::lround(width * scale); height = (int)std::lround(height * scale);
    fx *= scale; fy *= scale; cx *= scale; cy *= scale;
    if (stage2_voxel <= 0) stage2_voxel = stage1_voxel;
    scaled = true;
  }
};

// A robust loss of the visual stage as `KIND[:A]`, KIND none|huber|cauchy (lvba_loss_kind), A a finite number > 0 (default
// `default_scale`).  Anything else is refused with a message in *err; kind / scale are then untouched.
inline bool parse_loss(const char* text, double default_scale, int32_t& kind, double& scale, std::string* err = nullptr) {
  const std::string s = text ? text : "";
  const size_t colon = s.find(':');
  const std::string name = s.substr(0, colon);
  int32_t k;
  if (name == "none") k = LVBA_LOSS_NONE;
  else if (name == "huber") k = LVBA_LOSS_HUBER;
  else if (name == "cauchy") k = LVBA_LOSS_CAUCHY;
  else { if (err) *err = "'" + s + "': the kind must be none, huber or cauchy"; return false; }
  double a = default_scale;
  if (colon != std::string::npos) {
    const std::string num = s.substr(colon + 1);
    char* end = nullptr;
    a = num.empty() ? 0.0 : std::strtod(num.c_str(), &end);
    if (num.empty() || *end != '\0' || !std::isfinite(a) || !(a > 0.0)) {
      if (err) *err = "'" + s + "': the scale after ':' must be a finite number > 0";
      return false;
    }
  }
  kind = k;
  scale = a;
  return true;
}

// A list of index ranges `A:B,C,D:E` (each A:B inclusive, A <= B, a single index C for C:C, indices decimal and >= 0) as a
// mask of n entries, 1 on every listed index.  Anything else, or an index >= n, is refused with a message in *err; mask is
// then untouched.  n < 0 checks the syntax only and leaves mask untouched.
inline bool parse_index_ranges(const char* text, int n, std::vector<uint8_t>& mask, std::string* err = nullptr) {
  const std::string s = text ? text : "";
  std::vector<uint8_t> m((size_t)std::max(n, 0), 0);
  auto index = [](const std::string& t, long& v) {
    if (t.empty() || t.size() > 9 || t.find_first_not_of("0123456789") != std::string::npos) return false;
    v = std::strtol(t.c_str(), nullptr, 10);
    return true;
  };
  size_t pos = 0;
  do {
    const size_t comma = s.find(',', pos);
    const std::string item = s.substr(pos, comma == std::string::npos ? std::string::npos : comma - pos);
    const size_t colon = item.find(':');
    long a = 0, b = 0;
    const bool ok = colon == std::string::npos ? index(item, a) && index(item, b)
                                               : index(item.substr(0, colon), a) && index(item.substr(colon + 1), b);
    if (!ok || a > b) { if (err) *err = "'" + s + "': '" + item + "' is not an index or a range A:B with A <= B"; return false; }
    if (n >= 0 && b >= n) { if (err) *err = "'" + s + "': index " + std::to_string(b) + " is past the last of " + std::to_string(n); return false; }
    if (n >= 0) for (long i = a; i <= b; ++i) m[(size_t)i] = 1;
    pos = comma == std::string::npos ? std::string::npos : comma + 1;
  } while (pos != std::string::npos);
  if (n >= 0) mask.swap(m);
  return true;
}

// The subset of YAML the reference's config files use: `section:` lines, `  key: value` lines, flow lists that may run over
// several lines, `#` comments, quoted strings.  Returns "section/key" -> raw value text (lists without the brackets).
inline bool read_yaml_subset(const std::string& file, std::map<std::string, std::string>& kv, std::string* err) {
  std::ifstream fin(file);
  if (!fin.is_open()) { if (err) *err = "cannot open " + file; return false; }
  std::string line, section, open_key, open_val;
  auto trim = [](std::string s) { const auto a = s.find_first_not_of(" \t\r"); if (a == std::string::npos) return std::string(); const auto b = s.find_last_not_of(" \t\r"); return s.substr(a, b - a + 1); };
  while (std::getline(fin, line)) {
    const auto hash = line.find('#');
    if (hash != std::string::npos) line.erase(hash);
    if (trim(line).empty()) continue;
    if (!open_key.empty()) {                                        // inside a multi-line flow list
      open_val += " " + trim(line);
      if (open_val.find(']') != std::string::npos) { open_val.erase(open_val.find(']')); kv[open_key] = trim(open_val); open_key.clear(); }
      continue;
    }
    const bool indented = line[0] == ' ' || line[0] == '\t';
    const auto colon = line.find(':');
    if (colon == std::string::npos) continue;
    const std::string key = trim(line.substr(0, colon));
    std::string val = trim(line.substr(colon + 1));
    if (!indented && val.empty()) { section = key; continue; }
    const std::string full = (indented && !section.empty()) ? section + "/" + key : key;
    if (!indented) section.clear();
    if (!val.empty() && val[0] == '[') {
      val.erase(0, 1);
      if (val.find(']') == std::string::npos) { open_key = full; open_val = val; continue; }
      val.erase(val.find(']'));
    } else if (val.size() >= 2 && (val.front() == '"' || val.front() == '\'') && val.back() == val.front()) {
      val = val.substr(1, val.size() - 2);
    }
    kv[full] = trim(val);
  }
  if (!open_key.empty()) { if (err) *err = "unterminated list for " + open_key; return false; }
  return true;
}

inline bool load_config(const std::string& file, Config& c, std::string* err = nullptr) {
  std::map<std::string, std::string> kv;
  if (!read_yaml_subset(file, kv, err)) return false;
  auto has = [&](const char* k) { return kv.count(k) != 0; };
  auto num = [&](const char* k, double& v) { if (has(k)) v = std::atof(kv[k].c_str()); };
  auto integer = [&](const char* k, int& v) { if (has(k)) v = std::atoi(kv[k].c_str()); };
  auto flag = [&](const char* k, bool& v) { if (has(k)) { const std::string& s = kv[k]; v = (s == "true" || s == "True" || s == "1"); } };
  auto text = [&](const char* k, std::string& v) { if (has(k)) v = kv[k]; };
  auto list = [&](const char* k, auto& v) {
    if (!has(k)) return;
    v.clear();
    std::string s = kv[k];
    for (char& ch : s) if (ch == ',') ch = ' ';
    std::istringstream iss(s);
    double x;
    while (iss >> x) v.push_back((typename std::decay_t<decltype(v)>::value_type)x);
  };
  text("data_config/data_path", c.data_path); text("data_config/colmap_db_path", c.colmap_db_path);
  integer("data_config/image_sample_step", c.image_stride);
  flag("data_config/enable_lidar_ba", c.enable_lidar_ba); flag("data_config/enable_visual_ba", c.enable_visual_ba);
  integer("cam_model/cam_width", c.width); integer("cam_model/cam_height", c.height); num("cam_model/scale", c.scale);
  num("cam_model/cam_fx", c.fx); num("cam_model/cam_fy", c.fy); num("cam_model/cam_cx", c.cx); num("cam_model/cam_cy", c.cy);
  num("cam_model/cam_d0", c.d0); num("cam_model/cam_d1", c.d1); num("cam_model/cam_d2", c.d2); num("cam_model/cam_d3", c.d3);
  list("extrin_calib/extrinsic_T", c.extrinT); list("extrin_calib/extrinsic_R", c.extrinR);
  list("extrin_calib/Pcl", c.Pcl); list("extrin_calib/Rcl", c.Rcl);
  flag("window_ba/enable", c.window_enable); integer("window_ba/size", c.window_size);
  num("window_ba/anchor_leaf_size", c.anchor_leaf); flag("window_ba/use_window_ba_rel", c.window_rel);
  num("BALM_stage1/root_voxel_size", c.stage1_voxel); flag("BALM_stage1/enable", c.stage1_enable);
  num("BALM_stage2/root_voxel_size", c.stage2_voxel);
  list("BALM_stage1/eigen_ratio_array", c.eigen1); list("BALM_stage2/eigen_ratio_array", c.eigen2);
  num("track_fusion/min_view_angle", c.min_view_angle); num("track_fusion/reproj_mean_thr", c.reproj_mean_thr);
  flag("colmap_output/enable", c.colmap_output); num("colmap_output/filter_size_points3D", c.filter_size_points3D);
  if (c.extrinT.size() != 3 || c.extrinR.size() != 9 || c.Pcl.size() != 3 || c.Rcl.size() != 9) {
    if (err) *err = "extrin_calib needs extrinsic_T[3], extrinsic_R[9], Pcl[3], Rcl[9]";
    return false;
  }
  if (c.image_stride <= 0) { if (err) *err = "image_sample_step must be positive"; return false; }     // handleImages :89-92
  return true;
}

// ------------------------------------------------------------------------------------------------ small 3x3 algebra (row-major)
struct M3 { double m[9]; double operator()(int r, int c) const { return m[3 * r + c]; } double& operator()(int r, int c) { return m[3 * r + c]; } };
struct V3 { double v[3]; double operator()(int r) const { return v[r]; } double& operator()(int r) { return v[r]; } };
inline M3 mul(const M3& a, const M3& b) { M3 o{}; for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) o(r, c) = a(r, 0) * b(0, c) + a(r, 1) * b(1, c) + a(r, 2) * b(2, c); return o; }
inline M3 tr(const M3& a) { M3 o{}; for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) o(r, c) = a(c, r); return o; }
inline V3 mul(const M3& a, const V3& x) { V3 o{}; for (int r = 0; r < 3; ++r) o(r) = a(r, 0) * x(0) + a(r, 1) * x(1) + a(r, 2) * x(2); return o; }
inline M3 to_m3(const dataset::Mat3& R) { M3 o{}; for (int k = 0; k < 9; ++k) o.m[k] = R.m[k]; return o; }
inline V3 to_v3(const dataset::Vec3& p) { return V3{{p.v[0], p.v[1], p.v[2]}}; }

// Rci_, tci_ of initFromDatasetIO (:486-506): camera <- LiDAR composed with LiDAR <- IMU
inline void camera_from_body(const Config& c, M3& Rci, V3& tci) {
  M3 Rcl{}, Ril{};
  for (int k = 0; k < 9; ++k) { Rcl.m[k] = c.Rcl[(size_t)k]; Ril.m[k] = c.extrinR[(size_t)k]; }
  const V3 tcl{{c.Pcl[0], c.Pcl[1], c.Pcl[2]}}, til{{c.extrinT[0], c.extrinT[1], c.extrinT[2]}};
  const M3 Rli = tr(Ril);
  V3 tli = mul(Rli, til);
  for (int k = 0; k < 3; ++k) tli(k) = -tli(k);
  Rci = mul(Rcl, Rli);
  tci = mul(Rcl, tli);
  for (int k = 0; k < 3; ++k) tci(k) += tcl(k);
}

// Rcw = Rci Rwi^T, tcw = -Rcw pwi + tci   (generateDepthWithVoxel :857-870)
inline void world_to_camera(const Pose& T_w_i, const M3& Rci, const V3& tci, M3& Rcw, V3& tcw) {
  Rcw = mul(Rci, tr(to_m3(T_w_i.R)));
  const V3 a = mul(Rcw, to_v3(T_w_i.p));
  for (int k = 0; k < 3; ++k) tcw(k) = -a(k) + tci(k);
}

// Eigen::Quaterniond(R) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other,3,3>): no sign normalisation
inline void eigen_quaternion(const M3& R, double q[4] /* w x y z */) {
  double t = R(0, 0) + R(1, 1) + R(2, 2);
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[0] = 0.5 * t; t = 0.5 / t;
    q[1] = (R(2, 1) - R(1, 2)) * t; q[2] = (R(0, 2) - R(2, 0)) * t; q[3] = (R(1, 0) - R(0, 1)) * t;
  } else {
    int i = 0;
    if (R(1, 1) > R(0, 0)) i = 1;
    if (R(2, 2) > R(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(R(i, i) - R(j, j) - R(k, k) + 1.0);
    q[1 + i] = 0.5 * t; t = 0.5 / t;
    q[0] = (R(k, j) - R(j, k)) * t; q[1 + j] = (R(j, i) + R(i, j)) * t; q[1 + k] = (R(k, i) + R(i, k)) * t;
  }
}

// ------------------------------------------------------------------------------------------------ images
// handleImages (:77-131): every .png/.jpg/.jpeg/.bmp of <data>/all_image with a number in its name, sorted, every stride-th
inline bool list_images(const std::string& data, int stride, std::vector<double>& images_ids, std::string* err = nullptr) {
  namespace fs = std::filesystem;
  images_ids.clear();
  const fs::path dir = fs::path(data) / "all_image";
  if (!fs::exists(dir) || !fs::is_directory(dir)) { if (err) *err = "image dir missing: " + dir.string(); return false; }
  if (stride <= 0) { if (err) *err = "image stride must be positive"; return false; }
  std::vector<double> all;
  for (const auto& e : fs::directory_iterator(dir)) {
    if (!e.is_regular_file()) continue;
    const std::string ext = e.path().extension().string();
    if (ext != ".png" && ext != ".jpg" && ext != ".jpeg" && ext != ".bmp") continue;
    double ts = 0.0;
    if (!dataset::parse_timestamp_from_name(e.path().filename().string(), ts)) continue;
    all.push_back(ts);
  }
  if (all.empty()) { if (err) *err = "no image files in " + dir.string(); return false; }
  std::sort(all.begin(), all.end());
  for (size_t i = 0; i < all.size(); i += (size_t)stride) images_ids.push_back(all[i]);
  return true;
}
// getImagePath (:2146-2148): std::to_string prints six decimals
inline std::string image_file_name(double image_id) { return std::to_string(image_id) + ".png"; }

// ------------------------------------------------------------------------------------------------ COLMAP database
struct Keypoint { float x = 0, y = 0, sigma = 0, extremum_val = 0; };
using KeypointImages = std::vector<std::vector<Keypoint>>;
using MatchTable = std::vector<std::vector<std::pair<int, int>>>;      // all_matches_[pairIndex(i, j, N)]

class SqliteApi {
 public:
  struct sqlite3;
  struct sqlite3_stmt;
  int (*open_v2)(const char*, sqlite3**, int, const char*) = nullptr;
  int (*close)(sqlite3*) = nullptr;
  int (*prepare_v2)(sqlite3*, const char*, int, sqlite3_stmt**, const char**) = nullptr;
  int (*step)(sqlite3_stmt*) = nullptr;
  int (*reset)(sqlite3_stmt*) = nullptr;
  int (*finalize)(sqlite3_stmt*) = nullptr;
  int (*bind_int64)(sqlite3_stmt*, int, long long) = nullptr;
  int (*column_int)(sqlite3_stmt*, int) = nullptr;
  long long (*column_int64)(sqlite3_stmt*, int) = nullptr;
  const unsigned char* (*column_text)(sqlite3_stmt*, int) = nullptr;
  const void* (*column_blob)(sqlite3_stmt*, int) = nullptr;
  int (*column_bytes)(sqlite3_stmt*, int) = nullptr;
  const char* (*errmsg)(sqlite3*) = nullptr;
  static constexpr int kOk = 0, kRow = 100, kOpenReadOnly = 1;
  bool load(std::string* err) {
    if (lib_) return true;
    for (const char* nm : {"libsqlite3.so.0", "libsqlite3.so"}) { lib_ = dlopen(nm, RTLD_NOW); if (lib_) break; }
    if (!lib_) { if (err) *err = std::string("cannot dlopen libsqlite3: ") + dlerror(); return false; }
    bool ok = true;
    auto sym = [&](auto& f, const char* name) { *(void**)(&f) = dlsym(lib_, name); if (!f) { ok = false; if (err) *err = std::string("libsqlite3 lacks ") + name; } };
    sym(open_v2, "sqlite3_open_v2"); sym(close, "sqlite3_close"); sym(prepare_v2, "sqlite3_prepare_v2"); sym(step, "sqlite3_step");
    sym(reset, "sqlite3_reset"); sym(finalize, "sqlite3_finalize"); sym(bind_int64, "sqlite3_bind_int64"); sym(column_int, "sqlite3_column_int");
    sym(column_int64, "sqlite3_column_int64"); sym(column_text, "sqlite3_column_text"); sym(column_blob, "sqlite3_column_blob");
    sym(column_bytes, "sqlite3_column_bytes"); sym(errmsg, "sqlite3_errmsg");
    return ok;
  }
 private:
  void* lib_ = nullptr;
};

// loadFromColmapDB (:510-685).  Returns false — as the reference does before it falls back to SiftGPU — when the database cannot
// be opened or its image count differs from images_ids.size().  all_matches has one list per image pair (i < j) in pairIndex order.
inline bool load_colmap_db(const std::string& db_path, const std::vector<double>& images_ids, KeypointImages& all_keypoints,
                           MatchTable& all_matches, std::string* err = nullptr) {
  namespace fs = std::filesystem;
  static SqliteApi sq;
  if (!sq.load(err)) return false;
  SqliteApi::sqlite3* db = nullptr;
  if (sq.open_v2(db_path.c_str(), &db, SqliteApi::kOpenReadOnly, nullptr) != SqliteApi::kOk) {
    if (err) *err = std::string("[DB] open failed: ") + (db ? sq.errmsg(db) : "out of memory");
    if (db) sq.close(db);
    return false;
  }
  const int N = (int)images_ids.size();
  std::unordered_map<std::string, uint32_t> name2id;
  size_t db_image_count = 0;
  SqliteApi::sqlite3_stmt* st = nullptr;
  if (sq.prepare_v2(db, "SELECT image_id, name FROM images;", -1, &st, nullptr) == SqliteApi::kOk) {
    while (sq.step(st) == SqliteApi::kRow) {
      const uint32_t id = (uint32_t)sq.column_int64(st, 0);
      const unsigned char* txt = sq.column_text(st, 1);
      if (!txt) continue;
      const std::string name((const char*)txt);
      name2id[name] = id;
      name2id[fs::path(name).filename().string()] = id;
      ++db_image_count;
    }
  }
  sq.finalize(st);
  if (db_image_count != (size_t)N) {                                                                   // :547-555
    if (err) *err = "[DB] images count (" + std::to_string(db_image_count) + ") != dataset images count (" + std::to_string(N) + ")";
    sq.close(db);
    return false;
  }
  std::vector<int> db_id((size_t)N, -1);
  for (int i = 0; i < N; ++i) {
    const auto it = name2id.find(image_file_name(images_ids[(size_t)i]));                              // imageIdOfTs (:562-568)
    if (it != name2id.end()) db_id[(size_t)i] = (int)it->second;
  }
  all_keypoints.assign((size_t)N, {});
  if (sq.prepare_v2(db, "SELECT rows, cols, data FROM keypoints WHERE image_id=?;", -1, &st, nullptr) == SqliteApi::kOk) {
    for (int i = 0; i < N; ++i) {
      if (db_id[(size_t)i] < 0) continue;
      sq.reset(st);
      sq.bind_int64(st, 1, db_id[(size_t)i]);
      if (sq.step(st) != SqliteApi::kRow) continue;
      const int rows = sq.column_int(st, 0), cols = sq.column_int(st, 1);
      const void* blob = sq.column_blob(st, 2);
      const int bytes = sq.column_bytes(st, 2);
      if (!blob || rows < 0 || cols < 2 || (long long)bytes != (long long)rows * cols * (long long)sizeof(float)) continue;   // :587 (cols < 2 would read past a row)
      const float* fp = (const float*)blob;
      auto& vec = all_keypoints[(size_t)i];
      vec.resize((size_t)rows);
      for (int r = 0; r < rows; ++r) {
        Keypoint kp;
        kp.x = fp[(size_t)r * cols]; kp.y = fp[(size_t)r * cols + 1];
        if (cols >= 3) kp.sigma = fp[(size_t)r * cols + 2];
        if (cols >= 4) kp.extremum_val = fp[(size_t)r * cols + 3];
        vec[(size_t)r] = kp;
      }
    }
  }
  sq.finalize(st);
  all_matches.assign((size_t)N * (size_t)(N > 0 ? N - 1 : 0) / 2, {});
  if (sq.prepare_v2(db, "SELECT rows, cols, data FROM two_view_geometries WHERE pair_id=?;", -1, &st, nullptr) == SqliteApi::kOk) {
    size_t k = 0;
    for (int i = 0; i < N; ++i)
      for (int j = i + 1; j < N; ++j, ++k) {                                                          // image_pairs_ (:462-466)
        const int id1 = db_id[(size_t)i], id2 = db_id[(size_t)j];
        if (id1 < 0 || id2 < 0) continue;
        const auto& k1 = all_keypoints[(size_t)i];
        const auto& k2 = all_keypoints[(size_t)j];
        if (k1.empty() || k2.empty()) continue;
        const bool swapped = id1 > id2;
        const uint64_t lo = (uint64_t)(swapped ? id2 : id1), hi = (uint64_t)(swapped ? id1 : id2);
        const uint64_t pair_id = lo * 2147483647ull + hi;                                             // kColmapMaxNumImages (:512-519)
        sq.reset(st);
        sq.bind_int64(st, 1, (long long)pair_id);
        if (sq.step(st) != SqliteApi::kRow) continue;
        const int rows = sq.column_int(st, 0), cols = sq.column_int(st, 1);
        const void* blob = sq.column_blob(st, 2);
        const int bytes = sq.column_bytes(st, 2);
        if (cols != 2 || !blob || rows <= 0 || (long long)bytes != (long long)rows * 2 * (long long)sizeof(uint32_t)) continue;
        const uint32_t* up = (const uint32_t*)blob;
        auto& vec = all_matches[k];
        vec.reserve((size_t)rows);
        for (int r = 0; r < rows; ++r) {
          int i1 = (int)up[2 * r], i2 = (int)up[2 * r + 1];
          if (swapped) std::swap(i1, i2);
          if (i1 >= 0 && i1 < (int)k1.size() && i2 >= 0 && i2 < (int)k2.size()) vec.emplace_back(i1, i2);
        }
      }
  }
  sq.finalize(st);
  sq.close(db);
  return true;
}

// ------------------------------------------------------------------------------------------------ camera poses from the LiDAR result
// updateCameraPosesFromLidar (:412-446): every image takes the correction T_opt * T_orig^-1 of the scan nearest in time
inline void update_camera_poses_from_lidar(const std::vector<Pose>& lidar_opt, const std::vector<Pose>& lidar_orig,
                                           const std::vector<Pose>& cam_orig, const std::vector<double>& images_ids, std::vector<Pose>& poses) {
  poses.clear();
  std::vector<double> ts;
  for (const auto& x : lidar_opt) ts.push_back(x.t);
  for (size_t i = 0; i < images_ids.size() && i < cam_orig.size(); ++i) {
    const double t_img = images_ids[i];
    const auto it = std::lower_bound(ts.begin(), ts.end(), t_img);
    size_t idx = (it == ts.end()) ? ts.size() - 1 : (size_t)(it - ts.begin());
    if (it != ts.begin() && it != ts.end()) {
      const size_t prev = idx - 1;
      if (std::abs(ts[prev] - t_img) < std::abs(ts[idx] - t_img)) idx = prev;
    }
    if (ts.empty() || idx >= lidar_opt.size() || idx >= lidar_orig.size()) { poses.push_back(cam_orig[i]); continue; }
    const M3 Ro = to_m3(lidar_opt[idx].R), Rb = to_m3(lidar_orig[idx].R);
    const M3 Rd = mul(Ro, tr(Rb));                                        // T_delta = T_opt * T_orig^-1
    const V3 a = mul(Rd, to_v3(lidar_orig[idx].p));
    Pose out = cam_orig[i];
    const M3 Rn = mul(Rd, to_m3(cam_orig[i].R));
    const V3 b = mul(Rd, to_v3(cam_orig[i].p));
    for (int k = 0; k < 9; ++k) out.R.m[k] = Rn.m[k];
    for (int k = 0; k < 3; ++k) out.p.v[k] = b(k) + lidar_opt[idx].p.v[k] - a(k);
    poses.push_back(out);
  }
}

// ------------------------------------------------------------------------------------------------ the visual stage
struct VisualResult {
  std::vector<M3> Rcw_before, Rcw_after;       // Rcw_all_ / Rcw_all_optimized_
  std::vector<V3> tcw_before, tcw_after;
  std::vector<FusedTrack> tracks;              // tracks_ (Xw_fused updated for the points the solver kept, :1658-1666)
  std::vector<uint8_t> track_used;             // per track: in the visual problem with a plane
  lvba_fuse_summary fuse{};
  lvba_depth_summary depth{};
  lvba_voxel_summary surf{};
  lvba_summary solve{};                        // the solve (with a reprojection filter: the second one)
  lvba_summary solve_first{};                  // with a reprojection filter: the solve before it
  int64_t obs_removed = 0, points_dropped = 0;  // with a reprojection filter: what it took out
  bool intr_refined = false;                   // with lvba_visual_opts::refine_intrinsics: intr holds the refined intrinsics
  double intr[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // fx fy cx cy d0 d1 d2 d3 after the solve (those of the config without refinement)
  int64_t usable_tracks = 0, points_kept = 0, keypoints = 0, matches = 0, anchor_points = 0, depth_valid = 0;
  int anchors = 0;
};

// The visual problem of one solve_visual call in a file, to re-run or inspect the solve elsewhere.  Native byte order:
//   char[8] "LVBAVP01"; int64 M, T, nnz; double intr[8], sigma_px, sigma_plane;
//   the state before the solve: double q[M*4] (w x y z), t[M*3], X[T*3]; double plane_nd[T*4]; int64 obs_ptr[T+1];
//   int32 obs_cam[nnz]; float obs_uv[nnz*2]; the state after the solve: double q[M*4], t[M*3], X[T*3]
// (the arguments of lvba_visual_lm, fixed_cam = 0).
inline bool write_visual_problem(const std::string& path, const std::vector<std::array<double, 4>>& q0,
                                 const std::vector<std::array<double, 3>>& t0, const std::vector<std::array<double, 3>>& X0,
                                 const std::vector<std::array<double, 3>>& plane_n, const std::vector<double>& plane_d,
                                 const std::vector<std::vector<Observation>>& obs, const double intr[8], double sigma_px,
                                 double sigma_plane, const std::vector<std::array<double, 4>>& q1,
                                 const std::vector<std::array<double, 3>>& t1, const std::vector<std::array<double, 3>>& X1) {
  std::ofstream f(path, std::ios::binary);
  if (!f) return false;
  auto put = [&](const void* p, size_t n) { if (n) f.write(static_cast<const char*>(p), (std::streamsize)n); };
  const int64_t M = (int64_t)q0.size(), T = (int64_t)X0.size();
  std::vector<int64_t> obs_ptr((size_t)T + 1, 0);
  std::vector<int32_t> obs_cam;
  std::vector<float> obs_uv;
  std::vector<double> plane_nd((size_t)T * 4);
  for (int64_t i = 0; i < T; ++i) {
    for (const auto& o : obs[(size_t)i]) { obs_cam.push_back(o.cam); obs_uv.push_back(o.u); obs_uv.push_back(o.v); }
    obs_ptr[(size_t)i + 1] = (int64_t)obs_cam.size();
    for (int k = 0; k < 3; ++k) plane_nd[4 * (size_t)i + k] = plane_n[(size_t)i][(size_t)k];
    plane_nd[4 * (size_t)i + 3] = plane_d[(size_t)i];
  }
  const int64_t nnz = (int64_t)obs_cam.size();
  const double sig[2] = {sigma_px, sigma_plane};
  put("LVBAVP01", 8); put(&M, 8); put(&T, 8); put(&nnz, 8); put(intr, 64); put(sig, 16);
  put(q0.data(), (size_t)M * 32); put(t0.data(), (size_t)M * 24); put(X0.data(), (size_t)T * 24);
  put(plane_nd.data(), plane_nd.size() * 8); put(obs_ptr.data(), obs_ptr.size() * 8);
  put(obs_cam.data(), obs_cam.size() * 4); put(obs_uv.data(), obs_uv.size() * 4);
  put(q1.data(), (size_t)M * 32); put(t1.data(), (size_t)M * 24); put(X1.data(), (size_t)T * 24);
  return (bool)f;
}

// the intrinsics of a config as the visual problem takes them: fx fy cx cy d0 d1 d2 d3
inline std::array<double, 8> cfg_intr(const Config& cfg) { return {cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3}; }

// A set of intrinsics groups as `focal,principal,distortion` (any non-empty comma-separated subset, each once) as an
// lvba_visual_opts::refine_intrinsics mask.  Anything else is refused with a message in *err; mask is then untouched.
inline bool parse_intr_groups(const char* text, uint32_t& mask, std::string* err = nullptr) {
  const std::string s = text ? text : "";
  uint32_t m = 0;
  size_t at = 0;
  while (true) {
    const size_t comma = s.find(',', at);
    const std::string g = s.substr(at, comma == std::string::npos ? std::string::npos : comma - at);
    uint32_t b;
    if (g == "focal") b = LVBA_INTR_FOCAL;
    else if (g == "principal") b = LVBA_INTR_PRINCIPAL;
    else if (g == "distortion") b = LVBA_INTR_DISTORTION;
    else { if (err) *err = "'" + s + "': a comma-separated list of focal, principal, distortion"; return false; }
    if (m & b) { if (err) *err = "'" + s + "': '" + g + "' is listed twice"; return false; }
    m |= b;
    if (comma == std::string::npos) break;
    at = comma + 1;
  }
  mask = m;
  return true;
}

// runVisualBAWithLidarAssist (:144-154) minus the drawing / publishing calls.  x_buf_opt / x_buf_before: the LiDAR poses after
// and before runLidarBA (equal when it was disabled); eigen_in_force: the eigen-ratio array the last set_eigen_ratio_array call
// left behind (stage 2's after runLidarBA, bavoxel.hpp:17 otherwise).  opts: the visual LM's options (null: the defaults).
// problem_path: when not empty, the problem of the solve and its result go there (write_visual_problem).
// reproj_filter_px > 0: solve_visual_remove_outliers(reproj_filter_px, min_track_len) instead of solve_visual; the landmarks it
// drops are treated as landmarks without a plane (neither written back nor listed as kept).  opts->refine_intrinsics != 0: the
// solve runs on a handle with the intrinsics a parameter block (solve_visual_refine_intrinsics, or the filter's handle) and
// res.intr gets the refined ones; otherwise res.intr is the config's.
inline int run_visual_ba(const Config& cfg, const std::vector<Cloud*>& pl_fulls, const std::vector<Pose>& x_buf_opt,
                         const std::vector<Pose>& x_buf_before, const std::vector<double>& images_ids, const std::vector<Pose>& image_poses,
                         const KeypointImages& all_keypoints, const MatchTable& all_matches, const float eigen_in_force[4],
                         VisualResult& res, std::string* err = nullptr, const lvba_visual_opts* opts = nullptr,
                         const std::string& problem_path = std::string(), double reproj_filter_px = 0.0, int32_t min_track_len = 3) {
  const int M = (int)images_ids.size();
  if ((int)image_poses.size() != M) { if (err) *err = "Number of images and poses do not match"; return LVBA_ERR_INVALID_ARG; }      // :458-461
  if ((int)all_keypoints.size() != M) { if (err) *err = "all_keypoints.size() must equal #cameras"; return LVBA_ERR_INVALID_ARG; }  // :1429
  M3 Rci; V3 tci;
  camera_from_body(cfg, Rci, tci);
  std::vector<Pose> poses;
  update_camera_poses_from_lidar(x_buf_opt, x_buf_before, image_poses, images_ids, poses);
  res.Rcw_before.resize((size_t)M); res.tcw_before.resize((size_t)M); res.Rcw_after.resize((size_t)M); res.tcw_after.resize((size_t)M);
  for (int i = 0; i < M; ++i) {
    world_to_camera(poses[(size_t)i], Rci, tci, res.Rcw_after[(size_t)i], res.tcw_after[(size_t)i]);
    world_to_camera(image_poses[(size_t)i], Rci, tci, res.Rcw_before[(size_t)i], res.tcw_before[(size_t)i]);
  }
  // buildGridMapFromOptimized + generateDepthWithVoxel + the depth candidates of BuildTracksAndFuse3D (:1020-1038)
  DepthRenderer renderer;
  int rc = renderer.buildGridMapFromOptimized(pl_fulls, x_buf_opt, 0.5, &res.depth);
  if (rc != LVBA_OK) { if (err) *err = std::string("depth grid: ") + lvba_last_error(); return rc; }
  std::vector<double> kp_Xw;
  std::vector<uint8_t> kp_valid;
  rc = renderer.backproject(res.Rcw_after, res.tcw_after, images_ids, all_keypoints, cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3,
                            cfg.width, cfg.height, kp_Xw, kp_valid, 0.5, &res.depth);
  if (rc != LVBA_OK) { if (err) *err = std::string("depth candidates: ") + lvba_last_error(); return rc; }
  renderer.clear();
  res.keypoints = (int64_t)kp_valid.size();
  for (uint8_t v : kp_valid) res.depth_valid += v != 0;
  for (const auto& m : all_matches) res.matches += (int64_t)m.size();
  // BuildTracksAndFuse3D
  lvba_fuse_opts fo;
  lvba_fuse_default_opts(&fo);
  fo.min_view_angle_deg = cfg.min_view_angle; fo.reproj_mean_thr_px = cfg.reproj_mean_thr; fo.map_order = cfg.fuse_map_order;
  rc = build_tracks_and_fuse_3d(all_keypoints, all_matches, res.Rcw_after, res.tcw_after, cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3,
                                kp_Xw, kp_valid, res.tracks, &fo, &res.fuse);
  if (rc != LVBA_OK) { if (err) *err = std::string("track fusion: ") + lvba_last_error(); return rc; }
  res.track_used.assign(res.tracks.size(), 0);
  // optimizeCameraPoses (:1422-1669)
  std::vector<int> track_ids;
  for (int i = 0; i < (int)res.tracks.size(); ++i) {
    const auto& t = res.tracks[(size_t)i];
    const bool zero = std::abs(t.Xw_fused[0]) <= 1e-12 && std::abs(t.Xw_fused[1]) <= 1e-12 && std::abs(t.Xw_fused[2]) <= 1e-12;
    const bool finite = std::isfinite(t.Xw_fused[0]) && std::isfinite(t.Xw_fused[1]) && std::isfinite(t.Xw_fused[2]);
    if ((int)t.observations.size() >= fo.obser_thr && !zero && finite) track_ids.push_back(i);       // :1434-1439
  }
  res.usable_tracks = (int64_t)track_ids.size();
  if (track_ids.empty()) return LVBA_OK;                                                               // :1441-1444: warning, poses unchanged
  const int total = (int)std::min(pl_fulls.size(), x_buf_opt.size());
  if (total == 0) return LVBA_OK;
  // anchors of the visual stage (:1470-1490): no window LM, the frames are merged with their optimised relative poses
  const int window = cfg.window_size > 0 ? cfg.window_size : 1;
  std::vector<int32_t> win_ptr{0};
  std::vector<int64_t> scan_ptr{0};
  std::vector<double> rel;
  std::vector<Pose> anchor_poses;
  for (int start = 0; start < total; start += window) {
    const int end = std::min(start + window, total);
    const M3 Ra_t = tr(to_m3(x_buf_opt[(size_t)start].R));
    for (int j = start; j < end; ++j) {
      const M3 Rr = mul(Ra_t, to_m3(x_buf_opt[(size_t)j].R));
      V3 d{};
      for (int k = 0; k < 3; ++k) d(k) = x_buf_opt[(size_t)j].p.v[k] - x_buf_opt[(size_t)start].p.v[k];
      const V3 pr = mul(Ra_t, d);
      rel.insert(rel.end(), Rr.m, Rr.m + 9);
      rel.insert(rel.end(), pr.v, pr.v + 3);
      scan_ptr.push_back(scan_ptr.back() + (int64_t)pl_fulls[(size_t)j]->points.size());
    }
    win_ptr.push_back((int32_t)scan_ptr.size() - 1);
    anchor_poses.push_back(x_buf_opt[(size_t)start]);
  }
  std::vector<float> xyz((size_t)scan_ptr.back() * 3);
  for (int j = 0; j < total; ++j) {
    float* dst = xyz.data() + 3 * (size_t)scan_ptr[(size_t)j];
    for (const auto& pt : pl_fulls[(size_t)j]->points) { *dst++ = pt.x; *dst++ = pt.y; *dst++ = pt.z; }
  }
  const int n_anchor = (int)anchor_poses.size();
  lvba_anchor_clouds* ac = nullptr;
  int64_t n_pts = 0;
  rc = lvba_anchor_clouds_create(n_anchor, win_ptr.data(), scan_ptr.data(), xyz.data(), 3, rel.data(), cfg.anchor_leaf, -1, &ac, &n_pts);
  if (rc != LVBA_OK) { if (err) *err = std::string("anchor clouds: ") + lvba_last_error(); return rc; }
  std::vector<int64_t> cloud_ptr((size_t)n_anchor + 1);
  std::vector<float> merged((size_t)n_pts * 3);
  rc = lvba_anchor_clouds_export(ac, cloud_ptr.data(), merged.data(), nullptr);
  lvba_anchor_clouds_destroy(ac);
  if (rc != LVBA_OK) { if (err) *err = std::string("anchor clouds: ") + lvba_last_error(); return rc; }
  res.anchors = n_anchor; res.anchor_points = n_pts;
  std::vector<AnchorCloud> clouds((size_t)n_anchor);
  std::vector<AnchorCloud*> cloud_ptrs;
  for (int a = 0; a < n_anchor; ++a) {
    for (int64_t q = cloud_ptr[(size_t)a]; q < cloud_ptr[(size_t)a + 1]; ++q) clouds[(size_t)a].points.push_back({merged[3 * q], merged[3 * q + 1], merged[3 * q + 2]});
    cloud_ptrs.push_back(&clouds[(size_t)a]);
  }
  // surf_map (:1498-1507) and the plane of every landmark (:1529-1569)
  SurfMap<std::vector<Pose>> surf;
  rc = surf.build(cloud_ptrs, anchor_poses, cfg.stage2_voxel, eigen_in_force, &res.surf);
  if (rc != LVBA_OK) { if (err) *err = std::string("surf map: ") + lvba_last_error(); return rc; }
  const int Npts = (int)track_ids.size();
  std::vector<std::array<double, 4>> qs((size_t)M);
  std::vector<std::array<double, 3>> ts((size_t)M), Xs((size_t)Npts), plane_n;
  std::vector<double> plane_d;
  for (int k = 0; k < M; ++k) {
    double q[4];
    eigen_quaternion(res.Rcw_after[(size_t)k], q);
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    qs[(size_t)k] = {q[0] / n, q[1] / n, q[2] / n, q[3] / n};
    ts[(size_t)k] = {res.tcw_after[(size_t)k](0), res.tcw_after[(size_t)k](1), res.tcw_after[(size_t)k](2)};
  }
  for (int pi = 0; pi < Npts; ++pi) Xs[(size_t)pi] = res.tracks[(size_t)track_ids[(size_t)pi]].Xw_fused;
  rc = surf.recompute_local_planes(Xs, plane_n, plane_d);
  if (rc != LVBA_OK) { if (err) *err = std::string("plane lookup: ") + lvba_last_error(); return rc; }
  surf.clear();
  // observation lists (:1610-1631): the inliers, each once, cameras in range
  std::vector<std::vector<Observation>> obs((size_t)Npts);
  for (int pi = 0; pi < Npts; ++pi) {
    const auto& t = res.tracks[(size_t)track_ids[(size_t)pi]];
    std::unordered_set<int> seen;
    for (int idx : t.inlier_indices) {
      if (idx < 0 || idx >= (int)t.observations.size() || !seen.insert(idx).second) continue;
      const int cam = t.observations[(size_t)idx].first, kp = t.observations[(size_t)idx].second;
      if (cam < 0 || cam >= M) continue;
      obs[(size_t)pi].push_back({cam, all_keypoints[(size_t)cam][(size_t)kp].x, all_keypoints[(size_t)cam][(size_t)kp].y});
    }
  }
  const std::vector<std::array<double, 4>> qs0 = qs;
  const std::vector<std::array<double, 3>> ts0 = ts, Xs0 = Xs;
  std::vector<uint8_t> dropped((size_t)Npts, 0);
  const uint32_t refine = opts ? opts->refine_intrinsics : 0u;
  double intr[8] = {cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3};
  if (reproj_filter_px > 0.0) {
    std::vector<std::vector<uint8_t>> removed;
    rc = solve_visual_remove_outliers(qs, ts, Xs, plane_n, plane_d, obs, cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3, 0.5, 0.01,
                                      opts, reproj_filter_px, min_track_len, &removed, &res.solve_first, &res.solve, nullptr,
                                      refine ? intr : nullptr);
    for (int pi = 0; rc == LVBA_OK && pi < Npts; ++pi) {
      const auto& r = removed[(size_t)pi];
      for (uint8_t b : r) res.obs_removed += b != 0;
      dropped[(size_t)pi] = !r.empty() && std::all_of(r.begin(), r.end(), [](uint8_t b) { return b != 0; });
      res.points_dropped += dropped[(size_t)pi];
    }
  } else if (refine) {
    rc = solve_visual_refine_intrinsics(qs, ts, Xs, plane_n, plane_d, obs, intr[0], intr[1], intr[2], intr[3], intr[4], intr[5], intr[6],
                                        intr[7], refine, 0.5, 0.01, opts, &res.solve);
  } else {
    rc = solve_visual(qs, ts, Xs, plane_n, plane_d, obs, cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3, 0.5, 0.01, opts, &res.solve);
  }
  if (rc != LVBA_OK) { if (err) *err = std::string("visual LM: ") + lvba_last_error(); return rc; }
  if (!problem_path.empty()) {
    const double intr[8] = {cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.d0, cfg.d1, cfg.d2, cfg.d3};
    if (!write_visual_problem(problem_path, qs0, ts0, Xs0, plane_n, plane_d, obs, intr, 0.5, 0.01, qs, ts, Xs)) {
      if (err) *err = "cannot write " + problem_path;
      return LVBA_ERR_INVALID_ARG;
    }
  }
  const std::array<double, 8> given = cfg_intr(cfg);
  std::copy(given.begin(), given.end(), res.intr);
  if (res.solve.termination == LVBA_TERM_INVALID_STEPS) return LVBA_OK;                                // ceres::FAILURE, :1647-1650: nothing written back
  if (refine) { std::copy(intr, intr + 8, res.intr); res.intr_refined = true; }
  for (int k = 0; k < M; ++k) {                                                                       // :1652-1656
    const auto& q = qs[(size_t)k];
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    double R[9];
    dataset::quat_to_R(q[0] / n, q[1] / n, q[2] / n, q[3] / n, R);
    for (int e = 0; e < 9; ++e) res.Rcw_after[(size_t)k].m[e] = R[e];
    for (int e = 0; e < 3; ++e) res.tcw_after[(size_t)k](e) = ts[(size_t)k][(size_t)e];
  }
  for (int pi = 0; pi < Npts; ++pi) {                                                                  // :1658-1666
    const auto& n = plane_n[(size_t)pi];
    const bool has_plane = std::isfinite(n[0]) && std::isfinite(n[1]) && std::isfinite(n[2]) && std::isfinite(plane_d[(size_t)pi]) &&
                           !(std::abs(n[0]) <= 1e-6 && std::abs(n[1]) <= 1e-6 && std::abs(n[2]) <= 1e-6);
    if (!has_plane || dropped[(size_t)pi]) continue;
    res.tracks[(size_t)track_ids[(size_t)pi]].Xw_fused = Xs[(size_t)pi];
    res.track_used[(size_t)track_ids[(size_t)pi]] = 1;
    ++res.points_kept;
  }
  return LVBA_OK;
}

// ------------------------------------------------------------------------------------------------ COLMAP text model
// images.txt as written at :2018-2024: `k qw qx qy qz tx ty tz 1 k.jpg` then the empty observation line `0.0 0.0 -1`
inline bool write_images_txt(const std::string& file, const std::vector<M3>& Rcw, const std::vector<V3>& tcw, const std::vector<uint8_t>* listed = nullptr) {
  FILE* f = std::fopen(file.c_str(), "w");
  if (!f) return false;
  for (size_t k = 0; k < Rcw.size(); ++k) {
    if (listed && k < listed->size() && !(*listed)[k]) continue;          // the reference skips an image without LiDAR in its window before this line (:1994-1997)
    double q[4];
    eigen_quaternion(Rcw[k], q);
    std::fprintf(f, "%zu %.6f %.6f %.6f %.6f %.6f %.6f %.6f 1 %zu.jpg\n0.0 0.0 -1\n", k, q[0], q[1], q[2], q[3], tcw[k](0), tcw[k](1), tcw[k](2), k);
  }
  return std::fclose(f) == 0;
}
// points3D.txt as written at :2125-2136: `i x y z r g b 0`.  The reference colours LiDAR points from the images (OpenCV); here the
// points are the fused landmarks the visual problem kept, in grey — image decoding is outside this library.
inline bool write_points3D_txt(const std::string& file, const std::vector<FusedTrack>& tracks, const std::vector<uint8_t>& used) {
  FILE* f = std::fopen(file.c_str(), "w");
  if (!f) return false;
  size_t i = 0;
  for (size_t t = 0; t < tracks.size(); ++t) {
    if (t < used.size() && !used[t]) continue;
    std::fprintf(f, "%zu %.6f %.6f %.6f 128 128 128 0\n", i++, tracks[t].Xw_fused[0], tracks[t].Xw_fused[1], tracks[t].Xw_fused[2]);
  }
  return std::fclose(f) == 0;
}

// ------------------------------------------------------------------------------------------------ the reference's points3D.txt
// VisualizeOptComparison (src/lvba_system.cpp:1932-2143) does not write the fused landmarks: per image it takes the scans within +-0.5 s (:1971-1974),
// moves them to the world with the optimised LiDAR poses and stores them as FLOAT (:1980-1986), keeps per pixel (rounded projection, :2043-2045) the point
// nearest to the camera (`zc + 1e-6f < zbuf`, :2050), appends the survivors in pixel order (:2064-2067), and after all images thins the union with
// down_sampling_voxel2 at colmap_output/filter_size_points3D (:2119).  The colour comes from the decoded image — image decoding is outside this library, so
// the rows below carry (128, 128, 128); positions and the choice of points are the reference's.  An image whose window holds no LiDAR point is skipped —
// in images.txt too (:1994-1997 precede the pose line): `written` reports which images the reference would list.
// The reference returns the thinned set in unordered_map order; here the rows follow ascending voxel key.
struct LidarPoint3D { float x, y, z; };
inline void colmap_points_from_lidar(const Config& cfg, const std::vector<Cloud*>& pl_fulls, const std::vector<Pose>& x_buf_opt, const std::vector<double>& images_ids,
                                     const std::vector<M3>& Rcw, const std::vector<V3>& tcw, std::vector<LidarPoint3D>& out, std::vector<uint8_t>* written = nullptr) {
  const int W = cfg.width, H = cfg.height;
  std::vector<LidarPoint3D> merged;
  if (written) written->assign(images_ids.size(), 0);
  std::vector<float> zbuf;
  std::vector<LidarPoint3D> pix;
  for (size_t k = 0; k < images_ids.size() && k < Rcw.size(); ++k) {
    std::vector<LidarPoint3D> cloud;
    for (size_t idx = 0; idx < x_buf_opt.size() && idx < pl_fulls.size(); ++idx) {
      if (std::fabs(x_buf_opt[idx].t - images_ids[k]) > 0.5) continue;
      const M3 R = to_m3(x_buf_opt[idx].R);
      const V3 p = to_v3(x_buf_opt[idx].p);
      for (const auto& pb : pl_fulls[idx]->points) {
        const V3 xb{{(double)pb.x, (double)pb.y, (double)pb.z}};
        const V3 xw = mul(R, xb);
        cloud.push_back(LidarPoint3D{(float)(xw(0) + p(0)), (float)(xw(1) + p(1)), (float)(xw(2) + p(2))});
      }
    }
    if (cloud.empty()) continue;
    if (written) (*written)[k] = 1;
    zbuf.assign((size_t)W * H, std::numeric_limits<float>::infinity());
    pix.assign((size_t)W * H, LidarPoint3D{0, 0, 0});
    const float eps = 1e-6f;
    for (const auto& q : cloud) {
      const V3 xw{{(double)q.x, (double)q.y, (double)q.z}};
      const V3 rc = mul(Rcw[k], xw);
      const double X = rc(0) + tcw[k](0), Y = rc(1) + tcw[k](1), Z = rc(2) + tcw[k](2);          // projectWorldToPixel, include/utils.hpp:183-205
      if (!(std::isfinite(X) && std::isfinite(Y) && std::isfinite(Z)) || Z <= 1e-12) continue;
      const double x = X / Z, y = Y / Z;
      const double r2 = x * x + y * y, r4 = r2 * r2;
      const double radial = 1.0 + cfg.d0 * r2 + cfg.d1 * r4;
      const double x_tan = 2.0 * cfg.d2 * x * y + cfg.d3 * (r2 + 2.0 * x * x);
      const double y_tan = cfg.d2 * (r2 + 2.0 * y * y) + 2.0 * cfg.d3 * x * y;
      const double xd = x * radial + x_tan, yd = y * radial + y_tan;
      if (!(std::isfinite(xd) && std::isfinite(yd))) continue;
      const double u = cfg.fx * xd + cfg.cx, v = cfg.fy * yd + cfg.cy;
      if (!(std::isfinite(u) && std::isfinite(v))) continue;
      const int uu = (int)std::round(u), vv = (int)std::round(v);
      if (uu < 0 || uu >= W || vv < 0 || vv >= H) continue;
      const size_t i = (size_t)vv * W + uu;
      if (Z + eps < zbuf[i]) { zbuf[i] = (float)Z; pix[i] = q; }
    }
    for (size_t i = 0; i < zbuf.size(); ++i) if (std::isfinite(zbuf[i])) merged.push_back(pix[i]);
  }
  // down_sampling_voxel2 (include/BALM/tools.hpp:301-359): per voxel the original point nearest to the voxel centre, the first one on ties
  out.clear();
  const double leaf = cfg.filter_size_points3D;
  if (leaf < 0.001) { out = merged; return; }
  struct Best { double d2; size_t i; };
  std::map<std::array<int64_t, 3>, Best> best;
  for (size_t i = 0; i < merged.size(); ++i) {
    const float c[3] = {merged[i].x, merged[i].y, merged[i].z};
    std::array<int64_t, 3> key; double d2 = 0.0, d[3];
    for (int j = 0; j < 3; ++j) {
      float loc = (float)(c[j] / leaf);
      if (loc < 0.f) loc -= 1.f;
      key[j] = (int64_t)loc;
      d[j] = (double)c[j] - ((double)key[j] + 0.5) * leaf;
    }
    d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    auto it = best.find(key);
    if (it == best.end()) best.emplace(key, Best{d2, i});
    else if (d2 < it->second.d2) it->second = Best{d2, i};
  }
  for (const auto& kv : best) out.push_back(merged[kv.second.i]);
}
inline bool write_points3D_lidar_txt(const std::string& file, const std::vector<LidarPoint3D>& pts) {
  FILE* f = std::fopen(file.c_str(), "w");
  if (!f) return false;
  for (size_t i = 0; i < pts.size(); ++i) std::fprintf(f, "%zu %.6f %.6f %.6f 128 128 128 0\n", i, pts[i].x, pts[i].y, pts[i].z);
  return std::fclose(f) == 0;
}

}  // namespace offline
}  // namespace lvba_b200
