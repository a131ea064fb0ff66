// ref_colorize_driver.cpp — TEST INFRASTRUCTURE: the reference's own VisualizeOptComparison (src/lvba_system.cpp:1932-2143, compiled
// where it lies through oracle/ref_system_driver.cpp and the stand-in headers of oracle/ref_shim/) run on caller-supplied images, so that
// the colour half of boundary B8 — BGR -> RGB (:2051-2055), img(vv, uu), the `before` cloud of x_buf_before_ under Rcw_all_ / tcw_all_
// (:2000-2001, :2079) — is held against the reference itself.  The stand-in cv::imread reads every file as empty or as one grey value;
// here cv::imread is routed to images registered per path, in the BGR byte order cv::Mat holds.  Never part of the product; built by
// tests/test_ref_colorize_pin.py where the reference source exists.
#include <opencv2/opencv.hpp>

#include <map>
#include <string>

namespace lvba_colorize_test {
inline std::map<std::string, cv::Mat>& images() { static std::map<std::string, cv::Mat> m; return m; }
}  // namespace lvba_colorize_test
namespace cv {
inline Mat colour_imread(const std::string& path, int = IMREAD_COLOR) {
  const auto it = lvba_colorize_test::images().find(path);
  return it == lvba_colorize_test::images().end() ? Mat() : it->second.clone();
}
}  // namespace cv
#define imread colour_imread
#include "../../oracle/ref_system_driver.cpp"
#undef imread

extern "C" {

void colz_clear_images() { lvba_colorize_test::images().clear(); }
// rows x cols pixels, 3 bytes each in B, G, R order (what cv::imread(IMREAD_COLOR) returns)
void colz_add_image(const char* path, int rows, int cols, const uint8_t* bgr) {
  cv::Mat m(rows, cols, CV_8UC3);
  for (int y = 0; y < rows; ++y)
    for (int x = 0; x < cols; ++x) {
      const uint8_t* p = bgr + 3 * ((size_t)y * cols + x);
      m.at<cv::Vec3b>(y, x) = cv::Vec3b(p[0], p[1], p[2]);
    }
  lvba_colorize_test::images()[path] = m;
}

// Sets what VisualizeOptComparison reads — pl_fulls_, x_buf_ (optimised), x_buf_before_, images_ids_, Rcw/tcw_all_optimized_ (after),
// Rcw/tcw_all_ (before), the camera model, colmap_output/filter_size_points3D — and runs it with dataset_path_ = `dir` (images are
// looked up as dir + "all_image/" + std::to_string(id) + ".png").  Returns the sizes of the after / before clouds it keeps.
void colz_run(void* h, const char* dir, int F, const int64_t* scan_ptr, const float* xyz, const double* frame_ts, const double* poses_after,
              const double* poses_before, int M, const double* image_ts, const double* cams_after, const double* cams_before, const double* intr,
              int width, int height, double leaf, int64_t* n_after, int64_t* n_before) {
  auto& s = *static_cast<Sys*>(h)->s;
  auto& d = *s.dataset_io_;
  d.x_buf_.clear(); d.x_buf_before_.clear(); d.pl_fulls_.clear();
  for (int j = 0; j < F; ++j) {
    d.x_buf_.push_back(pose_in(poses_after + 12 * j, frame_ts[j]));
    d.x_buf_before_.push_back(pose_in(poses_before + 12 * j, frame_ts[j]));
    pcl::PointCloud<PointType>::Ptr pl(new pcl::PointCloud<PointType>());
    for (int64_t k = scan_ptr[j]; k < scan_ptr[j + 1]; ++k) { PointType p; p.x = xyz[3 * k]; p.y = xyz[3 * k + 1]; p.z = xyz[3 * k + 2]; pl->push_back(p); }
    d.pl_fulls_.push_back(pl);
  }
  s.images_ids_.assign(image_ts, image_ts + M);
  s.Rcw_all_optimized_.assign(M, Eigen::Matrix3d()); s.tcw_all_optimized_.assign(M, Eigen::Vector3d());
  s.Rcw_all_.assign(M, Eigen::Matrix3d()); s.tcw_all_.assign(M, Eigen::Vector3d());
  for (int k = 0; k < M; ++k) {
    const IMUST a = pose_in(cams_after + 12 * k, 0), b = pose_in(cams_before + 12 * k, 0);
    s.Rcw_all_optimized_[k] = a.R; s.tcw_all_optimized_[k] = a.p; s.Rcw_all_[k] = b.R; s.tcw_all_[k] = b.p;
  }
  s.image_width_ = width; s.image_height_ = height; s.scale_ = 1.0;
  s.fx_ = intr[0]; s.fy_ = intr[1]; s.cx_ = intr[2]; s.cy_ = intr[3]; s.d0_ = intr[4]; s.d1_ = intr[5]; s.d2_ = intr[6]; s.d3_ = intr[7];
  s.colmap_output_enable_ = true; s.filter_size_points3D_ = leaf;
  s.dataset_path_ = dir;
  s.VisualizeOptComparison(s.images_ids_, true);
  s.fout_poses_after.close(); s.fout_points_after.close();
  *n_after = s.pub_cloud_ ? (int64_t)s.pub_cloud_->size() : 0;
  *n_before = s.pub_cloud_b_ ? (int64_t)s.pub_cloud_b_->size() : 0;
}

// which = 0: the after cloud (colored_merged_after.pcd, points3D.txt), 1: the before cloud; rgb in R, G, B order
void colz_cloud(void* h, int which, float* xyz, uint8_t* rgb) {
  auto& s = *static_cast<Sys*>(h)->s;
  const auto& c = which == 0 ? s.pub_cloud_ : s.pub_cloud_b_;
  for (size_t i = 0; i < c->size(); ++i) {
    const auto& p = c->points[i];
    xyz[3 * i] = p.x; xyz[3 * i + 1] = p.y; xyz[3 * i + 2] = p.z;
    rgb[3 * i] = p.r; rgb[3 * i + 1] = p.g; rgb[3 * i + 2] = p.b;
  }
}

}  // extern "C"
