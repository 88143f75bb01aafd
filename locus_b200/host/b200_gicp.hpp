// b200_gicp.hpp -- C++ host-side mirror of the reference's registration / filter interface
// above the C ABI (include/locus_b200.h).  Header-only, no PCL / ROS / Eigen needed.
//
// The reference's callers hold a pcl::Registration<PointF,PointF>::Ptr
// (point_cloud_odometry/include/point_cloud_odometry/PointCloudOdometry.h:154,
//  point_cloud_localization/include/point_cloud_localization/PointCloudLocalization.h:228)
// and call exactly this surface on it (PointCloudOdometry.cc:147-155,265-269;
// PointCloudLocalization.cc:234-245,306-336).  B200Gicp keeps the same method names, argument
// meaning and error behaviour; shim/b200_gicp_pcl.hpp wraps it into a real
// pcl::Registration subclass when PCL is available.
#pragma once

#include <array>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/locus_b200.h"

namespace locus_b200 {

// Byte-compatible with pcl::PointXYZINormal (= PointF of frontend_utils): 48 bytes.
struct PointF {
  float x, y, z, data3;
  float normal_x, normal_y, normal_z, normal3;
  float intensity, curvature, pad0, pad1;
};
static_assert(sizeof(PointF) == 48, "PointF must match pcl::PointXYZINormal");

using Matrix4f = std::array<float, 16>;  // row-major

class B200Gicp {
 public:
  explicit B200Gicp(int device = 0) {
    if (lb_gicp_create(device, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
    lb_gicp_default_params(&p_);
  }
  ~B200Gicp() { lb_gicp_destroy(h_); }
  B200Gicp(const B200Gicp&) = delete;
  B200Gicp& operator=(const B200Gicp&) = delete;

  // ---- configuration: same names as gicp.h:134-143,264-298 and pcl::Registration
  void setTransformationEpsilon(double e) { p_.transformation_epsilon = e; apply(); }
  void setMaxCorrespondenceDistance(double d) { p_.max_correspondence_distance = d; apply(); }
  void setMaximumIterations(int n) { p_.max_iterations = n; apply(); }
  void setRANSACIterations(int n) { p_.ransac_iterations = n; apply(); }
  void setMaximumOptimizerIterations(int n) { p_.max_optimizer_iterations = n; apply(); }
  void setNumThreads(int n) { p_.num_threads = n; apply(); }          // accepted; the GPU path ignores it
  void enableTimingOutput(bool e) { p_.enable_timing_output = e; apply(); }
  void RecomputeTargetCovariance(bool r) { p_.recompute_target_covariance = r; apply(); }
  void RecomputeSourceCovariance(bool r) { p_.recompute_source_covariance = r; apply(); }
  void setEuclideanFitnessEpsilon(double e) { p_.euclidean_fitness_epsilon = e; apply(); }
  void setRotationEpsilon(double e) { p_.rotation_epsilon = e; apply(); }
  void setCorrespondenceRandomness(int k) { p_.k_correspondences = k; apply(); }
  double getTransformationEpsilon() const { return p_.transformation_epsilon; }
  double getMaxCorrespondenceDistance() const { return p_.max_correspondence_distance; }
  int getMaximumIterations() const { return p_.max_iterations; }
  int getMaximumOptimizerIterations() const { return p_.max_optimizer_iterations; }
  int getCorrespondenceRandomness() const { return p_.k_correspondences; }
  double getRotationEpsilon() const { return p_.rotation_epsilon; }
  std::string getClassName() const { return "B200GeneralizedIterativeClosestPoint"; }

  // ---- clouds (borrowed for the duration of the call)
  // gicp.h:162-179: an empty source is an error and leaves the previous input in place.
  bool setInputSource(const PointF* pts, size_t n, bool has_normals = true) {
    n_src_ = n;
    return lb_gicp_set_source(h_, pts, n, sizeof(PointF), 0, has_normals ? 16 : LB_NO_NORMALS, LB_MEM_HOST) == LB_OK;
  }
  bool setInputTarget(const PointF* pts, size_t n, bool has_normals = true) {
    return lb_gicp_set_target(h_, pts, n, sizeof(PointF), 0, has_normals ? 16 : LB_NO_NORMALS, LB_MEM_HOST, nullptr) == LB_OK;
  }

  // align(output, guess): output = final_transformation * input (gicp.hpp:586).  Returns false and keeps the
  // last good transform on failure (gicp.hpp:542-547).
  bool align(std::vector<PointF>* output, const Matrix4f* guess = nullptr) {
    int s = lb_gicp_align(h_, guess ? guess->data() : nullptr, &r_);
    if (s != LB_OK) return false;
    if (output) {
      // the caller's cloud keeps every non-geometric field; only xyz / normals are rewritten
      if (output->size() != n_src_) output->resize(n_src_);
      lb_gicp_transform_source(h_, nullptr, output->data(), sizeof(PointF), 0, LB_NO_NORMALS, LB_MEM_HOST);
    }
    return true;
  }
  Matrix4f getFinalTransformation() const {
    Matrix4f m;
    for (int i = 0; i < 16; i++) m[i] = r_.final_transformation[i];
    return m;
  }
  bool hasConverged() const { return r_.converged != 0; }
  double getFitnessScore(double max_range = 1.7976931348623157e308) {
    double s = 0;
    lb_gicp_fitness(h_, nullptr, max_range, &s);
    return s;
  }
  // getSearchMethodTarget()->nearestKSearch(point, 1, idx, d2) for a batch (PointCloudLocalization.cc:327-336)
  bool nearestKSearchTarget(const PointF* pts, size_t n, int32_t* idx, float* d2) {
    return lb_gicp_nn_target(h_, pts, n, sizeof(PointF), idx, d2, LB_MEM_HOST) == LB_OK;
  }
  // the ICP covariance after align (PointCloudLocalization.cc:325-336,398-421): the final transformation, the 1-NN of
  // every aligned point and the target's normals (rotated by normal_rotation, 3x3 row-major, when given)
  bool icpCovariance(lb_icp_covariance* out, double max_covariance = 0.01, const float* normal_rotation = nullptr) {
    return lb_gicp_icp_covariance(h_, nullptr, nullptr, LB_MEM_HOST, normal_rotation, max_covariance, out) == LB_OK;
  }
  // point_cloud_filter::NormalComputation::filter, k-NN mode (normal_computation.cc:26-59): writes normal_x/y/z of
  // every point of `cloud` (the curvature field is left alone, as the nodelet does).  3 <= k <= 20.
  bool computeNormals(PointF* cloud, size_t n, int k = 20) {
    if (lb_gicp_set_source(h_, cloud, n, sizeof(PointF), 0, LB_NO_NORMALS, LB_MEM_HOST) != LB_OK) return false;
    n_src_ = n;
    std::vector<float> nrm(4 * n);
    if (lb_gicp_compute_normals(h_, 0, k, nullptr, nrm.data(), LB_MEM_HOST) != LB_OK) return false;
    for (size_t i = 0; i < n; i++) {
      cloud[i].normal_x = nrm[4 * i]; cloud[i].normal_y = nrm[4 * i + 1]; cloud[i].normal_z = nrm[4 * i + 2];
    }
    return true;
  }
  // pcl::StatisticalOutlierRemoval (PointCloudFilter.cc:126-133) / pcl::RadiusOutlierRemoval (PointCloudFilter.cc:135-143,
  // PointCloudMerger.cc:112-117) on `cloud`, in place: the kept points stay, in input order.  `dense` is the cloud's
  // is_dense (PCL's branch of the radius filter).  Like computeNormals, the cloud becomes the handle's source.
  bool statisticalOutlierRemoval(std::vector<PointF>& cloud, int mean_k = 10, double std_mul = 1.0, bool negative = false) {
    return filterInPlace(cloud, [&](int32_t* kept, size_t* m) {
      return lb_gicp_statistical_outlier_removal(h_, 0, mean_k, std_mul, negative ? 1 : 0, kept, m, nullptr, nullptr, LB_MEM_HOST);
    });
  }
  bool radiusOutlierRemoval(std::vector<PointF>& cloud, double radius = 0.15, int min_neighbors = 3, bool dense = true,
                            bool negative = false) {
    return filterInPlace(cloud, [&](int32_t* kept, size_t* m) {
      return lb_gicp_radius_outlier_removal(h_, 0, radius, min_neighbors, dense ? 1 : 0, negative ? 1 : 0, kept, m, LB_MEM_HOST);
    });
  }
  const lb_gicp_result& result() const { return r_; }
  lb_gicp* handle() { return h_; }

 private:
  void apply() {
    if (lb_gicp_set_params(h_, &p_) != LB_OK) throw std::invalid_argument(lb_last_error_string());
  }
  template <class Run>
  bool filterInPlace(std::vector<PointF>& cloud, Run&& run) {
    if (lb_gicp_set_source(h_, cloud.data(), cloud.size(), sizeof(PointF), 0, LB_NO_NORMALS, LB_MEM_HOST) != LB_OK) return false;
    n_src_ = cloud.size();
    std::vector<int32_t> kept(cloud.size());
    size_t m = 0;
    if (run(kept.data(), &m) != LB_OK) return false;
    for (size_t j = 0; j < m; j++) cloud[j] = cloud[(size_t)kept[j]];    // kept[j] >= j: a forward pass is safe
    cloud.resize(m);
    return true;
  }
  lb_gicp* h_ = nullptr;
  lb_gicp_params p_{};
  lb_gicp_result r_{};
  size_t n_src_ = 0;
};

// Mirror of pclomp::NormalDistributionsTransform<PointF, PointF> as LOCUS sets it up when `registration_method: ndt`
// (PointCloudOdometry.cc:182-195, PointCloudLocalization.cc:267-280; setters of multithreaded_ndt/ndt_omp.h:116-196).
// Same call sequence as B200Gicp: setInputSource / setInputTarget / align / getFinalTransformation.
class B200Ndt {
 public:
  explicit B200Ndt(int device = 0) {
    lb_ndt_default_params(&p_);
    if (lb_ndt_create(device, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
  }
  ~B200Ndt() { lb_ndt_destroy(h_); }
  B200Ndt(const B200Ndt&) = delete;
  B200Ndt& operator=(const B200Ndt&) = delete;

  void setTransformationEpsilon(double e) { p_.transformation_epsilon = e; apply(); }
  void setMaxCorrespondenceDistance(double d) { p_.max_correspondence_distance = d; apply(); }   // accepted; NDT has no gate
  void setMaximumIterations(int n) { p_.max_iterations = n; apply(); }
  void setRANSACIterations(int n) { p_.ransac_iterations = n; apply(); }
  void setNumThreads(int n) { p_.num_threads = n; apply(); }                                      // accepted; the GPU path ignores it
  void enableTimingOutput(bool e) { p_.enable_timing_output = e; apply(); }
  void setResolution(float r) { p_.resolution = r; apply(); }          // re-initialises the current target's voxels (ndt_omp.h:124-131)
  void setStepSize(double s) { p_.step_size = s; apply(); }
  void setOulierRatio(double r) { p_.outlier_ratio = r; apply(); }     // the reference's spelling (ndt_omp.h:166)
  void setNeighborhoodSearchMethod(int m) { p_.search_method = m; apply(); }   // 0 KDTREE, 1 DIRECT26, 2 DIRECT7, 3 DIRECT1
  float getResolution() const { return p_.resolution; }
  double getStepSize() const { return p_.step_size; }
  double getOulierRatio() const { return p_.outlier_ratio; }
  std::string getClassName() const { return "B200NormalDistributionsTransform"; }

  bool setInputSource(const PointF* pts, size_t n) { return lb_ndt_set_source(h_, pts, n, sizeof(PointF), 0, LB_MEM_HOST) == LB_OK; }
  bool setInputTarget(const PointF* pts, size_t n) { return lb_ndt_set_target(h_, pts, n, sizeof(PointF), 0, LB_MEM_HOST) == LB_OK; }
  // the resident submap's points as the target, gathered on the device; call again after the map changed (a no-op while
  // it is unchanged)
  bool setInputTargetSubmap(lb_submap* m) { return lb_ndt_set_target_submap(h_, m) == LB_OK; }
  bool align(const Matrix4f* guess = nullptr) { return lb_ndt_align(h_, guess ? guess->data() : nullptr, &r_) == LB_OK; }
  Matrix4f getFinalTransformation() const {
    Matrix4f m;
    for (int i = 0; i < 16; i++) m[i] = r_.final_transformation[i];
    return m;
  }
  bool hasConverged() const { return r_.converged != 0; }
  double getTransformationProbability() const { return r_.trans_probability; }
  int getFinalNumIteration() const { return r_.nr_iterations; }
  const lb_ndt_result& result() const { return r_; }
  lb_ndt* handle() { return h_; }

 private:
  void apply() {
    if (lb_ndt_set_params(h_, &p_) != LB_OK) throw std::invalid_argument(lb_last_error_string());
  }
  lb_ndt* h_ = nullptr;
  lb_ndt_params p_{};
  lb_ndt_result r_{};
};

// Mirror of the `impl_` object inside point_cloud_filter::CustomVoxelGrid
// (custom_voxel_grid.h:25): the pcl::VoxelGrid<pcl::PCLPointCloud2> setters that
// config_callback / ChangeLeafSizeRostopic drive, and filter().
class B200VoxelGrid {
 public:
  explicit B200VoxelGrid(int device = 0) {
    if (lb_voxel_create(device, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
  }
  ~B200VoxelGrid() { lb_voxel_destroy(h_); }
  B200VoxelGrid(const B200VoxelGrid&) = delete;
  B200VoxelGrid& operator=(const B200VoxelGrid&) = delete;

  void setLeafSize(float lx, float ly, float lz) { lb_voxel_set_leaf_size(h_, lx, ly, lz); }
  std::array<float, 3> getLeafSize() const { std::array<float, 3> l{}; lb_voxel_get_leaf_size(h_, l.data()); return l; }
  void setFilterFieldName(const std::string& n) { field_ = n; push(); }
  std::string getFilterFieldName() const { return field_; }
  void setFilterLimits(double lo, double hi) { lo_ = lo; hi_ = hi; push(); }
  void getFilterLimits(double& lo, double& hi) const { lo = lo_; hi = hi_; }
  void setFilterLimitsNegative(bool n) { neg_ = n; push(); }
  bool getFilterLimitsNegative() const { return neg_; }
  void setMinimumPointsNumberPerVoxel(unsigned m) { lb_voxel_set_min_points_per_voxel(h_, (int)m); }
  void setDownsampleAllData(bool a) { lb_voxel_set_downsample_all_data(h_, a); }

  // filter(): `data` is the PointCloud2 blob (width*height points of point_step bytes).
  // Returns the number of output points written to `out` (same field layout, height 1, dense).
  long filter(const uint8_t* data, size_t n_pts, uint32_t point_step, const std::vector<lb_field>& fields,
              std::vector<uint8_t>* out) {
    out->resize(n_pts * point_step);
    size_t n_out = 0;
    int s = lb_voxel_filter(h_, data, n_pts, point_step, fields.data(), (int)fields.size(), nullptr, 0, out->data(), n_pts,
                            &n_out, nullptr, LB_MEM_HOST, LB_MEM_HOST);
    if (s != LB_OK) { out->clear(); return s; }
    out->resize(n_out * point_step);
    return (long)n_out;
  }

  // The `filtering/extract_features` branch of PointCloudFilter::Filter (PointCloudFilter.cc:144-173, SURVEY 8f row
  // f6): sharp, less-sharp, flat and less-flat points, rotated.  `out` gets x, y, z and intensity with zero normals and
  // curvature, like the reference's default-constructed PointF.  params: nullptr = the reference's defaults.
  // Returns LB_OK or the C ABI's status (out is then empty).
  int extractFeatures(const PointF* in, size_t n, std::vector<PointF>& out, const lb_features_params* params = nullptr,
                      lb_features_result* result = nullptr) {
    lb_features_params p;
    if (params) p = *params; else lb_features_default_params(&p);
    lb_features_result r{};
    std::vector<float> buf(8 * n);               // the output never exceeds 2n points
    const int s = lb_voxel_extract_features(h_, in, n, sizeof(PointF), offsetof(PointF, x), LB_MEM_HOST, &p, buf.data(),
                                            2 * n, &r, LB_MEM_HOST);
    if (result) *result = r;
    out.clear();
    if (s != LB_OK) return s;
    out.resize(r.n_out);
    for (size_t i = 0; i < r.n_out; i++) {
      PointF q{};
      q.x = buf[4 * i]; q.y = buf[4 * i + 1]; q.z = buf[4 * i + 2]; q.intensity = buf[4 * i + 3];
      out[i] = q;
    }
    return LB_OK;
  }

 private:
  void push() { lb_voxel_set_filter_limits(h_, field_.empty() ? nullptr : field_.c_str(), lo_, hi_, neg_); }
  lb_voxel* h_ = nullptr;
  std::string field_;
  double lo_ = -3.4028234663852886e38, hi_ = 3.4028234663852886e38;
  bool neg_ = false;
};

// The per-scan chain of the lidar callback (locus/src/Locus.cc:451-453: odometry_.SetLidar(filtered) +
// odometry_.UpdateEstimate(); PointCloudOdometry.cc:221-274) as the library's pipeline: submit raw PointCloud2 blobs
// in order, take results in order; scan k+1 is filtered while scan k is registered, `depth` registrations in flight.
class B200Odometry {
 public:
  B200Odometry(int device, int depth, size_t max_points, uint32_t max_point_step) {
    if (lb_odometry_create(device, depth, max_points, max_point_step, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
    lb_gicp_default_params(&p_);
  }
  ~B200Odometry() { lb_odometry_destroy(h_); }
  B200Odometry(const B200Odometry&) = delete;
  B200Odometry& operator=(const B200Odometry&) = delete;

  void setLeafSize(float l) { lb_voxel_set_leaf_size(lb_odometry_voxel(h_), l, l, l); }
  void setFilterLimits(const std::string& field, double lo, double hi) {
    lb_voxel_set_filter_limits(lb_odometry_voxel(h_), field.c_str(), lo, hi, 0);
  }
  lb_gicp_params& params() { return p_; }                       // edit, then applyParams() while the pipeline is idle
  bool applyParams() { return lb_odometry_set_gicp_params(h_, &p_) == LB_OK; }
  // normals stage (k = 0: off): every filtered scan gets its k-NN normals; idle pipeline, before the first scan
  bool setNormals(int k, const float* viewpoint = nullptr) { return lb_odometry_set_normals(h_, k, viewpoint) == LB_OK; }
  // registration_method: LB_REG_GICP (default) or LB_REG_NDT with its params (nullptr = lb_ndt_default_params); idle
  // pipeline, before the first scan
  bool setRegistration(int method, const lb_ndt_params* ndt = nullptr) {
    lb_ndt_params p;
    if (ndt) p = *ndt; else lb_ndt_default_params(&p);
    return lb_odometry_set_registration(h_, method, &p) == LB_OK;
  }

  // scan (and filtered_out, if given) must stay valid until next() has returned this ticket
  bool submit(const uint8_t* scan, size_t n_pts, uint32_t point_step, const std::vector<lb_field>& fields,
              const Matrix4f* prior = nullptr, uint8_t* filtered_out = nullptr, uint64_t* ticket = nullptr) {
    return lb_odometry_submit(h_, scan, n_pts, point_step, fields.data(), (int)fields.size(), LB_MEM_HOST,
                              prior ? prior->data() : nullptr, filtered_out, LB_MEM_HOST, ticket) == LB_OK;
  }
  // one scan of 1..3 lidars merged in the VoxelGrid stage, in the merger's alive_keys_ order (lb_odometry_submit_merged:
  // each input's transform is copied here, its points must stay valid until the result is returned)
  bool submitMerged(const std::vector<lb_voxel_input>& inputs, uint32_t point_step, const std::vector<lb_field>& fields,
                    const Matrix4f* prior = nullptr, uint8_t* filtered_out = nullptr, uint64_t* ticket = nullptr) {
    return lb_odometry_submit_merged(h_, inputs.data(), (int)inputs.size(), point_step, fields.data(), (int)fields.size(),
                                     LB_MEM_HOST, prior ? prior->data() : nullptr, filtered_out, LB_MEM_HOST, ticket) == LB_OK;
  }
  // false when nothing is ready (block == false) or nothing is pending
  bool next(lb_odometry_result* r, bool block = true) { return lb_odometry_next(h_, r, block ? 1 : 0) == LB_OK; }
  size_t pending() const { size_t n = 0; lb_odometry_pending(h_, &n); return n; }
  lb_odometry* handle() { return h_; }

 private:
  lb_odometry* h_ = nullptr;
  lb_gicp_params p_{};
};

// The whole lidar callback (locus/src/Locus.cc:450-543) as the library's pipeline: VoxelGrid, odometry, localization
// against `map` (the caller's lb_submap, updated with keyframes and cropped to the window), pose bookkeeping.
class B200Locus {
 public:
  B200Locus(int device, int depth, size_t max_points, uint32_t max_point_step, lb_submap* map) {
    if (lb_locus_create(device, depth, max_points, max_point_step, map, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
    lb_locus_default_params(&p_);
  }
  ~B200Locus() { lb_locus_destroy(h_); }
  B200Locus(const B200Locus&) = delete;
  B200Locus& operator=(const B200Locus&) = delete;

  void setLeafSize(float l) { lb_voxel_set_leaf_size(lb_locus_voxel(h_), l, l, l); }
  void setFilterLimits(const std::string& field, double lo, double hi) {
    lb_voxel_set_filter_limits(lb_locus_voxel(h_), field.c_str(), lo, hi, 0);
  }
  lb_locus_params& params() { return p_; }                      // edit, then applyParams() while nothing is in flight
  bool applyParams() { return lb_locus_set_params(h_, &p_) == LB_OK; }
  // params().front_end: normals and adaptive input voxelization (off by default; shipped values in locus_b200.h)
  // params().odometry_method / localization_method (LB_REG_GICP or LB_REG_NDT) with odometry_ndt / localization_ndt:
  // each package's registration_method; set before the first scan
  bool setRegistration(int odometry_method, int localization_method) {
    p_.odometry_method = odometry_method;
    p_.localization_method = localization_method;
    return applyParams();
  }

  // scan (and filtered_out, if given) must stay valid until next() has returned this ticket
  bool submit(const uint8_t* scan, size_t n_pts, uint32_t point_step, const std::vector<lb_field>& fields,
              const Matrix4f* prior = nullptr, uint8_t* filtered_out = nullptr, uint64_t* ticket = nullptr) {
    return lb_locus_submit(h_, scan, n_pts, point_step, fields.data(), (int)fields.size(), LB_MEM_HOST,
                           prior ? prior->data() : nullptr, filtered_out, LB_MEM_HOST, ticket) == LB_OK;
  }
  // as B200Odometry::submitMerged (lb_locus_submit_merged); the keyframe the map receives is the merged filtered scan
  bool submitMerged(const std::vector<lb_voxel_input>& inputs, uint32_t point_step, const std::vector<lb_field>& fields,
                    const Matrix4f* prior = nullptr, uint8_t* filtered_out = nullptr, uint64_t* ticket = nullptr) {
    return lb_locus_submit_merged(h_, inputs.data(), (int)inputs.size(), point_step, fields.data(), (int)fields.size(),
                                  LB_MEM_HOST, prior ? prior->data() : nullptr, filtered_out, LB_MEM_HOST, ticket) == LB_OK;
  }
  bool next(lb_locus_result* r, bool block = true) { return lb_locus_next(h_, r, block ? 1 : 0) == LB_OK; }
  size_t pending() const { size_t n = 0; lb_locus_pending(h_, &n); return n; }
  lb_locus* handle() { return h_; }

 private:
  lb_locus* h_ = nullptr;
  lb_locus_params p_{};
};

}  // namespace locus_b200
