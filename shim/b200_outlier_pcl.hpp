// b200_outlier_pcl.hpp -- drop-ins for the two PCL outlier filters LOCUS can switch on (SURVEY 8f row f5), backed by
// liblocus_b200.so.  Meant for a LOCUS catkin workspace; compiled here against the PCL mock under tests/pcl_stub/ and
// run on the GPU by tests/outlier_shim_harness.cpp.  See INTEGRATION.md 2d.
//
//   pcl::StatisticalOutlierRemoval<PointF>  -> pcl::B200StatisticalOutlierRemoval<PointF>   PointCloudFilter.cc:126-133
//   pcl::RadiusOutlierRemoval<PointF>       -> pcl::B200RadiusOutlierRemoval<PointF>        PointCloudFilter.cc:135-143,
//                                                                      PointCloudMerger.cc:112-117,139-144,169-174
// Same setters as PCL's (setInputCloud, setMeanK, setStddevMulThresh, setRadiusSearch, setMinNeighborsInRadius,
// setNegative) and the same filter(PointCloud&), which also works in place as the reference calls it
// (sor.setInputCloud(points_filtered); sor.filter(*points_filtered)).  The output is what pcl::copyPointCloud(*input,
// kept_indices, output) leaves: the kept points in input order, the input's header and is_dense, height 1.
//  * The radius filter takes its branch from input->is_dense, as PCL does (see lb_gicp_radius_outlier_removal).
//  * The callers construct a filter object per scan, so the objects share one lb_gicp handle per device (created on first
//    use, guarded by a mutex, kept until the process exits) instead of creating a CUDA stream per scan.
//  * A refused input (empty, a non-finite point, fewer than mean_k + 1 points, radius <= 0) is reported with PCL_ERROR
//    and gives an empty output, which is what PCL does for its own argument errors.
//  * Without a CUDA device the constructor throws: there is no CPU path behind the seam.
#pragma once

#include <cstddef>
#include <cstdint>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include <pcl/console/print.h>
#include <pcl/point_cloud.h>

#include "locus_b200.h"

namespace pcl {

template <typename PointT>
class B200OutlierFilterBase {
 public:
  using PointCloud = pcl::PointCloud<PointT>;
  using PointCloudConstPtr = typename PointCloud::ConstPtr;

  explicit B200OutlierFilterBase(int device) : device_(device) { handle(device_); }   // throws without a CUDA device
  virtual ~B200OutlierFilterBase() = default;

  void setInputCloud(const PointCloudConstPtr& cloud) { input_ = cloud; }
  PointCloudConstPtr getInputCloud() const { return input_; }
  void setNegative(bool negative) { negative_ = negative; }
  bool getNegative() const { return negative_; }

  void filter(PointCloud& output) {
    std::vector<int32_t> kept;
    bool ok = false;
    if (!input_ || input_->points.empty()) {
      PCL_ERROR("[pcl::%s::filter] Invalid or empty point cloud dataset given!\n", getClassName().c_str());
    } else {
      std::lock_guard<std::mutex> lk(mutex());
      lb_gicp* h = handle(device_);
      kept.resize(input_->size());
      size_t m = 0;
      if (lb_gicp_set_source(h, input_->points.data(), input_->size(), sizeof(PointT), offsetof(PointT, x), LB_NO_NORMALS,
                             LB_MEM_HOST) == LB_OK &&
          run(h, kept.data(), &m) == LB_OK) {
        kept.resize(m);
        ok = true;
      } else {
        PCL_ERROR("[pcl::%s::filter] %s\n", getClassName().c_str(), lb_last_error_string());
      }
    }
    std::vector<PointT> pts;
    if (ok) {
      pts.reserve(kept.size());
      for (int32_t i : kept) pts.push_back(input_->points[(size_t)i]);
    }
    if (input_) { output.header = input_->header; output.is_dense = input_->is_dense; }   // output may be *input_
    output.points.swap(pts);
    output.width = (unsigned)output.points.size();
    output.height = 1;
  }

  virtual std::string getClassName() const = 0;

 protected:
  virtual int run(lb_gicp* h, int32_t* kept, size_t* n_kept) = 0;

  PointCloudConstPtr input_;
  bool negative_ = false;

 private:
  static std::mutex& mutex() {
    static std::mutex mu;
    return mu;
  }
  // one handle per device for every filter object of the process; never destroyed (the CUDA runtime may already be torn
  // down when static destructors run)
  static lb_gicp* handle(int device) {
    static std::mutex create_mu;
    static std::vector<lb_gicp*> handles;
    std::lock_guard<std::mutex> lk(create_mu);
    if (device < 0) throw std::invalid_argument("B200 outlier filter: bad device");
    if ((size_t)device >= handles.size()) handles.resize((size_t)device + 1, nullptr);
    if (!handles[(size_t)device]) {
      lb_gicp* h = nullptr;
      if (lb_gicp_create(device, &h) != LB_OK) throw std::runtime_error(lb_last_error_string());
      handles[(size_t)device] = h;
    }
    return handles[(size_t)device];
  }

  int device_;
};

// pcl::StatisticalOutlierRemoval<PointT> (filters/impl/statistical_outlier_removal.hpp, PCL 1.10)
template <typename PointT>
class B200StatisticalOutlierRemoval : public B200OutlierFilterBase<PointT> {
 public:
  explicit B200StatisticalOutlierRemoval(int device = 0) : B200OutlierFilterBase<PointT>(device) {}
  void setMeanK(int nr_k) { mean_k_ = nr_k; }
  int getMeanK() const { return mean_k_; }
  void setStddevMulThresh(double stddev_mult) { std_mul_ = stddev_mult; }
  double getStddevMulThresh() const { return std_mul_; }
  std::string getClassName() const override { return "B200StatisticalOutlierRemoval"; }

 protected:
  int run(lb_gicp* h, int32_t* kept, size_t* n_kept) override {
    return lb_gicp_statistical_outlier_removal(h, 0, mean_k_, std_mul_, this->negative_ ? 1 : 0, kept, n_kept, nullptr,
                                               nullptr, LB_MEM_HOST);
  }

 private:
  int mean_k_ = 1;          // PCL's defaults
  double std_mul_ = 0.0;
};

// pcl::RadiusOutlierRemoval<PointT> (filters/impl/radius_outlier_removal.hpp, PCL 1.10)
template <typename PointT>
class B200RadiusOutlierRemoval : public B200OutlierFilterBase<PointT> {
 public:
  explicit B200RadiusOutlierRemoval(int device = 0) : B200OutlierFilterBase<PointT>(device) {}
  void setRadiusSearch(double radius) { radius_ = radius; }
  double getRadiusSearch() const { return radius_; }
  void setMinNeighborsInRadius(int min_pts) { min_pts_ = min_pts; }
  int getMinNeighborsInRadius() const { return min_pts_; }
  std::string getClassName() const override { return "B200RadiusOutlierRemoval"; }

 protected:
  int run(lb_gicp* h, int32_t* kept, size_t* n_kept) override {
    return lb_gicp_radius_outlier_removal(h, 0, radius_, min_pts_, this->input_->is_dense ? 1 : 0, this->negative_ ? 1 : 0,
                                          kept, n_kept, LB_MEM_HOST);
  }

 private:
  double radius_ = 0.0;     // PCL's defaults
  int min_pts_ = 1;
};

}  // namespace pcl
