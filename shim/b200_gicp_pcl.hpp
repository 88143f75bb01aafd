// b200_gicp_pcl.hpp -- pcl::Registration subclass backed by liblocus_b200.so.
// Meant for a LOCUS catkin workspace (PCL + frontend_utils); this repository's image has neither, so here the
// header is compiled against the minimal PCL mock under tests/pcl_stub/ (tests/test_cabi_cpu.py, tests/test_gicp_gpu.py::test_pcl_shim_runs: it parses, links and
// -- on a GPU box -- runs through pcl::Registration::align()).  See INTEGRATION.md.
//
// Drop-in for pcl::MultithreadedGeneralizedIterativeClosestPoint<PointF, PointF>
// (multithreaded_gicp/include/multithreaded_gicp/gicp.h:64-426): same setters, and
// computeTransformation() -- the one pure virtual of pcl::Registration -- forwards to the C ABI.
//
// What the subclass takes care of, beyond forwarding:
//  * No CPU kd-tree per scan.  pcl::Registration::initCompute() rebuilds the target's FLANN kd-tree whenever the
//    target changed unless force_no_recompute_ is set; the constructor installs a LAZY search tree with
//    setSearchMethodTarget(tree, /*force_no_recompute=*/true).  The tree is only built when somebody actually searches
//    it through getSearchMethodTarget() (PointCloudLocalization.cc:327-336 does, PointCloudOdometry never does); the
//    batched replacement of that loop is nearestTarget() = lb_gicp_nn_target on the index already resident on the GPU.
//  * Status propagation.  A refused cloud (empty, non-finite points, out of memory) is reported with PCL_ERROR and
//    leaves BOTH the PCL base and the device handle on their previous input, like gicp.h:164-171.
//  * Covariance mode.  recompute_*_covariance = false (the reference default, gicp.h:115-116) takes the covariances
//    from the normals PointF carries (gicp.hpp:81-82); true passes LB_NO_NORMALS so that the k-NN branch
//    (gicp.hpp:85-154) runs.
//  * transformation_ / previous_transformation_ are the guess-free increment, final_transformation_ = it * guess
//    (gicp.hpp:518,583), as the reference leaves them.
#pragma once

#include <stdexcept>
#include <vector>

#include <frontend_utils/CommonStructs.h>   // PointF = pcl::PointXYZINormal
#include <pcl/registration/registration.h>
#include <pcl/search/kdtree.h>

#include "locus_b200.h"

namespace pcl {

// pcl::search::KdTree whose FLANN index is built on first use instead of in setInputCloud().
template <typename PointT>
class B200LazyKdTree : public search::KdTree<PointT> {
 public:
  using Base = search::KdTree<PointT>;
  using PointCloudConstPtr = typename Base::PointCloudConstPtr;
  using IndicesConstPtr = typename Base::IndicesConstPtr;

  void setInputCloud(const PointCloudConstPtr& cloud, const IndicesConstPtr& indices = IndicesConstPtr()) override {
    pending_cloud_ = cloud; pending_indices_ = indices; built_ = false;
  }
  int nearestKSearch(const PointT& p, int k, std::vector<int>& k_indices, std::vector<float>& k_sqr_distances) const override {
    build();
    return Base::nearestKSearch(p, k, k_indices, k_sqr_distances);
  }
  int radiusSearch(const PointT& p, double radius, std::vector<int>& k_indices, std::vector<float>& k_sqr_distances,
                   unsigned int max_nn = 0) const override {
    build();
    return Base::radiusSearch(p, radius, k_indices, k_sqr_distances, max_nn);
  }
  bool built() const { return built_; }

 private:
  void build() const {
    if (built_ || !pending_cloud_) return;
    const_cast<B200LazyKdTree*>(this)->Base::setInputCloud(pending_cloud_, pending_indices_);
    built_ = true;
  }
  PointCloudConstPtr pending_cloud_;
  IndicesConstPtr pending_indices_;
  mutable bool built_ = false;
};

class B200GeneralizedIterativeClosestPoint : public Registration<PointF, PointF> {
 public:
  using Base = Registration<PointF, PointF>;
  using Ptr = boost::shared_ptr<B200GeneralizedIterativeClosestPoint>;

  explicit B200GeneralizedIterativeClosestPoint(int device = 0) {
    reg_name_ = "B200GeneralizedIterativeClosestPoint";
    if (lb_gicp_create(device, &h_) != LB_OK) throw std::runtime_error(lb_last_error_string());
    lb_gicp_default_params(&p_);
    // same defaults as gicp.h:111-127
    max_iterations_ = 200; transformation_epsilon_ = 5e-4; corr_dist_threshold_ = 5.0;
    p_.recompute_source_covariance = 0; p_.recompute_target_covariance = 0;   // reference default (gicp.h:115-116)
    // initCompute() must not build a FLANN tree of the target for every scan: lazy tree + force_no_recompute
    lazy_tree_.reset(new B200LazyKdTree<PointF>());
    setSearchMethodTarget(lazy_tree_, /*force_no_recompute=*/true);
  }
  ~B200GeneralizedIterativeClosestPoint() override { lb_gicp_destroy(h_); }

  // extra setters of the reference class (gicp.h:134-143,264-298)
  void setNumThreads(int n) { p_.num_threads = n; }
  void enableTimingOutput(bool e) { p_.enable_timing_output = e; }
  void RecomputeTargetCovariance(bool r) { p_.recompute_target_covariance = r; target_dirty_ = true; }
  void RecomputeSourceCovariance(bool r) { p_.recompute_source_covariance = r; source_dirty_ = true; }
  void setMaximumOptimizerIterations(int n) { p_.max_optimizer_iterations = n; }
  int getMaximumOptimizerIterations() { return p_.max_optimizer_iterations; }
  void setRotationEpsilon(double e) { p_.rotation_epsilon = e; }
  double getRotationEpsilon() { return p_.rotation_epsilon; }
  void setCorrespondenceRandomness(int k) { p_.k_correspondences = k; }
  int getCorrespondenceRandomness() { return p_.k_correspondences; }

  // gicp.h:162-179.  The device upload happens first: when it is refused, the PCL base keeps its previous input too.
  void setInputSource(const PointCloudSourceConstPtr& cloud) override {
    if (!cloud || cloud->points.empty()) {
      PCL_ERROR("[pcl::%s::setInputSource] Invalid or empty point cloud dataset given!\n", getClassName().c_str());
      return;
    }
    if (!upload(*cloud, /*target=*/false)) return;
    Base::setInputSource(cloud);
    source_dirty_ = false;
  }
  // gicp.h:196-200
  void setInputTarget(const PointCloudTargetConstPtr& cloud) override {
    if (!cloud || cloud->points.empty()) {
      PCL_ERROR("[pcl::%s::setInputTarget] Invalid or empty point cloud dataset given!\n", getClassName().c_str());
      return;
    }
    if (!upload(*cloud, /*target=*/true)) return;
    Base::setInputTarget(cloud);
    lazy_tree_->setInputCloud(cloud);      // stored, not indexed: built only if getSearchMethodTarget() is searched
    target_dirty_ = false;
  }

  // Batched form of the loop at PointCloudLocalization.cc:327-336 (one nearestKSearch(pt, 1, ..) per aligned point):
  // exact nearest target point of every point of `cloud`, original target indices, squared distances.
  bool nearestTarget(const PointCloudSource& cloud, std::vector<int>& indices, std::vector<float>& sqr_distances) {
    indices.resize(cloud.size()); sqr_distances.resize(cloud.size());
    if (cloud.points.empty()) return true;
    static_assert(sizeof(int) == sizeof(int32_t), "int32 indices");
    if (lb_gicp_nn_target(h_, cloud.points.data(), cloud.size(), sizeof(PointF), reinterpret_cast<int32_t*>(indices.data()),
                          sqr_distances.data(), LB_MEM_HOST) != LB_OK) {
      PCL_ERROR("[pcl::%s::nearestTarget] %s\n", getClassName().c_str(), lb_last_error_string());
      return false;
    }
    return true;
  }

  // PointCloudLocalization.cc:325-336 + :398-421 in one call after align(): transform the source by the final
  // transformation, 1-NN of every aligned point in the target, then ComputePoint2PlaneICPCovariance with the target's
  // normals.  Mat6 is the caller's Eigen::Matrix<double, 6, 6> (icp_covariance_).  *condition_number is left as it was
  // when the reference returns early (the D-NaN fallback), as condition_number_ is.  false on an error.  The target's
  // normals reach the GPU only with RecomputeTargetCovariance(false) (what LOCUS ships, recompute_covariance_local_map:
  // false); otherwise the call is refused rather than answered without normals.
  template <class Mat6>
  bool computePoint2PlaneICPCovariance(double max_covariance, Mat6* covariance, double* condition_number) {
    if (!target_normals_) {
      PCL_ERROR("[pcl::%s::computePoint2PlaneICPCovariance] the target was uploaded without its normals "
                "(RecomputeTargetCovariance(true)); set it to false\n", getClassName().c_str());
      return false;
    }
    lb_icp_covariance r;
    if (lb_gicp_icp_covariance(h_, nullptr, nullptr, LB_MEM_HOST, nullptr, max_covariance, &r) != LB_OK) {
      PCL_ERROR("[pcl::%s::computePoint2PlaneICPCovariance] %s\n", getClassName().c_str(), lb_last_error_string());
      return false;
    }
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) (*covariance)(i, j) = r.covariance[6 * i + j];
    if (!(r.flags & LB_ICPCOV_D_NAN)) *condition_number = r.condition_number;
    return true;
  }

  const lb_gicp_result& getLastResult() const { return res_; }
  lb_gicp* handle() { return h_; }

 protected:
  // gicp.hpp:405-617
  void computeTransformation(PointCloudSource& output, const Eigen::Matrix4f& guess) override {
    // a covariance mode changed after the clouds were set: the normal offset handed to the library depends on it
    if (source_dirty_ && input_ && !upload(*input_, false)) return;
    if (target_dirty_ && target_ && !upload(*target_, true)) return;
    source_dirty_ = target_dirty_ = false;
    p_.transformation_epsilon = transformation_epsilon_;
    p_.max_correspondence_distance = corr_dist_threshold_;
    p_.max_iterations = max_iterations_;
    if (lb_gicp_set_params(h_, &p_) != LB_OK) {
      PCL_ERROR("[pcl::%s::computeTransformation] %s\n", getClassName().c_str(), lb_last_error_string());
      return;
    }
    float g[16];
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) g[r * 4 + c] = guess(r, c);
    if (lb_gicp_align(h_, g, &res_) != LB_OK) {
      PCL_ERROR("[pcl::%s::computeTransformation] %s\n", getClassName().c_str(), lb_last_error_string());
      return;   // converged_ stays false, final_transformation_ stays the identity align() reset it to
    }
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) {
        final_transformation_(r, c) = res_.final_transformation[r * 4 + c];       // previous * guess (gicp.hpp:583)
        transformation_(r, c) = res_.transformation[r * 4 + c];                   // the guess-free increment
      }
    previous_transformation_ = transformation_;
    nr_iterations_ = res_.iterations;
    converged_ = res_.converged != 0;
    // output = final_transformation_ * input (gicp.hpp:586); non-geometric fields were copied by align()
    if (lb_gicp_transform_source(h_, nullptr, output.points.data(), sizeof(PointF), offsetof(PointF, x), LB_NO_NORMALS,
                                 LB_MEM_HOST) != LB_OK)
      PCL_ERROR("[pcl::%s::computeTransformation] %s\n", getClassName().c_str(), lb_last_error_string());
  }

 private:
  bool upload(const PointCloud<PointF>& cloud, bool target) {
    const bool recompute = target ? p_.recompute_target_covariance : p_.recompute_source_covariance;
    const ptrdiff_t normal_off = recompute ? LB_NO_NORMALS : (ptrdiff_t)offsetof(PointF, normal_x);
    const int s = target ? lb_gicp_set_target(h_, cloud.points.data(), cloud.size(), sizeof(PointF), offsetof(PointF, x), normal_off,
                                              LB_MEM_HOST, nullptr)
                         : lb_gicp_set_source(h_, cloud.points.data(), cloud.size(), sizeof(PointF), offsetof(PointF, x), normal_off,
                                              LB_MEM_HOST);
    if (s == LB_OK && target) target_normals_ = !recompute;
    if (s != LB_OK) {
      PCL_ERROR("[pcl::%s::%s] %s -- previous input kept\n", getClassName().c_str(), target ? "setInputTarget" : "setInputSource",
                lb_last_error_string());
      return false;
    }
    return true;
  }

  lb_gicp* h_ = nullptr;
  lb_gicp_params p_;
  lb_gicp_result res_{};
  boost::shared_ptr<B200LazyKdTree<PointF>> lazy_tree_;
  bool source_dirty_ = false, target_dirty_ = false;
  bool target_normals_ = false;      // the handle's target was uploaded with its normals
};

}  // namespace pcl
