// b200_feature_extraction_pcl.hpp -- the `filtering/extract_features` branch of PointCloudFilter::Filter (SURVEY 8f
// row f6) on the GPU, backed by liblocus_b200.so.  Meant for a LOCUS catkin workspace; compiled here against the PCL mock
// under tests/pcl_stub/ and run on the GPU by tests/features_shim_harness.cpp.  See INTEGRATION.md 2e.
//
// b200::extractFeatures(in, out) replaces PointCloudFilter.cc:145-173 (arrangePCLInScanLines, extractFeatures, the
// concatenation of the four feature clouds and the fixed rotation) with the reference's hard-coded parameters.  out gets
// the input's header; its points carry x, y, z and intensity, with zero normals and curvature (the reference builds them
// from a default-constructed PointF).  Returns false, with an empty output, for an empty input, as the reference cannot
// handle one (it reads point 0 unconditionally), and for a negative device.  The output is dense, as the reference's.
//  * The calls share one lb_voxel handle per device (created on first use, guarded by a mutex, kept until the process
//    exits).  Its VoxelGrid settings are not used by this call.
//  * Without a CUDA device the first call throws: there is no CPU path behind the seam.
#pragma once

#include <cstddef>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include <pcl/console/print.h>
#include <pcl/point_cloud.h>

#include "locus_b200.h"

namespace b200 {

namespace detail {
inline std::mutex& features_mutex() { static std::mutex m; return m; }
inline lb_voxel* features_handle(int device) {
  static std::vector<lb_voxel*> handles;
  if ((int)handles.size() <= device) handles.resize(device + 1, nullptr);
  if (!handles[device]) {
    lb_voxel* h = nullptr;
    const int s = lb_voxel_create(device, &h);
    if (s != LB_OK) throw std::runtime_error(std::string("b200::extractFeatures: ") + lb_last_error_string() + " (no CPU fallback)");
    handles[device] = h;
  }
  return handles[device];
}
}  // namespace detail

template <typename PointT>
bool extractFeatures(const pcl::PointCloud<PointT>& in, pcl::PointCloud<PointT>& out, int device = 0) {
  if (device < 0) {
    PCL_ERROR("[b200::extractFeatures] invalid device %d\n", device);
    out.points.clear(); out.width = 0; out.height = 1; out.header = in.header;
    return false;
  }
  std::vector<float> buf;
  lb_features_params p;
  lb_features_default_params(&p);
  lb_features_result r;
  int s;
  {
    std::lock_guard<std::mutex> lk(detail::features_mutex());
    lb_voxel* h = detail::features_handle(device);
    if (in.points.empty()) { out.points.clear(); out.width = 0; out.height = 1; out.header = in.header; return false; }
    buf.resize(8 * in.size());                    // the output never exceeds 2n points
    s = lb_voxel_extract_features(h, in.points.data(), in.size(), sizeof(PointT), offsetof(PointT, x), LB_MEM_HOST, &p,
                                  buf.data(), 2 * in.size(), &r, LB_MEM_HOST);
  }
  out.header = in.header;
  out.points.clear();
  if (s != LB_OK) { out.width = 0; out.height = 1; return false; }
  out.points.resize(r.n_out);
  for (size_t i = 0; i < r.n_out; i++) {
    PointT q{};
    q.x = buf[4 * i]; q.y = buf[4 * i + 1]; q.z = buf[4 * i + 2]; q.intensity = buf[4 * i + 3];
    out.points[i] = q;
  }
  out.width = (unsigned)r.n_out;
  out.height = 1;
  out.is_dense = true;                            // the reference's output is a default-constructed cloud, transformed
  return true;
}

}  // namespace b200
