// example_odometry.cpp -- compile/link check of the C++ host mirror, and a tiny end-to-end use
// that reads like PointCloudOdometry::UpdateICP (PointCloudOdometry.cc:249-269).
// Built by __graft_entry__.build(); needs a GPU to run.
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <vector>

#include "b200_gicp.hpp"

using namespace locus_b200;

int main() {
  int ndev = 0;
  lb_device_count(&ndev);
  if (ndev <= 0) { std::printf("no CUDA device: nothing to run (the library has no CPU path)\n"); return 0; }
  // hollow cube of test_point_cloud_odometry.cpp:60-97, shifted by (+0.05,+0.05,0)
  std::vector<PointF> reference, query;
  for (int ix = 0; ix < 10; ix++)
    for (int iy = 0; iy < 10; iy++)
      for (int iz = 0; iz < 10; iz++)
        if (ix == 0 || iy == 0 || ix == 9 || iy == 9) {
          PointF p{};
          p.x = ix * 0.1f; p.y = iy * 0.1f; p.z = iz * 0.1f; p.data3 = 1.f;
          reference.push_back(p);
          p.x += 0.05f; p.y += 0.05f;
          query.push_back(p);
        }
  B200Gicp icp;
  icp.setTransformationEpsilon(1e-3);
  icp.setMaxCorrespondenceDistance(1.0);
  icp.setMaximumIterations(20);
  icp.setRANSACIterations(0);
  icp.RecomputeSourceCovariance(true);
  icp.RecomputeTargetCovariance(true);
  icp.setInputSource(query.data(), query.size(), false);
  icp.setInputTarget(reference.data(), reference.size(), false);
  std::vector<PointF> aligned;
  if (!icp.align(&aligned)) { std::printf("align failed: %s\n", lb_last_error_string()); return 1; }
  Matrix4f T = icp.getFinalTransformation();
  std::printf("converged=%d t=(%.4f %.4f %.4f) fitness=%.3g\n", (int)icp.hasConverged(), T[3], T[7], T[11], icp.getFitnessScore());
  if (!(icp.hasConverged() && std::fabs(T[3] + 0.05f) < 1e-2f && std::fabs(T[7] + 0.05f) < 1e-2f)) return 2;

  // NormalComputation (row f2): the wall x = 0 of the cube has normals (+-1, 0, 0), flipped towards the origin
  B200Gicp ne;
  if (!ne.computeNormals(reference.data(), reference.size(), 12)) { std::printf("normals failed: %s\n", lb_last_error_string()); return 3; }
  int bad = 0;
  for (const PointF& p : reference)
    if (p.x > 0.85f && p.y > 0.25f && p.y < 0.65f && p.z > 0.25f && p.z < 0.65f && !(p.normal_x < -0.99f)) bad++;
  std::printf("normals: %d interior points of the wall x = 0.9 not facing the origin\n", bad);
  if (bad) return 4;

  // `registration_method: ndt` (row f4): the same pair through the NDT mirror (0.5 m voxels on the 0.9 m cube)
  B200Ndt ndt;
  ndt.setTransformationEpsilon(1e-3);
  ndt.setMaximumIterations(20);
  ndt.setResolution(0.5f);
  if (!ndt.setInputSource(query.data(), query.size()) || !ndt.setInputTarget(reference.data(), reference.size()) || !ndt.align()) {
    std::printf("ndt failed: %s\n", lb_last_error_string());
    return 8;
  }
  Matrix4f Tn = ndt.getFinalTransformation();
  std::printf("ndt: converged=%d t=(%.4f %.4f %.4f) after %d Newton steps\n", (int)ndt.hasConverged(), Tn[3], Tn[7], Tn[11], ndt.getFinalNumIteration());
  if (!(ndt.hasConverged() && std::fabs(Tn[3] + 0.05f) < 1e-2f && std::fabs(Tn[7] + 0.05f) < 1e-2f)) return 9;

  // `filtering/extract_features` (row f6) on the cube: its rings are short, so few points come out, but the call runs
  B200VoxelGrid features;
  std::vector<PointF> feats;
  lb_features_result fr{};
  if (features.extractFeatures(reference.data(), reference.size(), feats, nullptr, &fr) != LB_OK) {
    std::printf("features failed: %s\n", lb_last_error_string());
    return 10;
  }
  std::printf("features: %zu arranged, %zu out\n", fr.n_arranged, fr.n_out);

  // the pipelined chain: the same two clouds as PointCloud2 blobs of PointF records
  B200Odometry odo(0, 2, reference.size(), sizeof(PointF));
  odo.setLeafSize(0.01f);                                     // finer than the 0.1 m lattice: every point survives
  odo.params().transformation_epsilon = 1e-3; odo.params().max_correspondence_distance = 1.0; odo.params().max_iterations = 20;
  if (!odo.applyParams()) return 5;
  std::vector<lb_field> fields(3);
  const char* names[3] = {"x", "y", "z"};
  for (int i = 0; i < 3; i++) {
    std::snprintf(fields[i].name, sizeof(fields[i].name), "%s", names[i]);
    fields[i].offset = 4u * i; fields[i].datatype = LB_FLOAT32; fields[i].count = 1;
  }
  odo.submit(reinterpret_cast<const uint8_t*>(reference.data()), reference.size(), sizeof(PointF), fields);
  odo.submit(reinterpret_cast<const uint8_t*>(query.data()), query.size(), sizeof(PointF), fields);
  lb_odometry_result r0, r1;
  if (!odo.next(&r0) || !odo.next(&r1) || r0.has_pose || !r1.has_pose || r1.status != LB_OK) {
    std::printf("pipeline failed: %s\n", r1.error);
    return 6;
  }
  std::printf("pipeline: n_filtered=%zu t=(%.4f %.4f)\n", r1.n_filtered, r1.gicp.final_transformation[3], r1.gicp.final_transformation[7]);
  if (!(std::fabs(r1.gicp.final_transformation[3] + 0.05f) < 1e-2f && std::fabs(r1.gicp.final_transformation[7] + 0.05f) < 1e-2f)) return 7;

  // the whole callback: the first scan seeds the map, the second is odometry-aligned and localized against it
  lb_submap* map = nullptr;
  if (lb_submap_create(0, 0.05f, &map) != LB_OK) return 11;
  int rc = 0;
  {
    B200Locus loc(0, 2, reference.size(), sizeof(PointF), map);
    loc.setLeafSize(0.01f);
    loc.params().odometry = odo.params();
    loc.params().localization.max_correspondence_distance = 1.0;
    if (!loc.applyParams()) rc = 12;
    loc.submit(reinterpret_cast<const uint8_t*>(reference.data()), reference.size(), sizeof(PointF), fields);
    loc.submit(reinterpret_cast<const uint8_t*>(query.data()), query.size(), sizeof(PointF), fields);
    lb_locus_result l0, l1;
    if (rc == 0 && (!loc.next(&l0) || !loc.next(&l1) || !l0.keyframe || !l1.has_localization || l1.status != LB_OK)) rc = 13;
    if (rc == 0) std::printf("locus: L t=(%.4f %.4f), map %zu points\n", l1.pose[3], l1.pose[7], l1.map_size);
  }
  // a robot with three lidars: one scan whose three clouds (x, y, z, intensity records) are merged, moved into
  // base_link and filtered in the VoxelGrid stage, in the merger's order; the first scan seeds the map
  if (rc == 0 && lb_submap_clear(map) != LB_OK) rc = 14;
  if (rc == 0) {
    std::vector<lb_field> xyzi(fields);
    xyzi.push_back(lb_field{});
    std::snprintf(xyzi[3].name, sizeof(xyzi[3].name), "intensity");
    xyzi[3].offset = offsetof(PointF, intensity); xyzi[3].datatype = LB_FLOAT32; xyzi[3].count = 1;
    B200Locus loc(0, 1, 3 * reference.size(), sizeof(PointF), map);
    loc.setLeafSize(0.05f);
    if (!loc.applyParams()) rc = 15;
    const Matrix4f mounts[3] = {{1, 0, 0, 0.3f, 0, 1, 0, 0, 0, 0, 1, 0.4f, 0, 0, 0, 1},
                                {-1, 0, 0, -0.2f, 0, -1, 0, 0.25f, 0, 0, 1, 0.3f, 0, 0, 0, 1},
                                {0, -1, 0, -0.2f, 1, 0, 0, -0.25f, 0, 0, 1, 0.3f, 0, 0, 0, 1}};
    std::vector<lb_voxel_input> lidars(3);
    for (int i = 0; i < 3; i++)
      lidars[(size_t)i] = lb_voxel_input{reinterpret_cast<const uint8_t*>(reference.data()), reference.size(), mounts[i].data()};
    lb_locus_result m0;
    if (rc == 0 && (!loc.submitMerged(lidars, sizeof(PointF), xyzi) || !loc.next(&m0) || m0.status != LB_OK || !m0.keyframe)) rc = 16;
    if (rc == 0) std::printf("locus, three lidars: %zu filtered points, map %zu points\n", m0.n_filtered, m0.map_size);
  }
  lb_submap_destroy(map);
  return rc;
}
