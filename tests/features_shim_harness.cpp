// features_shim_harness.cpp -- TEST-ONLY driver of shim/b200_feature_extraction_pcl.hpp compiled against the PCL mock
// (tests/pcl_stub).  Reads a cloud from argv[1] (n x 3 float32, raw) into a PointCloudF, runs b200::extractFeatures the
// way PointCloudFilter::Filter would, and writes x, y, z, intensity (m x 4 float32) of the output to argv[2] for
// tests/test_features_gpu.py to compare with the oracle.  Without arguments it only makes one call on a tiny cloud.
// Exit code 3 = no CUDA device (the shim has no CPU path).
#include <cstdio>
#include <stdexcept>

#include <frontend_utils/CommonStructs.h>   // PointF = pcl::PointXYZINormal
#include "b200_feature_extraction_pcl.hpp"

int main(int argc, char** argv) {
  PointCloudF in, out;
  if (argc >= 3) {
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    float xyz[3];
    while (std::fread(xyz, sizeof(float), 3, f) == 3) {
      PointF p{};
      p.x = xyz[0]; p.y = xyz[1]; p.z = xyz[2];
      in.push_back(p);
    }
    std::fclose(f);
  } else {
    PointF p{};
    p.x = 1.f; p.y = 0.f; p.z = 0.f;
    in.push_back(p);
  }
  try {
    if (!b200::extractFeatures(in, out)) return 1;
  } catch (const std::exception& e) {
    std::printf("no_device=%s\n", e.what());
    return 3;
  }
  if (argc < 3) { std::printf("points=%zu\n", out.size()); return 0; }
  FILE* f = std::fopen(argv[2], "wb");
  if (!f) return 2;
  for (const PointF& p : out.points) {
    if (p.normal_x != 0.f || p.normal_y != 0.f || p.normal_z != 0.f || p.curvature != 0.f) return 4;
    const float v[4] = {p.x, p.y, p.z, p.intensity};
    std::fwrite(v, sizeof(float), 4, f);
  }
  std::fclose(f);
  std::printf("points=%zu\n", out.size());
  return 0;
}
