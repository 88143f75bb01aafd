// features_mirror_harness.cpp -- TEST-ONLY driver of B200VoxelGrid::extractFeatures (locus_b200/host/b200_gicp.hpp):
// reads argv[1] (n x 3 float32) into PointF records, writes x, y, z, intensity of the output (m x 4 float32) to argv[2]
// for tests/test_features_gpu.py to compare with the oracle.  Exit code 3 = no CUDA device.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "b200_gicp.hpp"

using namespace locus_b200;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::vector<PointF> in;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  float xyz[3];
  while (std::fread(xyz, sizeof(float), 3, f) == 3) {
    PointF p{};
    p.x = xyz[0]; p.y = xyz[1]; p.z = xyz[2]; p.data3 = 1.f;
    in.push_back(p);
  }
  std::fclose(f);
  std::vector<PointF> out;
  try {
    B200VoxelGrid vg;
    if (vg.extractFeatures(in.data(), in.size(), out) != LB_OK) { std::printf("error=%s\n", lb_last_error_string()); return 1; }
  } catch (const std::exception& e) {
    std::printf("no_device=%s\n", e.what());
    return 3;
  }
  f = std::fopen(argv[2], "wb");
  if (!f) return 2;
  for (const PointF& p : out) {
    if (p.normal_x != 0.f || p.normal_y != 0.f || p.normal_z != 0.f || p.curvature != 0.f) return 4;
    const float v[4] = {p.x, p.y, p.z, p.intensity};
    std::fwrite(v, sizeof(float), 4, f);
  }
  std::fclose(f);
  std::printf("points=%zu\n", out.size());
  return 0;
}
