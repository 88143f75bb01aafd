// outlier_shim_harness.cpp -- TEST-ONLY driver of shim/b200_outlier_pcl.hpp compiled against the PCL mock (tests/pcl_stub).
// Runs the filters the way LOCUS's callers do (PointCloudFilter.cc:126-143: setInputCloud, setters, filter in place;
// PointCloudMerger.cc:112-117: the radius filter on the merged cloud) on a cloud read from argv[1] (n x 3 float32, raw),
// and writes the kept points (n_kept x 3 float32) of each run to argv[2]<name>.bin for
// tests/test_outliers_gpu.py::test_outlier_shim_runs to compare with the oracle.  Without arguments it only constructs
// the filters.  Exit code 3 = no CUDA device (the shim has no CPU path).
#include <cstdio>
#include <string>
#include <vector>

#include <frontend_utils/CommonStructs.h>   // PointF = pcl::PointXYZINormal
#include "b200_outlier_pcl.hpp"

using Cloud = pcl::PointCloud<PointF>;

static bool write_xyz(const std::string& path, const Cloud& c) {
  FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  for (const PointF& p : c.points) {
    const float xyz[3] = {p.x, p.y, p.z};
    std::fwrite(xyz, sizeof(float), 3, f);
  }
  std::fclose(f);
  return true;
}

int main(int argc, char** argv) {
  try {
    pcl::B200StatisticalOutlierRemoval<PointF> probe;
  } catch (const std::exception& e) {
    std::printf("no_device=%s\n", e.what());
    return 3;
  }
  if (argc < 3) { std::printf("constructed=1\n"); return 0; }
  Cloud::Ptr in(new Cloud);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  float xyz[3];
  while (std::fread(xyz, sizeof(float), 3, f) == 3) {
    PointF p{};
    p.x = xyz[0]; p.y = xyz[1]; p.z = xyz[2]; p.intensity = 1.0f;
    in->push_back(p);
  }
  std::fclose(f);
  const std::string pre = argv[2];
  bool ok = true;

  // PointCloudFilter::Filter: the statistical filter (outlier_knn 10, outlier_std 1.0), then the radius filter
  // (0.15 m, 3), each in place on the same cloud
  Cloud::Ptr work(new Cloud(*in));
  pcl::B200StatisticalOutlierRemoval<PointF> sor;
  sor.setInputCloud(work);
  sor.setMeanK(10);
  sor.setStddevMulThresh(1.0);
  sor.filter(*work);
  ok = ok && write_xyz(pre + "sor.bin", *work);
  pcl::B200RadiusOutlierRemoval<PointF> rad;
  rad.setInputCloud(work);
  rad.setRadiusSearch(0.15);
  rad.setMinNeighborsInRadius(3);
  rad.filter(*work);
  ok = ok && write_xyz(pre + "sor_rad.bin", *work);
  std::printf("sor_then_radius=%zu\n", work->size());

  // out of place, negative, and the radius-search branch (a cloud whose is_dense is false)
  Cloud outliers;
  sor.setInputCloud(in);
  sor.setNegative(true);
  sor.filter(outliers);
  ok = ok && write_xyz(pre + "sor_neg.bin", outliers) && in->size() > outliers.size();
  Cloud::Ptr sparse(new Cloud(*in));
  sparse->is_dense = false;
  Cloud rad_out;
  rad.setInputCloud(sparse);
  rad.setRadiusSearch(0.1);
  rad.filter(rad_out);
  ok = ok && write_xyz(pre + "rad_sparse.bin", rad_out) && !rad_out.is_dense;
  std::printf("ok=%d\n", ok ? 1 : 0);
  return ok ? 0 : 1;
}
