// icp_covariance_cpp_harness.cpp -- TEST-ONLY driver of the ICP covariance through the C++ mirror
// (locus_b200/host/b200_gicp.hpp: B200Gicp::icpCovariance) and the PCL shim (shim/b200_gicp_pcl.hpp:
// computePoint2PlaneICPCovariance, compiled against the PCL mock of tests/pcl_stub with a 6x6 matrix type of its own).
// Each is compared with lb_gicp_icp_covariance called on an identically configured handle: three orthogonal planes
// (the reference's covariance fixture, offset by a small motion) and one plane (the D-NaN fallback, where the shim must
// leave *condition_number untouched).  Prints key=value lines that tests/test_icp_covariance_gpu.py checks; exit code 3
// = no CUDA device.  Built by tests/test_icp_covariance_cpu.py (compile and link) and the GPU test.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "b200_gicp.hpp"
#include "b200_gicp_pcl.hpp"

struct Mat6 {                        // the (i, j) access the shim needs from Eigen::Matrix<double, 6, 6>
  double v[36];
  double& operator()(int i, int j) { return v[6 * i + j]; }
};

// planes of 10 x 10 points, 0.1 apart: z = 0 (normal z), and with `three` also y = 0 (normal y) and x = 0 (normal x)
static std::vector<PointF> planes(bool three, float dx, float dy) {
  std::vector<PointF> out;
  for (int p = 0; p < (three ? 3 : 1); p++)
    for (int i = 0; i < 10; i++)
      for (int j = 0; j < 10; j++) {
        PointF q{};
        const float a = i * 0.1f + 0.05f, b = j * 0.1f + 0.05f;
        float xyz[3] = {a, b, 0.f}, n[3] = {0.f, 0.f, 1.f};
        if (p == 1) { xyz[0] = a; xyz[1] = 0.f; xyz[2] = b; n[1] = 1.f; n[2] = 0.f; }
        if (p == 2) { xyz[0] = 0.f; xyz[1] = a; xyz[2] = b; n[0] = 1.f; n[2] = 0.f; }
        q.x = xyz[0] + dx; q.y = xyz[1] + dy; q.z = xyz[2];
        q.normal_x = n[0]; q.normal_y = n[1]; q.normal_z = n[2];
        out.push_back(q);
      }
  return out;
}

static bool same(const lb_icp_covariance& a, const double* cov, double cond, bool cond_checked) {
  return memcmp(a.covariance, cov, sizeof(a.covariance)) == 0 &&
         (!cond_checked || memcmp(&a.condition_number, &cond, sizeof(cond)) == 0);
}

// the C call on a fresh handle with default parameters (what B200Gicp and the shim start from), after one align
static int c_call(const std::vector<PointF>& src, const std::vector<PointF>& tgt, int max_iterations, lb_icp_covariance* r) {
  lb_gicp* h = nullptr;
  if (lb_gicp_create(0, &h) != LB_OK) return -1;
  lb_gicp_params p;
  lb_gicp_default_params(&p);
  p.recompute_source_covariance = 0; p.recompute_target_covariance = 0;
  p.max_iterations = max_iterations;
  int s = lb_gicp_set_params(h, &p);
  if (s == LB_OK) s = lb_gicp_set_target(h, tgt.data(), tgt.size(), sizeof(PointF), 0, offsetof(PointF, normal_x), LB_MEM_HOST, nullptr);
  if (s == LB_OK) s = lb_gicp_set_source(h, src.data(), src.size(), sizeof(PointF), 0, offsetof(PointF, normal_x), LB_MEM_HOST);
  lb_gicp_result res;
  if (s == LB_OK) s = lb_gicp_align(h, nullptr, &res);
  if (s == LB_OK) s = lb_gicp_icp_covariance(h, nullptr, nullptr, LB_MEM_HOST, nullptr, 0.01, r);
  lb_gicp_destroy(h);
  return s;
}

int main() {
  int n_dev = 0;
  if (lb_device_count(&n_dev) != LB_OK || n_dev <= 0) { std::printf("no_device=1\n"); return 3; }
  for (int three = 1; three >= 0; three--) {
    const char* tag = three ? "planes3" : "plane1";
    const std::vector<PointF> tgt = planes(three, 0.f, 0.f), src = planes(three, 0.01f, -0.005f);
    lb_icp_covariance ref;
    const int s_ref = c_call(src, tgt, 20, &ref);
    std::printf("%s_c_status=%d\n%s_c_flags=%d\n", tag, s_ref, tag, ref.flags);

    // the C++ mirror, with the same parameters
    locus_b200::B200Gicp g(0);
    g.setMaximumIterations(20);
    g.RecomputeSourceCovariance(false); g.RecomputeTargetCovariance(false);
    std::vector<locus_b200::PointF> s2(src.size()), t2(tgt.size());
    static_assert(sizeof(locus_b200::PointF) == sizeof(PointF), "layouts");
    memcpy(s2.data(), src.data(), src.size() * sizeof(PointF));
    memcpy(t2.data(), tgt.data(), tgt.size() * sizeof(PointF));
    g.setInputTarget(t2.data(), t2.size()); g.setInputSource(s2.data(), s2.size());
    g.align(nullptr);
    lb_icp_covariance mr;
    const bool ok_m = g.icpCovariance(&mr, 0.01);
    const bool eq_m = ok_m && memcmp(&mr.Ap, &ref.Ap, sizeof(ref.Ap)) == 0 && mr.flags == ref.flags &&
                      same(ref, mr.covariance, mr.condition_number, !(ref.flags & LB_ICPCOV_D_NAN));
    std::printf("%s_mirror_equal=%d\n", tag, eq_m ? 1 : 0);

    // the PCL shim, through pcl::Registration as LOCUS holds it
    auto gicp = boost::make_shared<pcl::B200GeneralizedIterativeClosestPoint>(0);
    gicp->setMaximumIterations(20);
    PointCloudF::Ptr ps(new PointCloudF), pt(new PointCloudF);
    for (const PointF& q : src) ps->push_back(q);
    for (const PointF& q : tgt) pt->push_back(q);
    gicp->setInputSource(ps); gicp->setInputTarget(pt);
    PointCloudF out;
    gicp->align(out);
    Mat6 cov;
    double cond = 123.0;                     // condition_number_ of the previous scan
    const bool ok_s = gicp->computePoint2PlaneICPCovariance(0.01, &cov, &cond);
    const bool eq_s = ok_s && same(ref, cov.v, cond, !(ref.flags & LB_ICPCOV_D_NAN));
    std::printf("%s_shim_equal=%d\n%s_shim_condition_kept=%d\n", tag, eq_s ? 1 : 0, tag, cond == 123.0 ? 1 : 0);
    // a target uploaded without its normals is refused instead of answered from no normals
    gicp->RecomputeTargetCovariance(true);
    gicp->setInputTarget(pt);
    gicp->align(out);
    std::printf("%s_shim_refuses_without_normals=%d\n", tag, gicp->computePoint2PlaneICPCovariance(0.01, &cov, &cond) ? 0 : 1);
  }
  return 0;
}
