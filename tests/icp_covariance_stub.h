// icp_covariance_stub.h -- TEST-ONLY stand-in for lb_gicp_icp_covariance, included by locus_b200/csrc/odometry.cu after
// locus_stub.h (lb_locus builds).  Every call is recorded with the arguments stage L passed (the source scan id, T, the
// normal rotation, max_covariance) and also logged in locus_stub.h's event list as kind 4, so that its order against the
// inserts (kinds 1 and 3) and crops (2) can be checked.  The fake result is a function of the scan id: covariance[i] =
// id + i / 64, condition number 100 + id, flags 0 -- or, for a scan marked with stub_ic::fallback(), max * I, NaN and
// LB_ICPCOV_D_NAN, what the reference's early return leaves.  Never linked into liblocus_b200.so.
#pragma once
#include <cmath>
#include <set>

namespace stub_ic {
struct Call { uint64_t id; float T[16]; float R[9]; double max_cov; int tgt_is_map; };
inline std::vector<Call>& calls() { static std::vector<Call> v; return v; }
inline std::set<uint64_t>& fallback() { static std::set<uint64_t> v; return v; }
}  // namespace stub_ic

extern "C" {
inline int lb_gicp_icp_covariance(lb_gicp* h, const float* T, const int32_t* correspondences, int, const float* R,
                                  double max_cov, lb_icp_covariance* out) {
  if (!T || !R || correspondences) { lb::set_error("stub: stage L passes T and a rotation, no correspondences"); return LB_ERR_INVALID_ARG; }
  stub_ic::Call k{h->src, {}, {}, max_cov, h->tgt_is_map ? 1 : 0};
  memcpy(k.T, T, sizeof(k.T));
  memcpy(k.R, R, sizeof(k.R));
  bool fb;
  {
    std::lock_guard<std::mutex> lk(stub::mu());
    stub_ic::calls().push_back(k);
    stub::Event e{4, h->src, {}, 0};
    stub::events().push_back(e);
    fb = stub_ic::fallback().count(h->src) > 0;
  }
  memset(out, 0, sizeof(*out));
  for (int i = 0; i < 36; i++) out->covariance[i] = fb ? (i % 7 == 0 ? max_cov : 0.0) : (double)h->src + i / 64.0;
  out->condition_number = fb ? NAN : 100.0 + (double)h->src;
  out->flags = fb ? LB_ICPCOV_D_NAN : 0;
  out->n_query = out->n_used = h->n_src;
  return LB_OK;
}
}
