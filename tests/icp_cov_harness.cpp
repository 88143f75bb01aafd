// icp_cov_harness.cpp -- TEST-ONLY g++ build of locus_b200/csrc/icp_cov.h (steps 5-9 of the ICP covariance) with the
// library's host flags, for tests/test_icp_covariance_cpu.py.
#include "../locus_b200/csrc/icp_cov.h"

#include <cstring>

extern "C" void ic_compute(const double* Ap, double max_cov, double* cov, double* cond, int* flags) {
  const icpcov::Result r = icpcov::compute(Ap, max_cov);
  memcpy(cov, r.cov, sizeof(r.cov));
  *cond = r.condition_number;
  *flags = r.flags;
}
