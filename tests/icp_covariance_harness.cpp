// icp_covariance_harness.cpp -- TEST-ONLY CPU build of lb_locus_* (locus_b200/csrc/odometry.cu) against the fake stages
// of tests/locus_stub.h and the fake lb_gicp_icp_covariance of tests/icp_covariance_stub.h.  Built with LB_LOCUS_STUB by
// tests/test_icp_covariance_cpu.py into tests/_build/.
#include "../locus_b200/csrc/odometry.cu"

extern "C" {
void ih_reset(void) {
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::events().clear(); stub::flags().clear(); stub::corrections().clear();
  stub_ic::calls().clear(); stub_ic::fallback().clear();
}
void ih_set_fallback(uint64_t id) { std::lock_guard<std::mutex> lk(stub::mu()); stub_ic::fallback().insert(id); }
void ih_set_correction(uint64_t id, const double* C16) {
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::corrections()[id] = std::vector<double>(C16, C16 + 16);
}
// calls: id, T (16 floats), R (9 floats), max_cov, tgt_is_map
size_t ih_calls(uint64_t* id, float* T, float* R, double* max_cov, int* is_map, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& v = stub_ic::calls();
  for (size_t i = 0; i < v.size() && i < cap; i++) {
    id[i] = v[i].id; memcpy(T + 16 * i, v[i].T, sizeof(v[i].T)); memcpy(R + 9 * i, v[i].R, sizeof(v[i].R));
    max_cov[i] = v[i].max_cov; is_map[i] = v[i].tgt_is_map;
  }
  return v.size();
}
size_t ih_events(int* kind, uint64_t* id, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& ev = stub::events();
  for (size_t i = 0; i < ev.size() && i < cap; i++) { kind[i] = ev[i].kind; id[i] = ev[i].id; }
  return ev.size();
}
lb_submap* ih_submap_create(int device, size_t n) { lb_submap* m = new lb_submap; m->device = device; m->n = n; return m; }
void ih_submap_destroy(lb_submap* m) { delete m; }
}
