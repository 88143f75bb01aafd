// ndt_pipeline_harness.cpp -- TEST-ONLY CPU build of lb_odometry_* / lb_locus_* (locus_b200/csrc/odometry.cu) against
// fake stages (tests/locus_stub.h, tests/ndt_stub.h), with the NDT and GICP call log on.  Built by
// tests/test_ndt_pipeline_cpu.py into tests/_build/.
#define LB_LOCUS_STUB 1
#include "locus_stub.h"
#include "../locus_b200/csrc/odometry.cu"

extern "C" {
lb_submap* nh_submap_create(int device, size_t n) { lb_submap* m = new lb_submap; m->device = device; m->n = n; return m; }
void nh_submap_destroy(lb_submap* m) { delete m; }
int nh_clouds_alive(void) { return stub::clouds_alive().load(); }
int nh_ndt_alive(void) { return stub_ndt::alive().load(); }
void nh_ndt_default_params(lb_ndt_params* p) { lb_ndt_default_params(p); }
void nh_reset(void) {
  {
    std::lock_guard<std::mutex> lk(stub::mu());
    stub::events().clear(); stub::flags().clear(); stub::corrections().clear();
    stub_ic::calls().clear(); stub_ic::fallback().clear();
  }
  { std::lock_guard<std::mutex> lk(stub_ndt::mu()); stub_ndt::log().clear(); stub_ndt::logging() = true; }
  { std::lock_guard<std::mutex> lk(stub_fe::mu()); stub_fe::log().clear(); stub_fe::logging() = true; }
}
void nh_set_correction(uint64_t id, const double* C16) {
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::corrections()[id] = std::vector<double>(C16, C16 + 16);
}
size_t nh_events(int* kind, uint64_t* id, double* v16, size_t* n, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& ev = stub::events();
  for (size_t i = 0; i < ev.size() && i < cap; i++) {
    kind[i] = ev[i].kind; id[i] = ev[i].id; n[i] = ev[i].n;
    memcpy(v16 + 16 * i, ev[i].v, sizeof(ev[i].v));
  }
  return ev.size();
}
// the NDT / GICP call log: kind, source id, target id, target is the map, guess
size_t nh_ndt_log(char* kind, uint64_t* src, uint64_t* tgt, int* is_map, float* guess16, size_t cap) {
  std::lock_guard<std::mutex> lk(stub_ndt::mu());
  const auto& L = stub_ndt::log();
  for (size_t i = 0; i < L.size() && i < cap; i++) {
    kind[i] = L[i].kind; src[i] = L[i].src; tgt[i] = L[i].tgt; is_map[i] = L[i].tgt_is_map;
    memcpy(guess16 + 16 * i, L[i].guess, sizeof(L[i].guess));
  }
  return L.size();
}
// the scan ids lb_gicp_prepare_source was called for, in order
size_t nh_prepared(uint64_t* id, size_t cap) {
  std::lock_guard<std::mutex> lk(stub_fe::mu());
  size_t k = 0;
  for (const auto& r : stub_fe::log())
    if (r.kind == 'P') { if (k < cap) id[k] = r.id; k++; }
  return k;
}
size_t nh_fe_count(char kind) {
  std::lock_guard<std::mutex> lk(stub_fe::mu());
  size_t k = 0;
  for (const auto& r : stub_fe::log()) k += r.kind == kind;
  return k;
}
// lb_gicp_icp_covariance calls: source id, T, target is the map
size_t nh_icp_calls(uint64_t* id, float* T16, int* is_map, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& v = stub_ic::calls();
  for (size_t i = 0; i < v.size() && i < cap; i++) { id[i] = v[i].id; memcpy(T16 + 16 * i, v[i].T, sizeof(v[i].T)); is_map[i] = v[i].tgt_is_map; }
  return v.size();
}
}
