// locus_front_end_harness.cpp -- TEST-ONLY CPU build of lb_locus_* / lb_odometry_* (locus_b200/csrc/odometry.cu) with
// the front end's entry points logged in order (tests/front_end_stub.h).  LB_LOCUS_STUB selects the fakes of
// tests/locus_stub.h, LB_ODOMETRY_STUB those of tests/odometry_stub.h (the one with a target upload, for the pipeline
// without cloud sharing).  Built by tests/test_locus_front_end_cpu.py into tests/_build/.
#if defined(LB_LOCUS_STUB)
#include "locus_stub.h"
#else
#include "odometry_stub.h"
#endif
#include "front_end_stub.h"
#include "../locus_b200/csrc/odometry.cu"

extern "C" {
void fh_reset(void) {
#if defined(LB_LOCUS_STUB)
  {
    std::lock_guard<std::mutex> lk(stub::mu());
    stub::events().clear(); stub::flags().clear(); stub::corrections().clear();
  }
#endif
  std::lock_guard<std::mutex> lk(stub_fe::mu());
  stub_fe::log().clear();
  stub_fe::logging() = true;
}
int fh_set_leaf(lb_voxel* v, float l) { return lb_voxel_set_leaf_size(v, l, l, l); }
size_t fh_log(char* kind, uint64_t* id, int* a, int* b, double* v, size_t cap) {
  std::lock_guard<std::mutex> lk(stub_fe::mu());
  const auto& L = stub_fe::log();
  for (size_t i = 0; i < L.size() && i < cap; i++) { kind[i] = L[i].kind; id[i] = L[i].id; a[i] = L[i].a; b[i] = L[i].b; v[i] = L[i].v; }
  return L.size();
}
#if defined(LB_LOCUS_STUB)
lb_submap* fh_submap_create(int device, size_t n) { lb_submap* m = new lb_submap; m->device = device; m->n = n; return m; }
void fh_submap_destroy(lb_submap* m) { delete m; }
size_t fh_events(int* kind, uint64_t* id, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& ev = stub::events();
  for (size_t i = 0; i < ev.size() && i < cap; i++) { kind[i] = ev[i].kind; id[i] = ev[i].id; }
  return ev.size();
}
#endif
}
