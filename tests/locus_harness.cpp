// locus_harness.cpp -- TEST-ONLY CPU build of lb_locus_* (locus_b200/csrc/odometry.cu: the pipeline core and the
// localization stage) against fake stages (tests/locus_stub.h).  Built by tests/test_locus_cpu.py into tests/_build/.
#define LB_LOCUS_STUB 1
#include "locus_stub.h"
#include "../locus_b200/csrc/odometry.cu"

extern "C" {
lb_submap* lh_submap_create(int device, size_t n) { lb_submap* m = new lb_submap; m->device = device; m->n = n; return m; }
void lh_submap_destroy(lb_submap* m) { delete m; }
int lh_clouds_alive(void) { return stub::clouds_alive().load(); }
void lh_reset(void) {
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::events().clear(); stub::flags().clear(); stub::corrections().clear();
}
void lh_set_correction(uint64_t id, const double* C16) {
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::corrections()[id] = std::vector<double>(C16, C16 + 16);
}
size_t lh_events(int* kind, uint64_t* id, double* v16, size_t* n, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& ev = stub::events();
  for (size_t i = 0; i < ev.size() && i < cap; i++) {
    kind[i] = ev[i].kind; id[i] = ev[i].id; n[i] = ev[i].n;
    memcpy(v16 + 16 * i, ev[i].v, sizeof(ev[i].v));
  }
  return ev.size();
}
}
