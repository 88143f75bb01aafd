// merged_harness.cpp -- TEST-ONLY CPU build of lb_odometry_* / lb_locus_* (locus_b200/csrc/odometry.cu) with the
// multi-lidar VoxelGrid stage recorded by tests/merged_stub.h.  LB_LOCUS_STUB selects the fakes of tests/locus_stub.h,
// LB_ODOMETRY_STUB those of tests/odometry_stub.h.  Built by tests/test_merged_pipeline_cpu.py into tests/_build/.
#if defined(LB_LOCUS_STUB)
#include "locus_stub.h"
#else
#include "odometry_stub.h"
#endif
#include "merged_stub.h"
#include "../locus_b200/csrc/odometry.cu"

extern "C" {
void mh_reset(void) {
  { std::lock_guard<std::mutex> lk(stub_mg::mu()); stub_mg::calls().clear(); stub_mg::reserves().clear(); }
#if defined(LB_LOCUS_STUB)
  std::lock_guard<std::mutex> lk(stub::mu());
  stub::events().clear(); stub::flags().clear(); stub::corrections().clear();
#else
  stub::max_sleep_us().store(200);
#endif
}
// the merged calls in the order stage V made them: n_inputs, then per input slot (3 per call) id, n, has_T, T[16]
size_t mh_calls(int* n_inputs, uint64_t* id, size_t* n, int* has_T, float* T, size_t cap) {
  std::lock_guard<std::mutex> lk(stub_mg::mu());
  const auto& v = stub_mg::calls();
  for (size_t c = 0; c < v.size() && c < cap; c++) {
    n_inputs[c] = v[c].n_inputs;
    for (int i = 0; i < 3; i++) {
      id[3 * c + i] = v[c].id[i]; n[3 * c + i] = v[c].n[i]; has_T[3 * c + i] = v[c].has_T[i];
      memcpy(T + 16 * (3 * c + i), v[c].T[i], 16 * sizeof(float));
    }
  }
  return v.size();
}
const char* mh_last_error(void) { return lb_last_error_string(); }
size_t mh_reserves(size_t* out, size_t cap) {
  std::lock_guard<std::mutex> lk(stub_mg::mu());
  const auto& v = stub_mg::reserves();
  for (size_t i = 0; i < v.size() && i < cap; i++) out[i] = v[i];
  return v.size();
}
#if defined(LB_LOCUS_STUB)
lb_submap* mh_submap_create(int device, size_t n) { lb_submap* m = new lb_submap; m->device = device; m->n = n; return m; }
void mh_submap_destroy(lb_submap* m) { delete m; }
// map events (locus_stub.h): kind (1 insert, 2 crop), scan id, points
size_t mh_events(int* kind, uint64_t* id, size_t* n, size_t cap) {
  std::lock_guard<std::mutex> lk(stub::mu());
  const auto& ev = stub::events();
  for (size_t i = 0; i < ev.size() && i < cap; i++) { kind[i] = ev[i].kind; id[i] = ev[i].id; n[i] = ev[i].n; }
  return ev.size();
}
#endif
}
