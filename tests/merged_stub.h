// merged_stub.h -- TEST-ONLY stand-ins for the VoxelGrid entry points of the pipelines' multi-lidar input
// (lb_voxel_filter_merged, and the scratch reservation lb::voxel_reserve), included by locus_b200/csrc/odometry.cu after
// locus_stub.h or odometry_stub.h.  Every merged call is recorded with what stage V handed it: the number of inputs and,
// per input in order, its scan id (the first 8 bytes of its data, ~0 for an empty input), its point count and its
// transform (identity when none was given; has_T says which).  The fake result is that of the branch's fake
// lb_voxel_filter applied to the first non-empty input with the merged point count, so the scan carries that input's id
// (and its flags: bit 0 makes the VoxelGrid fail).  A scan whose inputs are all empty filters to nothing, as the real
// call does.  Never linked into liblocus_b200.so.
#pragma once
#include <mutex>
#include <vector>

namespace stub_mg {
struct Call { int n_inputs; uint64_t id[3]; size_t n[3]; int has_T[3]; float T[3][16]; };
inline std::mutex& mu() { static std::mutex m; return m; }
inline std::vector<Call>& calls() { static std::vector<Call> v; return v; }
inline std::vector<size_t>& reserves() { static std::vector<size_t> v; return v; }
}  // namespace stub_mg

namespace lb {
inline int voxel_reserve(lb_voxel*, size_t n_pts, uint32_t) {
  std::lock_guard<std::mutex> lk(stub_mg::mu());
  stub_mg::reserves().push_back(n_pts);
  return LB_OK;
}
}  // namespace lb

extern "C" {
inline int lb_voxel_filter_merged(lb_voxel* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step,
                                  const lb_field* fields, int n_fields, uint8_t* out, size_t cap, size_t* n_out,
                                  int32_t* vidx, int mem_in, int mem_out) {
  *n_out = 0;
  if (!inputs || n_inputs < 1 || n_inputs > 3) { lb::set_error("stub: 1 to 3 input clouds"); return LB_ERR_INVALID_ARG; }
  stub_mg::Call k{};
  k.n_inputs = n_inputs;
  size_t total = 0;
  int first = -1;
  for (int i = 0; i < n_inputs; i++) {
    k.n[i] = inputs[i].n_pts;
    k.id[i] = ~0ull;
    if (inputs[i].n_pts) {
      memcpy(&k.id[i], inputs[i].data, 8);
      if (first < 0) first = i;
    }
    k.has_T[i] = inputs[i].transform != nullptr;
    for (int e = 0; e < 16; e++) k.T[i][e] = inputs[i].transform ? inputs[i].transform[e] : (e % 5 == 0 ? 1.f : 0.f);
    total += inputs[i].n_pts;
  }
  { std::lock_guard<std::mutex> lk(stub_mg::mu()); stub_mg::calls().push_back(k); }
  if (total == 0) return LB_OK;
  return lb_voxel_filter(h, inputs[first].data, total, point_step, fields, n_fields, nullptr, 0, out, cap, n_out, vidx,
                         mem_in, mem_out);
}
}
