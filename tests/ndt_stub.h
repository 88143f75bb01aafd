// ndt_stub.h -- TEST-ONLY stand-ins for the lb_ndt_* entry points the pipelines call (lb_odometry's NDT workers,
// lb_locus's NDT localization), included by locus_b200/csrc/odometry.cu after locus_stub.h or odometry_stub.h.  The fakes
// do no geometry, like the GICP fakes of those files:
//   * set_source / set_target read the scan id from the cloud's first point (and refuse a torn cloud);
//     set_target_submap (lb_locus builds) marks the target as the map and refuses an empty one;
//   * align returns guess * C as final_transformation, C = the localization correction of the source scan when the
//     target is the map (locus_stub.h's corrections) and identity otherwise -- what the GICP fakes return -- and fails
//     like them on the scan's flags (lb_locus builds: bit 1 with a scan target, bit 2 with the map);
//     the other result fields are functions of the source id (nr_iterations = max_iterations).
// With logging on (tests/ndt_pipeline_harness.cpp turns it on), every call of these fakes is appended to one ordered
// log, together with the pipelines' GICP aligns and lb_gicp_set_target_submap calls (wrapped below):
//   'S' ndt set_source   'T' ndt set_target   'M' ndt set_target_submap   'A' ndt align (guess recorded)
//   'G' lb_gicp_align    'g' lb_gicp_set_target_submap
// Never linked into liblocus_b200.so.
#pragma once
#include <atomic>
#include <mutex>
#include <vector>

namespace stub_ndt {
struct Rec { char kind; uint64_t src, tgt; int tgt_is_map; float guess[16]; };
inline std::mutex& mu() { static std::mutex m; return m; }
inline bool& logging() { static bool on = false; return on; }
inline std::vector<Rec>& log() { static std::vector<Rec> v; return v; }
inline std::vector<size_t>& reserves() { static std::vector<size_t> v; return v; }
inline std::atomic<int>& alive() { static std::atomic<int> v{0}; return v; }
inline void add(char kind, uint64_t src, uint64_t tgt, int tgt_is_map, const float* guess) {
  std::lock_guard<std::mutex> lk(mu());
  if (!logging()) return;
  Rec r{kind, src, tgt, tgt_is_map, {}};
  for (int i = 0; i < 16; i++) r.guess[i] = guess ? guess[i] : ((i % 5 == 0) ? 1.f : 0.f);
  log().push_back(r);
}
}  // namespace stub_ndt

struct lb_ndt { uint64_t src = ~0ull, tgt = ~0ull; bool tgt_is_map = false; uint64_t launches = 0; lb_ndt_params P; };

namespace lb {
inline int ndt_check_params(const lb_ndt_params* p, const char* who) {
  if (!(p->resolution > 0) || !(p->step_size > 0) || !(p->outlier_ratio > 0) || !(p->outlier_ratio < 1) ||
      !(p->transformation_epsilon > 0) || p->max_iterations < 0 || p->min_points_per_voxel < 3 || !(p->min_covar_eigvalue_mult > 0)) {
    set_error("%s: stub: invalid NDT params", who);
    return LB_ERR_INVALID_ARG;
  }
  if (p->search_method < 0 || p->search_method > 3) { set_error("%s: stub: invalid search method", who); return LB_ERR_UNSUPPORTED; }
  return LB_OK;
}
inline int ndt_reserve(lb_ndt*, size_t max_points) {
  std::lock_guard<std::mutex> lk(stub_ndt::mu());
  stub_ndt::reserves().push_back(max_points);
  return LB_OK;
}
}  // namespace lb

extern "C" {
inline void lb_ndt_default_params(lb_ndt_params* p) {
  memset(p, 0, sizeof(*p));
  p->resolution = 1.0f; p->step_size = 0.1; p->outlier_ratio = 0.55; p->transformation_epsilon = 0.1; p->max_iterations = 35;
  p->min_points_per_voxel = 6; p->min_covar_eigvalue_mult = 0.01;
}
inline int lb_ndt_create(int, lb_ndt** h) { *h = new lb_ndt; lb_ndt_default_params(&(*h)->P); ++stub_ndt::alive(); return LB_OK; }
inline int lb_ndt_destroy(lb_ndt* h) { delete h; --stub_ndt::alive(); return LB_OK; }
inline int lb_ndt_set_params(lb_ndt* h, const lb_ndt_params* p) {
  LB_TRY(lb::ndt_check_params(p, "lb_ndt_set_params"));
  h->P = *p;
  return LB_OK;
}
inline int lb_ndt_launch_count(lb_ndt* h, uint64_t* n) { *n = h->launches; return LB_OK; }
inline int stub_ndt_cloud_id(const void* pts, size_t n, size_t stride, uint64_t* id) {
  if (n == 0) { lb::set_error("stub: empty NDT cloud"); return LB_ERR_EMPTY_SOURCE; }
  uint64_t last;
  memcpy(id, pts, 8);
  memcpy(&last, (const uint8_t*)pts + (n - 1) * stride, 8);
  if (last != *id) { lb::set_error("stub: torn NDT cloud"); return LB_ERR_INVALID_ARG; }
  return LB_OK;
}
inline int lb_ndt_set_source(lb_ndt* h, const void* pts, size_t n, size_t stride, size_t, int) {
  LB_TRY(stub_ndt_cloud_id(pts, n, stride, &h->src));
  stub_ndt::add('S', h->src, h->tgt, h->tgt_is_map, nullptr);
  return LB_OK;
}
inline int lb_ndt_set_target(lb_ndt* h, const void* pts, size_t n, size_t stride, size_t, int) {
  LB_TRY(stub_ndt_cloud_id(pts, n, stride, &h->tgt));
  h->tgt_is_map = false;
  stub_ndt::add('T', h->src, h->tgt, 0, nullptr);
  return LB_OK;
}
#if defined(LB_LOCUS_STUB)
inline int lb_ndt_set_target_submap(lb_ndt* h, lb_submap* m) {
  if (m->n == 0) { lb::set_error("stub: the map is empty"); return LB_ERR_NO_TARGET; }
  h->tgt_is_map = true;
  h->tgt = ~0ull;
  stub_ndt::add('M', h->src, h->tgt, 1, nullptr);
  return LB_OK;
}
#endif
inline int lb_ndt_align(lb_ndt* h, const float* guess, lb_ndt_result* out) {
  stub_ndt::add('A', h->src, h->tgt, h->tgt_is_map ? 1 : 0, guess);
  std::vector<double> C(16, 0.0);
  for (int i = 0; i < 4; i++) C[(size_t)(5 * i)] = 1.0;
#if defined(LB_LOCUS_STUB)
  stub::nap(h->src * 5 + 2);
  if (stub::flags_of(h->src) & (h->tgt_is_map ? 4u : 2u)) {
    lb::set_error("stub NDT align failure for scan %llu", (unsigned long long)h->src);
    return LB_ERR_NO_TARGET;
  }
  if (h->tgt_is_map) {
    std::lock_guard<std::mutex> lk(stub::mu());
    auto it = stub::corrections().find(h->src);
    if (it != stub::corrections().end()) C = it->second;
  }
#endif
  memset(out, 0, sizeof(*out));
  float G[16];
  for (int i = 0; i < 16; i++) G[i] = guess ? guess[i] : ((i % 5 == 0) ? 1.f : 0.f);
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      double s = 0;
      for (int k = 0; k < 4; k++) s += (double)G[4 * r + k] * C[(size_t)(4 * k + c)];
      out->final_transformation[4 * r + c] = (float)s;
    }
  out->converged = 1;
  out->nr_iterations = h->P.max_iterations;
  out->n_evaluations = 3 + (int)(h->src % 7);
  out->n_target_voxels = h->tgt_is_map ? -1 : (int)h->tgt;
  out->trans_probability = (double)h->src + 0.25;
  for (int i = 0; i < 6; i++) out->pose[i] = 0.5 * (double)h->src + i;
  out->t_total_s = 1e-3 * (double)h->src;
  h->launches += 30;
  return LB_OK;
}
}

// the pipelines' GICP aligns and map targets, logged in order with the NDT calls
inline int stub_ndt_gicp_align(lb_gicp* h, const float* guess, lb_gicp_result* out) {
#if defined(LB_LOCUS_STUB)
  stub_ndt::add('G', h->src, h->tgt, h->tgt_is_map ? 1 : 0, guess);
#else
  stub_ndt::add('G', h->src, h->tgt, 0, guess);
#endif
  return lb_gicp_align(h, guess, out);
}
#define lb_gicp_align stub_ndt_gicp_align
#if defined(LB_LOCUS_STUB)
inline int stub_ndt_gicp_set_target_submap(lb_gicp* h, lb_submap* m) {
  stub_ndt::add('g', h->src, ~0ull, 1, nullptr);
  return lb_gicp_set_target_submap(h, m);
}
#define lb_gicp_set_target_submap stub_ndt_gicp_set_target_submap
#endif
