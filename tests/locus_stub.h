// locus_stub.h -- TEST-ONLY stand-ins so that the host logic of lb_locus_* (locus_b200/csrc/odometry.cu: the
// pipeline core plus the localization stage) can be compiled and exercised without CUDA.  The fakes do no geometry:
//   * a "scan" is a buffer whose first 8 bytes hold its id and bytes 8..11 its flags (bit 0: the VoxelGrid fails,
//     bit 1: the odometry align fails, bit 2: the localization align fails); the fake VoxelGrid copies the id into
//     every output point and remembers the flags;
//   * the odometry align returns its guess as final_transformation, so a test chooses I_k through the prior;
//   * the localization align (a handle whose target is the submap) returns guess * C(id), C set per scan id by the
//     test (identity by default);
//   * transform_source writes the source id and T into the output buffer, and the fake submap logs every insert
//     (id, T, points) and crop (centre, half size; it removes half of the map).
// Never linked into liblocus_b200.so.
#pragma once
#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "../include/locus_b200.h"

// ---- the few CUDA runtime calls odometry.cu makes
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaStreamNonBlocking = 1 };
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = malloc(n); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, int) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, int, int) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -1; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t) { return "stub"; }

struct lb_submap { int device = 0; size_t n = 0; };

namespace lb {
inline char* err_buf() { static thread_local char b[512] = ""; return b; }
inline void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(err_buf(), 512, fmt, ap); va_end(ap);
}
inline int submap_device(const lb_submap* m) { return m->device; }
}  // namespace lb
#define LB_TRY(call) do { int s__ = (call); if (s__ != LB_OK) return s__; } while (0)

namespace stub {
struct Event { int kind; uint64_t id; double v[16]; size_t n; };   // kind 1: insert (v = T), 2: crop (v = centre, half)
inline std::mutex& mu() { static std::mutex m; return m; }
inline std::vector<Event>& events() { static std::vector<Event> v; return v; }
inline std::map<uint64_t, uint32_t>& flags() { static std::map<uint64_t, uint32_t> v; return v; }
inline std::map<uint64_t, std::vector<double>>& corrections() { static std::map<uint64_t, std::vector<double>> v; return v; }
inline std::atomic<int>& clouds_alive() { static std::atomic<int> v{0}; return v; }
inline uint32_t flags_of(uint64_t id) { std::lock_guard<std::mutex> lk(mu()); auto it = flags().find(id); return it == flags().end() ? 0u : it->second; }
inline void nap(uint64_t seed) { std::this_thread::sleep_for(std::chrono::microseconds((seed * 2654435761u >> 7) % 300)); }
}  // namespace stub

struct lb_voxel { uint64_t launches = 0; };
struct lb_gicp { uint64_t src = ~0ull, tgt = ~0ull; bool tgt_is_map = false; size_t n_src = 0; lb_gicp_params P; };
struct lb_cloud { uint64_t id; size_t n; };

extern "C" {
inline const char* lb_last_error_string(void) { return lb::err_buf(); }
inline int lb_voxel_create_on_stream(int, void*, lb_voxel** h) { *h = new lb_voxel; return LB_OK; }
inline int lb_voxel_destroy(lb_voxel* h) { delete h; return LB_OK; }
inline int lb_voxel_launch_count(lb_voxel* h, uint64_t* n) { *n = h->launches; return LB_OK; }
inline int lb_voxel_filter(lb_voxel*, const uint8_t* data, size_t n_pts, uint32_t point_step, const lb_field*, int,
                           const int32_t*, size_t, uint8_t* out, size_t cap, size_t* n_out, int32_t*, int, int) {
  uint64_t id; uint32_t flags;
  memcpy(&id, data, 8); memcpy(&flags, data + 8, 4);
  { std::lock_guard<std::mutex> lk(stub::mu()); stub::flags()[id] = flags; }
  stub::nap(id * 3 + 1);
  if (flags & 1u) { lb::set_error("stub voxel failure for scan %llu", (unsigned long long)id); return LB_ERR_INVALID_ARG; }
  if (n_pts > cap) return LB_ERR_CAPACITY;
  for (size_t i = 0; i < n_pts; i++) memcpy(out + i * point_step, &id, 8);
  *n_out = n_pts;
  return LB_OK;
}
inline int lb_gicp_default_params(lb_gicp_params* p) {
  memset(p, 0, sizeof(*p));
  p->k_correspondences = 20; p->gicp_epsilon = 1e-3; p->max_iterations = 200;
  return LB_OK;
}
inline int lb_gicp_create(int, lb_gicp** h) { *h = new lb_gicp; lb_gicp_default_params(&(*h)->P); return LB_OK; }
inline int lb_gicp_destroy(lb_gicp* h) { delete h; return LB_OK; }
inline int lb_gicp_reserve(lb_gicp*, size_t, int) { return LB_OK; }
inline int lb_gicp_set_params(lb_gicp* h, const lb_gicp_params* p) { h->P = *p; return LB_OK; }
inline int lb_gicp_launch_count(lb_gicp*, uint64_t* n) { *n = 0; return LB_OK; }
inline int lb_gicp_set_source(lb_gicp* h, const void* pts, size_t n, size_t stride, size_t, ptrdiff_t, int) {
  memcpy(&h->src, pts, 8); h->n_src = n;
  uint64_t last; memcpy(&last, (const uint8_t*)pts + (n - 1) * stride, 8);
  if (last != h->src) { lb::set_error("stub: torn source cloud"); return LB_ERR_INVALID_ARG; }
  return LB_OK;
}
inline int lb_gicp_set_target(lb_gicp*, const void*, size_t, size_t, size_t, ptrdiff_t, int, uint64_t*) { return LB_ERR_UNSUPPORTED; }
inline int lb_gicp_prepare_source(lb_gicp* h) { stub::nap(h->src * 11 + 3); return LB_OK; }
inline int lb_gicp_share_source(lb_gicp* h, lb_cloud** out) { *out = new lb_cloud{h->src, h->n_src}; ++stub::clouds_alive(); return LB_OK; }
inline int lb_cloud_release(lb_cloud* c) { delete c; --stub::clouds_alive(); return LB_OK; }
inline int lb_gicp_set_target_cloud(lb_gicp* h, lb_cloud* c) { h->tgt = c->id; h->tgt_is_map = false; return LB_OK; }
inline int lb_gicp_set_source_cloud(lb_gicp* h, lb_cloud* c) { h->src = c->id; h->n_src = c->n; return LB_OK; }
inline int lb_gicp_set_target_submap(lb_gicp* h, lb_submap* m) {
  if (m->n == 0) { lb::set_error("stub: the map is empty"); return LB_ERR_NO_TARGET; }
  h->tgt_is_map = true;
  return LB_OK;
}
inline int lb_gicp_align(lb_gicp* h, const float* guess, lb_gicp_result* out) {
  memset(out, 0, sizeof(*out));
  stub::nap(h->src * 7 + 5);
  const uint32_t fl = stub::flags_of(h->src);
  if (fl & (h->tgt_is_map ? 4u : 2u)) { lb::set_error("stub align failure for scan %llu", (unsigned long long)h->src); return LB_ERR_NO_TARGET; }
  float G[16];
  for (int i = 0; i < 16; i++) G[i] = guess ? guess[i] : ((i % 5 == 0) ? 1.f : 0.f);
  std::vector<double> C(16, 0.0);
  for (int i = 0; i < 4; i++) C[(size_t)(5 * i)] = 1.0;
  if (h->tgt_is_map) {
    std::lock_guard<std::mutex> lk(stub::mu());
    auto it = stub::corrections().find(h->src);
    if (it != stub::corrections().end()) C = it->second;
  }
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      double s = 0;
      for (int k = 0; k < 4; k++) s += (double)G[4 * r + k] * C[(size_t)(4 * k + c)];
      out->final_transformation[4 * r + c] = (float)s;
    }
  out->iterations = h->P.max_iterations; out->converged = 1;
  out->n_correspondences = (int)h->src;        // which scan was registered
  return LB_OK;
}
inline int lb_gicp_transform_source(lb_gicp* h, const float* T, void* out, size_t, size_t, ptrdiff_t, int) {
  memcpy(out, &h->src, 8);
  memcpy((uint8_t*)out + 8, T, 16 * sizeof(float));
  return LB_OK;
}
inline int lb_submap_insert(lb_submap* m, const void* pts, size_t n, size_t, size_t, int, size_t* n_inserted, float*) {
  stub::Event e{1, 0, {}, n};
  memcpy(&e.id, pts, 8);
  float T[16]; memcpy(T, (const uint8_t*)pts + 8, sizeof(T));
  for (int i = 0; i < 16; i++) e.v[i] = T[i];
  { std::lock_guard<std::mutex> lk(stub::mu()); stub::events().push_back(e); }
  m->n += n;
  if (n_inserted) *n_inserted = n;
  return LB_OK;
}
inline int lb_submap_crop_box(lb_submap* m, const float* c3, float half, size_t* n_removed) {
  stub::Event e{2, 0, {c3[0], c3[1], c3[2], half}, m->n / 2};
  { std::lock_guard<std::mutex> lk(stub::mu()); stub::events().push_back(e); }
  m->n -= m->n / 2;
  if (n_removed) *n_removed = e.n;
  return LB_OK;
}
inline int lb_submap_size(lb_submap* m, size_t* n) { *n = m->n; return LB_OK; }
}
