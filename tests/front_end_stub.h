// front_end_stub.h -- TEST-ONLY stand-ins for the entry points the pipeline's front end calls (normals stage, adaptive
// input voxelization, keyframe insert with normals), included by locus_b200/csrc/odometry.cu after locus_stub.h or
// odometry_stub.h.  With logging on (tests/locus_front_end_harness.cpp turns it on), every call is appended to one
// ordered log:
//   'N'  lb_gicp_estimate_normals   id = the cloud's scan id, a = which, b = k
//   'P'  lb_gicp_prepare_source     id = the source's scan id
//   'S'  lb_voxel_set_leaf_size     id = the last scan the fake VoxelGrid has filtered (lb_locus builds), v = leaf x
//   'I'  lb_submap_insert_with_normals (lb_locus builds)  id = the keyframe's scan id, a = stride, b = normal offset
// and the insert is also logged in locus_stub.h's event list as kind 3.  The VoxelGrid leaf is one value per handle.
// Never linked into liblocus_b200.so.
#pragma once
#include <map>
#include <mutex>
#include <vector>

namespace stub_fe {
struct Rec { char kind; uint64_t id; int a, b; double v; };
inline std::mutex& mu() { static std::mutex m; return m; }
inline bool& logging() { static bool on = false; return on; }
inline std::vector<Rec>& log() { static std::vector<Rec> v; return v; }
inline std::map<const lb_voxel*, float>& leaf() { static std::map<const lb_voxel*, float> v; return v; }
inline void add(char kind, uint64_t id, int a, int b, double v) {
  std::lock_guard<std::mutex> lk(mu());
  if (logging()) log().push_back(Rec{kind, id, a, b, v});
}
}  // namespace stub_fe

extern "C" {
inline int lb_gicp_estimate_normals(lb_gicp* h, int which, int k, const float*) {
  stub_fe::add('N', which == 0 ? h->src : h->tgt, which, k, 0.0);
  return LB_OK;
}
inline int lb_voxel_set_leaf_size(lb_voxel* h, float lx, float, float) {
  uint64_t last = ~0ull;
#if defined(LB_LOCUS_STUB)
  {
    std::lock_guard<std::mutex> lk(stub::mu());
    if (!stub::flags().empty()) last = stub::flags().rbegin()->first;
  }
#endif
  { std::lock_guard<std::mutex> lk(stub_fe::mu()); stub_fe::leaf()[h] = lx; }
  stub_fe::add('S', last, 0, 0, lx);
  return LB_OK;
}
inline int lb_voxel_get_leaf_size(lb_voxel* h, float* leaf3) {
  std::lock_guard<std::mutex> lk(stub_fe::mu());
  auto it = stub_fe::leaf().find(h);
  const float l = it == stub_fe::leaf().end() ? 0.25f : it->second;
  leaf3[0] = leaf3[1] = leaf3[2] = l;
  return LB_OK;
}
#if defined(LB_LOCUS_STUB)
inline int lb_submap_insert_with_normals(lb_submap* m, const void* pts, size_t n, size_t stride, size_t, size_t normal_off,
                                         int, size_t* n_inserted, float*) {
  stub::Event e{3, 0, {}, n};
  memcpy(&e.id, pts, 8);
  float T[16]; memcpy(T, (const uint8_t*)pts + 8, sizeof(T));
  for (int i = 0; i < 16; i++) e.v[i] = T[i];
  { std::lock_guard<std::mutex> lk(stub::mu()); stub::events().push_back(e); }
  stub_fe::add('I', e.id, (int)stride, (int)normal_off, 0.0);
  m->n += n;
  if (n_inserted) *n_inserted = n;
  return LB_OK;
}
#endif
}

// the prepare calls of the pipeline, logged in order with the normals calls
inline int stub_fe_prepare_source(lb_gicp* h) {
  stub_fe::add('P', h->src, 0, 0, 0.0);
  return lb_gicp_prepare_source(h);
}
#define lb_gicp_prepare_source stub_fe_prepare_source
