// submap.cuh -- SURVEY 8f row f3: the GPU-resident rolling submap (included by gicp.cu: same translation unit, it
// reuses the handle internals -- Cloud, the index build, the k-NN covariance kernels).
//
// What it replaces: the external point_cloud_mapper object LOCUS drives from its lidar callback
// (locus/src/Locus.cc:464-465,479-486,522-543; locus/config/lo_settings.yaml:49-62):
//   mapper_->InsertPoints(cloud_in_fixed_frame, incremental)   keyframe insert: a point enters the map iff no map
//                                                              point occupies its octree voxel yet  -> lb_submap_insert
//   mapper_->ApproxNearestNeighbors(scan, neighbors)           one map point per scan point          -> lb_submap_neighbors
//   mapper_->Refresh(current_pose)                             sliding window: box crop (box_filter_size: 20 m)
//                                                                                                     -> lb_submap_crop_box
// and what the GPU adds: the map never leaves HBM, and it IS the GICP target (lb_gicp_set_target_submap): its
// voxel-hash index is rebuilt only when the map changed (a keyframe or a crop, not every scan), and the k-NN
// covariance of a map point is computed ONCE, when the first registration after its insertion needs it, and cached
// for as long as the point lives -- instead of 500 k covariances per scan.
//
// The mapper package is not vendored in the reference tree (README.md:57-60), so its octree details are "parity
// unpinned": here a voxel is world-anchored (floor(p / resolution)), and "approximate nearest" is exact nearest.
// oracle/submap_oracle.py restates exactly these semantics on the CPU for the tests.
#pragma once
#include <algorithm>
#include <limits>

struct lb_submap {
  lb_gicp* eng = nullptr;              // index / k-NN engine (its stream orders all submap work)
  float res = 0.05f;
  size_t n = 0;                        // map points (insertion order)
  size_t n_cov = 0;                    // points [0, n_cov) have a cached covariance
  int cov_k = 0; double cov_eps = 0;   // parameters the cache was computed with
  DBuf<f4> pts[2];                     // ping-pong (crop compacts into the other one)
  DBuf<double> cov[2];                 // covariance cache, insertion order, 6 per point
  DBuf<f4> nrm[2];                     // normals paired with pts[] (from the first insert with normals on): w = 0 with
                                       // a normal, every word NaN without one
  bool nrm_on = false;
  size_t n_plain = 0;                  // map points inserted without a normal
  bool cov_from_normals = false;       // the engine cloud's covariances came from the normals ...
  double nrm_cov_eps = 0;              // ... with this gicp_epsilon
  int cur = 0;
  DBuf<unsigned long long> keys;       // occupancy hash
  DBuf<uint32_t> owner;
  uint32_t cap = 0;                    // table slots (power of two)
  DBuf<uint32_t> slot_of, flags, pos;
  DBuf<uint8_t> stage;
  DBuf<int32_t> nn_idx; DBuf<float> nn_d2; DBuf<float> out_xyz;
  ScanWork scan;
  uint32_t* d_count = nullptr; uint32_t* h_count = nullptr;   // [0] scan totals, [1] crop survivors without a normal
  uint64_t generation = 0;             // bumps on every change of the point set
  uint64_t indexed_generation = ~0ull; // generation the engine's cloud was built from
};

namespace lb {
int submap_device(const lb_submap* m) { return m->eng->c.device; }   // lb_locus_create checks it against its own
int submap_target_normals(const lb_submap* m, uint64_t generation, const f4** nrm) {
  if (m->generation != generation) {
    set_error("lb_submap: the map changed since lb_gicp_set_target_submap; call it again");
    return LB_ERR_INVALID_ARG;
  }
  *nrm = m->nrm_on ? m->nrm[m->cur].p : nullptr;
  return LB_OK;
}
// the map's current points for lb_ndt_set_target_submap (ndt.cu): float4 records (stride 16, w unused), insertion order
void submap_points_view(const lb_submap* m, const f4** pts, size_t* n, uint64_t* generation, cudaStream_t* stream) {
  *pts = m->pts[m->cur].p; *n = m->n; *generation = m->generation; *stream = m->eng->c.stream;
}
}  // namespace lb

namespace {

template <class T>
int grow_preserving(DBuf<T>& b, size_t need, size_t used, cudaStream_t st) {
  if (need <= b.cap) return LB_OK;
  size_t nc = b.cap ? b.cap : 4096;
  while (nc < need) nc = nc + nc / 2 + 4096;
  T* np = nullptr;
  LB_CUDA(cudaMalloc((void**)&np, nc * sizeof(T)));
  if (b.p && used) LB_CUDA(cudaMemcpyAsync(np, b.p, used * sizeof(T), cudaMemcpyDeviceToDevice, st));
  LB_CUDA(cudaStreamSynchronize(st));
  if (b.p) cudaFree(b.p);
  b.p = np; b.cap = nc;
  return LB_OK;
}

int submap_rehash(lb_submap* m, uint32_t want_slots) {
  Ctx& c = m->eng->c;
  uint32_t cap = 1u << 16;
  while (cap < want_slots) cap <<= 1;
  LB_TRY(m->keys.ensure(cap)); LB_TRY(m->owner.ensure(cap));
  m->cap = cap;
  LB_CUDA(cudaMemsetAsync(m->keys.p, 0xff, (size_t)cap * sizeof(unsigned long long), c.stream));
  LB_CUDA(cudaMemsetAsync(m->owner.p, 0xff, (size_t)cap * sizeof(uint32_t), c.stream));
  if (m->n) {
    sm_rehash_kernel<<<cdiv(m->n, 256), 256, 0, c.stream>>>(m->pts[m->cur].p, (uint32_t)m->n, m->res, m->keys.p, m->owner.p, cap - 1);
    c.launches++;
  }
  return LB_OK;
}

// the engine's SOURCE cloud = the map (index only); rebuilt when the point set changed
int submap_ensure_index(lb_submap* m) {
  if (m->indexed_generation == m->generation && m->eng->src->valid) return LB_OK;
  if (m->n == 0) { set_error("lb_submap: the map is empty"); return LB_ERR_NO_TARGET; }
  LB_TRY(replace_cloud(m->eng, m->eng->src, 0, m->pts[m->cur].p, m->n, sizeof(f4), 0, LB_NO_NORMALS, LB_MEM_DEVICE, "lb_submap"));
  LB_TRY(finish_index(m->eng, *m->eng->src, 0));
  m->eng->src->map = m; m->eng->src->map_generation = m->generation;
  m->indexed_generation = m->generation;
  return LB_OK;
}

int submap_adopt(lb_gicp* h, lb_submap* m);

}  // namespace

extern "C" {

int lb_submap_create(int device, float resolution, lb_submap** out) {
  if (!out) { set_error("lb_submap_create: null handle pointer"); return LB_ERR_INVALID_ARG; }
  if (!(resolution > 0.f)) { set_error("lb_submap_create: resolution must be > 0"); return LB_ERR_INVALID_ARG; }
  lb_submap* m = new lb_submap;
  int s = lb_gicp_create(device, &m->eng);
  if (s != LB_OK) { delete m; return s; }
  m->res = resolution;
  if (cudaMalloc((void**)&m->d_count, 2 * sizeof(uint32_t)) != cudaSuccess || cudaMallocHost((void**)&m->h_count, 2 * sizeof(uint32_t)) != cudaSuccess) {
    set_error("lb_submap_create: allocation failed");
    lb_gicp_destroy(m->eng); delete m;
    return LB_ERR_CUDA;
  }
  s = submap_rehash(m, 1u << 16);
  if (s != LB_OK) { lb_gicp_destroy(m->eng); delete m; return s; }
  *out = m;
  return LB_OK;
}

int lb_submap_destroy(lb_submap* m) {
  if (!m) return LB_OK;
  cudaSetDevice(m->eng->c.device);
  cudaStreamSynchronize(m->eng->c.stream);
  for (int i = 0; i < 2; i++) { m->pts[i].release(); m->cov[i].release(); m->nrm[i].release(); }
  m->keys.release(); m->owner.release(); m->slot_of.release(); m->flags.release(); m->pos.release(); m->stage.release();
  m->nn_idx.release(); m->nn_d2.release(); m->out_xyz.release(); m->scan.sums.release();
  if (m->d_count) cudaFree(m->d_count);
  if (m->h_count) cudaFreeHost(m->h_count);
  lb_gicp_destroy(m->eng);
  delete m;
  return LB_OK;
}

int lb_submap_size(lb_submap* m, size_t* n) {
  if (!m || !n) return LB_ERR_INVALID_ARG;
  *n = m->n;
  return LB_OK;
}

int lb_submap_generation(lb_submap* m, uint64_t* g) {
  if (!m || !g) return LB_ERR_INVALID_ARG;
  *g = m->generation;
  return LB_OK;
}

int lb_submap_clear(lb_submap* m) {
  if (!m) return LB_ERR_INVALID_ARG;
  LB_CUDA(cudaSetDevice(m->eng->c.device));
  m->n = 0; m->n_cov = 0; m->n_plain = 0; m->generation++;
  return submap_rehash(m, 1u << 16);
}

}  // extern "C"

namespace {

// lb_submap_insert (normal_off < 0) and lb_submap_insert_with_normals
int submap_insert(lb_submap* m, const void* pts, size_t n, size_t stride, size_t xyz_off, ptrdiff_t normal_off, int mem,
                  size_t* n_inserted, float* inserted_xyz, const char* who) {
  if (!m) { set_error("%s: null handle", who); return LB_ERR_INVALID_ARG; }
  if (n_inserted) *n_inserted = 0;
  if (n == 0) return LB_OK;
  if (!pts) { set_error("%s: null cloud", who); return LB_ERR_INVALID_ARG; }
  if ((stride & 3u) || (xyz_off & 3u) || xyz_off + 12 > stride || (normal_off >= 0 && ((normal_off & 3) || (size_t)normal_off + 12 > stride))) {
    set_error("%s: bad stride/offset", who);
    return LB_ERR_INVALID_ARG;
  }
  if (m->n + n > 0x7ffffff0ull) { set_error("%s: too many points", who); return LB_ERR_INVALID_ARG; }
  Ctx& c = m->eng->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)n;
  const uint8_t* d_src = (const uint8_t*)pts;
  if (mem == LB_MEM_HOST) {
    LB_TRY(m->stage.ensure(n * stride));
    LB_CUDA(cudaMemcpyAsync(m->stage.p, pts, n * stride, cudaMemcpyHostToDevice, c.stream));
    d_src = m->stage.p;
  }
  // room for every candidate: points, and a table that stays at most half full
  LB_TRY(grow_preserving(m->pts[m->cur], m->n + n, m->n, c.stream));
  if (normal_off >= 0 && !m->nrm_on) {
    // the first insert with normals: the points already in the map have none
    LB_TRY(grow_preserving(m->nrm[m->cur], m->n + n, 0, c.stream));
    if (m->n) LB_CUDA(cudaMemsetAsync(m->nrm[m->cur].p, 0xff, m->n * sizeof(f4), c.stream));
    m->nrm_on = true;
  }
  if (m->nrm_on) LB_TRY(grow_preserving(m->nrm[m->cur], m->n + n, m->n, c.stream));
  if ((m->n + n) * 2 > m->cap) LB_TRY(submap_rehash(m, (uint32_t)((m->n + n) * 2 + 1)));
  LB_TRY(m->slot_of.ensure(n)); LB_TRY(m->flags.ensure(n)); LB_TRY(m->pos.ensure(n));
  float* d_ins = nullptr;
  if (inserted_xyz) {
    if (mem == LB_MEM_HOST) { LB_TRY(m->out_xyz.ensure(3 * n)); d_ins = m->out_xyz.p; } else d_ins = inserted_xyz;
  }
  sm_claim_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_src, N, (uint32_t)stride, (uint32_t)xyz_off, m->res, m->keys.p, m->owner.p,
                                                      m->cap - 1, m->slot_of.p);
  sm_decide_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->slot_of.p, m->owner.p, N, m->flags.p);
  c.launches += 2;
  LB_TRY(exclusive_scan_u32(c, m->scan, m->flags.p, m->pos.p, n, m->d_count));
  sm_commit_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_src, N, (uint32_t)stride, (uint32_t)xyz_off, m->slot_of.p, m->flags.p, m->pos.p,
                                                       (uint32_t)m->n, m->pts[m->cur].p, m->owner.p, d_ins, (int)normal_off,
                                                       m->nrm_on ? m->nrm[m->cur].p : nullptr);
  c.launches++;
  LB_CUDA(cudaMemcpyAsync(m->h_count, m->d_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  LB_CUDA(cudaGetLastError());
  const size_t added = *m->h_count;
  if (inserted_xyz && mem == LB_MEM_HOST && added) {
    LB_CUDA(cudaMemcpyAsync(inserted_xyz, d_ins, added * 3 * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  if (added) { m->n += added; m->generation++; }
  if (normal_off < 0) m->n_plain += added;
  if (n_inserted) *n_inserted = added;
  return LB_OK;
}

}  // namespace

extern "C" {

int lb_submap_insert(lb_submap* m, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem, size_t* n_inserted,
                     float* inserted_xyz) {
  return submap_insert(m, pts, n, stride, xyz_off, -1, mem, n_inserted, inserted_xyz, "lb_submap_insert");
}

int lb_submap_insert_with_normals(lb_submap* m, const void* pts, size_t n, size_t stride, size_t xyz_off, size_t normal_off,
                                  int mem, size_t* n_inserted, float* inserted_xyz) {
  if (normal_off > 0x7fffffffull) { set_error("lb_submap_insert_with_normals: bad normal offset"); return LB_ERR_INVALID_ARG; }
  return submap_insert(m, pts, n, stride, xyz_off, (ptrdiff_t)normal_off, mem, n_inserted, inserted_xyz, "lb_submap_insert_with_normals");
}

int lb_submap_crop_box(lb_submap* m, const float* center3, float half_size, size_t* n_removed) {
  if (!m || !center3 || !(half_size >= 0.f)) { set_error("lb_submap_crop_box: bad argument"); return LB_ERR_INVALID_ARG; }
  if (n_removed) *n_removed = 0;
  if (m->n == 0) return LB_OK;
  Ctx& c = m->eng->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)m->n;
  const int o = m->cur ^ 1;
  LB_TRY(m->flags.ensure(m->n)); LB_TRY(m->pos.ensure(m->n));
  LB_TRY(m->pts[o].ensure(m->pts[m->cur].cap));
  if (m->n_cov) LB_TRY(m->cov[o].ensure(6 * m->n_cov));
  if (m->nrm_on) LB_TRY(m->nrm[o].ensure(m->nrm[m->cur].cap));
  // survivors without a normal: counted only when the map mixes points with and without one
  const bool count_plain = m->nrm_on && m->n_plain > 0 && m->n_plain < m->n;
  if (count_plain) LB_CUDA(cudaMemsetAsync(m->d_count + 1, 0, sizeof(uint32_t), c.stream));
  sm_crop_flags_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->pts[m->cur].p, N, center3[0], center3[1], center3[2], half_size, m->flags.p);
  c.launches++;
  LB_TRY(exclusive_scan_u32(c, m->scan, m->flags.p, m->pos.p, m->n, m->d_count));
  sm_compact_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->pts[m->cur].p, m->n_cov ? m->cov[m->cur].p : nullptr, N, (uint32_t)m->n_cov,
                                                        m->flags.p, m->pos.p, m->pts[o].p, m->n_cov ? m->cov[o].p : nullptr,
                                                        m->nrm_on ? m->nrm[m->cur].p : nullptr, m->nrm_on ? m->nrm[o].p : nullptr,
                                                        count_plain ? m->d_count + 1 : nullptr);
  c.launches++;
  // survivors among the points that had a cached covariance: they stay a prefix (the compaction is stable)
  uint32_t* h2 = m->h_count;
  LB_CUDA(cudaMemcpyAsync(h2, m->d_count, (count_plain ? 2 : 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const size_t kept = h2[0];
  const size_t kept_plain = m->n_plain == 0 ? 0 : (count_plain ? h2[1] : kept);
  size_t kept_cov = 0;
  if (m->n_cov) {
    if (m->n_cov == m->n) kept_cov = kept;
    else {
      uint32_t v = 0;
      LB_CUDA(cudaMemcpyAsync(&v, m->pos.p + m->n_cov, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));   // exclusive prefix at n_cov
      LB_CUDA(cudaStreamSynchronize(c.stream));
      kept_cov = v;
    }
  }
  if (n_removed) *n_removed = m->n - kept;
  if (kept == m->n) return LB_OK;                 // nothing left the window
  m->cur = o; m->n = kept; m->n_cov = kept_cov; m->n_plain = kept_plain; m->generation++;
  return submap_rehash(m, (uint32_t)(kept * 2 + 1));
}

int lb_submap_points(lb_submap* m, float* xyz_out, size_t capacity_points, int mem) {
  if (!m || !xyz_out) { set_error("lb_submap_points: null argument"); return LB_ERR_INVALID_ARG; }
  if (capacity_points < m->n) { set_error("lb_submap_points: capacity too small"); return LB_ERR_CAPACITY; }
  if (m->n == 0) return LB_OK;
  Ctx& c = m->eng->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)m->n;
  float* d = xyz_out;
  if (mem == LB_MEM_HOST) { LB_TRY(m->out_xyz.ensure(3 * m->n)); d = m->out_xyz.p; }
  // identity gather: xyz of every map point in insertion order
  LB_TRY(m->nn_idx.ensure(m->n));
  iota_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->nn_idx.p, N);
  sm_gather_xyz_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->pts[m->cur].p, m->nn_idx.p, N, d);
  c.launches += 2;
  if (mem == LB_MEM_HOST) LB_CUDA(cudaMemcpyAsync(xyz_out, d, 3 * m->n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  return LB_OK;
}

int lb_submap_normals(lb_submap* m, float* xyz_out, size_t capacity_points, int mem) {
  if (!m || !xyz_out) { set_error("lb_submap_normals: null argument"); return LB_ERR_INVALID_ARG; }
  if (capacity_points < m->n) { set_error("lb_submap_normals: capacity too small"); return LB_ERR_CAPACITY; }
  if (m->n == 0) return LB_OK;
  Ctx& c = m->eng->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)m->n;
  if (!m->nrm_on) {         // no point has a normal
    if (mem == LB_MEM_HOST) std::fill(xyz_out, xyz_out + 3 * m->n, std::numeric_limits<float>::quiet_NaN());
    else {
      LB_CUDA(cudaMemsetAsync(xyz_out, 0xff, 3 * m->n * sizeof(float), c.stream));
      LB_CUDA(cudaStreamSynchronize(c.stream));
    }
    return LB_OK;
  }
  float* d = xyz_out;
  if (mem == LB_MEM_HOST) { LB_TRY(m->out_xyz.ensure(3 * m->n)); d = m->out_xyz.p; }
  LB_TRY(m->nn_idx.ensure(m->n));
  iota_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->nn_idx.p, N);
  sm_gather_xyz_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->nrm[m->cur].p, m->nn_idx.p, N, d);
  c.launches += 2;
  if (mem == LB_MEM_HOST) LB_CUDA(cudaMemcpyAsync(xyz_out, d, 3 * m->n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  return LB_OK;
}

int lb_submap_neighbors(lb_submap* m, const void* query, size_t n, size_t stride, size_t xyz_off, float* neighbors_xyz,
                        int32_t* idx, float* d2, int mem) {
  if (!m || !query) { set_error("lb_submap_neighbors: null argument"); return LB_ERR_INVALID_ARG; }
  if (n == 0) return LB_OK;
  if ((stride & 3u) || (xyz_off & 3u) || xyz_off + 12 > stride) { set_error("lb_submap_neighbors: bad stride/offset"); return LB_ERR_INVALID_ARG; }
  Ctx& c = m->eng->c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(submap_ensure_index(m));
  const uint32_t N = (uint32_t)n;
  const uint8_t* dq = (const uint8_t*)query;
  if (mem == LB_MEM_HOST) {
    LB_TRY(m->stage.ensure(n * stride));
    LB_CUDA(cudaMemcpyAsync(m->stage.p, query, n * stride, cudaMemcpyHostToDevice, c.stream));
    dq = m->stage.p;
  }
  int32_t* di = idx; float* dd = d2; float* dx = neighbors_xyz;
  if (mem == LB_MEM_HOST || !idx) { LB_TRY(m->nn_idx.ensure(n)); di = m->nn_idx.p; }
  if (mem == LB_MEM_HOST || !d2) { LB_TRY(m->nn_d2.ensure(n)); dd = m->nn_d2.p; }
  if (neighbors_xyz && mem == LB_MEM_HOST) { LB_TRY(m->out_xyz.ensure(3 * n)); dx = m->out_xyz.p; }
  int blocks = cdiv(N, 8);
  if (blocks > c.sm_count * 8) blocks = c.sm_count * 8;
  nn_query_warp_kernel<<<blocks, 256, 0, c.stream>>>(m->eng->src->view(), dq + xyz_off, N, (uint32_t)stride, di, dd, 3.0e38f);
  c.launches++;
  if (neighbors_xyz) {
    sm_gather_xyz_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(m->pts[m->cur].p, di, N, dx);
    c.launches++;
  }
  if (mem == LB_MEM_HOST) {
    if (idx) LB_CUDA(cudaMemcpyAsync(idx, di, n * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    if (d2) LB_CUDA(cudaMemcpyAsync(d2, dd, n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
    if (neighbors_xyz) LB_CUDA(cudaMemcpyAsync(neighbors_xyz, dx, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  }
  LB_CUDA(cudaStreamSynchronize(c.stream));
  LB_CUDA(cudaGetLastError());
  return LB_OK;
}

int lb_gicp_set_target_submap(lb_gicp* h, lb_submap* m) {
  if (!h || !m) { set_error("lb_gicp_set_target_submap: null argument"); return LB_ERR_INVALID_ARG; }
  if (m->eng->c.device != h->c.device) { set_error("lb_gicp_set_target_submap: submap on device %d, handle on %d", m->eng->c.device, h->c.device); return LB_ERR_INVALID_ARG; }
  if (m->n == 0) { set_error("lb_gicp_set_target_submap: the map is empty"); return LB_ERR_NO_TARGET; }
  const int k = h->P.k_correspondences;
  if (k > 20) { set_error("lb_gicp_set_target_submap: k_correspondences > 20 is not supported for a resident submap"); return LB_ERR_UNSUPPORTED; }
  if ((size_t)k > m->n) { set_error("lb_gicp_set_target_submap: the map holds %zu points, fewer than k_correspondences (%d)", m->n, k); return LB_ERR_TOO_FEW_POINTS; }
  lb_gicp* e = m->eng;
  Ctx& c = e->c;
  LB_CUDA(cudaSetDevice(c.device));
  const bool reindexed = !(m->indexed_generation == m->generation && e->src->valid);
  LB_TRY(submap_ensure_index(m));
  Cloud& cl = *e->src;
  if (h->P.recompute_target_covariance == 0 && m->nrm_on && m->n_plain == 0) {
    // from the stored normals (gicp.hpp:81-82 for a target with normals), as normal_cov_kernel does for an uploaded
    // cloud; the k-NN cache is left alone
    if (reindexed || !cl.cov_valid || !m->cov_from_normals || m->nrm_cov_eps != h->P.gicp_epsilon) {
      LB_TRY(cl.cov.ensure(6 * cl.n));
      normal_cov_kernel<<<cdiv(cl.n, 256), 256, 0, c.stream>>>(cl.pts.p, m->nrm[m->cur].p, (uint32_t)cl.n, h->P.gicp_epsilon, cl.cov.p);
      c.launches++;
      cl.cov_valid = true;
      m->cov_from_normals = true; m->nrm_cov_eps = h->P.gicp_epsilon;
    }
    return submap_adopt(h, m);
  }
  // covariance cache: everything again when the parameters changed, otherwise only the points inserted since
  if (m->cov_k != k || m->cov_eps != h->P.gicp_epsilon) { m->n_cov = 0; m->cov_k = k; m->cov_eps = h->P.gicp_epsilon; }
  const bool new_cov = m->n_cov < m->n;
  if (new_cov) {
    LB_TRY(grow_preserving(m->cov[m->cur], 6 * m->n, 6 * m->n_cov, c.stream));
    Scratch& S = e->sc[0];
    const uint32_t N = (uint32_t)cl.n;
    LB_TRY(S.worklist.ensure(N));
    uint32_t* d_wl = S.d_u32 + 4;
    LB_CUDA(cudaMemsetAsync(d_wl, 0, 2 * sizeof(uint32_t), c.stream));
    CovFinIncr fin;
    fin.eps = h->P.gicp_epsilon; fin.cache = m->cov[m->cur].p; fin.first_new = (int)m->n_cov;
    static const int ring_cap = [] { const char* ev = getenv("LB_RING_CAP"); return ev ? atoi(ev) : 6; }();
    knn_cov_quadreg_kernel<20, CovFinIncr><<<cdiv(4ll * N, KQ_THREADS), KQ_THREADS, 0, c.stream>>>(cl.view(), cl.raw.p, k, fin, 99, ring_cap,
                                                                                              S.worklist.p, d_wl, nullptr);
    knn_cov_tail_kernel<20, CovFinIncr><<<c.sm_count * 2, 128, 0, c.stream>>>(cl.view(), k, fin, S.worklist.p, d_wl);
    c.launches += 2;
    m->n_cov = m->n;
  }
  if (reindexed || new_cov || !cl.cov_valid || m->cov_from_normals) {
    LB_TRY(cl.cov.ensure(6 * cl.n));
    cov_gather_kernel<<<cdiv(6ll * cl.n, 256), 256, 0, c.stream>>>(cl.pts.p, (uint32_t)cl.n, m->cov[m->cur].p, cl.cov.p);
    c.launches++;
    cl.cov_valid = true;
    m->cov_from_normals = false;
  }
  return submap_adopt(h, m);
}

}  // extern "C"

namespace {

// the engine's cloud, its covariances enqueued, becomes h's target
int submap_adopt(lb_gicp* h, lb_submap* m) {
  lb_gicp* e = m->eng;
  Ctx& c = e->c;
  Cloud& cl = *e->src;
  LB_CUDA(cudaGetLastError());
  if (!cl.ready) LB_CUDA(cudaEventCreateWithFlags(&cl.ready, cudaEventDisableTiming));
  LB_CUDA(cudaEventRecord(cl.ready, c.stream));
  // adopt the engine's cloud as this handle's target (shared, immutable: the engine switches to another object when
  // the map changes while somebody still holds this one)
  if (h->tgt != e->src) {
    if (h->tgt.use_count() > 1) pool_release(h, h->tgt);
    h->tgt = e->src;
  }
  LB_CUDA(cudaSetDevice(h->c.device));
  LB_CUDA(cudaStreamWaitEvent(h->c.stream, cl.ready, 0));
  return LB_OK;
}

}  // namespace

extern "C" {

int lb_submap_launch_count(lb_submap* m, uint64_t* n) {
  if (!m || !n) return LB_ERR_INVALID_ARG;
  return lb_gicp_launch_count(m->eng, n);
}

}  // extern "C"
