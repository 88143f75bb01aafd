// gicp_kernels.cuh -- CUDA kernels of the GICP hot path (K2-K6 of SURVEY.md 2.3).
//
//   gather_cloud_kernel      strided caller cloud -> packed float4 (+ normals)
//   grid_keys_kernel         K2: cell key per point
//   grid_reorder_kernel      K2: cell-contiguous float4 copy + cell histogram
//   knn_cov_quadreg_kernel   K3: k-NN(20) -> moments -> Jacobi -> regularised covariance (+ knn_cov_tail_kernel,
//                            knn_cov_quad_kernel for k > 20)
//   normal_cov_kernel        K3': covariance from normals (reference default mode)
//   prep_source_kernel       K6: output = guess * input (gicp.hpp:440)
//   nn_corr_kernel           K4: transform, exact 1-NN in the voxel hash, gate, Mahalanobis
//   objective_kernel<NV>     K5: 13 (BFGS) / 28 (GN) double sums, warp-shuffle + fixed-shape tree
//   align_persistent_kernel  K4+K5+BFGS+outer loop resident on the device (cooperative launch)
//   transform_kernel, nn_query_kernel, fitness_kernel   accessor surface (a8/a9)
#pragma once

#include <type_traits>

#include "bfgs.h"
#include "grid.h"
#include "nn_staged.cuh"
#include "prims.cuh"

namespace lb {

constexpr int AL_THREADS = 256;      // threads per CTA of the align kernels (255 registers for the leader warp)
#ifndef AL_ACC_WARPS_CFG
#define AL_ACC_WARPS_CFG 4
#endif
constexpr int AL_ACC_WARPS = AL_ACC_WARPS_CFG;   // warps that accumulate objective terms (shuffle throughput bounds the reduce)
constexpr int AL_ACC = AL_ACC_WARPS * 32;
constexpr int AL_PPC = AL_ACC * 4;   // source points per CTA (4 per accumulating lane, register-resident)
constexpr int AL_MAXV = 28;          // widest reduction (Gauss-Newton)
constexpr int AL_PSTRIDE = 32;       // words per CTA slot
constexpr int AL_MAXB = 8;           // slots per polling lane: supports up to 256 CTAs
// loop_solve_kernel runs no correspondence search, so its CTA can be the leader warp and the accumulating warps only:
// 160 threads at <= 168 registers (registers are allocated per SM sub-partition: 3 warps of 168 fit in one of the
// four, 2 of 200), two CTAs per SM
constexpr int AL_SOLVE_THREADS = 32 + AL_ACC;
constexpr int AL_SOLVE_POLL = 8;     // slot words one thread of the solve kernel polls at a time

// ------------------------------------------------------------------ cloud upload
__global__ void __launch_bounds__(256)
gather_cloud_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off, int normal_off,
                    f4* __restrict__ raw, f4* __restrict__ nrm, BBoxAcc* __restrict__ acc,
                    const f4* __restrict__ same_raw, const f4* __restrict__ same_nrm, uint32_t* __restrict__ differs) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  float x = 0.f, y = 0.f, z = 0.f;
  if (i < n) {
    const uint8_t* p = base + (size_t)i * stride;
    const float* q = reinterpret_cast<const float*>(p + xyz_off);
    x = q[0]; y = q[1]; z = q[2];
    raw[i] = f4{x, y, z, 1.0f};
    bool diff = false;
    if (same_raw) {                       // is this the cloud `same_raw` was gathered from, bit for bit?
      const f4 o = same_raw[i];
      diff = __float_as_uint(o.x) != __float_as_uint(x) || __float_as_uint(o.y) != __float_as_uint(y) || __float_as_uint(o.z) != __float_as_uint(z);
    }
    if (normal_off >= 0) {
      const float* m = reinterpret_cast<const float*>(p + normal_off);
      nrm[i] = f4{m[0], m[1], m[2], 0.0f};
      if (same_nrm) {
        const f4 o = same_nrm[i];
        diff = diff || __float_as_uint(o.x) != __float_as_uint(m[0]) || __float_as_uint(o.y) != __float_as_uint(m[1]) || __float_as_uint(o.z) != __float_as_uint(m[2]);
      }
    }
    if (diff) *differs = 1u;
    ok = isfinite(x) && isfinite(y) && isfinite(z);
  }
  bbox_warp_accumulate(ok, x, y, z, acc);   // finite-point bounding box + count (accumulator was reset by the previous build)
}

// ------------------------------------------------------------------ K2 index build
struct GridGeom {
  float ox, oy, oz, inv_h, h;
  int nx, ny, nz;
};

__device__ __forceinline__ uint32_t cell_of(const GridGeom& g, float x, float y, float z) {
  int cx = (int)floorf((x - g.ox) * g.inv_h);
  int cy = (int)floorf((y - g.oy) * g.inv_h);
  int cz = (int)floorf((z - g.oz) * g.inv_h);
  cx = min(max(cx, 0), g.nx - 1); cy = min(max(cy, 0), g.ny - 1); cz = min(max(cz, 0), g.nz - 1);
  return (uint32_t)((cz * g.ny + cy) * g.nx + cx);
}

__global__ void __launch_bounds__(256)
grid_keys_kernel(const f4* __restrict__ raw, uint32_t n, GridGeom g, uint32_t* __restrict__ keys, BBoxAcc* acc_to_reset) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && acc_to_reset) bbox_reset(acc_to_reset);   // the host has consumed it: ready for the next build
  if (i >= n) return;
  f4 p = raw[i];
  keys[i] = cell_of(g, p.x, p.y, p.z);
}

// occupancy probe for the automatic cell size: marks cells, counts first touches
__global__ void __launch_bounds__(256)
grid_occupancy_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ cell_cnt, uint32_t* n_occ) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t first = 0;
  if (i < n) first = (atomicAdd(&cell_cnt[keys[i]], 1u) == 0u) ? 1u : 0u;
  uint32_t b = __ballot_sync(0xffffffffu, first);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_occ, (uint32_t)__popc(b));
}

__global__ void __launch_bounds__(256)
grid_reorder_kernel(const f4* __restrict__ raw, const uint32_t* __restrict__ sorted_keys,
                    const uint32_t* __restrict__ sorted_vals, uint32_t n, f4* __restrict__ pts,
                    uint32_t* __restrict__ cell_cnt) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  uint32_t i = sorted_vals[s];
  f4 p = raw[i];
  pts[s] = f4{p.x, p.y, p.z, bits_to_float((int32_t)i)};
  if (cell_cnt) atomicAdd(&cell_cnt[sorted_keys[s]], 1u);   // null: the occupancy probe already counted
}

// ------------------------------------------------------------------ K3 covariances
// K3, quad-per-query variant with local-memory lists (k > 20, and the A/B baseline behind LB_KNN=quadlocal): the 4 lanes of a quad scan every cell run of the probe block
// cooperatively (lane q takes points s+q, s+q+4, ... of each contiguous run: 64-byte coalesced reads),
// each keeping its own sorted top-K; a quad-wide K-round merge (shuffle min on (d2, index)) yields the
// exact union top-K in ascending order and accumulates the moments in that order -- the same order the
// one-thread kernel and the oracle use, so results are bit-identical.  4x the resident warps of the
// thread-per-point kernel and a quarter of the insertion work per lane.
template <int K>
struct QuadList {
  float d2[K];
  int oi[K];
  int si[K];
  int cnt;
  __device__ __forceinline__ void init() { cnt = 0; }
  __device__ __forceinline__ void push(float d, int o, int s) {
    if (cnt == K) {
      if (!better(d, o, d2[K - 1], oi[K - 1])) return;
    } else {
      cnt++;
    }
    int j = cnt - 1;
    while (j > 0 && better(d, o, d2[j - 1], oi[j - 1])) {
      d2[j] = d2[j - 1]; oi[j] = oi[j - 1]; si[j] = si[j - 1];
      j--;
    }
    d2[j] = d; oi[j] = o; si[j] = s;
  }
};

// per-row hook of quad_scan_shell: lists without a shared gate do nothing
template <int K>
__device__ __forceinline__ void quad_row_done(QuadList<K>&, unsigned) {}
// RegList: tighten the rejection gate to the quad-wide maximum of the lanes' (K/4)-th best keys.  The union of the
// four lists then holds at least K >= k candidates that are not worse than the gate, so a candidate beyond it
// can never be one of the k nearest.  Lanes hold disjoint quarters of the candidates, so the single-lane
// threshold key[K-1] alone prunes 4x less than one list over all candidates would.
template <int K>
__device__ __forceinline__ void quad_row_done(RegList<K>& L, unsigned qmask) {
  unsigned long long t = L.key[K / 4 - 1];
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    unsigned hi = __shfl_xor_sync(qmask, (unsigned)(t >> 32), o);
    unsigned lo = __shfl_xor_sync(qmask, (unsigned)t, o);
    unsigned long long u = ((unsigned long long)hi << 32) | lo;
    t = u > t ? u : t;
  }
  L.gate = t;
}

template <int K, class List>
__device__ __forceinline__ void quad_scan_shell(const GridView& g, int cx, int cy, int cz, int r, float qx, float qy,
                                                float qz, int sub, List& L, int split_from, unsigned qmask = 0u) {
  int z0 = imax_(cz - r, 0), z1 = imin_(cz + r, g.nz - 1);
  int y0 = imax_(cy - r, 0), y1 = imin_(cy + r, g.ny - 1);
  // r <= 1: the 4 lanes split the POINTS of every run (64-byte coalesced reads of dense cells);
  // r >= 2: the lanes split the ROWS (shells of sparse neighbourhoods are mostly empty rows, whose cost is the
  //         dependent cell_start look-ups: four of them now overlap)
  const bool split_rows = r >= split_from;
  if (r == 1 && !split_rows) {
    // nearest rows first (centre row, then the four face-adjacent rows, then the four corner rows): the k-th
    // best distance tightens early, so fewer of the later candidates have to be inserted into the sorted lists
    const int DZ[9] = {0, 0, 0, -1, 1, -1, -1, 1, 1};
    const int DY[9] = {0, -1, 1, 0, 0, -1, 1, -1, 1};
#pragma unroll 1
    for (int j = 0; j < 9; j++) {
      int z = cz + DZ[j], y = cy + DY[j];
      if (z < 0 || z >= g.nz || y < 0 || y >= g.ny) continue;
      int base = (z * g.ny + y) * g.nx;
      bool face = (j != 0);
      int nseg = face ? 1 : 2;
      for (int k = 0; k < nseg; k++) {
        int xa, xb;
        if (face) { xa = imax_(cx - 1, 0); xb = imin_(cx + 1, g.nx - 1); }
        else { xa = xb = (k == 0) ? cx - 1 : cx + 1; if (xa < 0 || xa >= g.nx) continue; }
        if (xa > xb) continue;
        uint32_t s = g.cell_start[base + xa], e = g.cell_start[base + xb + 1];
        for (uint32_t i = s + sub; i < e; i += 4) {
          f4 p = g.pts[i];
          L.push(dist2(qx, qy, qz, p.x, p.y, p.z), float_to_bits(p.w), (int)i);
        }
      }
      if (qmask) quad_row_done(L, qmask);
    }
    return;
  }
  int row = 0;
  for (int z = z0; z <= z1; z++) {
    bool zface = (iabs_(z - cz) == r);
    for (int y = y0; y <= y1; y++, row++) {
      if (split_rows && (row & 3) != sub) continue;
      bool face = zface || (iabs_(y - cy) == r);
      int base = (z * g.ny + y) * g.nx;
      int nseg = face ? 1 : 2;
      for (int k = 0; k < nseg; k++) {
        int xa, xb;
        if (face) { xa = imax_(cx - r, 0); xb = imin_(cx + r, g.nx - 1); }
        else { xa = xb = (k == 0) ? cx - r : cx + r; if (xa < 0 || xa >= g.nx) continue; }
        if (xa > xb) continue;
        uint32_t s = g.cell_start[base + xa], e = g.cell_start[base + xb + 1];
        for (uint32_t i = s + (split_rows ? 0 : sub); i < e; i += (split_rows ? 1 : 4)) {
          f4 p = g.pts[i];
          L.push(dist2(qx, qy, qz, p.x, p.y, p.z), float_to_bits(p.w), (int)i);
        }
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(128)
knn_cov_quad_kernel(GridView g, int k, double eps, double* __restrict__ cov, int ring_cap,
                    uint32_t* __restrict__ worklist, uint32_t* __restrict__ wl_count, int split_from, int lazy_merge) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t s = t >> 2;
  const int sub = threadIdx.x & 3;
  const unsigned qmask = 0xFu << ((threadIdx.x & 31) & ~3);
  if (s >= (uint32_t)g.n) return;   // whole quads exit together (n is checked per quad)
  f4 q = g.pts[s];
  QuadList<K> L;
  L.init();
  int cx, cy, cz; float minfrac;
  query_cell(g, q.x, q.y, q.z, cx, cy, cz, minfrac);
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  double sum[3], m2[6];
  bool done = false;
  if (r1 > ring_cap) r1 = ring_cap;   // sparse neighbourhoods are finished by knn_cov_tail_kernel (a warp per query)
  for (int r = r0; r <= r1; r++) {
    quad_scan_shell<K>(g, cx, cy, cz, r, q.x, q.y, q.z, sub, L, split_from);
    if (lazy_merge) {
      int total = L.cnt;
      total += __shfl_xor_sync(qmask, total, 1);
      total += __shfl_xor_sync(qmask, total, 2);
      if (total < k && r < r1) continue;   // not even k candidates yet: next shell
    }
    // K-round merge of the four sorted lists
    int p = 0, found = 0;
    float kth = 3.0e38f;
    sum[0] = sum[1] = sum[2] = 0.0;
    m2[0] = m2[1] = m2[2] = m2[3] = m2[4] = m2[5] = 0.0;
    for (int round = 0; round < k; round++) {
      float hd = (p < L.cnt) ? L.d2[p] : 3.0e38f;
      int ho = (p < L.cnt) ? L.oi[p] : 0x7fffffff;
      int hs = (p < L.cnt) ? L.si[p] : -1;
      float bd = hd; int bo = ho; int bs = hs;
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        float od = __shfl_xor_sync(qmask, bd, o);
        int oo = __shfl_xor_sync(qmask, bo, o);
        int os = __shfl_xor_sync(qmask, bs, o);
        if (better(od, oo, bd, bo)) { bd = od; bo = oo; bs = os; }
      }
      if (bs < 0) break;          // fewer than k points in everything scanned so far
      if (bo == ho && hs >= 0) p++;
      found++;
      kth = bd;
      f4 pt = g.pts[bs];
      sum[0] += pt.x; sum[1] += pt.y; sum[2] += pt.z;
      m2[0] += pt.x * pt.x; m2[1] += pt.y * pt.x; m2[2] += pt.y * pt.y;
      m2[3] += pt.z * pt.x; m2[4] += pt.z * pt.y; m2[5] += pt.z * pt.z;
    }
    if (found == k && kth < ring_bound2(g, r, minfrac)) { done = true; break; }
  }
  // the whole grid was covered (r1 not capped): the union top-k is final even without the bound test
  {
    int rr0, rr1;
    ring_range(g, cx, cy, cz, rr0, rr1);
    if (rr1 <= ring_cap) done = true;
  }
  if (!done) {
    if (sub == 0) worklist[atomicAdd(wl_count, 1u)] = s;
    return;
  }
  double out[6];
  cov_from_moments(sum, m2, k, eps, out);
  if (sub == 0) {
    double* d = cov + 6 * (size_t)s;
#pragma unroll
    for (int e = 0; e < 6; e++) d[e] = out[e];
  }
}

// What a k-NN kernel does with the k neighbours of a query, visited in ascending (d2, index) order:
// CovFin  -> GICP covariance (gicp.hpp:85-154): double moments -> Jacobi -> regularised, written in sorted order;
// NormalFin -> PCL NormalEstimation (SURVEY 8f row f2, hd.h): nine float accumulators -> eigen33 -> flipped normal +
//              curvature, written at the point's ORIGINAL index.
struct CovFin {
  double eps;
  double* cov;
  double sum[3], m2[6];
  __device__ __forceinline__ bool skip(const f4&) const { return false; }
  __device__ __forceinline__ void reset() {
    sum[0] = sum[1] = sum[2] = 0.0;
    m2[0] = m2[1] = m2[2] = m2[3] = m2[4] = m2[5] = 0.0;
  }
  __device__ __forceinline__ void add(const f4& pt) {
    sum[0] += pt.x; sum[1] += pt.y; sum[2] += pt.z;
    m2[0] += pt.x * pt.x; m2[1] += pt.y * pt.x; m2[2] += pt.y * pt.y;
    m2[3] += pt.z * pt.x; m2[4] += pt.z * pt.y; m2[5] += pt.z * pt.z;
  }
  __device__ __forceinline__ void finish(uint32_t s, const f4&, int k, bool writer) {
    double out[6];
    cov_from_moments(sum, m2, k, eps, out);
    if (writer) {
      double* d = cov + 6 * (size_t)s;
#pragma unroll
      for (int e = 0; e < 6; e++) d[e] = out[e];
    }
  }
};

// Rolling submap (row f3): covariances only for the points inserted since the last pass (original index >= first_new),
// written into the submap's per-point cache in ORIGINAL (insertion) order; the other queries leave at once.
struct CovFinIncr {
  double eps;
  double* cache;       // insertion order, 6 per point
  int first_new;
  double sum[3], m2[6];
  __device__ __forceinline__ bool skip(const f4& q) const { return float_to_bits(q.w) < first_new; }
  __device__ __forceinline__ void reset() {
    sum[0] = sum[1] = sum[2] = 0.0;
    m2[0] = m2[1] = m2[2] = m2[3] = m2[4] = m2[5] = 0.0;
  }
  __device__ __forceinline__ void add(const f4& pt) {
    sum[0] += pt.x; sum[1] += pt.y; sum[2] += pt.z;
    m2[0] += pt.x * pt.x; m2[1] += pt.y * pt.x; m2[2] += pt.y * pt.y;
    m2[3] += pt.z * pt.x; m2[4] += pt.z * pt.y; m2[5] += pt.z * pt.z;
  }
  __device__ __forceinline__ void finish(uint32_t, const f4& q, int k, bool writer) {
    double out[6];
    cov_from_moments(sum, m2, k, eps, out);
    if (writer) {
      double* d = cache + 6 * (size_t)float_to_bits(q.w);
#pragma unroll
      for (int e = 0; e < 6; e++) d[e] = out[e];
    }
  }
};

struct NormalFin {
  float vp[3];
  f4* out;            // original order: (nx, ny, nz, curvature)
  NormalAccum acc;
  __device__ __forceinline__ bool skip(const f4&) const { return false; }
  __device__ __forceinline__ void reset() { acc.reset(); }
  __device__ __forceinline__ void add(const f4& pt) { acc.add(pt.x, pt.y, pt.z); }
  __device__ __forceinline__ void finish(uint32_t, const f4& q, int k, bool writer) {
    float o[4];
    pcl_normal_from_accum(acc, k, q.x, q.y, q.z, vp, o);
    if (writer) out[float_to_bits(q.w)] = f4{o[0], o[1], o[2], o[3]};
  }
};

// K3, register-resident variant (the default for k <= 20).  Same quad-per-query scan, same (d2, index) order and
// same summation order as knn_cov_quad_kernel, hence the same bits; what changes is where the candidate lists
// live.  Each lane's sorted list is a RegList (static indexing, fully unrolled: ~60 registers), so an insertion is
// ~100 independent select instructions instead of a chain of dependent local-memory loads and stores -- the
// long-scoreboard stalls that held the old kernel at ~16 % of the issue rate.  The 4-way merge needs a moving
// head per lane, i.e. dynamic indexing: the lists are copied once per merge into shared memory ([entry][thread]
// layout, conflict-free) and popped from there.  Lists hold keys only; the k selected points are re-read through
// their original index (`raw`, the original-order copy of the cloud: same coordinates as the sorted copy).
constexpr int KQ_THREADS = 128;
template <int K, class Fin>
__device__ __forceinline__ void knn_quad_query(const GridView& g, const f4* __restrict__ raw, int k, Fin& fin, int split_from,
                                               int ring_cap, uint32_t* __restrict__ worklist,
                                               uint32_t* __restrict__ wl_count, uint32_t s, int sub, unsigned qmask, int tid,
                                               uint32_t* m_d, uint32_t* m_o);
#ifndef KQ_MINB
#define KQ_MINB 4
#endif
template <int K, class Fin>
__global__ void __launch_bounds__(KQ_THREADS, KQ_MINB)
knn_cov_quadreg_kernel(GridView g, const f4* __restrict__ raw, int k, Fin fin, int split_from,
                       int ring_cap, uint32_t* __restrict__ worklist, uint32_t* __restrict__ wl_count,
                       uint32_t* __restrict__ next_query /*nullable: dynamic distribution of 8-query batches*/) {
  __shared__ uint32_t m_d[(K + 1) * KQ_THREADS];
  __shared__ uint32_t m_o[(K + 1) * KQ_THREADS];
  const int sub = threadIdx.x & 3;
  const int lane = threadIdx.x & 31;
  const unsigned qmask = 0xFu << (lane & ~3);
  const int tid = threadIdx.x;
  m_d[K * KQ_THREADS + tid] = 0xffffffffu; m_o[K * KQ_THREADS + tid] = 0xffffffffu;   // sentinel behind every list
  // Static mode (next_query == nullptr): one batch per warp, taken from the thread index.  Dynamic mode: a
  // resident grid whose warps pull batches of 8 consecutive queries from a counter until the cloud is done -- the
  // per-query cost varies a lot (rings scanned), and a static grid of ~1.6 waves ends with a long, mostly idle tail.
  uint32_t wbase = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8;
  for (;; ) {
    if (next_query) {
      uint32_t b = 0;
      if (lane == 0) b = atomicAdd(next_query, 8u);
      wbase = __shfl_sync(0xffffffffu, b, 0);
    }
    if (wbase >= (uint32_t)g.n) return;
    knn_quad_query<K>(g, raw, k, fin, split_from, ring_cap, worklist, wl_count, wbase + (uint32_t)(lane >> 2), sub, qmask,
                      tid, m_d, m_o);
    if (!next_query) return;
    __syncwarp();
  }
}

template <int K, class Fin>
__device__ __forceinline__ void knn_quad_query(const GridView& g, const f4* __restrict__ raw, int k, Fin& fin, int split_from,
                                               int ring_cap, uint32_t* __restrict__ worklist,
                                               uint32_t* __restrict__ wl_count, uint32_t s, int sub, unsigned qmask, int tid,
                                               uint32_t* m_d, uint32_t* m_o) {
  if (s >= (uint32_t)g.n) return;   // whole quads exit together
  f4 q = g.pts[s];
  if (fin.skip(q)) return;          // (the four lanes of a quad share the query)
  RegList<K> L;
  L.init();
  int cx, cy, cz; float minfrac;
  query_cell(g, q.x, q.y, q.z, cx, cy, cz, minfrac);
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  // Shell r of a query in a sparse corner of the grid is (2r+1)^2 mostly empty rows of dependent look-ups: past
  // ring_cap the query goes to knn_cov_tail_kernel, where a whole warp shares the rows of each shell.
  bool done = r1 <= ring_cap;          // the whole grid gets scanned below: final even without the bound test
  const int r_last = r1 < ring_cap ? r1 : ring_cap;
  for (int r = r0; r <= r_last; r++) {
    quad_scan_shell<K>(g, cx, cy, cz, r, q.x, q.y, q.z, sub, L, split_from, qmask);
    quad_row_done(L, qmask);
    int total = L.cnt;
    total += __shfl_xor_sync(qmask, total, 1);
    total += __shfl_xor_sync(qmask, total, 2);
    if (total < k && r < r_last) continue;   // not even k candidates yet: next shell
    if (total < k && !done) break;           // capped and still short of k: the tail kernel finishes this query
#pragma unroll
    for (int j = 0; j < K; j++) {
      m_d[j * KQ_THREADS + tid] = (uint32_t)(L.key[j] >> 32);
      m_o[j * KQ_THREADS + tid] = (uint32_t)L.key[j];
    }
    int p = 0, found = 0;
    float kth = 3.0e38f;
    fin.reset();
    for (int round = 0; round < k; round++) {
      const uint32_t hd = m_d[p * KQ_THREADS + tid], ho = m_o[p * KQ_THREADS + tid];
      uint32_t bd = hd, bo = ho;
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        uint32_t od = __shfl_xor_sync(qmask, bd, o);
        uint32_t oo = __shfl_xor_sync(qmask, bo, o);
        if (od < bd || (od == bd && oo < bo)) { bd = od; bo = oo; }
      }
      if (bd == 0xffffffffu && bo == 0xffffffffu) break;   // fewer than k points in everything scanned so far
      if (bd == hd && bo == ho) p++;                       // original indices are unique: exactly one lane pops
      found++;
      kth = bits_to_float((int32_t)bd);
      fin.add(raw[bo]);
    }
    if (found == k && kth < ring_bound2(g, r, minfrac)) { done = true; break; }
  }
  if (!done) {
    if (sub == 0) worklist[atomicAdd(wl_count, 1u)] = s;
    return;
  }
  fin.finish(s, q, k, sub == 0);
}

// K3 tail: one WARP per query for the sparse neighbourhoods the quad kernel gave up on.  The rows of each
// shell are spread over the 32 lanes (a shell of radius r has (2r+1)^2 rows, most of them empty: the cost is
// the dependent cell_start -> points loads, which now overlap 32-wide); a 32-way merge on packed
// (d2, index) keys yields the exact top-k in ascending order.
template <int K, class Fin>
__global__ void __launch_bounds__(128)
knn_cov_tail_kernel(GridView g, int k, Fin fin, const uint32_t* __restrict__ worklist,
                    const uint32_t* __restrict__ wl_count) {
  const int lane = threadIdx.x & 31;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t count = *wl_count;
  for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < count; w += nwarps) {
    const uint32_t s = worklist[w];
    f4 q = g.pts[s];
    QuadList<K> L;
    L.init();
    int cx, cy, cz; float minfrac;
    query_cell(g, q.x, q.y, q.z, cx, cy, cz, minfrac);
    int r0, r1;
    ring_range(g, cx, cy, cz, r0, r1);
    for (int r = r0; r <= r1; r++) {
      // rows of the shell, lane-strided
      const int side = 2 * r + 1;
      for (int j = lane; j < side * side; j += 32) {
        int dz = j / side - r, dy = j % side - r;
        int z = cz + dz, y = cy + dy;
        if (z < 0 || z >= g.nz || y < 0 || y >= g.ny) continue;
        bool face = (iabs_(dz) == r) || (iabs_(dy) == r);
        int base = (z * g.ny + y) * g.nx;
        int nseg = face ? 1 : 2;
        for (int sgm = 0; sgm < nseg; sgm++) {
          int xa, xb;
          if (face) { xa = imax_(cx - r, 0); xb = imin_(cx + r, g.nx - 1); }
          else { xa = xb = (sgm == 0) ? cx - r : cx + r; if (xa < 0 || xa >= g.nx) continue; }
          if (xa > xb) continue;
          uint32_t a = g.cell_start[base + xa], e = g.cell_start[base + xb + 1];
          for (uint32_t i = a; i < e; i++) {
            f4 p = g.pts[i];
            L.push(dist2(q.x, q.y, q.z, p.x, p.y, p.z), float_to_bits(p.w), (int)i);
          }
        }
      }
      __syncwarp();
      // enough candidates in total?  (cheap test before the 32-way merge)
      int total = L.cnt;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
      if (total < k && r < r1) continue;
      // k-round merge on packed keys: (float bits of d2 (non-negative: order preserving) << 32) | original index
      int p = 0, found = 0;
      float kth = 3.0e38f;
      fin.reset();
      for (int round = 0; round < k; round++) {
        unsigned long long key = (p < L.cnt)
            ? (((unsigned long long)__float_as_uint(L.d2[p]) << 32) | (unsigned)L.oi[p])
            : 0xffffffffffffffffull;
        unsigned long long best = key;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
          best = other < best ? other : best;
        }
        if (best == 0xffffffffffffffffull) break;
        unsigned owner = __ballot_sync(0xffffffffu, key == best);
        int src_lane = __ffs(owner) - 1;
        int bs = __shfl_sync(0xffffffffu, (p < L.cnt) ? L.si[p] : -1, src_lane);
        if (lane == src_lane) p++;
        found++;
        kth = __uint_as_float((unsigned)(best >> 32));
        fin.add(g.pts[bs]);
      }
      if (found == k && kth < ring_bound2(g, r, minfrac)) break;
    }
    fin.finish(s, q, k, lane == 0);
    __syncwarp();
  }
}

// Row f2, radius mode of the NormalComputation nodelet (normal_computation.cc:73-77: norm_est_.setRadiusSearch): the
// neighbourhood of a point is EVERY point closer than the radius (FLANN RadiusResultSet: d2 < float(radius^2), strict),
// visited in ascending (d2, index) order -- the order PCL's nine float32 accumulators see them in, so it defines the
// rounding.  One warp per query: the lanes scan the rows of the shells that can reach the radius and append their hits
// (packed (d2, index) keys) to a list in shared memory; the warp sorts the list (bitonic), then lanes 0-8 each run one
// of the nine accumulators over the sorted neighbours (staged 32 at a time) and lane 0 finishes the normal.  Fewer than
// three neighbours -> NaN normal (pcl::computePointNormal), which the nodelet then drops (:53-57): `valid` flags them.
constexpr int NR_CAP = 2048;          // neighbours per query held in shared memory (16 KB per warp)
constexpr int NR_WARPS = 4;
__global__ void __launch_bounds__(NR_WARPS * 32)
normals_radius_kernel(GridView g, const f4* __restrict__ raw, float r2, float vp0, float vp1, float vp2, f4* __restrict__ out,
                      uint32_t* __restrict__ valid, int* __restrict__ overflow) {
  extern __shared__ unsigned long long nr_keys[];       // [NR_WARPS][NR_CAP]
  __shared__ int cnt[NR_WARPS];
  __shared__ float ptbuf[NR_WARPS][32][3];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long* keys = nr_keys + (size_t)w * NR_CAP;
  const uint32_t nwarps = gridDim.x * NR_WARPS;
  const float vp[3] = {vp0, vp1, vp2};
  for (uint32_t s = blockIdx.x * NR_WARPS + w; s < (uint32_t)g.n; s += nwarps) {
    const f4 q = g.pts[s];
    if (lane == 0) cnt[w] = 0;
    __syncwarp();
    int cx, cy, cz; float minfrac;
    query_cell(g, q.x, q.y, q.z, cx, cy, cz, minfrac);
    int r0, r1;
    ring_range(g, cx, cy, cz, r0, r1);
    for (int r = r0; r <= r1; r++) {
      const int side = 2 * r + 1;
      for (int j = lane; j < side * side; j += 32) {
        const int dz = j / side - r, dy = j % side - r;
        const int z = cz + dz, y = cy + dy;
        if (z < 0 || z >= g.nz || y < 0 || y >= g.ny) continue;
        const bool face = (iabs_(dz) == r) || (iabs_(dy) == r);
        const int base = (z * g.ny + y) * g.nx;
        const int nseg = face ? 1 : 2;
        for (int sgm = 0; sgm < nseg; sgm++) {
          int xa, xb;
          if (face) { xa = imax_(cx - r, 0); xb = imin_(cx + r, g.nx - 1); }
          else { xa = xb = (sgm == 0) ? cx - r : cx + r; if (xa < 0 || xa >= g.nx) continue; }
          if (xa > xb) continue;
          const uint32_t a = g.cell_start[base + xa], e = g.cell_start[base + xb + 1];
          for (uint32_t i = a; i < e; i++) {
            const f4 p = g.pts[i];
            const float d2 = dist2(q.x, q.y, q.z, p.x, p.y, p.z);
            if (d2 < r2) {
              const int pos = atomicAdd(&cnt[w], 1);
              if (pos < NR_CAP) keys[pos] = RegList<1>::make_key(d2, float_to_bits(p.w));
            }
          }
        }
      }
      __syncwarp();
      if (ring_bound2(g, r, minfrac) >= r2) break;      // nothing beyond the scanned block can be inside the radius
    }
    __syncwarp();
    int M = cnt[w];
    if (M > NR_CAP) { if (lane == 0) atomicExch(overflow, 1); M = 0; }      // reported by the host as LB_ERR_CAPACITY
    // bitonic sort of the M keys (ascending (d2, index)), padded to a power of two with all-ones keys
    int P = 32;
    while (P < M) P <<= 1;
    for (int i = M + lane; i < P; i += 32) keys[i] = ~0ull;
    __syncwarp();
    for (int k = 2; k <= P; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = lane; i < P; i += 32) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = keys[i], b = keys[ixj];
            const bool up = (i & k) == 0;
            if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
          }
        }
        __syncwarp();
      }
    // the nine float32 accumulators of computeMeanAndCovarianceMatrix, one per lane, in neighbour order
    float acc = 0.f;
    for (int base = 0; base < M; base += 32) {
      if (base + lane < M) {
        const f4 p = raw[(uint32_t)keys[base + lane]];
        ptbuf[w][lane][0] = p.x; ptbuf[w][lane][1] = p.y; ptbuf[w][lane][2] = p.z;
      }
      __syncwarp();
      if (lane < 9) {
        const int m = min(32, M - base);
        for (int t = 0; t < m; t++) {
          const float x = ptbuf[w][t][0], y = ptbuf[w][t][1], z = ptbuf[w][t][2];
          float term;
          switch (lane) {
            case 0: term = x * x; break; case 1: term = x * y; break; case 2: term = x * z; break;
            case 3: term = y * y; break; case 4: term = y * z; break; case 5: term = z * z; break;
            case 6: term = x; break; case 7: term = y; break; default: term = z; break;
          }
          acc = acc + term;
        }
      }
      __syncwarp();
    }
    NormalAccum A;
#pragma unroll
    for (int c = 0; c < 9; c++) A.a[c] = __shfl_sync(0xffffffffu, acc, c);
    if (lane == 0) {
      float o[4];
      const float qnan = __int_as_float(0x7fc00000);
      if (M < 3) { o[0] = o[1] = o[2] = o[3] = qnan; }
      else pcl_normal_from_accum(A, M, q.x, q.y, q.z, vp, o);
      const int orig = float_to_bits(q.w);
      out[orig] = f4{o[0], o[1], o[2], o[3]};
      valid[orig] = (isfinite(o[0]) && isfinite(o[1]) && isfinite(o[2])) ? 1u : 0u;
    }
    __syncwarp();
  }
}

// pcl::removeNaNNormalsFromPointCloud: the indices of the points that stay, ascending
__global__ void __launch_bounds__(256)
compact_indices_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t n, int32_t* __restrict__ out_idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flags[i]) out_idx[pos[i]] = (int32_t)i;
}

// K3': covariance from a stored normal (the reference's default mode when normals are present)
__global__ void __launch_bounds__(256)
normal_cov_kernel(const f4* __restrict__ pts, const f4* __restrict__ nrm, uint32_t n, double eps, double* __restrict__ cov) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  int i = float_to_bits(pts[s].w);
  f4 m = nrm[i];
  double out[6];
  cov_from_normal(m.x, m.y, m.z, eps, out);
  double* d = cov + 6 * (size_t)s;
#pragma unroll
  for (int e = 0; e < 6; e++) d[e] = out[e];
}

// ------------------------------------------------------------------ K6 transforms
struct Mat34 { float m[12]; };
struct Mat33d { double m[9]; };

__global__ void __launch_bounds__(256)
prep_source_kernel(const f4* __restrict__ pts, uint32_t n, Mat34 G, f4* __restrict__ work) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  f4 p = pts[s];
  float x, y, z;
  xform_pcl(G.m, p.x, p.y, p.z, x, y, z);
  work[s] = f4{x, y, z, p.w};
}

// out[i] = T * raw[i]  (original order), written into a strided layout; normals rotated if present
__global__ void __launch_bounds__(256)
transform_kernel(const f4* __restrict__ raw, const f4* __restrict__ nrm, uint32_t n, Mat34 T, uint8_t* __restrict__ out,
                 uint32_t stride, uint32_t xyz_off, int normal_off) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  f4 p = raw[i];
  float x, y, z;
  xform_pcl(T.m, p.x, p.y, p.z, x, y, z);
  float* q = reinterpret_cast<float*>(out + (size_t)i * stride + xyz_off);
  q[0] = x; q[1] = y; q[2] = z;
  if (normal_off >= 0 && nrm) {
    f4 m = nrm[i];
    // pcl::transformPointCloudWithNormals: rotation only (so3), p0 + (p1 + p2)
    float* r = reinterpret_cast<float*>(out + (size_t)i * stride + normal_off);
    r[0] = T.m[0] * m.x + (T.m[1] * m.y + T.m[2] * m.z);
    r[1] = T.m[4] * m.x + (T.m[5] * m.y + T.m[6] * m.z);
    r[2] = T.m[8] * m.x + (T.m[9] * m.y + T.m[10] * m.z);
  }
}

// exact 1-NN of arbitrary queries in a grid (PointCloudLocalization.cc:327-336)
__global__ void __launch_bounds__(128)
nn_query_kernel(GridView g, const uint8_t* __restrict__ q, uint32_t n, uint32_t stride, int32_t* __restrict__ idx,
                float* __restrict__ d2, float max_d2) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = reinterpret_cast<const float*>(q + (size_t)i * stride);
  int bo; float bd;
  int s = nn1(g, p[0], p[1], p[2], max_d2, bo, bd);
  idx[i] = (s >= 0) ? bo : -1;
  d2[i] = bd;
}

// Exact 1-NN, warp-per-query (the HBM-resident regime: big maps, many queries).  The rows of the probe block are
// looked up by different lanes at once, then the candidate points of all rows are fetched FLATTENED: lane l takes
// candidates l, l+32, ... of the concatenated runs, so every load instruction moves 32 independent 16-byte points
// (512 contiguous bytes where the runs are dense).  Each lane keeps its best packed key (d2 bits << 32 | original
// index); one 64-bit warp-min per shell decides.  First step = the whole 3x3x3 block (nine 3-cell runs).
struct NnWarpSmem { uint32_t a0[32], a1[32]; int n0[32], off[33]; };

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long other = __shfl_xor_sync(0xffffffffu, v, o);
    v = other < v ? other : v;
  }
  return v;
}

// returns the best packed key (all lanes), 0xffff... when nothing is within max_d2
__device__ __forceinline__ unsigned long long nn1_warp(const GridView& g, float qx, float qy, float qz, float max_d2,
                                                      NnWarpSmem& w) {
  const int lane = threadIdx.x & 31;
  int cx, cy, cz; float minfrac;
  query_cell(g, qx, qy, qz, cx, cy, cz, minfrac);
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  unsigned long long best = 0xffffffffffffffffull;
  const unsigned long long gate = ((unsigned long long)__float_as_uint(max_d2)) << 32;   // keys >= gate fail d2 < max_d2
  bool first = true;
  if (r0 > 1 && ring_bound2(g, r0 - 1, minfrac) >= max_d2) return 0xffffffffffffffffull;   // query far outside the grid
  for (int r = (r0 <= 1 ? 1 : r0); r <= (r1 < 1 ? 1 : r1); r++) {
    // rows of this step: the full (2r+1)^2 block when it is the first step with r == 1, else the shell of radius r;
    // only rows that intersect the grid are enumerated
    const bool block = first && r == 1;
    first = false;
    const int z0 = imax_(cz - r, 0), z1 = imin_(cz + r, g.nz - 1);
    const int y0 = imax_(cy - r, 0), y1 = imin_(cy + r, g.ny - 1);
    const int ny_c = y1 - y0 + 1;
    const int nrows = (z1 >= z0 && y1 >= y0) ? (z1 - z0 + 1) * ny_c : 0;
    for (int rowbase = 0; rowbase < nrows; rowbase += 32) {
      uint32_t a0 = 0, a1 = 0; int n0 = 0, n1 = 0;
      int j = rowbase + lane;
      if (j < nrows) {
        int z = z0 + j / ny_c, y = y0 + j % ny_c;
        int base = (z * g.ny + y) * g.nx;
        bool face = block || (iabs_(z - cz) == r) || (iabs_(y - cy) == r);
        if (face) {
          int xa = imax_(cx - r, 0), xb = imin_(cx + r, g.nx - 1);
          if (xa <= xb) { a0 = g.cell_start[base + xa]; n0 = (int)(g.cell_start[base + xb + 1] - a0); }
        } else {
          int x0 = cx - r, x1 = cx + r;
          if (x0 >= 0 && x0 < g.nx) { a0 = g.cell_start[base + x0]; n0 = (int)(g.cell_start[base + x0 + 1] - a0); }
          if (x1 >= 0 && x1 < g.nx) { a1 = g.cell_start[base + x1]; n1 = (int)(g.cell_start[base + x1 + 1] - a1); }
        }
      }
      int len = n0 + n1;
      int incl = len;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      if (total == 0) continue;
      __syncwarp();
      w.a0[lane] = a0; w.a1[lane] = a1; w.n0[lane] = n0; w.off[lane] = incl - len;
      if (lane == 31) w.off[32] = total;
      __syncwarp();
#ifndef NNW_UNROLL
#define NNW_UNROLL 2
#endif
#if NNW_UNROLL == 2
      // two candidates per lane and trip: both point loads are in flight before either is used
      int cur = 0;
      for (int idx = lane; idx < total; idx += 64) {
        while (idx >= w.off[cur + 1]) cur++;
        int local = idx - w.off[cur];
        int nn0 = w.n0[cur];
        uint32_t pi = (local < nn0) ? (w.a0[cur] + (uint32_t)local) : (w.a1[cur] + (uint32_t)(local - nn0));
        const int idx2 = idx + 32;
        const bool two = idx2 < total;
        uint32_t pj = pi;
        if (two) {
          while (idx2 >= w.off[cur + 1]) cur++;
          int local2 = idx2 - w.off[cur];
          int nn2 = w.n0[cur];
          pj = (local2 < nn2) ? (w.a0[cur] + (uint32_t)local2) : (w.a1[cur] + (uint32_t)(local2 - nn2));
        }
        f4 p = g.pts[pi];
        f4 p2 = g.pts[pj];
        unsigned long long key = ((unsigned long long)__float_as_uint(dist2(qx, qy, qz, p.x, p.y, p.z)) << 32) |
                                 (unsigned)float_to_bits(p.w);
        unsigned long long key2 = ((unsigned long long)__float_as_uint(dist2(qx, qy, qz, p2.x, p2.y, p2.z)) << 32) |
                                  (unsigned)float_to_bits(p2.w);
        best = key < best ? key : best;
        best = key2 < best ? key2 : best;       // pj == pi when there is no second candidate: harmless duplicate
      }
#else
      int cur = 0;
      for (int idx = lane; idx < total; idx += 32) {
        while (idx >= w.off[cur + 1]) cur++;
        int local = idx - w.off[cur];
        int nn0 = w.n0[cur];
        uint32_t pi = (local < nn0) ? (w.a0[cur] + (uint32_t)local) : (w.a1[cur] + (uint32_t)(local - nn0));
        f4 p = g.pts[pi];
        unsigned long long key = ((unsigned long long)__float_as_uint(dist2(qx, qy, qz, p.x, p.y, p.z)) << 32) |
                                 (unsigned)float_to_bits(p.w);
        best = key < best ? key : best;
      }
#endif
    }
    unsigned long long wbest = warp_min_u64(best);
    float lb2 = ring_bound2(g, r, minfrac);
    if (lb2 >= max_d2) { best = wbest; break; }
    if (wbest < gate && __uint_as_float((unsigned)(wbest >> 32)) < lb2) { best = wbest; break; }
    if (r == (r1 < 1 ? 1 : r1)) best = wbest;
  }
  // every exit of the loop leaves the warp-wide minimum in `best` (the loop body runs at least once)
  return best < gate ? best : 0xffffffffffffffffull;
}

__global__ void __launch_bounds__(256)
nn_query_warp_kernel(GridView g, const uint8_t* __restrict__ q, uint32_t n, uint32_t stride, int32_t* __restrict__ idx,
                     float* __restrict__ d2, float max_d2) {
  __shared__ NnWarpSmem sm[8];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t nwarps = gridDim.x * 8;
  for (uint32_t i = blockIdx.x * 8 + wib; i < n; i += nwarps) {
    const float* p = reinterpret_cast<const float*>(q + (size_t)i * stride);
    float qx = p[0], qy = p[1], qz = p[2];   // (prefetching the next query here was slower)
    unsigned long long best = nn1_warp(g, qx, qy, qz, max_d2, sm[wib]);
    if (lane == 0) {
      bool ok = best != 0xffffffffffffffffull;
      idx[i] = ok ? (int32_t)(unsigned)(best & 0xffffffffull) : -1;
      d2[i] = ok ? __uint_as_float((unsigned)(best >> 32)) : max_d2;
    }
  }
}

// candidate-scan statistics of the same search (profiling aid for the NN roofline, SURVEY 8d: B_nn = Nq (16 + 16 c + 8)):
// counts the target points a query visits.
__global__ void __launch_bounds__(128)
nn_count_kernel(GridView g, const uint8_t* __restrict__ q, uint32_t n, uint32_t stride, float max_d2,
                unsigned long long* __restrict__ total) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned cnt = 0;
  if (i < n) {
    const float* p = reinterpret_cast<const float*>(q + (size_t)i * stride);
    float qx = p[0], qy = p[1], qz = p[2];
    int cx, cy, cz; float minfrac;
    query_cell(g, qx, qy, qz, cx, cy, cz, minfrac);
    int r0, r1;
    ring_range(g, cx, cy, cz, r0, r1);
    float bd2 = max_d2; bool found = false; int bi = 0x7fffffff;
    for (int r = r0; r <= r1; r++) {
      if (r > r0 || r0 > 0) {
        float lb2 = ring_bound2(g, r - 1, minfrac);
        if (lb2 >= max_d2) break;
        if (found && bd2 < lb2) break;
      }
      visit_shell(g, cx, cy, cz, r, [&](float x, float y, float z, int oi, int si) {
        cnt++;
        float d = dist2(qx, qy, qz, x, y, z);
        if (!found) { if (d < max_d2) { found = true; bd2 = d; bi = oi; } }
        else if (better(d, oi, bd2, bi)) { bd2 = d; bi = oi; }
      });
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(total, (unsigned long long)cnt);
}

// ------------------------------------------------------------------ block / grid reductions
// Fixed-shape, bitwise run-to-run deterministic reduction of NV doubles held by the threads of the first
// NWARPS warps [W0, W0+NWARPS): warp shuffle tree -> per-warp slots in shared memory -> lane e of warp 0 adds the NWARPS
// slots of value e in warp order.  Lane e (< NV) of warp 0 returns total e; every other thread gets 0.
// (Only NWARPS warps shuffle: SHFL issues at one warp-instruction per cycle per SM, so the cost is
// NWARPS * NV * 10 cycles.)  All threads of the CTA must call it (two CTA barriers inside).
template <int NV, int NWARPS, int W0 = 0>
__device__ __forceinline__ double block_reduce(double* v, double* red /*[NWARPS][NV]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp >= W0 && warp < W0 + NWARPS) {
#pragma unroll
    for (int e = 0; e < NV; e++) {
      double x = v[e];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
      if (lane == 0) red[(warp - W0) * NV + e] = x;
    }
  }
  __syncthreads();
  double tot = 0.0;
  if (warp == 0 && lane < NV) {
#pragma unroll
    for (int w = 0; w < NWARPS; w++) tot += red[w * NV + lane];
  }
  __syncthreads();
  return tot;
}

// One published value of a CTA slot: the double is split in two 32-bit halves, each packed with the low 32
// bits of the collective's epoch into an 8-byte word (8-byte accesses are single L2 transactions).  A reader
// loads both words at once and retries until both tags match: ONE round trip, no fences (a gpu-scope fence
// would invalidate L1, where the leader warp keeps its BFGS state), no reliance on 16-byte atomicity.
struct __align__(16) SlotWord { unsigned long long lo, hi; };

__device__ __forceinline__ void slot_store(SlotWord* p, double v, unsigned long long epoch) {
  unsigned long long bits = (unsigned long long)__double_as_longlong(v);
  unsigned long long tag = (epoch & 0xffffffffull) << 32;
  unsigned long long lo = tag | (bits & 0xffffffffull), hi = tag | (bits >> 32);
  // published with atomic exchanges: atomics are performed at L2 immediately, whereas a plain store can sit in
  // the SM's write path for microseconds when no fence pushes it out
  atomicExch(&p->lo, lo);
  atomicExch(&p->hi, hi);
}
__device__ __forceinline__ bool slot_try(const SlotWord* p, unsigned long long epoch, double& v) {
  unsigned long long lo, hi;
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "l"(p) : "memory");
  unsigned long long tag = epoch & 0xffffffffull;
  if ((lo >> 32) != tag || (hi >> 32) != tag) return false;
  v = __longlong_as_double((long long)((hi << 32) | (lo & 0xffffffffull)));
  return true;
}
// Gather the NV published words of all `ncta` slots and sum each value over the slots in a fixed order.
// Every (slot, value) pair is polled by exactly one thread of the CTA, all pairs in flight at once (one L2
// round trip when nobody is late); the values land in a shared matrix and warp w then sums rows e = w,
// w + nwarps, ... lane-strided + shuffle tree.  out[e] (shared) valid after the trailing CTA barrier.
// A thread holds at most CHUNK words in registers: with fewer than all of its pairs (the solve kernel's register
// budget), the pairs are gathered CHUNK per thread at a time, one after the other.
constexpr int AL_MAXCTA = 160;
constexpr long long AL_POLL_DELAY = 400;   // cycles before the first poll; chosen on an earlier GPU, not re-tuned for the H100
template <int NV, int THREADS, int CHUNK = (AL_MAXCTA * NV + THREADS - 1) / THREADS>
__device__ __forceinline__ void slots_all_sum(const SlotWord* buf, int ncta, unsigned long long epoch,
                                              double* mat /*[NV][AL_MAXCTA] shared*/, double* out /*shared [NV]*/,
                                              long long* prof_rounds = nullptr, long long poll_delay = AL_POLL_DELAY) {
  static_assert(CHUNK >= 1 && CHUNK <= 32, "one bit of the pending mask per word in flight");
  const int npairs = ncta * NV;
  // every CTA publishes at about the same time and a publication takes a while to land in L2: polling at once
  // wastes a full round trip on words that are not there yet, so hold the first poll back a little
  {
    const long long t_start = clock64();
    while (clock64() - t_start < poll_delay) {}
  }
  int rounds = 0;
  for (int first = 0; first < npairs; first += CHUNK * THREADS) {
    unsigned pending = 0;
#pragma unroll
    for (int k = 0; k < CHUNK; k++)
      if (first + (int)threadIdx.x + k * THREADS < npairs) pending |= 1u << k;
    while (pending) {
      rounds++;
      // issue every pending load first, then look at the tags: the loads of one round overlap (one L2 round trip)
      unsigned long long lo[CHUNK], hi[CHUNK];
#pragma unroll
      for (int k = 0; k < CHUNK; k++) {
        lo[k] = 0; hi[k] = 0;
        if (pending & (1u << k)) {
          int pr = first + threadIdx.x + k * THREADS;
          int b = pr / NV, e = pr - b * NV;
          const SlotWord* p = &buf[(size_t)b * AL_PSTRIDE + e];
          asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(lo[k]), "=l"(hi[k]) : "l"(p));
        }
      }
      const unsigned long long tag = epoch & 0xffffffffull;
#pragma unroll
      for (int k = 0; k < CHUNK; k++)
        if ((pending & (1u << k)) && (lo[k] >> 32) == tag && (hi[k] >> 32) == tag) {
          int pr = first + threadIdx.x + k * THREADS;
          int b = pr / NV, e = pr - b * NV;
          mat[e * AL_MAXCTA + b] = __longlong_as_double((long long)((hi[k] << 32) | (lo[k] & 0xffffffffull)));
          pending &= ~(1u << k);
        }
    }
  }
  if (prof_rounds) { prof_rounds[0] += rounds; prof_rounds[1] += clock64(); }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = warp; e < NV; e += THREADS / 32) {
    double x = 0.0;
    for (int b = lane; b < ncta; b += 32) x += mat[e * AL_MAXCTA + b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if (lane == 0) out[e] = x;
  }
  __syncthreads();
}

// ------------------------------------------------------------------ K4 correspondences
struct CorrArgs {
  GridView tgt;
  const double* tgt_cov;   // sorted-target order, 6 per point
  const f4* src;           // guess-transformed source, sorted order
  const double* src_cov;   // 6 per point
  int n_src;
  float max_d2;            // gate, float-exact equivalent of corr_dist^2 (gicp.hpp:438,483)
  f4* corr;                // matched target point, w = sorted target index or -1
  double* M;               // 6 per source point
  int nn_mode;             // search of the correspondence step: 0 each thread on its own, 1 staged (cp.async), 2 staged (TMA)
  int nn_cap;              // staged: candidate points per warp stage
  float nn_r0;             // staged: radius of the first look in cells (NNS_R0; LB_NN_R0 overrides it for A/B runs)
  NnsFarItem* far_items;   // staged: queue of the undecided queries of one correspondence step (n_src entries) ...
  int* far_count;          // ... and its two counters (steps alternate between them)
  long long* prof;         // tuning aid (LB_NNPROF): 8 words per group of 32 source points, or null
};

// second half of one correspondence: j = sorted position of the nearest target point (or -1): the matched point and
// M = (R C1 R' + C2)^-1 are written for source point s.  returns 1 when matched.
__device__ __forceinline__ int correspond_finish(const CorrArgs& a, const double* R, int s, int j) {
  double M[6] = {0., 0., 0., 0., 0., 0.};
  f4 c = f4{0.f, 0.f, 0.f, bits_to_float(-1)};
  if (j >= 0) {
    f4 t = a.tgt.pts[j];
    c = f4{t.x, t.y, t.z, bits_to_float(j)};
    double C1[6], C2[6];
    const double* c1 = a.src_cov + 6 * (size_t)s;
    const double* c2 = a.tgt_cov + 6 * (size_t)j;
#pragma unroll
    for (int e = 0; e < 6; e++) { C1[e] = c1[e]; C2[e] = c2[e]; }
    mahalanobis(R, C1, C2, M);
  }
  a.corr[s] = c;
  double* m = a.M + 6 * (size_t)s;
#pragma unroll
  for (int e = 0; e < 6; e++) m[e] = M[e];
  return j >= 0 ? 1 : 0;
}

__device__ __forceinline__ int correspond_point(const CorrArgs& a, const float* T, const double* R, int s, long long* prof = nullptr) {
  const long long t0 = prof ? clock64() : 0;
  f4 p = a.src[s];
  float qx, qy, qz;
  xform(T, p.x, p.y, p.z, qx, qy, qz);
  int bo; float bd;
  int j = nn1_pruned(a.tgt, qx, qy, qz, a.max_d2, bo, bd);
  const long long t1 = prof ? clock64() : 0;
  const int r = correspond_finish(a, R, s, j);
  if (prof) { prof[0] += t1 - t0; prof[1] += clock64() - t1; prof[2] += 1; }
  return r;
}

// The correspondence step over the source points [begin, end) by all threads of a CTA; returns this thread's number of
// matched points.  Serial form: every thread searches on its own (nn1_pruned).  (A two-phase variant -- 3x3x3 block per
// thread, then a whole warp per undecided query -- was measured slower.)
__device__ __forceinline__ int correspond_slice(const CorrArgs& a, const float* T, const double* R, int begin, int end,
                                                long long* prof = nullptr) {
  int hits = 0;
  for (int s = begin + (int)threadIdx.x; s < end; s += (int)blockDim.x) hits += correspond_point(a, T, R, s, prof);
  return hits;
}

// Staged form (nn_staged.cuh): the same points go to the same threads, but the 32 searches of a warp run together and
// fetch their candidates through the warp's shared-memory stage.  have_prev: a.corr still holds the matches of the
// previous outer iteration of THIS align() (same target), which bound the new search.  All threads of the CTA call it.
struct NnsCta { unsigned char* base; int cap; };     // dynamic shared memory: per warp cap points + one mbarrier
__device__ __forceinline__ size_t nns_warp_bytes(int cap) { return (size_t)cap * sizeof(f4) + 16; }
__device__ __forceinline__ NnsWarp nns_warp_view(const NnsCta& c) {
  NnsWarp w;
  w.stage = reinterpret_cast<f4*>(c.base + (size_t)(threadIdx.x >> 5) * nns_warp_bytes(c.cap));
  w.cap = c.cap;
  w.mbar = reinterpret_cast<unsigned long long*>(w.stage + c.cap);
  w.phase = 0;
  return w;
}
// once per kernel, by every warp, before the first staged search
__device__ __forceinline__ void nns_warp_init(NnsWarp& w) {
  if ((threadIdx.x & 31) == 0) nns_mbar_init(w.mbar);
  __syncwarp();
}
template <bool TMA>
__device__ __forceinline__ int correspond_slice_staged(const CorrArgs& a, const float* T, const double* R, int begin, int end,
                                                       bool have_prev, NnsWarp& w, int step_parity) {
  int hits = 0;
  const int lane = threadIdx.x & 31;
  const NnsFarQueue fq{a.far_items, a.far_count + step_parity};
  for (int base = begin + (int)(threadIdx.x - lane); base < end; base += (int)blockDim.x) {
    const int s = base + lane;
    const bool active = s < end;
    float qx = 0.f, qy = 0.f, qz = 0.f, ub2 = 0.f;
    bool have_ub = false;
    if (active) {
      const f4 p = a.src[s];
      xform(T, p.x, p.y, p.z, qx, qy, qz);
      if (have_prev) {
        const float4 c = __ldcg(reinterpret_cast<const float4*>(a.corr + s));  // possibly written by another SM (far queue)
        if (float_to_bits(c.w) >= 0) { have_ub = true; ub2 = dist2(qx, qy, qz, c.x, c.y, c.z); }
      }
    }
    int bo; float bd;
    long long* wp = a.prof ? a.prof + 8 * (size_t)(base >> 5) : nullptr;     // tuning aid: per-warp cycle counters
    const int j = nn1_staged<TMA>(a.tgt, active, qx, qy, qz, a.max_d2, have_ub, ub2, w, bo, bd, a.far_items ? &fq : nullptr, s, wp, a.nn_r0);
    const long long tf0 = wp ? clock64() : 0;
    if (active && j != NNS_DEFERRED) hits += correspond_finish(a, R, s, j);
    if (wp && lane == 0) wp[3] = clock64() - tf0;
  }
  return hits;
}

// The queued (far) queries of one correspondence step, one per warp: warp `gwarp` of `nwarps` takes items gwarp,
// gwarp + nwarps, ... and searches each one's remaining ball with all its lanes (nn1_far_item).  Returns this thread's
// number of matched points (lane 0 counts).  (A lane-per-item variant -- the compacted items through the staged pass
// again, rows in batches of 9 -- was measured slower.)
__device__ __forceinline__ int correspond_far(const CorrArgs& a, const float* T, const double* R, int nfar, int gwarp, int nwarps,
                                              uint32_t* scratch) {
  int hits = 0;
  const int lane = threadIdx.x & 31;
  for (int i = gwarp; i < nfar; i += nwarps) {
    const NnsFarItem it = a.far_items[i];
    const f4 p = a.src[it.s];
    float qx, qy, qz;
    xform(T, p.x, p.y, p.z, qx, qy, qz);
    const int j = nn1_far_item(a.tgt, it, qx, qy, qz, a.max_d2, scratch);
    if (lane == 0) hits += correspond_finish(a, R, it.s, j);
    __syncwarp();
  }
  return hits;
}

// nn_mode: 0 = serial, 1 = staged with cp.async, 2 = staged with TMA bulk copies
__device__ __forceinline__ int correspond_slice_mode(const CorrArgs& a, const float* T, const double* R, int begin, int end,
                                                     bool have_prev, NnsWarp& w, int step_parity, long long* prof = nullptr) {
  if (a.nn_mode == 1) return correspond_slice_staged<false>(a, T, R, begin, end, have_prev, w, step_parity);
  if (a.nn_mode == 2) return correspond_slice_staged<true>(a, T, R, begin, end, have_prev, w, step_parity);
  return correspond_slice(a, T, R, begin, end, prof);
}

extern __shared__ __align__(16) unsigned char nns_dyn_smem[];

__global__ void __launch_bounds__(128)
nn_corr_kernel(CorrArgs a, Mat34 T, Mat33d R, int have_prev, int* __restrict__ m_count) {
  const int begin = min(a.n_src, (int)(blockIdx.x * blockDim.x)), end = min(a.n_src, begin + (int)blockDim.x);
  NnsCta nc{nns_dyn_smem, a.nn_cap};
  NnsWarp w = nns_warp_view(nc);
  if (a.nn_mode) nns_warp_init(w);
  int hits = correspond_slice_mode(a, T.m, R.m, begin, end, have_prev != 0, w, 0);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
  if ((threadIdx.x & 31) == 0 && hits) atomicAdd(m_count, hits);
}

// How uneven the cloud is over its voxel hash: points that sit in cells holding more than `thresh` points.  The staged
// search scans a lane's candidates sequentially, which is the right shape for voxel-filtered clouds (a handful of
// points per cell) and the wrong one for raw, locally very dense maps, where the warp-per-query kernel shares a
// query's candidates among 32 lanes.
__global__ void cell_density_kernel(const uint32_t* __restrict__ cell_start, size_t ncells, uint32_t thresh, unsigned long long* __restrict__ out) {
  unsigned long long dense = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < ncells; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t c = cell_start[i + 1] - cell_start[i];
    if (c > thresh) dense += c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dense += __shfl_xor_sync(0xffffffffu, dense, o);
  if ((threadIdx.x & 31) == 0 && dense) atomicAdd(out, dense);
}

// Exact 1-NN of arbitrary query points (lb_gicp_nn_target), two kernels: 32 queries per warp through the staged search
// -- first look = half a cell around the query -- with the undecided queries queued; then one warp per queued query:
// the ball of its best candidate so far (nn1_ball_warp), or, when the first look found nothing, the ring-by-ring search
// of the warp-per-query kernel (nn1_warp).
template <bool TMA>
__global__ void __launch_bounds__(128)
nn_query_staged_kernel(GridView g, const uint8_t* __restrict__ q, uint32_t n, uint32_t stride, int32_t* __restrict__ idx,
                       float* __restrict__ d2, float max_d2, int cap, NnsFarItem* __restrict__ far_items, int* __restrict__ far_count,
                       long long* __restrict__ count) {
  NnsCta nc{nns_dyn_smem, cap};
  NnsWarp w = nns_warp_view(nc);
  nns_warp_init(w);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = i < n;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (active) {
    const float* p = reinterpret_cast<const float*>(q + (size_t)i * stride);
    qx = p[0]; qy = p[1]; qz = p[2];
  }
  int bo; float bd;
  long long wp[8];                                // profiling launch only: wp[5] = candidates the warp staged
  const NnsFarQueue fq{far_items, far_count};
  const int j = nn1_staged<TMA>(g, active, qx, qy, qz, max_d2, false, 0.f, w, bo, bd, &fq, (int)i, count ? wp : nullptr);
  if (active && j != NNS_DEFERRED) { idx[i] = j >= 0 ? bo : -1; d2[i] = j >= 0 ? bd : max_d2; }
  if (count && (threadIdx.x & 31) == 0) atomicAdd(reinterpret_cast<unsigned long long*>(count), (unsigned long long)wp[5]);
}

__global__ void __launch_bounds__(256)
nn_query_far_kernel(GridView g, const uint8_t* __restrict__ q, uint32_t stride, int32_t* __restrict__ idx, float* __restrict__ d2,
                    float max_d2, const NnsFarItem* __restrict__ far_items, const int* __restrict__ far_count) {
  __shared__ NnWarpSmem sm[8];
  const int nfar = *far_count;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const unsigned long long gate_key = (unsigned long long)__float_as_uint(max_d2) << 32;
  for (int k = blockIdx.x * 8 + wib; k < nfar; k += gridDim.x * 8) {
    const NnsFarItem it = far_items[k];
    const float* p = reinterpret_cast<const float*>(q + (size_t)it.s * stride);
    const float qx = p[0], qy = p[1], qz = p[2];
    int oi = -1; float od = max_d2;
    bool done = false;
    if (it.best < gate_key) {                     // a candidate is known: everything that matters lies within its distance
      int rbs, rbi; float rbd;
      done = nn1_ball_warp(g, qx, qy, qz, max_d2, it.ball2, true, __uint_as_float((unsigned)(it.best >> 32)),
                           (int)(unsigned)(it.best & 0xffffffffull), it.bs, reinterpret_cast<uint32_t*>(&sm[wib]), rbs, rbi, rbd);
      oi = rbi; od = rbd;
    }
    if (!done) {
      const unsigned long long best = nn1_warp(g, qx, qy, qz, max_d2, sm[wib]);
      const bool ok = best != 0xffffffffffffffffull;
      oi = ok ? (int)(unsigned)(best & 0xffffffffull) : -1;
      od = ok ? __uint_as_float((unsigned)(best >> 32)) : max_d2;
    }
    if (lane == 0) { idx[it.s] = oi; d2[it.s] = od; }
    __syncwarp();
  }
}

// second kernel of a staged correspondence step outside the persistent kernels: the queued queries
constexpr int NN_FAR_THREADS = 128;
__global__ void __launch_bounds__(NN_FAR_THREADS)
nn_far_kernel(CorrArgs a, Mat34 T, Mat33d R, int* __restrict__ m_count) {
  __shared__ uint32_t scratch[NN_FAR_THREADS / 32][66];
  const int nfar = a.far_count[0];
  const int wib = threadIdx.x >> 5;
  int hits = correspond_far(a, T.m, R.m, nfar, blockIdx.x * (NN_FAR_THREADS / 32) + wib, gridDim.x * (NN_FAR_THREADS / 32), scratch[wib]);
  if ((threadIdx.x & 31) == 0 && hits) atomicAdd(m_count, hits);
}

// ------------------------------------------------------------------ K5 objective
struct ObjArgs {
  const f4* src;
  const f4* corr;
  const double* M;
  int n_src;
};

// accumulate the NV sums of this thread's points.  NV = 13: BFGS objective; 28: Gauss-Newton.
// CTA c owns the contiguous chunk [c*chunk, (c+1)*chunk) of the (cell-sorted) source.  The objective terms are
// accumulated by the 128 lanes of warps 1..4 (warp 0 is the leader of the persistent kernel): lane t takes points
// begin + t + 128*j, j = 0, 1, ...  in that order.
constexpr int AL_ACC_W0 = 1;                 // first accumulating warp
constexpr int AL_PPL = AL_PPC / AL_ACC;      // points per accumulating lane held in registers (4)

__device__ __forceinline__ void cta_chunk(int n, int& begin, int& end) {
  int chunk = (n + (int)gridDim.x - 1) / (int)gridDim.x;
  begin = min(n, (int)blockIdx.x * chunk);
  end = min(n, begin + chunk);
}
__device__ __forceinline__ int acc_lane() { return (int)threadIdx.x - 32 * AL_ACC_W0; }   // 0..127 for accumulating lanes

// A lane's correspondences, register-resident across all objective evaluations of one outer iteration
// (the correspondences are fixed during the inner solve, gicp.hpp:518-524): zero memory traffic per evaluation.
template <int PPL>
struct PointCacheT {
  static constexpr int kPPL = PPL;
  float px[PPL], py[PPL], pz[PPL], qx[PPL], qy[PPL], qz[PPL];
  double M[PPL][6];
};
using PointCache = PointCacheT<AL_PPL>;

// The same correspondences in dynamic shared memory, for loop_solve_kernel: registers held for the whole solve would
// not leave room for two CTAs per SM.  Lane-fastest ([field][point][lane]): a warp's accesses are conflict-free.
// The accessors address the dynamic shared array directly (no pointer members): the compiler then emits shared-window
// loads with immediate offsets instead of keeping 64-bit generic addresses live.
extern __shared__ __align__(16) unsigned char al_cache_smem[];
template <int PPL>
struct SmemCacheT {
  static constexpr int kPPL = PPL;
  static constexpr size_t kBytes = (size_t)6 * PPL * AL_ACC * (sizeof(double) + sizeof(float));
  // M: [6][PPL][AL_ACC] doubles, then [6][PPL][AL_ACC] floats px, py, pz, qx, qy, qz
  __device__ __forceinline__ double& m(int e, int j, int t) const {
    return reinterpret_cast<double*>(al_cache_smem)[(e * PPL + j) * AL_ACC + t];
  }
  __device__ __forceinline__ float& f(int c, int j, int t) const {
    return reinterpret_cast<float*>(al_cache_smem + (size_t)6 * PPL * AL_ACC * sizeof(double))[(c * PPL + j) * AL_ACC + t];
  }
};

// point j of accumulating lane t of the chunk [begin, end): source point p, matched point c, M.  Points past the end
// and unmatched points come back as zeros, whose M = 0 adds exact zeros.
__device__ __forceinline__ void cache_fetch(const ObjArgs& a, int begin, int end, int t, int j, f4& p, f4& c, double* M) {
  int s = begin + t + AL_ACC * j;
  bool ok = (t >= 0 && t < AL_ACC && s < end);
  // corr / M may have been written by a warp of another SM (far queue of the staged search): read them from L2
  c = f4{0.f, 0.f, 0.f, bits_to_float(-1)};
  if (ok) { const float4 cc = __ldcg(reinterpret_cast<const float4*>(a.corr + s)); c = f4{cc.x, cc.y, cc.z, cc.w}; }
  ok = ok && float_to_bits(c.w) >= 0;
  p = ok ? a.src[s] : f4{0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int e = 0; e < 6; e++) M[e] = ok ? __ldcg(a.M + 6 * (size_t)s + e) : 0.0;
}

template <int PPL>
__device__ __forceinline__ void cache_load(const ObjArgs& a, int begin, int end, PointCacheT<PPL>& pc) {
  const int t = acc_lane();
#pragma unroll
  for (int j = 0; j < PPL; j++) {
    f4 p, c;
    cache_fetch(a, begin, end, t, j, p, c, pc.M[j]);
    pc.px[j] = p.x; pc.py[j] = p.y; pc.pz[j] = p.z;
    pc.qx[j] = c.x; pc.qy[j] = c.y; pc.qz[j] = c.z;
  }
}

template <int PPL>
__device__ __forceinline__ void cache_load(const ObjArgs& a, int begin, int end, SmemCacheT<PPL>& pc) {
  const int t = acc_lane();
#pragma unroll
  for (int j = 0; j < PPL; j++) {
    f4 p, c;
    double M[6];
    cache_fetch(a, begin, end, t, j, p, c, M);
    pc.f(0, j, t) = p.x; pc.f(1, j, t) = p.y; pc.f(2, j, t) = p.z;
    pc.f(3, j, t) = c.x; pc.f(4, j, t) = c.y; pc.f(5, j, t) = c.z;
#pragma unroll
    for (int e = 0; e < 6; e++) pc.m(e, j, t) = M[e];
  }
}

template <int NV, int PPL>
__device__ __forceinline__ void objective_from_cache(const PointCacheT<PPL>& pc, const float* T, const double* dP, const double* dT,
                                                     const double* dS, double* acc) {
#pragma unroll
  for (int j = 0; j < PPL; j++) {
    if constexpr (NV == 13) objective_terms(T, pc.px[j], pc.py[j], pc.pz[j], pc.qx[j], pc.qy[j], pc.qz[j], pc.M[j], acc);
    else gn_terms(T, dP, dT, dS, pc.px[j], pc.py[j], pc.pz[j], pc.qx[j], pc.qy[j], pc.qz[j], pc.M[j], acc);
  }
}

template <int NV, int PPL>
__device__ __forceinline__ void objective_from_cache(const SmemCacheT<PPL>& pc, const float* T, const double* dP, const double* dT,
                                                     const double* dS, double* acc) {
  const int t = acc_lane();
#pragma unroll 1
  for (int j = 0; j < PPL; j++) {
    double M[6];
#pragma unroll
    for (int e = 0; e < 6; e++) M[e] = pc.m(e, j, t);
    const float px = pc.f(0, j, t), py = pc.f(1, j, t), pz = pc.f(2, j, t);
    const float qx = pc.f(3, j, t), qy = pc.f(4, j, t), qz = pc.f(5, j, t);
    if constexpr (NV == 13) objective_terms(T, px, py, pz, qx, qy, qz, M, acc);
    else gn_terms(T, dP, dT, dS, px, py, pz, qx, qy, qz, M, acc);
  }
}

// same lane -> points mapping and order, straight from global memory (chunks larger than AL_PPC, and the
// host-driven kernel).  Unmatched points carry M = 0 and add exact zeros, like the padded cache entries.
template <int NV>
__device__ __forceinline__ void objective_from_global(const ObjArgs& a, const float* T, const double* dP, const double* dT,
                                                      const double* dS, int begin, int end, double* acc) {
  const int t = acc_lane();
  if (t < 0 || t >= AL_ACC) return;
  for (int s = begin + t; s < end; s += AL_ACC) {
    const float4 cc = __ldcg(reinterpret_cast<const float4*>(a.corr + s));     // L2: possibly written by another SM
    f4 c = f4{cc.x, cc.y, cc.z, cc.w};
    f4 p = a.src[s];
    double M[6];
    const double* m = a.M + 6 * (size_t)s;
#pragma unroll
    for (int e = 0; e < 6; e++) M[e] = __ldcg(m + e);
    if (float_to_bits(c.w) < 0) { c = f4{0.f, 0.f, 0.f, 0.f}; p = c; }
    if constexpr (NV == 13) objective_terms(T, p.x, p.y, p.z, c.x, c.y, c.z, M, acc);
    else gn_terms(T, dP, dT, dS, p.x, p.y, p.z, c.x, c.y, c.z, M, acc);
  }
}

struct Vec6d { double v[6]; };

// Host-driven objective: every CTA reduces its chunk into its slot; the last CTA to finish sums the slots
// in fixed order and writes the NV totals to `out` (mapped pinned memory).  Same chunking, block_reduce and
// slot summation order as the persistent kernel, so both execution modes produce identical bits.
template <int NV>
__global__ void __launch_bounds__(AL_THREADS)
objective_kernel(ObjArgs a, Vec6d x, SlotWord* __restrict__ slots, unsigned* __restrict__ ticket, double* __restrict__ out) {
  __shared__ double red[AL_ACC_WARPS * NV];
  __shared__ double mat[NV * AL_MAXCTA];
  __shared__ double tot_s[NV];
  __shared__ float sT[12];
  __shared__ double sD[27];
  __shared__ bool last;
  if (threadIdx.x == 0) {
    apply_state(x.v, sT);
    if (NV != 13) r_derivatives(x.v, sD, sD + 9, sD + 18);
  }
  __syncthreads();
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = sT[i];
  double acc[NV];
#pragma unroll
  for (int e = 0; e < NV; e++) acc[e] = 0.0;
  int begin, end;
  cta_chunk(a.n_src, begin, end);
  objective_from_global<NV>(a, T, sD, sD + 9, sD + 18, begin, end, acc);
  double tot = block_reduce<NV, AL_ACC_WARPS, AL_ACC_W0>(acc, red);
  if (threadIdx.x < NV) slot_store(&slots[(size_t)blockIdx.x * AL_PSTRIDE + threadIdx.x], tot, 1ull);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = atomicAdd(ticket, 1u);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    slots_all_sum<NV, AL_THREADS>(slots, gridDim.x, 1ull, mat, tot_s);
    if (threadIdx.x < NV) out[threadIdx.x] = tot_s[threadIdx.x];
    // reset the tags and the ticket for the next launch
    for (int i = threadIdx.x; i < (int)gridDim.x * NV; i += AL_THREADS)
      slot_store(&slots[(size_t)(i / NV) * AL_PSTRIDE + (i % NV)], 0.0, 0ull);
    if (threadIdx.x == 0) *ticket = 0;
  }
}

// ------------------------------------------------------------------ persistent align
// One cooperative launch per align(): the whole computeTransformation loop (gicp.hpp:445-583) stays on
// the device.  Per CTA, warp 0 is the LEADER: its 32 lanes run the scalar outer-loop / BFGS code of
// bfgs.h convergently (state in registers / a few hundred bytes of L1-resident local memory); the other
// warps are WORKERS parked on the CTA barrier until the leader posts a command (correspond / objective /
// Gauss-Newton terms / exit) in shared memory.  Every data-parallel command ends in a grid-wide
// deterministic all-reduce: each CTA publishes its partials as (value, epoch) words in its slot with
// single 16-byte L2 stores; every CTA polls the words of all slots and sums them in a fixed order -- no
// atomics, no fences (so L1 is never invalidated), and every CTA obtains bitwise identical totals, so all
// leaders take identical decisions.  Slots are double-buffered; epochs are unique across launches.
struct AlignArgs {
  CorrArgs c;
  SlotWord* slots;        // [2][gridDim.x][AL_PSTRIDE] (value, epoch) words
  unsigned long long epoch_base;   // unique per launch, so stale epochs of earlier launches never match
  int poll_delay;                  // cycles to hold back the first poll of a collective
  long long* debug;       // nullable: [8] cycle counters written by CTA 0 (profiling aid)
  OuterParams P;
  float guess[16];
  OuterResult* result;
};

enum { OP_NONE = 0, OP_CORR = 1, OP_FDF = 2, OP_GN = 3, OP_EXIT = 4, OP_LOAD = 5 };

struct AlignShared {
  int op;
  int m;
  int corr_calls;                                          // correspondence steps done by this launch
  unsigned nn_phase[AL_THREADS / 32];                      // staged search: mbarrier parity of every warp
  long long t_reduce, t_wait, n_coll, t_scalar, t_mark, t_corr;   // CTA 0 / thread 0 cycle counters
  long long poll[2];                                       // poll rounds of thread 0, sum of clock at poll completion
  float T[12];
  double R[9];
  double D[27];
  double red[AL_ACC_WARPS * AL_MAXV];
  double bc[AL_MAXV + 4];
  double mat[AL_MAXV * AL_MAXCTA];
};

struct Collective {   // per-thread copy; advances in lockstep in every thread of the grid
  unsigned long long epoch;
  int flip;
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// grid-wide deterministic sum of the NV doubles held by the accumulating lanes; totals land in
// sh.bc[0..NV-1] (visible to all threads after return).  THREADS: the CTA size of the calling kernel.
template <int NV, int THREADS>
__device__ __forceinline__ void grid_all_reduce(const AlignArgs& a, AlignShared& sh, Collective& co, double* acc) {
  constexpr int all_pairs = (AL_MAXCTA * NV + THREADS - 1) / THREADS;
  constexpr int chunk = THREADS == AL_THREADS ? all_pairs : (all_pairs < AL_SOLVE_POLL ? all_pairs : AL_SOLVE_POLL);
  const bool prof = (blockIdx.x == 0 && threadIdx.x == 0);
  long long t0 = prof ? clock64() : 0;
  double tot = block_reduce<NV, AL_ACC_WARPS, AL_ACC_W0>(acc, sh.red);
  co.epoch++;
  const int ncta = gridDim.x;
  SlotWord* buf = a.slots + (size_t)co.flip * ncta * AL_PSTRIDE;
  if (threadIdx.x < NV) slot_store(&buf[(size_t)blockIdx.x * AL_PSTRIDE + threadIdx.x], tot, co.epoch);
  long long t1 = prof ? clock64() : 0;
  const bool snap = a.debug && threadIdx.x == 0 && (co.epoch - a.epoch_base) == 100;   // one collective, all CTAs
  if (snap) a.debug[16 + blockIdx.x] = (long long)globaltimer_ns();
  slots_all_sum<NV, THREADS, chunk>(buf, ncta, co.epoch, sh.mat, sh.bc, prof ? sh.poll : nullptr, (long long)a.poll_delay);
  if (prof) sh.poll[1] -= t1;   // accumulates (poll completion - publish) for thread 0
  if (snap) a.debug[16 + AL_MAXCTA + blockIdx.x] = (long long)globaltimer_ns();
  co.flip ^= 1;
  if (prof) { long long t2 = clock64(); sh.t_reduce += t1 - t0; sh.t_wait += t2 - t1; sh.n_coll++; sh.t_mark = t2; }
}

// (the persistent kernel only: its 256-thread CTA runs the search)
template <int PPL>
__device__ __forceinline__ void do_correspond(const AlignArgs& a, AlignShared& sh, Collective& co, PointCacheT<PPL>& pc) {
  float T[12]; double R[9];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = sh.T[i];
#pragma unroll
  for (int i = 0; i < 9; i++) R[i] = sh.R[i];
  int begin, end;
  cta_chunk(a.c.n_src, begin, end);
  const bool cprof = a.debug && blockIdx.x == 0 && threadIdx.x == 0;
  const long long p0 = cprof ? clock64() : 0;
  NnsCta nc{nns_dyn_smem, a.c.nn_cap};
  NnsWarp w = nns_warp_view(nc);
  w.phase = sh.nn_phase[threadIdx.x >> 5];
  const int calls = sh.corr_calls;                 // correspondence steps of this launch before this one
  const bool have_prev = calls > 0;                // a.c.corr holds the matches of the previous outer iteration
  int hits = correspond_slice_mode(a.c, T, R, begin, end, have_prev, w, calls & 1, cprof ? a.debug + 11 : nullptr);
  if ((threadIdx.x & 31) == 0) sh.nn_phase[threadIdx.x >> 5] = w.phase;
  if (a.c.nn_mode && a.c.far_items) {
    // the undecided queries of ALL CTAs were queued: once everybody has queued (grid-wide exchange), every warp of the
    // grid takes its share of them
    __threadfence();
    double zero[1] = {0.0};
    grid_all_reduce<1, AL_THREADS>(a, sh, co, zero);
    const int nfar = *(volatile int*)(a.c.far_count + (calls & 1));
    if (blockIdx.x == 0 && threadIdx.x == 0) a.c.far_count[(calls & 1) ^ 1] = 0;      // the next step's counter
    hits += correspond_far(a.c, T, R, nfar, (int)blockIdx.x * (AL_THREADS / 32) + (int)(threadIdx.x >> 5),
                           (int)gridDim.x * (AL_THREADS / 32), reinterpret_cast<uint32_t*>(w.stage));
    __threadfence();
  }
  const long long q0 = cprof ? clock64() : 0;
  if (cprof) a.debug[10] += q0 - p0;
  // The correspondence arrays may have been written by other CTAs (far queue): they are re-read (L2) after the exchange below.
  __shared__ int s_hits[AL_THREADS];
  s_hits[threadIdx.x] = hits;
  __syncthreads();
  if (threadIdx.x == 0) sh.corr_calls++;
  double cnt[1] = {0.0};
  const int t = acc_lane();
  if (t >= 0 && t < AL_ACC) {
    int h = 0;
    for (int k = t; k < AL_THREADS; k += AL_ACC) h += s_hits[k];
    cnt[0] = (double)h;
  }
  const long long q1 = cprof ? clock64() : 0;
  grid_all_reduce<1, AL_THREADS>(a, sh, co, cnt);
  if (end - begin <= PPL * AL_ACC && t >= 0 && t < AL_ACC) {
    ObjArgs oa{a.c.src, a.c.corr, a.c.M, a.c.n_src};
    cache_load<PPL>(oa, begin, end, pc);
  }
  if (cprof) { a.debug[14] += q1 - q0; a.debug[15] += clock64() - q1; }
}

// Cache: PointCacheT (registers) or SmemCacheT (shared memory); THREADS: the CTA size of the calling kernel
template <int NV, int THREADS, class Cache>
__device__ __forceinline__ void do_objective(const AlignArgs& a, AlignShared& sh, Collective& co, const Cache& pc) {
  constexpr int PPL = Cache::kPPL;
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = sh.T[i];
  double acc[NV];
#pragma unroll
  for (int e = 0; e < NV; e++) acc[e] = 0.0;
  int begin, end;
  cta_chunk(a.c.n_src, begin, end);
  const int t = acc_lane();
  if (end - begin <= PPL * AL_ACC) {
    if (t >= 0 && t < AL_ACC) objective_from_cache<NV, PPL>(pc, T, sh.D, sh.D + 9, sh.D + 18, acc);
  } else {
    ObjArgs oa{a.c.src, a.c.corr, a.c.M, a.c.n_src};
    objective_from_global<NV>(oa, T, sh.D, sh.D + 9, sh.D + 18, begin, end, acc);
  }
  grid_all_reduce<NV, THREADS>(a, sh, co, acc);
}

// Backend of bfgs.h for the leader warp (all 32 lanes call every method together).
template <class Cache, int THREADS>
struct DeviceBackendT {
  static constexpr int PPL = Cache::kPPL;
  const AlignArgs& a;
  AlignShared& sh;
  Collective& co;
  Cache& pc;     // warp 0 never accumulates: its cache is never read
  int m;

  __device__ DeviceBackendT(const AlignArgs& a_, AlignShared& sh_, Collective& co_, Cache& pc_)
      : a(a_), sh(sh_), co(co_), pc(pc_), m(0) {}

  // the 12 trigonometric values of a state, one per lane, broadcast to the warp
  __device__ __forceinline__ void warp_trig(const double* x, Trig& t) {
    const int lane = threadIdx.x & 31;
    const int k = lane % 3;
    double sv = 0.0, cv = 0.0;
    if (lane < 6) {                      // lanes 0-2: half angles (float-rounded argument), lanes 3-5: full angles
      double ang = (lane < 3) ? (double)half_angle(x, k) : x[3 + k];
      sv = sin(ang);
      cv = cos(ang);
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
      t.ch[i] = (float)__shfl_sync(0xffffffffu, cv, i);
      t.sh[i] = (float)__shfl_sync(0xffffffffu, sv, i);
      t.c[i] = __shfl_sync(0xffffffffu, cv, 3 + i);
      t.s[i] = __shfl_sync(0xffffffffu, sv, 3 + i);
    }
  }

  __device__ int correspond(const float* T, const double* R) {
    const int lane = threadIdx.x & 31;
    if (lane < 12) sh.T[lane] = T[lane];
    if (lane < 9) sh.R[lane] = R[lane];
    if (lane == 0) sh.op = OP_CORR;
    const long long tc0 = clock64();
    __syncthreads();
    do_correspond<PPL>(a, sh, co, pc);
    m = (int)sh.bc[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) { const long long tc1 = clock64(); sh.t_corr += tc1 - tc0; sh.t_mark = tc1; }
    return m;
  }

  __device__ void fdf(const double* x, double* f, double* g) {
    const int lane = threadIdx.x & 31;
    Trig t;
    warp_trig(x, t);
    float T[12];
    apply_state_trig(x, t, T);
    if (lane < 12) sh.T[lane] = T[lane];
    if (lane == 0) sh.op = OP_FDF;
    if (blockIdx.x == 0 && threadIdx.x == 0) sh.t_scalar += clock64() - sh.t_mark;   // leader time since the last collective
    __syncthreads();
    do_objective<13, THREADS>(a, sh, co, pc);
    double sums[13];
#pragma unroll
    for (int e = 0; e < 13; e++) sums[e] = sh.bc[e];
    objective_finish_trig(sums, m, t, f, g);
  }

  __device__ int gn(const double* x, double* f, double* b, double* H) {
    const int lane = threadIdx.x & 31;
    Trig t;
    warp_trig(x, t);
    float T[12];
    double D[27];
    apply_state_trig(x, t, T);
    r_derivatives_trig(t, D, D + 9, D + 18);
    if (lane < 12) sh.T[lane] = T[lane];
    if (lane < 27) sh.D[lane] = D[lane];
    if (lane == 0) sh.op = OP_GN;
    __syncthreads();
    do_objective<28, THREADS>(a, sh, co, pc);
    *f = sh.bc[0] / (double)m;
#pragma unroll
    for (int e = 0; e < 6; e++) b[e] = sh.bc[1 + e];
#pragma unroll
    for (int e = 0; e < 21; e++) H[e] = sh.bc[7 + e];
    return 0;
  }
};

#ifndef AL_MINB
#define AL_MINB 1
#endif
// PPL = source points per accumulating lane kept in registers: 4 (512 points per CTA: lowest latency) or 8 (1024
// points per CTA: half the SMs per align, what the odometry pipeline's workers use)
template <int PPL>
__global__ void __launch_bounds__(AL_THREADS, AL_MINB)
align_persistent_kernel(const __grid_constant__ AlignArgs a) {
  __shared__ AlignShared sh;
  Collective co;
  co.epoch = a.epoch_base; co.flip = 0;
  const long long t_begin = clock64();
  if (a.debug && blockIdx.x == 0 && threadIdx.x == 0) { for (int i = 10; i < 16; i++) a.debug[i] = 0; }
  if (threadIdx.x == 0) { sh.t_reduce = 0; sh.t_wait = 0; sh.n_coll = 0; sh.t_scalar = 0; sh.t_corr = 0; sh.t_mark = clock64(); sh.poll[0] = 0; sh.poll[1] = 0; sh.corr_calls = 0; }
  if ((threadIdx.x & 31) == 0) sh.nn_phase[threadIdx.x >> 5] = 0;
  if (a.c.nn_mode) { NnsCta nc{nns_dyn_smem, a.c.nn_cap}; NnsWarp w0 = nns_warp_view(nc); nns_warp_init(w0); }
  if (threadIdx.x < 32) {
    PointCacheT<PPL> pc_unused;   // warp 0 does not accumulate; kept apart from the workers' register-resident cache
    DeviceBackendT<PointCacheT<PPL>, AL_THREADS> be(a, sh, co, pc_unused);
    OuterResult r;
    gicp_outer_loop(be, a.P, a.guess, r);
    if (threadIdx.x == 0) sh.op = OP_EXIT;
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      *a.result = r;
      if (a.debug) {
        a.debug[0] = clock64() - t_begin; a.debug[1] = sh.t_reduce; a.debug[2] = sh.t_wait; a.debug[3] = sh.n_coll;
        a.debug[6] = sh.t_scalar; a.debug[7] = sh.poll[0]; a.debug[8] = sh.poll[1]; a.debug[9] = sh.t_corr;
      }
    }
  } else {
    PointCacheT<PPL> pc;
    for (;;) {
      __syncthreads();
      const int op = sh.op;
      if (op == OP_EXIT) break;
      if (op == OP_CORR) do_correspond<PPL>(a, sh, co, pc);
      else if (op == OP_FDF) do_objective<13, AL_THREADS>(a, sh, co, pc);
      else do_objective<28, AL_THREADS>(a, sh, co, pc);
    }
  }
}

// ------------------------------------------------------------------ stream-ordered align (LB_EXEC_STREAM_ORDERED)
// The correspondence step wants the whole GPU at full occupancy (thousands of independent exact searches, the far ones
// ~600 candidates each); the inner solve wants a small co-resident grid with everything in registers.  Inside ONE
// persistent kernel the search runs on the solve's 8 warps per SM, far below full occupancy.  Here one
// outer iteration is two launches on the handle's stream -- loop_nn_kernel (plain grid, 128-thread CTAs, the search at
// full occupancy) and loop_solve_kernel (the cooperative grid: BFGS / GN solve, convergence test, next rotation) -- with
// the state of computeTransformation (gicp.hpp:445-583) kept in device memory between them.  The host enqueues a few
// iterations ahead; kernels of iterations after convergence return at once.  Same device functions, same reduction
// shape as the single persistent kernel: identical bits.
constexpr int LOOP_K = 4;            // outer iterations enqueued per batch
struct LoopState {
  OuterState s;
  double R[9];                       // rotation of the next correspondence step (gicp.hpp:450-460)
  int m[LOOP_K];                     // correspondences found by the search of iteration k of the batch
  OuterResult result;
};

__global__ void __launch_bounds__(128)
loop_nn_kernel(CorrArgs a, LoopState* __restrict__ st, int k) {
  if (st->s.done) return;
  float T[12]; double R[9];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = st->s.T[i];
#pragma unroll
  for (int i = 0; i < 9; i++) R[i] = st->R[i];
  const int begin = min(a.n_src, (int)(blockIdx.x * blockDim.x)), end = min(a.n_src, begin + (int)blockDim.x);
  NnsCta nc{nns_dyn_smem, a.nn_cap};
  NnsWarp w = nns_warp_view(nc);
  if (a.nn_mode) nns_warp_init(w);
  int hits = correspond_slice_mode(a, T, R, begin, end, st->s.nr > 0, w, k & 1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
  if ((threadIdx.x & 31) == 0 && hits) atomicAdd(&st->m[k], hits);
}

// the queued queries of iteration k's search (staged search only), one per warp of a fixed grid
__global__ void __launch_bounds__(NN_FAR_THREADS)
loop_far_kernel(CorrArgs a, LoopState* __restrict__ st, int k) {
  if (st->s.done) return;
  float T[12]; double R[9];
#pragma unroll
  for (int i = 0; i < 12; i++) T[i] = st->s.T[i];
#pragma unroll
  for (int i = 0; i < 9; i++) R[i] = st->R[i];
  const int nfar = a.far_count[k & 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) a.far_count[(k & 1) ^ 1] = 0;       // the next iteration's counter
  __shared__ uint32_t scratch[NN_FAR_THREADS / 32][66];
  const int wib = threadIdx.x >> 5;
  int hits = correspond_far(a, T, R, nfar, blockIdx.x * (NN_FAR_THREADS / 32) + wib, gridDim.x * (NN_FAR_THREADS / 32), scratch[wib]);
  if ((threadIdx.x & 31) == 0 && hits) atomicAdd(&st->m[k], hits);
}

// Two shapes, chosen by the host from the points per CTA:
//   THREADS = AL_THREADS (4 points per lane: the lowest latency of one align): the persistent kernel's CTA, one per SM,
//     255 registers, correspondences in registers (PointCacheT);
//   THREADS = AL_SOLVE_THREADS (8 points per lane: the odometry pipeline's workers): the leader warp and the
//     accumulating warps only, 168 registers, correspondences in dynamic shared memory (SmemCacheT<PPL>::kBytes per
//     CTA), two CTAs per SM -- twice the aligns in flight under the per-device budget.
// Same reduction shape and summation order in both: identical bits.
template <int PPL, int THREADS>
__global__ void __launch_bounds__(THREADS, THREADS == AL_SOLVE_THREADS ? 2 : AL_MINB)
loop_solve_kernel(const __grid_constant__ AlignArgs a, LoopState* __restrict__ st, int k) {
  using Cache = typename std::conditional<THREADS == AL_SOLVE_THREADS, SmemCacheT<PPL>, PointCacheT<PPL>>::type;
  __shared__ AlignShared sh;
  if (st->s.done) return;                      // converged in an earlier launch of this batch (uniform for the grid)
  Collective co;
  co.epoch = a.epoch_base; co.flip = 0;
  if (threadIdx.x == 0) { sh.t_reduce = 0; sh.t_wait = 0; sh.n_coll = 0; sh.t_scalar = 0; sh.t_corr = 0; sh.t_mark = clock64(); sh.poll[0] = 0; sh.poll[1] = 0; }
  if (threadIdx.x < 32) {
    Cache pc_unused;
    DeviceBackendT<Cache, THREADS> be(a, sh, co, pc_unused);
    OuterState s = st->s;
    const int m = st->m[k];
    be.m = m;
    if (threadIdx.x == 0) sh.op = OP_LOAD;      // workers: this CTA's correspondences -> the cache
    __syncthreads();
    outer_step(s, be, a.P, m);
    if (threadIdx.x == 0) sh.op = OP_EXIT;
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0) {   // every leader holds the same state: CTA 0 publishes it
      if (!s.done) {
        double R[9];
        outer_rotation(s, a.guess, R);
#pragma unroll
        for (int i = 0; i < 9; i++) st->R[i] = R[i];
      } else {
        OuterResult r;
        outer_finish(s, a.guess, r);
        st->result = r;
      }
      st->m[k] = 0;                              // ready for the next batch
      st->s = s;
    }
  } else {
    Cache pc;
    for (;;) {
      __syncthreads();
      const int op = sh.op;
      if (op == OP_EXIT) break;
      if (op == OP_LOAD) {
        int begin, end;
        cta_chunk(a.c.n_src, begin, end);
        const int t = acc_lane();
        if (end - begin <= PPL * AL_ACC && t >= 0 && t < AL_ACC) {
          ObjArgs oa{a.c.src, a.c.corr, a.c.M, a.c.n_src};
          cache_load<PPL>(oa, begin, end, pc);
        }
      }
      else if (op == OP_FDF) do_objective<13, THREADS>(a, sh, co, pc);
      else do_objective<28, THREADS>(a, sh, co, pc);
    }
  }
}

// ------------------------------------------------------------------ row f1: point-to-plane information matrix
// PointCloudLocalization.cc:694-750 (ComputeAp_ForPoint2PlaneICP) after src/utils.cc:106-128 (normalizePCloud).
// Three small reductions (double, fixed-shape block trees; per-CTA partials are summed on the host in CTA order).
// normalizePCloud's two reductions exactly as the reference computes them (utils.cc:106-118): pcl::compute3DCentroid
// into an Eigen::Vector4f and `float dist` are both float32 sums accumulated IN POINT ORDER, so a parallel tree would
// give different bits (~1e-4 relative on 30 k points).  One CTA: all 256 threads stage a tile of 256 points in shared
// memory (coalesced), three lanes of warp 0 add the tile's x / y / z (pass 1) or one lane adds the 256 norms (pass 2)
// sequentially while the other warps already load the next tile.
// out4 = {cx, cy, cz, dist}.
__global__ void __launch_bounds__(256)
ap_normalize_seq_kernel(const uint8_t* __restrict__ q, uint32_t n, uint32_t stride, uint32_t xyz_off, float* __restrict__ out4) {
  __shared__ float tile[2][3][256];
  __shared__ float cen[3];
  const int tid = threadIdx.x;
  float acc = 0.f;
  for (int pass = 0; pass < 2; pass++) {
    float cx = 0.f, cy = 0.f, cz = 0.f;
    if (pass == 1) { cx = cen[0]; cy = cen[1]; cz = cen[2]; }
    acc = 0.f;
    const uint32_t ntiles = (n + 255u) / 256u;
    for (uint32_t t = 0; t <= ntiles; t++) {
      if (t < ntiles) {                           // stage tile t
        const uint32_t i = t * 256u + (uint32_t)tid;
        float x = 0.f, y = 0.f, z = 0.f;
        if (i < n) {
          const float* p = reinterpret_cast<const float*>(q + (size_t)i * stride + xyz_off);
          x = p[0]; y = p[1]; z = p[2];
        }
        if (pass == 1) {
          const float dx = x - cx, dy = y - cy, dz = z - cz;
          x = sqrtf((dx * dx + dy * dy) + dz * dz);          // Eigen's (a_i - centroid).norm()
        }
        tile[t & 1][0][tid] = x; tile[t & 1][1][tid] = y; tile[t & 1][2][tid] = z;
      }
      if (t > 0 && tid < (pass == 0 ? 3 : 1)) {    // add tile t - 1 in point order
        const uint32_t base = (t - 1) * 256u;
        const int cnt = (int)min(256u, n - base);
        const float* src = tile[(t - 1) & 1][tid];
        for (int k = 0; k < cnt; k++) acc = acc + src[k];
      }
      __syncthreads();
    }
    if (pass == 0) {
      if (tid < 3) { cen[tid] = acc / (float)n; out4[tid] = acc / (float)n; }
    } else if (tid == 0) {
      out4[3] = acc;
    }
    __syncthreads();
  }
}

struct ApArgs {
  const uint8_t* q; uint32_t n, q_stride, q_xyz_off;
  const uint8_t* ref; uint32_t n_ref, r_stride, r_normal_off;
  const int32_t* corr;
  const float* norm;             // device {cx, cy, cz, dist} of ap_normalize_seq_kernel, or null: no normalisation
  double R[9]; int use_R;        // PointNormal variant rotates the reference normal by R (PointCloudLocalization.cc:715-718)
};

__global__ void __launch_bounds__(256)
ap_accumulate_kernel(ApArgs a, double* __restrict__ partials /*[grid][21]*/) {
  __shared__ double red[8 * 21];
  double acc[21];
#pragma unroll
  for (int e = 0; e < 21; e++) acc[e] = 0.0;
  // normalizePCloud: a = factor * p - factor * centroid, factor = n / sum |p - centroid| (float32, utils.cc:119-124)
  float factor = 1.f, tx = 0.f, ty = 0.f, tz = 0.f;
  if (a.norm) {
    factor = (float)a.n / a.norm[3];
    tx = -factor * a.norm[0]; ty = -factor * a.norm[1]; tz = -factor * a.norm[2];
  }
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(a.q + (size_t)i * a.q_stride + a.q_xyz_off);
    int j = a.corr[i];
    if (j < 0 || (uint32_t)j >= a.n_ref) continue;
    const float* nr = reinterpret_cast<const float*>(a.ref + (size_t)j * a.r_stride + a.r_normal_off);
    double ai[3] = {(double)(factor * p[0] + tx), (double)(factor * p[1] + ty), (double)(factor * p[2] + tz)};
    double ni[3] = {(double)nr[0], (double)nr[1], (double)nr[2]};
    if (isnan(ai[0]) || isnan(ai[1]) || isnan(ai[2]) || isnan(ni[0]) || isnan(ni[1]) || isnan(ni[2])) continue;
    if (a.use_R) {
      double r0 = a.R[0] * ni[0] + a.R[1] * ni[1] + a.R[2] * ni[2];
      double r1 = a.R[3] * ni[0] + a.R[4] * ni[1] + a.R[5] * ni[2];
      double r2 = a.R[6] * ni[0] + a.R[7] * ni[1] + a.R[8] * ni[2];
      ni[0] = r0; ni[1] = r1; ni[2] = r2;
    }
    double H[6] = {ai[1] * ni[2] - ai[2] * ni[1], ai[2] * ni[0] - ai[0] * ni[2], ai[0] * ni[1] - ai[1] * ni[0],
                   ni[0], ni[1], ni[2]};
    int e = 0;
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
      for (int c = r; c < 6; c++) acc[e++] += H[r] * H[c];
  }
  double tot = block_reduce<21, 8, 0>(acc, red);
  if (threadIdx.x < 21) partials[21 * (size_t)blockIdx.x + threadIdx.x] = tot;
}

// ------------------------------------------------------------------ row f3: resident rolling submap
// cell-sorted covariances of a cloud from a per-point cache kept in original (insertion) order
__global__ void __launch_bounds__(256)
cov_gather_kernel(const f4* __restrict__ pts, uint32_t n, const double* __restrict__ cache, double* __restrict__ cov) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t s = t / 6, e = t - 6 * s;
  if (s >= n) return;
  cov[6 * (size_t)s + e] = cache[6 * (size_t)float_to_bits(pts[s].w) + e];
}

// Occupancy hash of the submap: one entry per occupied voxel of edge `res` (world-anchored: voxel = floor(p / res)),
// open addressing, 64-bit key = the three voxel coordinates (21 bits each, offset 2^20), owner = map index of the
// point that occupies the voxel.  InsertPoints semantics of the reference's mapper (Locus.cc:465,532: a point enters
// the map iff no map point occupies its voxel yet; points are visited in input order) made parallel: candidates claim
// their voxel with atomicMin on (0x80000000 | input index) -- a committed owner (< 2^31) always wins, otherwise the
// lowest input index does, which is what the sequential loop yields.
constexpr unsigned long long SM_EMPTY = ~0ull;
__device__ __forceinline__ bool sm_voxel_key(float x, float y, float z, float res, unsigned long long& key) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
  const float fx = floorf(x / res), fy = floorf(y / res), fz = floorf(z / res);
  const float LIM = 1048575.0f;      // 2^20 - 1
  if (fx < -LIM || fx > LIM || fy < -LIM || fy > LIM || fz < -LIM || fz > LIM) return false;
  const unsigned long long cx = (unsigned long long)((int)fx + 1048576), cy = (unsigned long long)((int)fy + 1048576),
                           cz = (unsigned long long)((int)fz + 1048576);
  key = (cx << 42) | (cy << 21) | cz;
  return true;
}
__device__ __forceinline__ uint32_t sm_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}
// slot of `key`, claiming an empty one when it is not in the table yet
__device__ __forceinline__ uint32_t sm_find_or_claim(unsigned long long* __restrict__ keys, uint32_t mask, unsigned long long key) {
  uint32_t slot = sm_hash(key) & mask;
  for (;;) {
    const unsigned long long cur = atomicCAS(&keys[slot], SM_EMPTY, key);
    if (cur == SM_EMPTY || cur == key) return slot;
    slot = (slot + 1) & mask;
  }
}

__global__ void __launch_bounds__(256)
sm_claim_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off, float res,
                unsigned long long* __restrict__ keys, uint32_t* __restrict__ owner, uint32_t mask, uint32_t* __restrict__ slot_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = reinterpret_cast<const float*>(base + (size_t)i * stride + xyz_off);
  unsigned long long key;
  uint32_t slot = 0xffffffffu;
  if (sm_voxel_key(p[0], p[1], p[2], res, key)) {
    slot = sm_find_or_claim(keys, mask, key);
    atomicMin(&owner[slot], 0x80000000u | i);
  }
  slot_of[i] = slot;
}

__global__ void __launch_bounds__(256)
sm_decide_kernel(const uint32_t* __restrict__ slot_of, const uint32_t* __restrict__ owner, uint32_t n, uint32_t* __restrict__ flags) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t s = slot_of[i];
  flags[i] = (s != 0xffffffffu && owner[s] == (0x80000000u | i)) ? 1u : 0u;
}

__global__ void __launch_bounds__(256)
sm_commit_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off, const uint32_t* __restrict__ slot_of,
                 const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t n_old, f4* __restrict__ pts,
                 uint32_t* __restrict__ owner, float* __restrict__ inserted_xyz /*nullable*/) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  const float* p = reinterpret_cast<const float*>(base + (size_t)i * stride + xyz_off);
  const uint32_t j = n_old + pos[i];
  pts[j] = f4{p[0], p[1], p[2], 1.0f};
  owner[slot_of[i]] = j;
  if (inserted_xyz) { inserted_xyz[3 * (size_t)pos[i]] = p[0]; inserted_xyz[3 * (size_t)pos[i] + 1] = p[1]; inserted_xyz[3 * (size_t)pos[i] + 2] = p[2]; }
}

// rebuild of the table from the map's points (after a crop, or when the table grows)
__global__ void __launch_bounds__(256)
sm_rehash_kernel(const f4* __restrict__ pts, uint32_t n, float res, unsigned long long* __restrict__ keys,
                 uint32_t* __restrict__ owner, uint32_t mask) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const f4 p = pts[j];
  unsigned long long key;
  if (!sm_voxel_key(p.x, p.y, p.z, res, key)) return;
  owner[sm_find_or_claim(keys, mask, key)] = j;      // one map point per voxel: no two writers
}

// Refresh(current_pose) of the sliding-window mapper (Locus.cc:537, lo_settings.yaml:58 box_filter_size): pcl::CropBox
// keeps min <= p <= max, box = centre +- half
__global__ void __launch_bounds__(256)
sm_crop_flags_kernel(const f4* __restrict__ pts, uint32_t n, float cx, float cy, float cz, float half, uint32_t* __restrict__ flags) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const f4 p = pts[j];
  const float mnx = cx - half, mny = cy - half, mnz = cz - half, mxx = cx + half, mxy = cy + half, mxz = cz + half;
  const bool out = (p.x < mnx || p.y < mny || p.z < mnz) || (p.x > mxx || p.y > mxy || p.z > mxz);
  flags[j] = out ? 0u : 1u;
}
__global__ void __launch_bounds__(256)
sm_compact_kernel(const f4* __restrict__ pts, const double* __restrict__ cov, uint32_t n, uint32_t n_cov,
                  const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, f4* __restrict__ pts_out,
                  double* __restrict__ cov_out) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || !flags[j]) return;
  const uint32_t d = pos[j];
  pts_out[d] = pts[j];
  if (j < n_cov) {
#pragma unroll
    for (int e = 0; e < 6; e++) cov_out[6 * (size_t)d + e] = cov[6 * (size_t)j + e];
  }
}
__global__ void __launch_bounds__(256) iota_kernel(int32_t* __restrict__ a, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (int32_t)i;
}
// neighbours[i] = xyz of map point idx[i] (ApproxNearestNeighbors output cloud, Locus.cc:479)
__global__ void __launch_bounds__(256)
sm_gather_xyz_kernel(const f4* __restrict__ pts, const int32_t* __restrict__ idx, uint32_t n, float* __restrict__ out_xyz) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t j = idx[i];
  f4 p = (j >= 0) ? pts[j] : f4{0.f, 0.f, 0.f, 0.f};
  out_xyz[3 * (size_t)i] = p.x; out_xyz[3 * (size_t)i + 1] = p.y; out_xyz[3 * (size_t)i + 2] = p.z;
}

// ------------------------------------------------------------------ fitness (a9)
// pcl::Registration::getFitnessScore: mean of squared 1-NN distances <= max_range.
__global__ void __launch_bounds__(128)
fitness_kernel(GridView g, const f4* __restrict__ raw, uint32_t n, Mat34 T, double max_range,
               double* __restrict__ partials /*[gridDim.x][2]*/) {
  __shared__ double red[(128 / 32) * 2];
  double acc[2] = {0.0, 0.0};
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    f4 p = raw[i];
    float x, y, z;
    xform_pcl(T.m, p.x, p.y, p.z, x, y, z);
    int bo; float bd;
    int s = nn1_pruned(g, x, y, z, 3.0e38f, bo, bd);
    if (s >= 0 && (double)bd <= max_range) { acc[0] = (double)bd; acc[1] = 1.0; }
  }
  double tot = block_reduce<2, 4, 0>(acc, red);
  if (threadIdx.x < 2) partials[2 * (size_t)blockIdx.x + threadIdx.x] = tot;
}

}  // namespace lb
