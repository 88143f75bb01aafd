// features.cu -- LOAM-style feature extraction of the point-cloud filter (SURVEY 8f row f6) on the lb_voxel handle's
// stream.  Semantics: features.h.  Three launches and one host synchronisation (a second one copies a host output):
//   feat_point_kernel    per input point: ring (or dropped), per-CTA ring histogram, and the halfPassed cut as one
//                        max-reduction of ~index over the points that switch it on (the smallest such index wins)
//   feat_ring_kernel     one CTA per ring: stable compaction of the ring's points in input order (their offset is the
//                        histogram's prefix), orientation / intensity, unreliable marks, curvature, a rank sort
//                        of every region, the pick walk of one warp (32 candidates per ballot, regions in order), the
//                        less-flat list and its VoxelGrid.  Rings of up to FEAT_SMEM_PTS points work in shared memory,
//                        larger ones in global scratch of the same layout (no ring-size cap below int32).
//   feat_out_kernel      one CTA per (ring, category): offsets from the per-ring counts, rotation, writes.  When the
//                        output does not fit the capacity nothing is written; CTA (0, 0) publishes the totals.
#include <float.h>
#include <math.h>

#include "features.h"
#include "prims.cuh"

namespace lb {

constexpr int FEAT_T = 256;              // threads of a ring CTA
constexpr int FEAT_SMEM_PTS = 2048;      // ring points staged in shared memory
constexpr int FEAT_CATS = 4;             // sharp, less-sharp, flat, less-flat

struct FeatState {
  unsigned cut_inv;                      // max of ~i over the points that switch halfPassed on; 0: none does
  uint32_t ring_cnt[FEAT_MAX_RINGS];
  uint32_t cat_cnt[FEAT_CATS][FEAT_MAX_RINGS];
  uint32_t total[FEAT_CATS + 2];         // arranged, sharp, less-sharp, flat, less-flat, out
};

// per-point scratch of the arranged cloud (a ring uses [start, start + cnt) of every array)
struct FeatScratch {
  int* ring_of;                          // input point -> ring, -1 dropped
  f4* pts;                               // arranged cloud (swapped axes, intensity)
  float* curv;                           // curvature; reused as voxel keys
  int* order;                            // sorted region positions; reused as the voxel sort
  int* lf;                               // less-flat positions
  unsigned char* picked;
  signed char* label;
  int* list[3];                          // sharp, less-sharp, flat picks (ring-local positions)
  f4* lf_out;                            // the ring's VoxelGrid output
};

__device__ __forceinline__ void feat_load(const uint8_t* in, uint32_t i, uint32_t stride, uint32_t xyz_off, float& x, float& y, float& z) {
  const float* q = reinterpret_cast<const float*>(in + (size_t)i * stride + xyz_off);
  x = q[0]; y = q[1]; z = q[2];
}

__device__ __forceinline__ void feat_bounds(const uint8_t* in, uint32_t n, uint32_t stride, uint32_t xyz_off, float& start, float& end) {
  float x0, y0, z0, xl, yl, zl;
  feat_load(in, 0, stride, xyz_off, x0, y0, z0);
  feat_load(in, n - 1, stride, xyz_off, xl, yl, zl);
  feat_scan_bounds(x0, y0, xl, yl, start, end);
}

__global__ void __launch_bounds__(256)
feat_point_kernel(const uint8_t* __restrict__ in, uint32_t n, uint32_t stride, uint32_t xyz_off, FeatParams p,
                  int* __restrict__ ring_of, FeatState* __restrict__ st) {
  __shared__ uint32_t hist[FEAT_MAX_RINGS];
  __shared__ float s_start, s_end;
  for (int r = threadIdx.x; r < FEAT_MAX_RINGS; r += blockDim.x) hist[r] = 0;
  if (threadIdx.x == 0) feat_bounds(in, n, stride, xyz_off, s_start, s_end);
  __syncthreads();
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    float ix, iy, iz, x, y, z;
    feat_load(in, i, stride, xyz_off, ix, iy, iz);
    const int ring = feat_ring(ix, iy, iz, p, x, y, z);
    ring_of[i] = ring;
    if (ring >= 0) {
      atomicAdd(&hist[ring], 1u);
      if (feat_half_passes(feat_ori_a(x, z, s_start), s_start)) atomicMax(&st->cut_inv, ~i);
    }
  }
  __syncthreads();
  for (int r = threadIdx.x; r < p.n_rings; r += blockDim.x)
    if (hist[r]) atomicAdd(&st->ring_cnt[r], hist[r]);
}

__device__ __forceinline__ uint32_t feat_ord_min(uint32_t v, uint32_t* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = sm[0];
  for (int w = 1; w < FEAT_T / 32; w++) r = min(r, sm[w]);
  __syncthreads();
  return r;
}

// the pick walk of one region, run by warp 0: candidates k, k -/+ 1, ... are tested 32 at a time; the first eligible
// one is taken, its marks are written, and the next window starts right after it
template <bool CORNER>
__device__ void feat_walk(const int* order, long long sp, long long m, const float* curv, unsigned char* picked, signed char* label,
                          const f4* P, const FeatParams& p, int** lists, uint32_t* n_list, int* list_base) {
  const int lane = threadIdx.x & 31;
  const int limit = CORNER ? p.max_less_sharp : p.max_flat;
  int taken = 0;
  long long k = CORNER ? m - 1 : 0;
  while ((CORNER ? k >= 0 : k < m) && taken < limit) {
    const long long kk = CORNER ? k - lane : k + lane;
    bool ok = false;
    int idx = 0;
    if (kk >= 0 && kk < m) {
      idx = order[sp + kk];
      ok = CORNER ? feat_corner_candidate(picked[idx], curv[idx], p.curv_thr) : feat_flat_candidate(picked[idx], curv[idx], p.curv_thr);
    }
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if (!b) { k = CORNER ? k - 32 : k + 32; continue; }
    const int f = __ffs(b) - 1;
    const int sel = __shfl_sync(0xffffffffu, idx, f);
    taken++;
    if (lane == 0) {
      if (CORNER) {
        const bool sharp = taken <= p.max_sharp;
        label[sel] = sharp ? FEAT_CORNER_SHARP : FEAT_CORNER_LESS_SHARP;
        if (sharp) lists[0][list_base[0] + n_list[0]++] = sel;
        lists[1][list_base[1] + n_list[1]++] = sel;
      } else {
        label[sel] = FEAT_SURFACE_FLAT;
        lists[2][list_base[2] + n_list[2]++] = sel;
      }
      feat_mark_as_picked(P, sel, p.cr, picked);
    }
    __syncwarp();
    k = CORNER ? k - f - 1 : k + f + 1;
  }
}

__global__ void __launch_bounds__(FEAT_T)
feat_ring_kernel(const uint8_t* __restrict__ in, uint32_t n, uint32_t stride, uint32_t xyz_off, FeatParams p, FeatScratch S,
                 FeatState* __restrict__ st) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint32_t scan_sm[FEAT_T / 32 + 1];
  __shared__ uint32_t red_sm[FEAT_T / 32];
  __shared__ uint32_t s_start, s_cnt, s_base;
  __shared__ float s_so, s_eo;
  __shared__ unsigned s_cut;
  const int r = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    uint32_t a = 0;
    for (int q = 0; q < r; q++) a += st->ring_cnt[q];
    s_start = a; s_cnt = st->ring_cnt[r];
    feat_bounds(in, n, stride, xyz_off, s_so, s_eo);
    s_cut = st->cut_inv ? ~st->cut_inv : 0xffffffffu;
    s_base = 0;
  }
  __syncthreads();
  const uint32_t start = s_start, cnt = s_cnt, cut = s_cut;
  const float so = s_so, eo = s_eo;
  // ---- arrangement: the ring's points in input order
  f4* G = S.pts + start;
  for (uint32_t t0 = 0; t0 < n; t0 += FEAT_T) {
    const uint32_t i = t0 + tid;
    const bool mine = i < n && S.ring_of[i] == r;
    uint32_t tot;
    const uint32_t o = block_excl_scan<FEAT_T>(mine ? 1u : 0u, &tot, scan_sm) + s_base;
    if (mine) {
      float ix, iy, iz, x, y, z;
      feat_load(in, i, stride, xyz_off, ix, iy, iz);
      feat_ring(ix, iy, iz, p, x, y, z);
      const float ori = (i <= cut) ? feat_ori_a(x, z, so) : feat_ori_b(x, z, eo);
      G[o] = f4{x, y, z, feat_intensity(r, ori, so, eo, p.scan_period)};
    }
    __syncthreads();
    if (tid == 0) s_base += tot;
    __syncthreads();
  }
  uint32_t* cat = &st->cat_cnt[0][r];        // category c of this ring: cat[c * FEAT_MAX_RINGS], zeroed before the call
  if (feat_ring_skipped(cnt, p.cr)) return;
  // ---- work arrays: shared memory for small rings, the global scratch otherwise
  const bool small = cnt <= (uint32_t)FEAT_SMEM_PTS;
  f4* P = G;
  float* curv = S.curv + start;
  int* order = S.order + start;
  int* lf = S.lf + start;
  unsigned char* picked = S.picked + start;
  signed char* label = S.label + start;
  if (small) {
    P = reinterpret_cast<f4*>(smem);
    curv = reinterpret_cast<float*>(P + FEAT_SMEM_PTS);
    order = reinterpret_cast<int*>(curv + FEAT_SMEM_PTS);
    lf = order + FEAT_SMEM_PTS;
    picked = reinterpret_cast<unsigned char*>(lf + FEAT_SMEM_PTS);
    label = reinterpret_cast<signed char*>(picked + FEAT_SMEM_PTS);
  }
  for (uint32_t k = tid; k < cnt; k += FEAT_T) {
    if (small) P[k] = G[k];
    picked[k] = 0;
    label[k] = FEAT_NO_REGION;
  }
  __syncthreads();
  const int cr = p.cr;
  for (long long i = cr + tid; i < (long long)cnt - 1 - cr; i += FEAT_T) feat_unreliable_marks(P, i, cr, picked);
  for (long long i = cr + tid; i <= (long long)cnt - 1 - cr; i += FEAT_T) curv[i] = feat_curvature(P, i, cr);
  __syncthreads();
  // ---- every region in the insertion sort's order (feat_region_rank: a permutation, NaN curvatures included)
  for (int j = 0; j < p.n_regions; j++) {
    long long sp, ep;
    feat_region(cnt, cr, p.n_regions, j, sp, ep);
    if (ep <= sp) continue;
    bool nan = false;
    for (long long a = sp + tid; a <= ep; a += FEAT_T) nan = nan || isnan(curv[a]);
    const bool no_nan = !__syncthreads_or(nan);
    for (long long a = sp + tid; a <= ep; a += FEAT_T) {
      order[sp + feat_region_rank(curv, sp, ep, a, no_nan)] = (int)a;
      label[a] = FEAT_SURFACE_LESS_FLAT;
    }
  }
  __syncthreads();
  // ---- the pick walk, regions in order
  if (tid < 32) {
    uint32_t n_list[3] = {0, 0, 0};
    int* lists[3] = {S.list[0], S.list[1], S.list[2]};
    int base[3] = {(int)start, (int)start, (int)start};
    for (int j = 0; j < p.n_regions; j++) {
      long long sp, ep;
      feat_region(cnt, cr, p.n_regions, j, sp, ep);
      if (ep <= sp) continue;
      feat_walk<true>(order, sp, ep - sp + 1, curv, picked, label, P, p, lists, n_list, base);
      feat_walk<false>(order, sp, ep - sp + 1, curv, picked, label, P, p, lists, n_list, base);
    }
    if (tid == 0) for (int c = 0; c < 3; c++) cat[c * FEAT_MAX_RINGS] = n_list[c];
  }
  __syncthreads();
  // ---- less-flat list: every unskipped-region point that is not a corner, in position order
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (uint32_t t0 = 0; t0 < cnt; t0 += FEAT_T) {
    const uint32_t k = t0 + tid;
    const bool in_lf = k < cnt && label[k] <= FEAT_SURFACE_LESS_FLAT;
    uint32_t tot;
    const uint32_t o = block_excl_scan<FEAT_T>(in_lf ? 1u : 0u, &tot, scan_sm) + s_base;
    if (in_lf) lf[o] = (int)k;
    __syncthreads();
    if (tid == 0) s_base += tot;
    __syncthreads();
  }
  const uint32_t m = s_base;
  f4* out = S.lf_out + start;
  if (m == 0) return;
  // ---- VoxelGrid<PointF> of the less-flat list
  uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
  for (uint32_t k = tid; k < m; k += FEAT_T) {
    const f4 q = P[lf[k]];
    const uint32_t o[3] = {f2ord(q.x), f2ord(q.y), f2ord(q.z)};
    for (int d = 0; d < 3; d++) { mn[d] = min(mn[d], o[d]); mx[d] = min(mx[d], ~o[d]); }
  }
  float fmn[3], fmx[3];
  for (int d = 0; d < 3; d++) { fmn[d] = ord2f(feat_ord_min(mn[d], red_sm)); fmx[d] = ord2f(~feat_ord_min(mx[d], red_sm)); }
  const FeatGrid g = feat_grid(fmn, fmx, p.leaf);
  if (g.overflow) {
    for (uint32_t k = tid; k < m; k += FEAT_T) out[k] = P[lf[k]];
    if (tid == 0) cat[3 * FEAT_MAX_RINGS] = m;
    return;
  }
  int* key = reinterpret_cast<int*>(curv);      // curvature and region order are no longer needed
  int* srt = order;
  for (uint32_t k = tid; k < m; k += FEAT_T) {
    const f4 q = P[lf[k]];
    key[k] = feat_voxel_key(g, q.x, q.y, q.z);
  }
  __syncthreads();
  for (uint32_t a = tid; a < m; a += FEAT_T) {
    const int ka = key[a];
    uint32_t rank = 0;
    for (uint32_t b = 0; b < m; b++) {
      const int kb = key[b];
      rank += (kb < ka || (kb == ka && b < a)) ? 1u : 0u;
    }
    srt[rank] = (int)a;
  }
  __syncthreads();
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (uint32_t t0 = 0; t0 < m; t0 += FEAT_T) {
    const uint32_t s = t0 + tid;
    const bool head = s < m && (s == 0 || key[srt[s]] != key[srt[s - 1]]);
    uint32_t tot;
    const uint32_t v = block_excl_scan<FEAT_T>(head ? 1u : 0u, &tot, scan_sm) + s_base;
    if (head) {
      const int kv = key[srt[s]];
      f4 acc = P[lf[srt[s]]];
      uint32_t e = s + 1;
      for (; e < m && key[srt[e]] == kv; e++) {
        const f4 q = P[lf[srt[e]]];
        acc.x = acc.x + q.x; acc.y = acc.y + q.y; acc.z = acc.z + q.z; acc.w = acc.w + q.w;
      }
      const float c = (float)(e - s);
      out[v] = f4{acc.x / c, acc.y / c, acc.z / c, acc.w / c};
    }
    __syncthreads();
    if (tid == 0) s_base += tot;
    __syncthreads();
  }
  if (tid == 0) cat[3 * FEAT_MAX_RINGS] = s_base;
}

struct FeatRot { float T[12]; };

// grid (n_rings, 4): CTA (r, c) writes ring r's points of category c at their place in the concatenated output
__global__ void __launch_bounds__(128)
feat_out_kernel(FeatScratch S, FeatRot R, int n_rings, size_t capacity, FeatState* __restrict__ st, float* __restrict__ out4) {
  __shared__ uint32_t s_base, s_start;
  __shared__ unsigned long long s_total;
  const int r = blockIdx.x, c = blockIdx.y;
  if (threadIdx.x == 0) {
    unsigned long long tot[FEAT_CATS] = {0, 0, 0, 0}, arranged = 0;
    uint32_t start = 0;
    for (int q = 0; q < n_rings; q++) {
      const uint32_t rc = st->ring_cnt[q];
      arranged += rc;
      if (q < r) start += rc;
      for (int k = 0; k < FEAT_CATS; k++) tot[k] += st->cat_cnt[k][q];
    }
    uint32_t base = 0;
    for (int k = 0; k < c; k++) base += (uint32_t)tot[k];
    for (int q = 0; q < r; q++) base += st->cat_cnt[c][q];
    s_base = base; s_start = start;
    s_total = tot[0] + tot[1] + tot[2] + tot[3];
    if (r == 0 && c == 0) {
      st->total[0] = (uint32_t)arranged;
      for (int k = 0; k < FEAT_CATS; k++) st->total[1 + k] = (uint32_t)tot[k];
      st->total[FEAT_CATS + 1] = (uint32_t)s_total;
    }
  }
  __syncthreads();
  if (s_total > capacity) return;
  const uint32_t m = st->cat_cnt[c][r], base = s_base, start = s_start;
  for (uint32_t k = threadIdx.x; k < m; k += blockDim.x) {
    const f4 q = (c == 3) ? S.lf_out[start + k] : S.pts[start + S.list[c][start + k]];
    float x, y, z;
    xform_pcl(R.T, q.x, q.y, q.z, x, y, z);
    reinterpret_cast<float4*>(out4)[base + k] = make_float4(x, y, z, q.w);
  }
}

// ------------------------------------------------------------------ host side
struct FeatWork {
  DBuf<uint8_t> in;
  DBuf<int> ring_of, order, lf, lists;
  DBuf<f4> pts, lf_out;
  DBuf<float> curv, out;
  DBuf<unsigned char> picked;
  FeatState* d_st = nullptr;
  FeatState* h_st = nullptr;
  bool smem_set = false;
};

FeatWork* feat_work_new() { return new FeatWork; }

void feat_work_free(FeatWork* w) {
  if (!w) return;
  w->in.release(); w->ring_of.release(); w->order.release(); w->lf.release(); w->lists.release();
  w->pts.release(); w->lf_out.release(); w->curv.release(); w->out.release(); w->picked.release();
  if (w->d_st) cudaFree(w->d_st);
  if (w->h_st) cudaFreeHost(w->h_st);
  delete w;
}

static int feat_check_params(const lb_features_params* q) {
  if (!q) { set_error("lb_voxel_extract_features: null params"); return LB_ERR_INVALID_ARG; }
  if (q->n_rings < 1 || q->n_rings > FEAT_MAX_RINGS) { set_error("lb_voxel_extract_features: n_rings must be 1..%d", FEAT_MAX_RINGS); return LB_ERR_INVALID_ARG; }
  if (!(q->upper_deg > q->lower_deg) || !isfinite(q->lower_deg) || !isfinite(q->upper_deg)) {
    set_error("lb_voxel_extract_features: need finite lower_deg < upper_deg"); return LB_ERR_INVALID_ARG;
  }
  if (q->curvature_region < 1 || q->curvature_region > FEAT_MAX_CURVATURE_REGION) {
    set_error("lb_voxel_extract_features: curvature_region must be 1..%d", FEAT_MAX_CURVATURE_REGION); return LB_ERR_INVALID_ARG;
  }
  if (q->n_feature_regions < 1 || q->n_feature_regions > FEAT_MAX_REGIONS) {
    set_error("lb_voxel_extract_features: n_feature_regions must be 1..%d", FEAT_MAX_REGIONS); return LB_ERR_INVALID_ARG;
  }
  if (!(q->less_flat_leaf > 0.f)) { set_error("lb_voxel_extract_features: less_flat_leaf must be > 0"); return LB_ERR_INVALID_ARG; }
  if (q->max_corner_sharp < 0 || q->max_corner_less_sharp < 0 || q->max_surface_flat < 0) {
    set_error("lb_voxel_extract_features: negative feature count"); return LB_ERR_INVALID_ARG;
  }
  return LB_OK;
}

int feat_extract(Ctx& c, FeatWork* w, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem_in,
                 const lb_features_params* q, float* out4, size_t out_capacity, lb_features_result* res, int mem_out) {
  if (!res) { set_error("lb_voxel_extract_features: null result"); return LB_ERR_INVALID_ARG; }
  memset(res, 0, sizeof(*res));
  LB_TRY(feat_check_params(q));
  if (n == 0) { set_error("lb_voxel_extract_features: empty input cloud"); return LB_ERR_EMPTY_SOURCE; }
  if (!pts || (!out4 && out_capacity > 0)) { set_error("lb_voxel_extract_features: null buffer"); return LB_ERR_INVALID_ARG; }
  if (n > 0x3ffffff0ull) { set_error("lb_voxel_extract_features: too many points"); return LB_ERR_INVALID_ARG; }
  if ((stride & 3u) || (xyz_off & 3u) || xyz_off + 12 > stride || (reinterpret_cast<uintptr_t>(pts) & 3u)) {
    set_error("lb_voxel_extract_features: x, y, z must be three aligned floats inside a stride that is a multiple of 4");
    return LB_ERR_INVALID_ARG;
  }
  if (mem_out == LB_MEM_DEVICE && out4 && (reinterpret_cast<uintptr_t>(out4) & 15u)) {
    set_error("lb_voxel_extract_features: a device output must be 16-byte aligned"); return LB_ERR_INVALID_ARG;
  }
  FeatParams p;
  p.n_rings = q->n_rings; p.lower = q->lower_deg; p.upper = q->upper_deg; p.scan_period = q->scan_period;
  p.cr = q->curvature_region; p.n_regions = q->n_feature_regions; p.max_sharp = q->max_corner_sharp;
  p.max_less_sharp = q->max_corner_less_sharp; p.max_flat = q->max_surface_flat; p.curv_thr = q->curvature_threshold;
  p.leaf = q->less_flat_leaf;
  p.factor = (float)(p.n_rings - 1) / (p.upper - p.lower);

  LB_CUDA(cudaSetDevice(c.device));
  if (!w->d_st) {
    LB_CUDA(cudaMalloc((void**)&w->d_st, sizeof(FeatState)));
    LB_CUDA(cudaMallocHost((void**)&w->h_st, sizeof(FeatState)));
  }
  const size_t smem = (size_t)FEAT_SMEM_PTS * (sizeof(f4) + sizeof(float) + 2 * sizeof(int) + 2);
  if (!w->smem_set) {
    LB_CUDA(cudaFuncSetAttribute(feat_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    w->smem_set = true;
  }
  const uint32_t nn = (uint32_t)n;
  LB_TRY(w->ring_of.ensure(n)); LB_TRY(w->pts.ensure(n)); LB_TRY(w->curv.ensure(n)); LB_TRY(w->order.ensure(n));
  LB_TRY(w->lf.ensure(n)); LB_TRY(w->picked.ensure(2 * n)); LB_TRY(w->lists.ensure(3 * n)); LB_TRY(w->lf_out.ensure(n));
  const uint8_t* d_in = static_cast<const uint8_t*>(pts);
  if (mem_in == LB_MEM_HOST) {
    LB_TRY(w->in.ensure(n * stride));
    LB_CUDA(cudaMemcpyAsync(w->in.p, pts, n * stride, cudaMemcpyHostToDevice, c.stream));
    d_in = w->in.p;
  }
  // every output fits 2n points: sharp <= corners, flat + less-flat <= 2 * non-corners
  float* d_out = out4;
  size_t cap = out4 ? out_capacity : 0;
  if (mem_out == LB_MEM_HOST) {
    LB_TRY(w->out.ensure(8 * n));
    d_out = w->out.p; cap = 2 * n;
  }
  FeatScratch S;
  S.ring_of = w->ring_of.p; S.pts = w->pts.p; S.curv = w->curv.p; S.order = w->order.p; S.lf = w->lf.p;
  S.picked = w->picked.p; S.label = reinterpret_cast<signed char*>(w->picked.p + n);
  S.list[0] = w->lists.p; S.list[1] = w->lists.p + n; S.list[2] = w->lists.p + 2 * n;
  S.lf_out = w->lf_out.p;
  FeatRot R;
  feat_rotation(R.T);
  LB_CUDA(cudaMemsetAsync(w->d_st, 0, sizeof(FeatState), c.stream));
  feat_point_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(d_in, nn, (uint32_t)stride, (uint32_t)xyz_off, p, S.ring_of, w->d_st);
  feat_ring_kernel<<<p.n_rings, FEAT_T, smem, c.stream>>>(d_in, nn, (uint32_t)stride, (uint32_t)xyz_off, p, S, w->d_st);
  feat_out_kernel<<<dim3(p.n_rings, FEAT_CATS), 128, 0, c.stream>>>(S, R, p.n_rings, cap, w->d_st, d_out);
  c.launches += 3;
  LB_CUDA(cudaGetLastError());
  LB_CUDA(cudaMemcpyAsync(w->h_st, w->d_st, sizeof(FeatState), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const uint32_t* t = w->h_st->total;
  res->n_arranged = t[0]; res->n_sharp = t[1]; res->n_less_sharp = t[2]; res->n_flat = t[3]; res->n_less_flat = t[4];
  res->n_out = t[5];
  if (res->n_out > out_capacity || (res->n_out > 0 && !out4)) {
    set_error("lb_voxel_extract_features: output capacity %zu < %zu points", out_capacity, res->n_out);
    return LB_ERR_CAPACITY;
  }
  if (mem_out == LB_MEM_HOST && res->n_out > 0) {
    LB_CUDA(cudaMemcpyAsync(out4, d_out, res->n_out * 4 * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  return LB_OK;
}

}  // namespace lb
