// ndt.cu -- NDT registration on the GPU (SURVEY 8f row f4): the C ABI `lb_ndt_*` replaces
// pclomp::NormalDistributionsTransform<PointF, PointF> behind LOCUS's `registration_method: ndt`
// (PointCloudOdometry.cc:182-195, PointCloudLocalization.cc:267-280).
//
//   lb_ndt_set_target    setInputTarget -> init() -> VoxelGridCovariance::filter(true)
//                        (ndt_omp.h:116-119,257-262; voxel_grid_covariance_omp_impl.hpp:48-370):
//                        ndt_gather -> ndt_keys -> stable radix sort (prims.cu) -> ndt_heads -> scan -> ndt_head_pos ->
//                        ndt_gaussians -> ndt_hash_insert.  One warp per voxel fetches its points 32 at a time and adds
//                        them in input order (the reference's accumulation order), so means / inverse covariances /
//                        centroids are reproducible bit for bit.
//   lb_ndt_align         computeTransformation (ndt_omp_impl.hpp:100-208) as a stream-ordered chain of
//                        [evaluation, ndt_ctl_kernel] steps.  An evaluation computes the score / gradient / Hessian terms
//                        of every source point against the voxels around it: float per-pair terms and double sums as in
//                        the reference, eight lanes per point (ndt_eval_group_kernel) for the float passes, one thread per
//                        point (ndt_eval_kernel) for the closing double-precision Hessian pass; one partial row per CTA.
//                        The one-CTA controller kernel adds the rows in a fixed shape and runs the Newton step (6x6
//                        Jacobi SVD on its first warp) / More-Thuente line search state machine of ndt.h, then posts the
//                        next request.  The host enqueues a batch of steps and reads the controller back once per batch;
//                        the specialisations a request does not name, and steps after the end, return at once.
//
// Latency-bound gather work over L1 / L2 resident data (96-byte voxel records behind a hash lookup, a few MB per pass); no
// contraction, no tensor cores.
#include <algorithm>
#include <chrono>
#include <new>
#include <vector>

#include "ndt.h"
#include "prims.cuh"

namespace lb {

// the resident submap (submap.cuh, compiled into gicp.cu): its current points, count, generation and stream
int submap_device(const lb_submap* m);
void submap_points_view(const lb_submap* m, const f4** pts, size_t* n, uint64_t* generation, cudaStream_t* stream);

constexpr int NDT_EVAL_THREADS = 128;
constexpr int NDT_BATCH = 8;            // [evaluation, controller] steps enqueued between two looks at the controller

__global__ void __launch_bounds__(256)
ndt_gather_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off, f4* __restrict__ out,
                  BBoxAcc* __restrict__ acc) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  float x = 0.f, y = 0.f, z = 0.f;
  if (i < n) {
    const float* q = reinterpret_cast<const float*>(base + (size_t)i * stride + xyz_off);
    x = q[0]; y = q[1]; z = q[2];
    out[i] = f4{x, y, z, 1.0f};
    ok = isfinite(x) && isfinite(y) && isfinite(z);
  }
  bbox_warp_accumulate(ok, x, y, z, acc);
}

__global__ void __launch_bounds__(256)
ndt_keys_kernel(const f4* __restrict__ pts, uint32_t n, NdtLattice L, uint32_t invalid_key, uint32_t* __restrict__ keys) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const f4 p = pts[i];
  const bool ok = isfinite(p.x) && isfinite(p.y) && isfinite(p.z);     // non-finite target points are skipped (:196-200)
  keys[i] = ok ? (uint32_t)ndt_voxel_key(L, p.x, p.y, p.z) : invalid_key;
}

// flag[i] = 1 when sorted position i opens a voxel with at least min_pts points
__global__ void __launch_bounds__(256)
ndt_heads_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t invalid_key, int min_pts, uint32_t* __restrict__ flag) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = keys[i];
  uint32_t f = 0;
  if (k != invalid_key && (i == 0 || keys[i - 1] != k)) {
    uint32_t j = i + 1;
    while (j < n && keys[j] == k && (int)(j - i) < min_pts) j++;
    f = (int)(j - i) >= min_pts ? 1u : 0u;
  }
  flag[i] = f;
}

// head_pos[slot] = sorted position at which the slot-th searchable voxel starts
__global__ void __launch_bounds__(256)
ndt_head_pos_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ slot_of, uint32_t n, uint32_t* __restrict__ head_pos) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) head_pos[slot_of[i]] = i;
}

// One warp per voxel.  The lanes fetch 32 points of the voxel at a time (the next batch while the current one is being
// added); the sums themselves run over the points one after the other in input order on every lane alike -- that order
// is what makes mean / covariance / centroid reproducible bit for bit (the reference adds them in its input loop,
// voxel_grid_covariance_omp_impl.hpp:218-225).  A thread per voxel instead was slower: two
// dependent gathers per point, and the voxel under the sensor holds thousands of points.
__global__ void __launch_bounds__(128)
ndt_gaussians_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t n, const uint32_t* __restrict__ head_pos,
                     uint32_t n_valid, const f4* __restrict__ pts, double eig_mult, NdtVoxel* __restrict__ vox, f4* __restrict__ cen,
                     int32_t* __restrict__ leaf_idx) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_valid) return;
  const uint32_t i0 = head_pos[w];
  const uint32_t k = keys[i0];
  double sum[3] = {0, 0, 0}, m2[6] = {0, 0, 0, 0, 0, 0};
  float csum[3] = {0.f, 0.f, 0.f};
  uint32_t total = 0;
  uint32_t j = i0 + lane;
  bool in = j < n && keys[j] == k;
  f4 p = in ? pts[vals[j]] : f4{0.f, 0.f, 0.f, 0.f};
  for (;;) {
    const int cnt = __popc(__ballot_sync(0xffffffffu, in));        // the voxel's points are contiguous: a prefix of the lanes
    const f4 cur = p;
    if (cnt == 32) {                                               // fetch the next batch before adding this one
      j += 32;
      in = j < n && keys[j] == k;
      p = in ? pts[vals[j]] : f4{0.f, 0.f, 0.f, 0.f};
    }
    for (int t = 0; t < cnt; t++) {
      const float x = __shfl_sync(0xffffffffu, cur.x, t), y = __shfl_sync(0xffffffffu, cur.y, t), z = __shfl_sync(0xffffffffu, cur.z, t);
      const double d0 = x, d1 = y, d2 = z;
      sum[0] += d0; sum[1] += d1; sum[2] += d2;
      csum[0] += x; csum[1] += y; csum[2] += z;
      m2[0] += d0 * d0; m2[1] += d0 * d1; m2[2] += d0 * d2; m2[3] += d1 * d1; m2[4] += d1 * d2; m2[5] += d2 * d2;
    }
    total += (uint32_t)cnt;
    if (cnt < 32) break;
  }
  if (lane != 0) return;
  NdtVoxel v;
  float c[3];
  const int nr = ndt_finish_voxel((int)total, sum, m2, csum, eig_mult, v, c);
  vox[w] = v;
  cen[w] = f4{c[0], c[1], c[2], __int_as_float(nr)};
  leaf_idx[w] = (int32_t)k;
}

__global__ void __launch_bounds__(256)
ndt_hash_insert_kernel(const int32_t* __restrict__ leaf_idx, uint32_t n_valid, uint32_t* __restrict__ hkey, int32_t* __restrict__ hval,
                       uint32_t hmask) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_valid) return;
  const uint32_t key = (uint32_t)leaf_idx[s];
  uint32_t h = ndt_hash(key) & hmask;
  for (;;) {
    const uint32_t prev = atomicCAS(&hkey[h], 0xffffffffu, key);
    if (prev == 0xffffffffu) { hval[h] = (int32_t)s; return; }
    h = (h + 1) & hmask;
  }
}

// One evaluation: every source point against the voxels around it; one partial (43 doubles) per CTA.  Which sums the
// controller wants (score + gradient / + Hessian / the double-precision Hessian alone) is only known on the device, so
// one specialisation per request is enqueued and the two that do not match return at once: the line search's trials
// (score + gradient, 7 sums) then run with a third of the registers of the 43-sum pass.
template <int WANT>
__global__ void __launch_bounds__(NDT_EVAL_THREADS)
ndt_eval_kernel(const NdtCtl* __restrict__ ctl, NdtTargetView tv, NdtGauss G, const f4* __restrict__ src, uint32_t n,
                double* __restrict__ partials) {
  constexpr int K0 = WANT == NDT_WANT_HESSIAN ? 7 : 0, K1 = WANT == NDT_WANT_DERIV ? 7 : NDT_NSUM;
  __shared__ NdtAngles sA;
  __shared__ float sT[12];
  __shared__ double sred[NDT_EVAL_THREADS / 32][K1 - K0];
  if (ctl->want != WANT) return;                           // another specialisation's turn, or the align has finished
  {
    const uint32_t* g = reinterpret_cast<const uint32_t*>(&ctl->ang);
    uint32_t* s = reinterpret_cast<uint32_t*>(&sA);
    for (uint32_t w = threadIdx.x; w < sizeof(NdtAngles) / 4; w += blockDim.x) s[w] = g[w];
    if (threadIdx.x < 12) sT[threadIdx.x] = ctl->T[threadIdx.x];
  }
  __syncthreads();
  double acc[NDT_NSUM];
#pragma unroll
  for (int k = 0; k < NDT_NSUM; k++) acc[k] = 0.0;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const f4 p = src[i];
    ndt_point_eval(tv, G, sA, sT, p.x, p.y, p.z, WANT, acc);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = K0; k < K1; k++) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sred[warp][k - K0] = v;
  }
  __syncthreads();
  if (threadIdx.x < NDT_NSUM) {
    const int k = threadIdx.x;
    double v = 0.0;
    if (k >= K0 && k < K1) {
#pragma unroll
      for (int w = 0; w < NDT_EVAL_THREADS / 32; w++) v += sred[w][k - K0];
    }
    partials[(size_t)blockIdx.x * NDT_NSUM + k] = v;       // sums this request does not produce are 0 (hessian.setZero())
  }
}

// The same evaluation with EIGHT lanes per source point (float passes only).  A 30 k-point scan is 918 warps of the
// kernel above -- six per SM, each a 3-4 k-instruction chain of dependent hash probes and double-precision exps, so the
// GPU idles on latency.  Here the eight lanes of a point probe its candidate cells side by side (hits appended to a
// shared-memory list, then ranked by (distance, slot) = the reference's visiting order), compute one (point, voxel) pair
// each, and add the pairs' float terms IN THAT ORDER into per-point double subtotals (lane s owns sums s, s + 8, ...):
// the same per-pair arithmetic (ndt.h) and the same per-point association as the kernel above, eight times the warps.
constexpr int NDT_GRP = 8;                                   // lanes per source point
constexpr int NDT_GPTS = NDT_EVAL_THREADS / NDT_GRP;         // points per batch of a CTA
constexpr int NDT_GBATCH = 2;                                // batches per CTA (one partial row per CTA)

template <int WANT>
__global__ void __launch_bounds__(NDT_EVAL_THREADS)
ndt_eval_group_kernel(const NdtCtl* __restrict__ ctl, NdtTargetView tv, NdtGauss G, const f4* __restrict__ src, uint32_t n,
                      double* __restrict__ partials) {
  constexpr bool HESS = WANT == NDT_WANT_DERIV_H;
  constexpr int NT = HESS ? NDT_NSUM : 7;                    // sums of this request
  constexpr int NC = (NT + NDT_GRP - 1) / NDT_GRP;           // of which one lane owns at most this many
  __shared__ NdtAngles sA;
  __shared__ float sT[12];
  __shared__ float sterm[NDT_GPTS][NDT_GRP][NT];
  __shared__ int shit_slot[NDT_GPTS][NDT_MAX_NB];
  __shared__ float shit_key[NDT_GPTS][NDT_MAX_NB];
  __shared__ int ssorted[NDT_GPTS][NDT_MAX_NB];
  __shared__ int shit_n[NDT_GPTS];
  __shared__ float sxj[NDT_GPTS][8], sxh[NDT_GPTS][16];
  __shared__ double sacc[NDT_GPTS][NT];
  if (ctl->want != WANT) return;
  {
    const uint32_t* g = reinterpret_cast<const uint32_t*>(&ctl->ang);
    uint32_t* sw = reinterpret_cast<uint32_t*>(&sA);
    for (uint32_t w = threadIdx.x; w < sizeof(NdtAngles) / 4; w += blockDim.x) sw[w] = g[w];
    if (threadIdx.x < 12) sT[threadIdx.x] = ctl->T[threadIdx.x];
  }
  __syncthreads();
  const int pt = threadIdx.x / NDT_GRP, sub = threadIdx.x % NDT_GRP;
  const unsigned gmask = 0xffu << (threadIdx.x & 24);        // the eight lanes of this point
  double total[NC];
#pragma unroll
  for (int ci = 0; ci < NC; ci++) total[ci] = 0.0;
  for (int b = 0; b < NDT_GBATCH; b++) {
    const uint32_t i = (blockIdx.x * NDT_GBATCH + b) * NDT_GPTS + pt;
    const bool valid = i < n;
    if (sub == 0) shit_n[pt] = 0;
    __syncwarp(gmask);
    float x0 = 0.f, x1 = 0.f, x2 = 0.f, q0 = 0.f, q1 = 0.f, q2 = 0.f;
    if (valid) {
      const f4 p = src[i];
      x0 = p.x; x1 = p.y; x2 = p.z;
      xform_pcl(sT, x0, x1, x2, q0, q1, q2);
      // 1. candidate voxels, eight at a time
      if (tv.method == NDT_KDTREE) {
        const float q[3] = {q0, q1, q2};
        int lo[3], hi[3];
        ndt_kd_range(tv, q, lo, hi);
        const int nx = hi[0] - lo[0] + 1, ny = hi[1] - lo[1] + 1, nz = hi[2] - lo[2] + 1;
        if (nx > 0 && ny > 0 && nz > 0) {
          const int ncell = nx * ny * nz, nxy = nx * ny;
          // at most 4 cells per axis: c / nxy and r / nx through float reciprocals (exact for these ranges: the + 0.5 keeps
          // the quotient away from an integer boundary)
          const float inv_nxy = 1.0f / (float)nxy, inv_nx = 1.0f / (float)nx;
          for (int c = sub; c < ncell; c += NDT_GRP) {
            const int iz = (int)(((float)c + 0.5f) * inv_nxy), rem = c - iz * nxy;
            const int iy = (int)(((float)rem + 0.5f) * inv_nx);
            const int cx = lo[0] + (rem - iy * nx), cy = lo[1] + iy, cz = lo[2] + iz;
            int sl;
            float d2;
            if (ndt_kd_probe(tv, cx, cy, cz, q0, q1, q2, sl, d2)) {
              const int pos = atomicAdd(&shit_n[pt], 1);
              if (pos < NDT_MAX_NB) { shit_slot[pt][pos] = sl; shit_key[pt][pos] = d2; }
            }
          }
        }
      } else {
        const int nrel = ndt_direct_count(tv.method);
        for (int r = sub; r < nrel; r += NDT_GRP) {
          const int sl = ndt_direct_probe(tv, r, q0, q1, q2);
          if (sl >= 0) {
            const int pos = atomicAdd(&shit_n[pt], 1);
            shit_slot[pt][pos] = sl; shit_key[pt][pos] = (float)r;        // visited in the order of the relative cells
          }
        }
      }
    }
    __syncwarp(gmask);
    const int k = min(shit_n[pt], NDT_MAX_NB);
    // 2. the reference's visiting order: ascending (distance, slot)
    for (int h = sub; h < k; h += NDT_GRP) {
      const float kh = shit_key[pt][h];
      const int sh = shit_slot[pt][h];
      int rank = 0;
      for (int o = 0; o < k; o++) {
        const float ko = shit_key[pt][o];
        rank += (ko < kh || (ko == kh && shit_slot[pt][o] < sh)) ? 1 : 0;
      }
      ssorted[pt][rank] = sh;
    }
    __syncwarp(gmask);
    // 3. one pair per lane, its terms through shared memory, the owners add them in order
    double acc[NC];
#pragma unroll
    for (int ci = 0; ci < NC; ci++) acc[ci] = 0.0;
    if (k > 0) {
      // the point's derivative rows: lane s computes row s of the gradient table (and rows s, s + 8 of the Hessian table)
      sxj[pt][sub] = ndt_row_dot(sA.jf, sub, x0, x1, x2);
      if (HESS) {
        sxh[pt][sub] = ndt_row_dot(sA.hf, sub, x0, x1, x2);
        if (sub + 8 < 15) sxh[pt][sub + 8] = ndt_row_dot(sA.hf, sub + 8, x0, x1, x2);
      }
      __syncwarp(gmask);
      float pg[3][6], ph[6][3];
      ndt_point_derivs_place(sxj[pt], sxh[pt], HESS, pg, ph);
      for (int base = 0; base < k; base += NDT_GRP) {
        const int j = base + sub;
        if (j < k) {
          float t[NT];
          const bool ok = ndt_pair_terms_f<HESS>(G, pg, ph, q0, q1, q2, tv.vox[ssorted[pt][j]], t);
#pragma unroll
          for (int e = 0; e < NT; e++) sterm[pt][sub][e] = ok ? t[e] : 0.0f;      // a dropped pair adds nothing
        }
        __syncwarp(gmask);
        const int m = min(NDT_GRP, k - base);
        for (int jj = 0; jj < m; jj++) {
#pragma unroll
          for (int ci = 0; ci < NC; ci++) {
            const int c = sub + NDT_GRP * ci;
            if (c < NT) acc[ci] += (double)sterm[pt][jj][c];
          }
        }
        __syncwarp(gmask);
      }
    }
#pragma unroll
    for (int ci = 0; ci < NC; ci++) total[ci] += acc[ci];
  }
  // 4. one partial row per CTA: the points' subtotals in point order
#pragma unroll
  for (int ci = 0; ci < NC; ci++) {
    const int c = sub + NDT_GRP * ci;
    if (c < NT) sacc[pt][c] = total[ci];
  }
  __syncthreads();
  if (threadIdx.x < NDT_NSUM) {
    const int c = threadIdx.x;
    double v = 0.0;
    if (c < NT) {
#pragma unroll
      for (int p = 0; p < NDT_GPTS; p++) v += sacc[p][c];
    }
    partials[(size_t)blockIdx.x * NDT_NSUM + c] = v;
  }
}

struct NdtRows { int thread, group; bool use_group; };        // partial rows (= CTAs) of the two kernel shapes
static inline int ndt_rows_of(const NdtRows& r, int want) { return (r.use_group && want != NDT_WANT_HESSIAN) ? r.group : r.thread; }

static void ndt_launch_eval(int want, const NdtRows& rows, cudaStream_t st, const NdtCtl* ctl, const NdtTargetView& tv, const NdtGauss& G,
                            const f4* src, uint32_t n, double* partials) {
  if (rows.use_group && want == NDT_WANT_DERIV_H)
    ndt_eval_group_kernel<NDT_WANT_DERIV_H><<<rows.group, NDT_EVAL_THREADS, 0, st>>>(ctl, tv, G, src, n, partials);
  else if (rows.use_group && want == NDT_WANT_DERIV)
    ndt_eval_group_kernel<NDT_WANT_DERIV><<<rows.group, NDT_EVAL_THREADS, 0, st>>>(ctl, tv, G, src, n, partials);
  else if (want == NDT_WANT_DERIV_H) ndt_eval_kernel<NDT_WANT_DERIV_H><<<rows.thread, NDT_EVAL_THREADS, 0, st>>>(ctl, tv, G, src, n, partials);
  else if (want == NDT_WANT_DERIV) ndt_eval_kernel<NDT_WANT_DERIV><<<rows.thread, NDT_EVAL_THREADS, 0, st>>>(ctl, tv, G, src, n, partials);
  else ndt_eval_kernel<NDT_WANT_HESSIAN><<<rows.thread, NDT_EVAL_THREADS, 0, st>>>(ctl, tv, G, src, n, partials);
}

// Adds the CTA partials (fixed shape: sixteen consecutive ranges of CTAs summed in CTA order, then the sixteen range sums
// in order -- run-to-run identical bits) and advances the controller.
constexpr int NDT_CTL_PARTS = 16;
constexpr int NDT_CTL_THREADS = 704;                       // >= NDT_NSUM * NDT_CTL_PARTS
__device__ __forceinline__ void ndt_sum_partials(const double* __restrict__ partials, int blocks, double (*part)[NDT_NSUM], double* sums) {
  const int t = threadIdx.x;
  if (t < NDT_NSUM * NDT_CTL_PARTS) {
    const int k = t % NDT_NSUM, r = t / NDT_NSUM;
    const int per = (blocks + NDT_CTL_PARTS - 1) / NDT_CTL_PARTS;
    const int b0 = r * per, b1 = min(blocks, b0 + per);
    double v = 0.0;
#pragma unroll 8
    for (int b = b0; b < b1; b++) v += partials[(size_t)b * NDT_NSUM + k];
    part[r][k] = v;
  }
  __syncthreads();
  if (t < NDT_NSUM) {
    double v = 0.0;
#pragma unroll
    for (int r = 0; r < NDT_CTL_PARTS; r++) v += part[r][t];
    sums[t] = v;
  }
  __syncthreads();
}

// The Newton solve of the controller on one warp: x = pinv(A) (-g).  The three disjoint column pairs of a round (ndt.h,
// ndt_svd6_pair) are rotated side by side, lane (grp, k) = (lane >> 3, lane & 7) holding row k of pair grp; the column
// norms / dot product of a pair are added in row order (as the serial loop does), so the bits equal ndt_svd6_solve's.
// The serial solve is a chain of dependent double-precision divisions and square roots per Newton step.
__device__ __forceinline__ void ndt_svd6_solve_warp(const double* A, const double* g, double (*U)[6], double (*V)[6], double* x) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  for (int e = lane; e < 36; e += 32) { U[e / 6][e % 6] = A[e]; V[e / 6][e % 6] = (e / 6 == e % 6) ? 1.0 : 0.0; }
  __syncwarp();
  const int grp = lane >> 3, k = lane & 7;
  const bool active = grp < 3 && k < 6;
  for (int sweep = 0; sweep < 60; sweep++) {
    bool any = false;
    for (int r = 0; r < 5; r++) {
      int p = 0, q = 1;
      if (grp < 3) ndt_svd6_pair(3 * r + grp, p, q);
      const double up = active ? U[k][p] : 0.0, uq = active ? U[k][q] : 0.0;
      const double vp = active ? V[k][p] : 0.0, vq = active ? V[k][q] : 0.0;
      const double a = up * up, bb = uq * uq, gm = up * uq;
      double alpha = 0, beta = 0, gamma = 0;
#pragma unroll
      for (int kk = 0; kk < 6; kk++) {
        const int from = grp * 8 + kk;
        alpha += __shfl_sync(FULL, a, from); beta += __shfl_sync(FULL, bb, from); gamma += __shfl_sync(FULL, gm, from);
      }
      double c = 1.0, s = 0.0;
      const bool rot = ndt_svd6_angle(alpha, beta, gamma, c, s) && active;
      if (rot) {
        U[k][p] = c * up - s * uq; U[k][q] = s * up + c * uq;
        V[k][p] = c * vp - s * vq; V[k][q] = s * vp + c * vq;
      }
      any = __any_sync(FULL, rot) || any;
      __syncwarp();
    }
    if (!any) break;
  }
  if (lane == 0) {
    double ng[6];
    for (int i = 0; i < 6; i++) ng[i] = -g[i];
    ndt_svd6_finish(U, V, ng, x);
  }
  __syncwarp();
}

__global__ void __launch_bounds__(NDT_CTL_THREADS)
ndt_ctl_kernel(NdtCtl* __restrict__ ctl, const double* __restrict__ partials, int rows_float, int rows_hessian) {
  __shared__ double part[NDT_CTL_PARTS][NDT_NSUM];
  __shared__ double sums[NDT_NSUM];
  __shared__ double sU[6][6], sV[6][6], sx[6];
  __shared__ NdtCtl sc;                // the controller works on a shared-memory copy: its scalar code is a chain of dependent
                                       // loads and stores of this state, 30 cycles each here, an L2 round trip each in global memory
  const int want = ctl->want;
  if (want == NDT_WANT_NONE) return;
  {
    const uint32_t* g = reinterpret_cast<const uint32_t*>(ctl);
    uint32_t* w = reinterpret_cast<uint32_t*>(&sc);
    for (uint32_t i = threadIdx.x; i < sizeof(NdtCtl) / 4; i += blockDim.x) w[i] = g[i];
  }
  ndt_sum_partials(partials, want == NDT_WANT_HESSIAN ? rows_hessian : rows_float, part, sums);     // the rows the request's kernel wrote; syncs the CTA
  if (threadIdx.x < 32) {
    // lane 0 runs the scalar controller; whenever it needs a Newton direction the whole warp computes it
    int need = 0;
    if (threadIdx.x == 0) need = ndt_ctl_run(sc, sums, nullptr) ? 1 : 0;
    need = __shfl_sync(0xffffffffu, need, 0);
    while (need) {
      __syncwarp();                                       // lane 0's writes of sc.H / sc.g are visible to the warp
      ndt_svd6_solve_warp(sc.H, sc.g, sU, sV, sx);
      if (threadIdx.x == 0) need = ndt_ctl_run(sc, sums, sx) ? 1 : 0;
      need = __shfl_sync(0xffffffffu, need, 0);
    }
    __syncwarp();
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&sc);
    uint32_t* g = reinterpret_cast<uint32_t*>(ctl);
    for (uint32_t i = threadIdx.x; i < sizeof(NdtCtl) / 4; i += 32) g[i] = w[i];
  }
}

// lb_ndt_derivatives: one evaluation at a caller-given pose, sums to out[43]
__global__ void __launch_bounds__(NDT_CTL_THREADS)
ndt_sum_kernel(const double* __restrict__ partials, int blocks, double* __restrict__ out) {
  __shared__ double part[NDT_CTL_PARTS][NDT_NSUM];
  __shared__ double sums[NDT_NSUM];
  ndt_sum_partials(partials, blocks, part, sums);
  if (threadIdx.x < NDT_NSUM) out[threadIdx.x] = sums[threadIdx.x];
}

}  // namespace lb

using namespace lb;

struct lb_ndt {
  Ctx c;
  lb_ndt_params P;
  NdtGauss G;
  // source
  DBuf<f4> src, src_spare;
  uint32_t n_src = 0;
  // target
  DBuf<f4> tgt, tgt_spare;
  uint32_t n_tgt = 0;
  float tgt_mn[3] = {0, 0, 0}, tgt_mx[3] = {0, 0, 0};
  bool tgt_dirty = false;               // the voxel structure has to be (re)built from tgt
  bool have_tgt = false;
  const lb_submap* tgt_map = nullptr;   // lb_ndt_set_target_submap: the map tgt was gathered from, at this generation
  uint64_t tgt_map_gen = 0;
  cudaEvent_t map_ready = nullptr;      // the map's stream -> this handle's stream
  DBuf<uint32_t> keys, flag, slot_of, head_pos;
  SortWork sort;
  ScanWork scan;
  DBuf<NdtVoxel> vox;
  DBuf<f4> cen;
  DBuf<int32_t> leaf_idx, hval;
  DBuf<uint32_t> hkey;
  NdtTargetView tv;
  NdtLattice L;
  // evaluation
  DBuf<uint8_t> io;
  DBuf<double> partials;
  NdtCtl* d_ctl = nullptr;
  NdtCtl* h_ctl = nullptr;              // pinned
  double* d_sums = nullptr;
  double* h_sums = nullptr;             // pinned
  BBoxAcc* d_acc = nullptr;
  BBoxAcc* h_acc = nullptr;             // pinned
  uint32_t* d_u32 = nullptr;
  uint32_t* h_u32 = nullptr;            // pinned
};

extern "C" {

void lb_ndt_default_params(lb_ndt_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->resolution = 1.0f;                  // ndt_omp_impl.hpp:50
  p->step_size = 0.1;                    // :51
  p->outlier_ratio = 0.55;               // :52
  p->transformation_epsilon = 0.1;       // :93
  p->max_iterations = 35;                // :94
  p->min_points_per_voxel = 6;           // voxel_grid_covariance_omp.h:186
  p->min_covar_eigvalue_mult = 0.01;     // :187
  p->search_method = NDT_KDTREE;         // ndt_omp_impl.hpp:96
  p->max_correspondence_distance = 0.0;
  p->ransac_iterations = 0;
  p->num_threads = 0;
  p->enable_timing_output = 0;
}

static int ndt_create_impl(int device, void* stream, bool ext, lb_ndt** out) {
  if (!out) { set_error("lb_ndt_create: null handle pointer"); return LB_ERR_INVALID_ARG; }
  lb_ndt* h = new (std::nothrow) lb_ndt;
  if (!h) { set_error("lb_ndt_create: out of memory"); return LB_ERR_CUDA; }
  int s = ctx_init(h->c, device, stream, ext);
  if (s != LB_OK) { delete h; return s; }
  lb_ndt_default_params(&h->P);
  ndt_gauss_constants(h->P.outlier_ratio, h->P.resolution, h->G);
  memset(&h->tv, 0, sizeof(h->tv));
  bool ok = cudaMalloc((void**)&h->d_ctl, sizeof(NdtCtl)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_ctl, sizeof(NdtCtl)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_sums, NDT_NSUM * sizeof(double)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_sums, NDT_NSUM * sizeof(double)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_acc, sizeof(BBoxAcc)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_acc, sizeof(BBoxAcc)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_u32, 8 * sizeof(uint32_t)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_u32, 8 * sizeof(uint32_t)) == cudaSuccess;
  if (!ok) {
    set_error("lb_ndt_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    lb_ndt_destroy(h);
    return LB_ERR_CUDA;
  }
  *out = h;
  return LB_OK;
}

int lb_ndt_create(int device, lb_ndt** h) { return ndt_create_impl(device, nullptr, false, h); }
int lb_ndt_create_on_stream(int device, void* stream, lb_ndt** h) { return ndt_create_impl(device, stream, true, h); }

int lb_ndt_destroy(lb_ndt* h) {
  if (!h) return LB_OK;
  cudaSetDevice(h->c.device);
  if (h->c.stream) cudaStreamSynchronize(h->c.stream);
  h->src.release(); h->src_spare.release(); h->tgt.release(); h->tgt_spare.release();
  h->keys.release(); h->flag.release(); h->slot_of.release(); h->head_pos.release();
  h->sort.ka.release(); h->sort.kb.release(); h->sort.va.release(); h->sort.vb.release(); h->sort.state.release();
  h->scan.sums.release();
  h->vox.release(); h->cen.release(); h->leaf_idx.release(); h->hval.release(); h->hkey.release();
  h->io.release(); h->partials.release();
  if (h->d_ctl) cudaFree(h->d_ctl);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  if (h->d_sums) cudaFree(h->d_sums);
  if (h->h_sums) cudaFreeHost(h->h_sums);
  if (h->d_acc) cudaFree(h->d_acc);
  if (h->h_acc) cudaFreeHost(h->h_acc);
  if (h->d_u32) cudaFree(h->d_u32);
  if (h->h_u32) cudaFreeHost(h->h_u32);
  if (h->map_ready) cudaEventDestroy(h->map_ready);
  ctx_destroy(h->c);
  delete h;
  return LB_OK;
}

}  // extern "C"

namespace lb {
// lb_ndt_set_params' refusals, shared with the pipelines that take NDT params (odometry.cu)
int ndt_check_params(const lb_ndt_params* p, const char* who) {
  if (!(p->resolution > 0) || !(p->step_size > 0) || !(p->outlier_ratio > 0) || !(p->outlier_ratio < 1) ||
      !(p->transformation_epsilon > 0) || p->max_iterations < 0 || p->min_points_per_voxel < 3 || !(p->min_covar_eigvalue_mult > 0)) {
    // setMinPointVoxel refuses fewer than 3 points (voxel_grid_covariance_omp.h:203-214)
    set_error("%s: resolution / step / outlier ratio / epsilon must be positive, min_points_per_voxel >= 3", who);
    return LB_ERR_INVALID_ARG;
  }
  if (p->search_method < NDT_KDTREE || p->search_method > NDT_DIRECT1) {
    set_error("%s: search_method must be 0 (KDTREE), 1 (DIRECT26), 2 (DIRECT7) or 3 (DIRECT1)", who);
    return LB_ERR_UNSUPPORTED;
  }
  return LB_OK;
}
}  // namespace lb

extern "C" {

int lb_ndt_set_params(lb_ndt* h, const lb_ndt_params* p) {
  if (!h || !p) { set_error("lb_ndt_set_params: null argument"); return LB_ERR_INVALID_ARG; }
  LB_TRY(ndt_check_params(p, "lb_ndt_set_params"));
  // setResolution re-initialises the voxel structure of the current target (ndt_omp.h:124-131); the same holds for the
  // two voxel parameters
  if (p->resolution != h->P.resolution || p->min_points_per_voxel != h->P.min_points_per_voxel ||
      p->min_covar_eigvalue_mult != h->P.min_covar_eigvalue_mult)
    h->tgt_dirty = h->n_tgt > 0;
  h->P = *p;
  ndt_gauss_constants(h->P.outlier_ratio, h->P.resolution, h->G);
  return LB_OK;
}

// caller cloud -> packed float4 in `dst` (+ bounding box and count of the finite points in h->h_acc); synchronous
static int ndt_upload(lb_ndt* h, DBuf<f4>& dst, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem, const char* who) {
  if (!pts || stride < 12 || xyz_off + 12 > stride || (stride & 3) || (xyz_off & 3) || n > 0x7fffffffull) {
    set_error("%s: bad cloud description (n %zu, stride %zu, xyz offset %zu)", who, n, stride, xyz_off);
    return LB_ERR_INVALID_ARG;
  }
  LB_CUDA(cudaSetDevice(h->c.device));
  const uint8_t* dev = (const uint8_t*)pts;
  if (mem == LB_MEM_HOST) {
    LB_TRY(h->io.ensure(n * stride));
    LB_CUDA(cudaMemcpyAsync(h->io.p, pts, n * stride, cudaMemcpyHostToDevice, h->c.stream));
    dev = h->io.p;
  } else if (mem != LB_MEM_DEVICE) {
    set_error("%s: mem must be LB_MEM_HOST or LB_MEM_DEVICE", who);
    return LB_ERR_INVALID_ARG;
  }
  LB_TRY(dst.ensure(n));
  bbox_init_kernel<<<1, 32, 0, h->c.stream>>>(h->d_acc);
  ndt_gather_kernel<<<cdiv((long long)n, 256), 256, 0, h->c.stream>>>(dev, (uint32_t)n, (uint32_t)stride, (uint32_t)xyz_off, dst.p, h->d_acc);
  h->c.launches += 2;
  LB_CUDA(cudaMemcpyAsync(h->h_acc, h->d_acc, sizeof(BBoxAcc), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaStreamSynchronize(h->c.stream));
  return LB_OK;
}

int lb_ndt_set_source(lb_ndt* h, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem) {
  if (!h) { set_error("lb_ndt_set_source: null handle"); return LB_ERR_INVALID_ARG; }
  if (n == 0) { set_error("lb_ndt_set_source: invalid or empty point cloud dataset given"); return LB_ERR_EMPTY_SOURCE; }
  LB_TRY(ndt_upload(h, h->src_spare, pts, n, stride, xyz_off, mem, "lb_ndt_set_source"));
  if (h->h_acc->count != (uint32_t)n) {
    set_error("lb_ndt_set_source: %zu of %zu points are not finite; the previous source is kept", n - h->h_acc->count, n);
    return LB_ERR_INVALID_ARG;
  }
  std::swap(h->src, h->src_spare);
  h->n_src = (uint32_t)n;
  return LB_OK;
}

// lb_ndt_set_target and lb_ndt_set_target_submap: upload into the spare buffer, then swap (any refusal keeps the target)
static int ndt_take_target(lb_ndt* h, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem, const char* who) {
  LB_TRY(ndt_upload(h, h->tgt_spare, pts, n, stride, xyz_off, mem, who));
  if (h->h_acc->count == 0) { set_error("%s: no finite point; the previous target is kept", who); return LB_ERR_NO_TARGET; }
  // lattice check before the swap: a grid the reference would refuse leaves the previous target in place
  float mn[3], mx[3];
  for (int a = 0; a < 3; a++) { mn[a] = ord2f(h->h_acc->mn[a]); mx[a] = ord2f(h->h_acc->mx[a]); }
  NdtLattice L;
  if (!ndt_lattice(mn, mx, h->P.resolution, L)) {
    set_error("%s: leaf size is too small for the input dataset, integer indices would overflow", who);
    return LB_ERR_VOXEL_OVERFLOW;
  }
  std::swap(h->tgt, h->tgt_spare);
  for (int a = 0; a < 3; a++) { h->tgt_mn[a] = mn[a]; h->tgt_mx[a] = mx[a]; }
  h->n_tgt = (uint32_t)n;
  h->tgt_dirty = true;
  h->have_tgt = false;
  h->tgt_map = nullptr;
  return LB_OK;
}

int lb_ndt_set_target(lb_ndt* h, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem) {
  if (!h) { set_error("lb_ndt_set_target: null handle"); return LB_ERR_INVALID_ARG; }
  if (n == 0) { set_error("lb_ndt_set_target: empty target cloud"); return LB_ERR_NO_TARGET; }
  return ndt_take_target(h, pts, n, stride, xyz_off, mem, "lb_ndt_set_target");
}

int lb_ndt_set_target_submap(lb_ndt* h, lb_submap* m) {
  if (!h || !m) { set_error("lb_ndt_set_target_submap: null argument"); return LB_ERR_INVALID_ARG; }
  if (submap_device(m) != h->c.device) {
    set_error("lb_ndt_set_target_submap: submap on device %d, handle on %d", submap_device(m), h->c.device);
    return LB_ERR_INVALID_ARG;
  }
  const f4* pts = nullptr;
  size_t n = 0;
  uint64_t gen = 0;
  cudaStream_t map_stream = nullptr;
  submap_points_view(m, &pts, &n, &gen, &map_stream);
  if (h->tgt_map == m && h->tgt_map_gen == gen) return LB_OK;      // unchanged map: the target (and its Gaussians) stand
  if (n == 0) { set_error("lb_ndt_set_target_submap: the map is empty"); return LB_ERR_NO_TARGET; }
  LB_CUDA(cudaSetDevice(h->c.device));
  // The gather reads the map's buffer on this handle's stream: an event recorded on the map's stream orders it after
  // whatever map work is still pending there (the map calls synchronise before they return today; the event keeps
  // that an implementation detail of the map).
  if (!h->map_ready) LB_CUDA(cudaEventCreateWithFlags(&h->map_ready, cudaEventDisableTiming));
  LB_CUDA(cudaEventRecord(h->map_ready, map_stream));
  LB_CUDA(cudaStreamWaitEvent(h->c.stream, h->map_ready, 0));
  LB_TRY(ndt_take_target(h, pts, n, sizeof(f4), 0, LB_MEM_DEVICE, "lb_ndt_set_target_submap"));
  h->tgt_map = m;
  h->tgt_map_gen = gen;
  return LB_OK;
}

// VoxelGridCovariance::filter(true) on the stored target
static int ndt_build_target(lb_ndt* h) {
  Ctx& c = h->c;
  const uint32_t n = h->n_tgt;
  const float* mn = h->tgt_mn;
  const float* mx = h->tgt_mx;      // bounding box of the finite points, kept from the upload (a resolution change rebuilds from it)
  if (!ndt_lattice(mn, mx, h->P.resolution, h->L)) {
    set_error("NDT target: leaf size is too small for the input dataset, integer indices would overflow");
    return LB_ERR_VOXEL_OVERFLOW;
  }
  const NdtLattice& L = h->L;
  const uint64_t cells = (uint64_t)L.div_b[0] * L.div_b[1] * L.div_b[2];
  const uint32_t invalid_key = (uint32_t)cells;                  // one past the last voxel: non-finite points sort to the end
  int key_bits = 1;
  while ((1ull << key_bits) <= cells) key_bits++;
  LB_TRY(h->keys.ensure(n)); LB_TRY(h->flag.ensure(n)); LB_TRY(h->slot_of.ensure(n));
  ndt_keys_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(h->tgt.p, n, L, invalid_key, h->keys.p);
  c.launches++;
  uint32_t *ks = nullptr, *vs = nullptr;
  LB_TRY(radix_sort_pairs(c, h->sort, h->keys.p, nullptr, n, key_bits, &ks, &vs));
  ndt_heads_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(ks, n, invalid_key, h->P.min_points_per_voxel, h->flag.p);
  c.launches++;
  LB_TRY(exclusive_scan_u32(c, h->scan, h->flag.p, h->slot_of.p, n, h->d_u32));
  LB_CUDA(cudaMemcpyAsync(h->h_u32, h->d_u32, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const uint32_t nv = h->h_u32[0];
  uint32_t cap = 16;
  while (cap < 2u * nv) cap <<= 1;
  LB_TRY(h->vox.ensure(nv + 1)); LB_TRY(h->cen.ensure(nv + 1)); LB_TRY(h->leaf_idx.ensure(nv + 1)); LB_TRY(h->head_pos.ensure(nv + 1));
  LB_TRY(h->hkey.ensure(cap)); LB_TRY(h->hval.ensure(cap));
  LB_CUDA(cudaMemsetAsync(h->hkey.p, 0xff, (size_t)cap * sizeof(uint32_t), c.stream));
  if (nv > 0) {
    ndt_head_pos_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(h->flag.p, h->slot_of.p, n, h->head_pos.p);
    ndt_gaussians_kernel<<<cdiv((long long)nv * 32, 128), 128, 0, c.stream>>>(ks, vs, n, h->head_pos.p, nv, h->tgt.p, h->P.min_covar_eigvalue_mult,
                                                                              h->vox.p, h->cen.p, h->leaf_idx.p);
    ndt_hash_insert_kernel<<<cdiv(nv, 256), 256, 0, c.stream>>>(h->leaf_idx.p, nv, h->hkey.p, h->hval.p, cap - 1);
    c.launches += 3;
  }
  LB_CUDA(cudaGetLastError());
  NdtTargetView& tv = h->tv;
  tv.vox = h->vox.p; tv.cen = h->cen.p; tv.hkey = h->hkey.p; tv.hval = h->hval.p; tv.hmask = cap - 1;
  tv.n_valid = (int)nv;
  for (int a = 0; a < 3; a++) { tv.min_b[a] = L.min_b[a]; tv.max_b[a] = L.max_b[a]; tv.div_b[a] = L.div_b[a]; }
  tv.leaf = h->P.resolution; tv.inv_leaf = L.inv_leaf;
  const double radius = (double)h->P.resolution;
  tv.r2 = (float)(radius * radius);
  h->tgt_dirty = false;
  h->have_tgt = true;
  return LB_OK;
}

static int ndt_ready(lb_ndt* h, const char* who) {
  if (!h) { set_error("%s: null handle", who); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  if (h->n_tgt == 0) { set_error("%s: no target set", who); return LB_ERR_NO_TARGET; }
  if (h->tgt_map) {
    const f4* pts = nullptr;
    size_t n = 0;
    uint64_t gen = 0;
    cudaStream_t st = nullptr;
    submap_points_view(h->tgt_map, &pts, &n, &gen, &st);
    if (gen != h->tgt_map_gen) {
      set_error("%s: the map changed since lb_ndt_set_target_submap; call it again", who);
      return LB_ERR_INVALID_ARG;
    }
  }
  if (h->tgt_dirty || !h->have_tgt) LB_TRY(ndt_build_target(h));
  h->tv.method = h->P.search_method;
  h->tv.min_pts = h->P.min_points_per_voxel;
  return LB_OK;
}

int lb_ndt_target_voxels(lb_ndt* h, size_t capacity, size_t* n_voxels, int32_t* leaf_idx, int32_t* nr_points, double* mean3,
                         double* icov9, float* centroid3) {
  LB_TRY(ndt_ready(h, "lb_ndt_target_voxels"));
  const size_t nv = (size_t)h->tv.n_valid;
  if (n_voxels) *n_voxels = nv;
  if (!leaf_idx && !nr_points && !mean3 && !icov9 && !centroid3) return LB_OK;
  if (capacity < nv) { set_error("lb_ndt_target_voxels: capacity %zu < %zu voxels", capacity, nv); return LB_ERR_CAPACITY; }
  std::vector<NdtVoxel> v(nv);
  std::vector<f4> c(nv);
  LB_CUDA(cudaMemcpyAsync(v.data(), h->vox.p, nv * sizeof(NdtVoxel), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaMemcpyAsync(c.data(), h->cen.p, nv * sizeof(f4), cudaMemcpyDeviceToHost, h->c.stream));
  if (leaf_idx) LB_CUDA(cudaMemcpyAsync(leaf_idx, h->leaf_idx.p, nv * sizeof(int32_t), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaStreamSynchronize(h->c.stream));
  for (size_t i = 0; i < nv; i++) {
    if (nr_points) nr_points[i] = float_to_bits(c[i].w);
    if (mean3) memcpy(mean3 + 3 * i, v[i].mean, 3 * sizeof(double));
    if (icov9) memcpy(icov9 + 9 * i, v[i].icov, 9 * sizeof(double));
    if (centroid3) { centroid3[3 * i] = c[i].x; centroid3[3 * i + 1] = c[i].y; centroid3[3 * i + 2] = c[i].z; }
  }
  return LB_OK;
}

static int ndt_source_ready(lb_ndt* h, const char* who, NdtRows* rows) {
  if (h->n_src == 0) { set_error("%s: no source set", who); return LB_ERR_EMPTY_SOURCE; }
  // LB_NDT_EVAL=thread: every pass with one thread per source point (A/B baseline); default: eight lanes per point for the float passes
  static const bool use_group = !(getenv("LB_NDT_EVAL") && !strcmp(getenv("LB_NDT_EVAL"), "thread"));
  rows->thread = cdiv(h->n_src, NDT_EVAL_THREADS);
  rows->group = cdiv(h->n_src, NDT_GPTS * NDT_GBATCH);
  rows->use_group = use_group;
  LB_TRY(h->partials.ensure((size_t)std::max(rows->thread, rows->group) * NDT_NSUM));
  return LB_OK;
}

int lb_ndt_derivatives(lb_ndt* h, const float* T16, const double* pose6, int compute_hessian, double* score, double* gradient6,
                       double* hessian36) {
  LB_TRY(ndt_ready(h, "lb_ndt_derivatives"));
  if (!T16 || !pose6 || compute_hessian < 0 || compute_hessian > 2) { set_error("lb_ndt_derivatives: bad argument"); return LB_ERR_INVALID_ARG; }
  NdtRows rows;
  LB_TRY(ndt_source_ready(h, "lb_ndt_derivatives", &rows));
  NdtCtl& c = *h->h_ctl;
  memset(&c, 0, sizeof(c));
  for (int i = 0; i < 12; i++) c.T[i] = T16[i];
  ndt_angles(pose6, c.ang);
  c.want = compute_hessian == 2 ? NDT_WANT_HESSIAN : (compute_hessian ? NDT_WANT_DERIV_H : NDT_WANT_DERIV);
  LB_CUDA(cudaMemcpyAsync(h->d_ctl, h->h_ctl, sizeof(NdtCtl), cudaMemcpyHostToDevice, h->c.stream));
  ndt_launch_eval(c.want, rows, h->c.stream, h->d_ctl, h->tv, h->G, h->src.p, h->n_src, h->partials.p);
  ndt_sum_kernel<<<1, NDT_CTL_THREADS, 0, h->c.stream>>>(h->partials.p, ndt_rows_of(rows, c.want), h->d_sums);
  h->c.launches += 2;
  LB_CUDA(cudaMemcpyAsync(h->h_sums, h->d_sums, NDT_NSUM * sizeof(double), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaStreamSynchronize(h->c.stream));
  if (score) *score = h->h_sums[0];
  if (gradient6) memcpy(gradient6, h->h_sums + 1, 6 * sizeof(double));
  if (hessian36) memcpy(hessian36, h->h_sums + 7, 36 * sizeof(double));
  return LB_OK;
}

int lb_ndt_align(lb_ndt* h, const float* guess16, lb_ndt_result* result) {
  LB_TRY(ndt_ready(h, "lb_ndt_align"));
  if (!result) { set_error("lb_ndt_align: null result"); return LB_ERR_INVALID_ARG; }
  NdtRows rows;
  LB_TRY(ndt_source_ready(h, "lb_ndt_align", &rows));
  const auto t0 = std::chrono::steady_clock::now();
  static const float I16[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  const float* g = guess16 ? guess16 : I16;
  for (int i = 0; i < 12; i++) if (!isfinite(g[i])) { set_error("lb_ndt_align: the guess is not finite"); return LB_ERR_INVALID_ARG; }
  NdtCtl& c = *h->h_ctl;
  ndt_ctl_begin(c, g, h->P.step_size, h->P.transformation_epsilon, h->P.max_iterations);
  LB_CUDA(cudaMemcpyAsync(h->d_ctl, h->h_ctl, sizeof(NdtCtl), cudaMemcpyHostToDevice, h->c.stream));
  // an align needs at most (max_iterations + 2) Newton steps of 1 + 10 + 1 evaluations each
  const long max_pairs = 1 + (long)(h->P.max_iterations + 3) * 12;
  long pairs = 0;
  for (;;) {
    for (int b = 0; b < NDT_BATCH; b++) {
      for (int want = NDT_WANT_DERIV_H; want <= NDT_WANT_HESSIAN; want++)
        ndt_launch_eval(want, rows, h->c.stream, h->d_ctl, h->tv, h->G, h->src.p, h->n_src, h->partials.p);
      ndt_ctl_kernel<<<1, NDT_CTL_THREADS, 0, h->c.stream>>>(h->d_ctl, h->partials.p, ndt_rows_of(rows, NDT_WANT_DERIV), ndt_rows_of(rows, NDT_WANT_HESSIAN));
    }
    h->c.launches += 4 * NDT_BATCH;
    pairs += NDT_BATCH;
    LB_CUDA(cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(NdtCtl), cudaMemcpyDeviceToHost, h->c.stream));
    LB_CUDA(cudaStreamSynchronize(h->c.stream));
    if (c.want == NDT_WANT_NONE) break;
    if (pairs > max_pairs) { set_error("lb_ndt_align: the controller did not finish within %ld evaluations", pairs); return LB_ERR_CUDA; }
  }
  memset(result, 0, sizeof(*result));
  for (int i = 0; i < 12; i++) result->final_transformation[i] = c.final_T[i];
  result->final_transformation[15] = 1.0f;
  result->converged = c.converged;
  result->nr_iterations = c.nr_iterations;
  result->n_evaluations = c.n_evals;
  result->trans_probability = c.score / (double)h->n_src;          // ndt_omp_impl.hpp:207
  for (int i = 0; i < 6; i++) result->pose[i] = c.p[i];
  result->n_target_voxels = h->tv.n_valid;
  result->t_total_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return LB_OK;
}

int lb_ndt_launch_count(lb_ndt* h, uint64_t* n) {
  if (!h || !n) { set_error("lb_ndt_launch_count: null argument"); return LB_ERR_INVALID_ARG; }
  *n = h->c.launches;
  return LB_OK;
}

}  // extern "C"

namespace lb {

// Pre-sizes every buffer an NDT registration of clouds of up to max_points device-resident points touches (source,
// target, voxel build, sort, scan, evaluation partials), so that lb_odometry's workers make no device allocation in
// steady state.  The host upload staging is not reserved: the pipelines hand device clouds only.
int ndt_reserve(lb_ndt* h, size_t max_points) {
  if (!h || max_points == 0 || max_points > 0x7fffffffull) { set_error("ndt_reserve: bad argument"); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  const size_t n = max_points;
  LB_TRY(h->src.ensure(n)); LB_TRY(h->src_spare.ensure(n)); LB_TRY(h->tgt.ensure(n)); LB_TRY(h->tgt_spare.ensure(n));
  LB_TRY(h->keys.ensure(n)); LB_TRY(h->flag.ensure(n)); LB_TRY(h->slot_of.ensure(n));
  LB_TRY(radix_sort_reserve(h->c, h->sort, n));
  LB_TRY(h->scan.sums.ensure(std::max<size_t>((n + 2047) / 2048, 16384)));    // exclusive_scan_u32's spine
  LB_TRY(h->vox.ensure(n + 1)); LB_TRY(h->cen.ensure(n + 1)); LB_TRY(h->leaf_idx.ensure(n + 1)); LB_TRY(h->head_pos.ensure(n + 1));
  uint32_t cap = 16;
  while (cap < 2u * (uint32_t)n) cap <<= 1;                           // ndt_build_target's table for n searchable voxels
  LB_TRY(h->hkey.ensure(cap)); LB_TRY(h->hval.ensure(cap));
  const size_t rows = std::max(cdiv((long long)n, NDT_EVAL_THREADS), cdiv((long long)n, NDT_GPTS * NDT_GBATCH));
  LB_TRY(h->partials.ensure(rows * NDT_NSUM));
  LB_CUDA(cudaStreamSynchronize(h->c.stream));
  return LB_OK;
}

}  // namespace lb
