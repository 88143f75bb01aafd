// voxel.cu -- VoxelGrid front-end (kernel K1): hash-and-centroid reduce.
//
// Replaces pcl::VoxelGrid<pcl::PCLPointCloud2>::applyFilter as driven by
// point_cloud_filter/src/custom_voxel_grid.cc:76-87 (index arithmetic cross-
// checked with multithreaded_ndt/voxel_grid_covariance_omp_impl.hpp:67-164).
//
// One call = one stream-ordered chain of kernels with NO host round trip in between: everything a later kernel needs
// from an earlier one (bounding box -> min_b / div_b / key width, voxel count) stays in a small device-resident state
// block; the host synchronises once, at the end, to learn the voxel count and the status.  3 + (sort passes) kernels:
//   vg_bbox_kernel     finite + filter-limit + body-box predicate, min/max reduce (two 16-byte loads per 32-byte
//                      record); the last CTA derives min_b, div_b, the overflow guard and the key width
//   vg_keys_kernel     int32 PCL leaf index per point (bit-exact float32 math) + a packed float4 record of the four
//                      averaged fields, so that no later kernel touches the raw cloud's strided layout again; also
//                      every sort pass's digit histogram, and the reset of the look-back state of the kernels after it
//   radix sort         one scatter kernel per pass of the stable LSD sort of (leaf index, point#); passes beyond the
//                      key width return at once
//   vg_segment_kernel  tiles of sorted positions: voxel heads, min_points_per_voxel, output slots by decoupled
//                      look-back, and one lane per voxel summing it in float32 in ascending point order, / count; the
//                      last tile writes the call's state into pinned host memory (no copy in the chain)
// Algorithmic bytes: N_in*point_step + N_out*point_step (SURVEY 8d).
#include <float.h>
#include <math.h>

#include "prims.cuh"

namespace lb {
const char* last_error();

// feature extraction (features.cu) runs on the handle's stream with scratch of its own
struct FeatWork;
FeatWork* feat_work_new();
void feat_work_free(FeatWork* w);
int feat_extract(Ctx& c, FeatWork* w, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem_in,
                 const lb_features_params* q, float* out4, size_t out_capacity, lb_features_result* res, int mem_out);

constexpr int VG_MAX_FIELDS = 16;

struct VoxelFieldsDev {
  int n_ff;                          // averaged FLOAT32 fields
  uint32_t ff_off[VG_MAX_FIELDS];
};

// device-resident state of one lb_voxel_filter call (written by the kernels; vg_segment_kernel hands it to the host)
struct VoxState {
  BBoxAcc acc;                 // bounding box of the surviving points; reset by the CTA that consumes it
  unsigned ticket;             // last-CTA detection of vg_bbox_kernel
  unsigned seg_ticket;         // tile ids of vg_segment_kernel; reset by vg_bbox_kernel
  int status;                  // LB_OK or LB_ERR_VOXEL_OVERFLOW
  int min_b[3], div_b[3];
  uint32_t sentinel;           // number of cells of the grid = key of a dropped point (sorts last)
  int key_bits;                // width of the sort key; 0: nothing to do (empty input / overflow)
  uint32_t count;              // surviving points
  uint32_t n_final;            // output points (occupied voxels after min_points_per_voxel)
};

struct VoxLimits {
  int ff_off;                  // byte offset of the filter field, < 0: none
  float fmin, fmax;            // getMinMax3D compares in float32
  double dmin, dmax;           // applyFilter compares the double limits
  int negative;
};

// Up to three input clouds taken as ONE cloud (row f4: the point_cloud_merger node concatenates the 2-3 lidars of a
// robot, a + (b + c), PointCloudMerger.cc:150-178) with, per cloud, what its pcl/PassThrough nodelet does first
// (locus.launch:90-133): drop non-finite points and points whose field lies outside the limits -- in the SENSOR frame --
// then transform into base_link (`output_frame`).  Both are folded into the loads of the voxel kernels.
constexpr int VG_MAX_INPUTS = 3;
struct VoxInputs {
  const uint8_t* base[VG_MAX_INPUTS];
  uint32_t start[VG_MAX_INPUTS + 1];     // global point number of the first point of every cloud; start[n] = total
  float T[VG_MAX_INPUTS][12];            // row-major 3x4 sensor -> base_link
  int has_T[VG_MAX_INPUTS];
  int n;
  VoxLimits pass;                        // PassThrough limits on the raw field (ff_off < 0: none)
};
__device__ __forceinline__ const uint8_t* vg_point(const VoxInputs& in, uint32_t i, uint32_t stride, int& c) {
  c = (in.n > 1 && i >= in.start[1]) ? ((in.n > 2 && i >= in.start[2]) ? 2 : 1) : 0;
  return in.base[c] + (size_t)(i - in.start[c]) * stride;
}
// PassThrough predicate (sensor frame) and the transform of one point; returns false when PassThrough drops the point
__device__ __forceinline__ bool vg_passthrough(const VoxInputs& in, int c, float v, float& x, float& y, float& z) {
  if (in.pass.ff_off >= 0) {
    if (!isfinite(x) || !isfinite(y) || !isfinite(z) || !isfinite(v)) return false;     // pcl::PassThrough removes NaNs
    const double dv = (double)v;
    const bool drop = in.pass.negative ? (dv < in.pass.dmax && dv > in.pass.dmin) : (dv > in.pass.dmax || dv < in.pass.dmin);
    if (drop) return false;
  }
  if (in.has_T[c]) {
    float ox, oy, oz;
    xform(in.T[c], x, y, z, ox, oy, oz);       // Eigen Matrix4f * Vector4f (pcl_ros::transformPointCloud)
    x = ox; y = oy; z = oz;
  }
  return true;
}

// the 8 words of a 32-byte record, fetched with two 16-byte loads
struct Rec32 { uint4 a, b; };
__device__ __forceinline__ Rec32 load_rec32(const uint8_t* p) {
  Rec32 r;
  r.a = __ldg(reinterpret_cast<const uint4*>(p));
  r.b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  return r;
}
__device__ __forceinline__ float rec32_word(const Rec32& r, uint32_t off) {
  const uint32_t w = off >> 2;
  uint32_t v = (w == 0) ? r.a.x : (w == 1) ? r.a.y : (w == 2) ? r.a.z : (w == 3) ? r.a.w
             : (w == 4) ? r.b.x : (w == 5) ? r.b.y : (w == 6) ? r.b.z : r.b.w;
  return __uint_as_float(v);
}

__device__ __forceinline__ bool vg_survives(bool lim_drop, float x, float y, float z, const BodyBox& body) {
  return !lim_drop && isfinite(x) && isfinite(y) && isfinite(z) && !body_box_drops(body, x, y, z);
}

// pcl::getMinMax3D over the points that pass the (float32) limits, the finite check and the body box; the last CTA to
// finish turns the box into the grid geometry exactly like applyFilter does on the host side of PCL
// (voxel_grid_covariance_omp_impl.hpp:75-103): dx*dy*dz overflow guard, min_b = floor(min_p * inv_leaf), div_b.
__global__ void __launch_bounds__(256)
vg_bbox_kernel(const __grid_constant__ VoxInputs in, uint32_t n, uint32_t stride, uint32_t xyz_off, VoxLimits lim, BodyBox body,
               float inv0, float inv1, float inv2, int vec32, VoxState* __restrict__ st) {
  uint32_t mn0 = 0xffffffffu, mn1 = 0xffffffffu, mn2 = 0xffffffffu, mx0 = 0, mx1 = 0, mx2 = 0, cnt = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int ci;
    const uint8_t* p = vg_point(in, i, stride, ci);
    float x, y, z, v = 0.f, pv = 0.f;
    if (vec32) {
      const Rec32 r = load_rec32(p);
      x = rec32_word(r, xyz_off); y = rec32_word(r, xyz_off + 4); z = rec32_word(r, xyz_off + 8);
      if (lim.ff_off >= 0) v = rec32_word(r, (uint32_t)lim.ff_off);
      if (in.pass.ff_off >= 0) pv = rec32_word(r, (uint32_t)in.pass.ff_off);
    } else {
      const float* q = reinterpret_cast<const float*>(p + xyz_off);
      x = q[0]; y = q[1]; z = q[2];
      if (lim.ff_off >= 0) v = *reinterpret_cast<const float*>(p + lim.ff_off);
      if (in.pass.ff_off >= 0) pv = *reinterpret_cast<const float*>(p + in.pass.ff_off);
    }
    if (!vg_passthrough(in, ci, pv, x, y, z)) continue;
    if (lim.ff_off >= 0 && in.has_T[ci] && (uint32_t)lim.ff_off >= xyz_off && (uint32_t)lim.ff_off < xyz_off + 12)
      v = ((uint32_t)lim.ff_off == xyz_off) ? x : (((uint32_t)lim.ff_off == xyz_off + 4) ? y : z);   // the grid's own limits see base_link coordinates
    bool drop = false;
    if (lim.ff_off >= 0) drop = lim.negative ? (v < lim.fmax && v > lim.fmin) : (v > lim.fmax || v < lim.fmin);
    if (!vg_survives(drop, x, y, z, body)) continue;
    const uint32_t ox = f2ord(x), oy = f2ord(y), oz = f2ord(z);
    mn0 = min(mn0, ox); mn1 = min(mn1, oy); mn2 = min(mn2, oz);
    mx0 = max(mx0, ox); mx1 = max(mx1, oy); mx2 = max(mx2, oz);
    cnt++;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  __shared__ uint32_t sm[8][7];
  __shared__ bool last;
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sm[w][0] = mn0; sm[w][1] = mn1; sm[w][2] = mn2; sm[w][3] = mx0; sm[w][4] = mx1; sm[w][5] = mx2; sm[w][6] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; i++) {
      mn0 = min(mn0, sm[i][0]); mn1 = min(mn1, sm[i][1]); mn2 = min(mn2, sm[i][2]);
      mx0 = max(mx0, sm[i][3]); mx1 = max(mx1, sm[i][4]); mx2 = max(mx2, sm[i][5]);
      cnt += sm[i][6];
    }
    if (cnt > 0) {       // one set of atomics per CTA (same-address atomics serialise in L2)
      atomicMin(&st->acc.mn[0], mn0); atomicMin(&st->acc.mn[1], mn1); atomicMin(&st->acc.mn[2], mn2);
      atomicMax(&st->acc.mx[0], mx0); atomicMax(&st->acc.mx[1], mx1); atomicMax(&st->acc.mx[2], mx2);
      atomicAdd(&st->acc.count, cnt);
    }
    __threadfence();
    last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  // ---- grid geometry (what pcl::VoxelGrid::applyFilter derives from min_p / max_p)
  const uint32_t count = atomicAdd(&st->acc.count, 0u);
  int status = LB_OK, key_bits = 0;
  uint32_t sentinel = 0;
  if (count > 0) {
    float min_p[3], max_p[3];
    const float inv[3] = {inv0, inv1, inv2};
    for (int d = 0; d < 3; d++) { min_p[d] = ord2f(atomicAdd(&st->acc.mn[d], 0u)); max_p[d] = ord2f(atomicAdd(&st->acc.mx[d], 0u)); }
    const long long dx = (long long)((max_p[0] - min_p[0]) * inv[0]) + 1;
    const long long dy = (long long)((max_p[1] - min_p[1]) * inv[1]) + 1;
    const long long dz = (long long)((max_p[2] - min_p[2]) * inv[2]) + 1;
    int min_b[3], div_b[3];
    for (int d = 0; d < 3; d++) {
      min_b[d] = (int)floorf(min_p[d] * inv[d]);
      const int max_b = (int)floorf(max_p[d] * inv[d]);
      div_b[d] = max_b - min_b[d] + 1;
      st->min_b[d] = min_b[d]; st->div_b[d] = div_b[d];
    }
    const long long ncells = (long long)div_b[0] * div_b[1] * div_b[2];
    if (dx * dy * dz > 2147483647ll || ncells > 2147483647ll) {
      status = LB_ERR_VOXEL_OVERFLOW;      // "Leaf size is too small for the input dataset. Integer indices would overflow."
    } else {
      sentinel = (uint32_t)ncells;
      key_bits = 1;
      while (key_bits < 32 && (1ull << key_bits) <= (unsigned long long)sentinel) key_bits++;
    }
  }
  st->status = status; st->sentinel = sentinel; st->key_bits = key_bits; st->count = count;
  st->n_final = 0;
  bbox_reset(&st->acc);            // consumed: clean for the next call
  st->ticket = 0;
  st->seg_ticket = 0;
}

// the sort key (PCL leaf index, or the sentinel for a dropped point) and the averaged record of point i
__device__ __forceinline__ uint32_t vg_point_key(const VoxInputs& in, uint32_t i, uint32_t stride, uint32_t xyz_off, const VoxLimits& lim,
                                                 const BodyBox& body, float inv0, float inv1, float inv2, int vec32,
                                                 const VoxelFieldsDev& F, const VoxState* __restrict__ st, float4* __restrict__ rec) {
  const uint32_t sentinel = st->sentinel;
  const int min_b0 = st->min_b[0], min_b1 = st->min_b[1], min_b2 = st->min_b[2];
  const int mul1 = st->div_b[0], mul2 = st->div_b[0] * st->div_b[1];
  int ci;
  const uint8_t* p = vg_point(in, i, stride, ci);
  float x, y, z, v = 0.f, pv = 0.f;
  float4 r4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (vec32) {
    const Rec32 r = load_rec32(p);
    x = rec32_word(r, xyz_off); y = rec32_word(r, xyz_off + 4); z = rec32_word(r, xyz_off + 8);
    if (lim.ff_off >= 0) v = rec32_word(r, (uint32_t)lim.ff_off);
    if (in.pass.ff_off >= 0) pv = rec32_word(r, (uint32_t)in.pass.ff_off);
    if (rec) r4 = make_float4(rec32_word(r, F.ff_off[0]), rec32_word(r, F.ff_off[1]), rec32_word(r, F.ff_off[2]), rec32_word(r, F.ff_off[3]));
  } else {
    x = *reinterpret_cast<const float*>(p + xyz_off);
    y = *reinterpret_cast<const float*>(p + xyz_off + 4);
    z = *reinterpret_cast<const float*>(p + xyz_off + 8);
    if (lim.ff_off >= 0) v = *reinterpret_cast<const float*>(p + lim.ff_off);
    if (in.pass.ff_off >= 0) pv = *reinterpret_cast<const float*>(p + in.pass.ff_off);
    if (rec) r4 = make_float4(*reinterpret_cast<const float*>(p + F.ff_off[0]), *reinterpret_cast<const float*>(p + F.ff_off[1]),
                              *reinterpret_cast<const float*>(p + F.ff_off[2]), *reinterpret_cast<const float*>(p + F.ff_off[3]));
  }
  const bool passed = vg_passthrough(in, ci, pv, x, y, z);
  if (in.has_T[ci]) {
    // the record the centroid sums holds the TRANSFORMED coordinates (the averaged fields are x, y, z, intensity here)
    if (rec) {
      if (F.ff_off[0] == xyz_off) r4.x = x; if (F.ff_off[1] == xyz_off + 4) r4.y = y; if (F.ff_off[2] == xyz_off + 8) r4.z = z;
    }
    if (lim.ff_off >= 0 && (uint32_t)lim.ff_off >= xyz_off && (uint32_t)lim.ff_off < xyz_off + 12)
      v = ((uint32_t)lim.ff_off == xyz_off) ? x : (((uint32_t)lim.ff_off == xyz_off + 4) ? y : z);
  }
  bool drop = !passed;
  if (!drop && lim.ff_off >= 0) {
    const double dv = (double)v;
    drop = lim.negative ? (dv < lim.dmax && dv > lim.dmin) : (dv > lim.dmax || dv < lim.dmin);
  }
  uint32_t key = sentinel;
  if (vg_survives(drop, x, y, z, body)) {          // BodyFilter folded into the load predicate (row f4)
    // static_cast<int>(floor(x * inv_leaf) - float(min_b))   (voxel_grid_covariance_omp_impl.hpp:159-161)
    const int ijk0 = (int)(floorf(x * inv0) - (float)min_b0);
    const int ijk1 = (int)(floorf(y * inv1) - (float)min_b1);
    const int ijk2 = (int)(floorf(z * inv2) - (float)min_b2);
    const int idx = ijk0 + ijk1 * mul1 + ijk2 * mul2;
    key = ((uint32_t)idx < sentinel) ? (uint32_t)idx : sentinel;
  }
  if (rec) rec[i] = r4;
  return key;
}

constexpr int VG_KEYS_ITEMS = 4;     // points per thread of vg_keys_kernel: 1024 per CTA, one histogram flush each

// Keys + records, and the digit histogram of every sort pass the key width needs (one atomic per non-zero digit and
// CTA, the last CTA turns them into digit offsets).  Also resets the look-back state of the sort's scatters and of
// vg_segment_kernel: every kernel after this one starts from clean status words.
__global__ void __launch_bounds__(256)
vg_keys_kernel(const __grid_constant__ VoxInputs in, uint32_t n, uint32_t stride, uint32_t xyz_off, VoxLimits lim, BodyBox body,
               float inv0, float inv1, float inv2, int vec32, VoxelFieldsDev F, const VoxState* __restrict__ st,
               uint32_t* __restrict__ keys, float4* __restrict__ rec /*nullable: only for 4 averaged fields*/,
               RsDev* __restrict__ rs, uint32_t* __restrict__ rs_status, uint32_t rs_tiles,
               uint32_t* __restrict__ seg_status, uint32_t seg_tiles) {
  __shared__ uint32_t sh[RS_PASSES_MAX][256];
  __shared__ uint32_t scan_sm[256 / 32 + 1];
  __shared__ bool last;
  const int key_bits = st->key_bits;
  if (key_bits == 0) return;              // empty input or overflow: nothing is sorted
  const int passes = (key_bits + 7) >> 3;
  for (int t = threadIdx.x; t < RS_PASSES_MAX * 256; t += 256) (&sh[0][0])[t] = 0;
  rs_reset_lookback(rs, rs_status, rs_tiles);
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < seg_tiles; t += gridDim.x * blockDim.x) seg_status[t] = LB_NOT_READY;
  __syncthreads();
#pragma unroll 1
  for (int u = 0; u < VG_KEYS_ITEMS; u++) {
    const uint32_t i = blockIdx.x * (256u * VG_KEYS_ITEMS) + u * 256u + threadIdx.x;
    uint32_t key = 0;
    if (i < n) {
      key = vg_point_key(in, i, stride, xyz_off, lim, body, inv0, inv1, inv2, vec32, F, st, rec);
      keys[i] = key;
    }
    rs_hist_warp_add(sh, key, i < n, passes);
  }
  rs_hist_flush(sh, rs, passes, scan_sm, &last);
}

// which ping-pong buffer holds the sorted pairs: A after an odd number of executed passes, B after an even number
__device__ __forceinline__ bool vg_sorted_in_a(int key_bits) { return (((key_bits + 7) >> 3) & 1) != 0; }

// lookback_prefix by a whole warp over consecutive status words, 32 tiles per step; every lane returns the prefix.
__device__ __forceinline__ uint32_t lookback_prefix_warp(const uint32_t* status, uint32_t tile) {
  const int lane = threadIdx.x & 31;
  uint32_t excl = 0;
  for (int64_t top = (int64_t)tile - 1;; top -= 32) {         // lane 0 reads the nearest earlier tile
    const int64_t j = top - lane;
    const volatile uint32_t* w = status + (j >= 0 ? j : 0);
    uint32_t s = (j >= 0) ? *w : LB_PREFIX;                    // before tile 0: a prefix of 0
    while (__any_sync(0xffffffffu, s == LB_NOT_READY))
      if (s == LB_NOT_READY) s = *w;
    const uint32_t pm = __ballot_sync(0xffffffffu, (s & LB_PREFIX) != 0);
    const int stop = pm ? __ffs(pm) - 1 : 31;                  // the nearest prefix ends the walk
    uint32_t v = (lane <= stop) ? (s & ~LB_PREFIX) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    excl += v;
    if (pm) return excl;
  }
}

constexpr int VG_SEG_TILE = 1024;    // sorted positions per CTA of vg_segment_kernel (256 threads x 4)

// One tile of sorted positions, taken in ticket order:
//   1. the positions where the key changes (voxel heads, and the start of the dropped points' sentinel run)
//   2. the end of the voxel that crosses the tile end: one warp reads on, 32 keys per step
//   3. FOUR: the packed float4 records of the tile and of that crossing tail (up to another tile's worth) staged in
//      shared memory (coalesced point numbers, 16-byte gathers, all in flight at once); and per voxel that STARTS in the tile: its end (the next head, or the crossing tail's end) and whether it holds
//      min_points_per_voxel points
//   4. output slots: the kept voxels of the tile in order, after those of every earlier tile (decoupled look-back)
//   5. one lane per voxel: float32 sum of its records in ascending input order (the order the stable sort produced;
//      it defines the rounding: PCL's centroid += point, then /= float(n)), records past the tile end read from
//      global memory; other layouts read the caller's bytes through the sorted point numbers
// The last tile knows the voxel count: it writes the call's whole state into pinned host memory.
template <bool FOUR>
__global__ void __launch_bounds__(256)
vg_segment_kernel(const __grid_constant__ VoxInputs in, uint32_t stride, const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb,
                  const uint32_t* __restrict__ va, const uint32_t* __restrict__ vb, const float4* __restrict__ rec,
                  VoxState* __restrict__ st, VoxState* __restrict__ h_st, uint32_t* __restrict__ seg_status, uint32_t n,
                  int min_points, VoxelFieldsDev F, uint32_t capacity, int vec32, uint8_t* __restrict__ out,
                  int32_t* __restrict__ out_voxel_idx) {
  __shared__ uint32_t bnd[VG_SEG_TILE];      // tile positions where the key changes, ascending
  __shared__ uint32_t endp[VG_SEG_TILE];     // end of the voxel starting at bnd[h]; 0: not an output voxel
  __shared__ uint32_t slot[VG_SEG_TILE];     // its rank among the tile's output voxels
  __shared__ float4 recs[FOUR ? 2 * VG_SEG_TILE : 1];   // sorted positions t0 .. staged end
  __shared__ uint32_t scan_sm[256 / 32 + 1];
  __shared__ uint32_t tile_sm, pre_sm, tail_sm;
  const int key_bits = st->key_bits;
  if (key_bits == 0) {                       // empty input or overflow: only the state goes back
    if (blockIdx.x == 0 && threadIdx.x == 0) { VoxState s = *st; s.n_final = 0; *h_st = s; }
    return;
  }
  if (threadIdx.x == 0) tile_sm = atomicAdd(&st->seg_ticket, 1u);
  __syncthreads();
  const uint32_t tile = tile_sm;
  const bool in_a = vg_sorted_in_a(key_bits);
  const uint32_t* keys = in_a ? ka : kb;
  const uint32_t* vals = in_a ? va : vb;
  const uint32_t sentinel = st->sentinel;
  const uint32_t t0 = tile * VG_SEG_TILE, t1 = min(n, t0 + VG_SEG_TILE);
  // 1.
  uint32_t nb;
  {
    const uint32_t base = t0 + threadIdx.x * 4;
    uint32_t bits = 0, c = 0;
    uint32_t prev = (base > 0 && base <= n) ? keys[base - 1] : 0xffffffffu;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint32_t i = base + j;
      if (i < n) {
        const uint32_t k = keys[i];
        if (i == 0 || k != prev) { bits |= 1u << j; c++; }
        prev = k;
      }
    }
    uint32_t q = block_excl_scan<256>(c, &nb, scan_sm);
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (bits & (1u << j)) bnd[q++] = base + j;
  }
  __syncthreads();
  // 2.
  if (threadIdx.x < 32) {
    uint32_t e = t1;
    if (nb > 0 && t1 < n) {
      const uint32_t k = keys[bnd[nb - 1]];
      if (k < sentinel) {
        for (;; e += 32) {
          const uint32_t i = e + threadIdx.x;
          const uint32_t other = __ballot_sync(0xffffffffu, !(i < n && keys[i] == k));
          if (other) { e += __ffs(other) - 1; break; }
        }
      }
    }
    if (threadIdx.x == 0) tail_sm = e;
  }
  __syncthreads();
  const uint32_t tail = tail_sm;
  const uint32_t staged = min(tail, t0 + 2 * VG_SEG_TILE);
  // 3.
  if (FOUR) {
    uint32_t pv[2 * VG_SEG_TILE / 256];
    float4 rv[2 * VG_SEG_TILE / 256];
#pragma unroll
    for (int u = 0; u < 2 * VG_SEG_TILE / 256; u++) {
      const uint32_t i = t0 + threadIdx.x + 256u * u;
      pv[u] = (i < staged) ? vals[i] : 0xffffffffu;
    }
#pragma unroll
    for (int u = 0; u < 2 * VG_SEG_TILE / 256; u++) rv[u] = (pv[u] != 0xffffffffu) ? rec[pv[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 2 * VG_SEG_TILE / 256; u++)
      if (pv[u] != 0xffffffffu) recs[threadIdx.x + 256u * u] = rv[u];
  }
  for (uint32_t h = threadIdx.x; h < nb; h += 256) {
    const uint32_t a = bnd[h];
    const uint32_t k = keys[a];
    uint32_t e = 0;
    if (k < sentinel) {
      e = (h + 1 < nb) ? bnd[h + 1] : tail;
      if (min_points > 1 && (int)(e - a) < min_points) e = 0;
    }
    endp[h] = e;
  }
  __syncthreads();
  // 4.
  {
    uint32_t kc = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) { const uint32_t h = threadIdx.x * 4 + j; if (h < nb && endp[h]) kc++; }
    uint32_t tot;
    uint32_t r = block_excl_scan<256>(kc, &tot, scan_sm);
#pragma unroll
    for (int j = 0; j < 4; j++) { const uint32_t h = threadIdx.x * 4 + j; if (h < nb && endp[h]) slot[h] = r++; }
    if (threadIdx.x < 32) {
      uint32_t* mine = seg_status + tile;
      if (threadIdx.x == 0) lookback_publish(mine, tile == 0 ? (LB_PREFIX | tot) : tot);
      const uint32_t pre = tile == 0 ? 0u : lookback_prefix_warp(seg_status, tile);
      if (threadIdx.x == 0 && tile > 0) lookback_publish(mine, LB_PREFIX | (pre + tot));
      if (threadIdx.x == 0) pre_sm = pre;
      if (threadIdx.x == 0 && tile == gridDim.x - 1) {           // every earlier tile is counted: the call's result is known
        st->n_final = pre + tot;
        VoxState s = *st;
        s.n_final = pre + tot;
        *h_st = s;
      }
    }
  }
  __syncthreads();
  // 5.
  const uint32_t pre = pre_sm;
  for (uint32_t h = threadIdx.x; h < nb; h += 256) {
    const uint32_t e = endp[h];
    if (!e) continue;
    const uint32_t o = pre + slot[h];
    if (o >= capacity) continue;
    const uint32_t a = bnd[h];
    int cfirst;
    const uint8_t* first = vg_point(in, vals[a], stride, cfirst);
    uint8_t* dst = out + (size_t)o * stride;
    const float cnt = (float)(e - a);
    if (FOUR) {
      float4 acc = recs[a - t0];                                  // the sum starts from the first record itself
      const uint32_t em = min(e, staged);
      uint32_t j = a + 1;
      for (; j < em; j++) {
        const float4 v = recs[j - t0];
        acc.x = acc.x + v.x; acc.y = acc.y + v.y; acc.z = acc.z + v.z; acc.w = acc.w + v.w;
      }
      for (; j + 4 <= e; j += 4) {                                // past the staged records: 4 gathers in flight, added in order
        const uint32_t p0 = vals[j], p1 = vals[j + 1], p2 = vals[j + 2], p3 = vals[j + 3];
        const float4 v0 = rec[p0], v1 = rec[p1], v2 = rec[p2], v3 = rec[p3];
        acc.x = acc.x + v0.x; acc.y = acc.y + v0.y; acc.z = acc.z + v0.z; acc.w = acc.w + v0.w;
        acc.x = acc.x + v1.x; acc.y = acc.y + v1.y; acc.z = acc.z + v1.z; acc.w = acc.w + v1.w;
        acc.x = acc.x + v2.x; acc.y = acc.y + v2.y; acc.z = acc.z + v2.z; acc.w = acc.w + v2.w;
        acc.x = acc.x + v3.x; acc.y = acc.y + v3.y; acc.z = acc.z + v3.z; acc.w = acc.w + v3.w;
      }
      for (; j < e; j++) {
        const float4 v = rec[vals[j]];
        acc.x = acc.x + v.x; acc.y = acc.y + v.y; acc.z = acc.z + v.z; acc.w = acc.w + v.w;
      }
      // bytes not covered by an averaged field come from the voxel's first point
      if (vec32 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0) {
        const uint4 w0 = reinterpret_cast<const uint4*>(first)[0], w1 = reinterpret_cast<const uint4*>(first)[1];
        reinterpret_cast<uint4*>(dst)[0] = w0; reinterpret_cast<uint4*>(dst)[1] = w1;
      } else {
        for (uint32_t w = 0; w < stride / 4; w++)
          reinterpret_cast<uint32_t*>(dst)[w] = reinterpret_cast<const uint32_t*>(first)[w];
      }
      *reinterpret_cast<float*>(dst + F.ff_off[0]) = acc.x / cnt;
      *reinterpret_cast<float*>(dst + F.ff_off[1]) = acc.y / cnt;
      *reinterpret_cast<float*>(dst + F.ff_off[2]) = acc.z / cnt;
      *reinterpret_cast<float*>(dst + F.ff_off[3]) = acc.w / cnt;
    } else {
      float acc[VG_MAX_FIELDS];
      const int nf = F.n_ff;
#pragma unroll
      for (int f = 0; f < VG_MAX_FIELDS; f++) acc[f] = (f < nf) ? *reinterpret_cast<const float*>(first + F.ff_off[f]) : 0.f;
      for (uint32_t j = a + 1; j < e; j++) {
        int cj;
        const uint8_t* p = vg_point(in, vals[j], stride, cj);
#pragma unroll
        for (int f = 0; f < VG_MAX_FIELDS; f++)
          if (f < nf) acc[f] = acc[f] + *reinterpret_cast<const float*>(p + F.ff_off[f]);
      }
      // bytes not covered by an averaged field come from the voxel's first point
      for (uint32_t w = 0; w < stride / 4; w++)
        reinterpret_cast<uint32_t*>(dst)[w] = reinterpret_cast<const uint32_t*>(first)[w];
#pragma unroll
      for (int f = 0; f < VG_MAX_FIELDS; f++)
        if (f < nf) *reinterpret_cast<float*>(dst + F.ff_off[f]) = acc[f] / cnt;
    }
    if (out_voxel_idx) out_voxel_idx[o] = (int32_t)keys[a];
  }
}

__global__ void vg_state_init_kernel(VoxState* st) {
  if (threadIdx.x == 0) {
    bbox_reset(&st->acc);
    st->ticket = 0; st->seg_ticket = 0; st->status = 0; st->sentinel = 0; st->key_bits = 0; st->count = 0; st->n_final = 0;
    for (int d = 0; d < 3; d++) { st->min_b[d] = 0; st->div_b[d] = 0; }
  }
}

}  // namespace lb

using namespace lb;

struct lb_voxel {
  Ctx c;
  float leaf[3] = {0.f, 0.f, 0.f};
  char filter_field[32] = "";
  double lim_min = -FLT_MAX, lim_max = FLT_MAX;
  int negative = 0;
  int min_points = 0;
  int downsample_all = 1;
  BodyBox body{0, 1.f, 0.f, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};   // BodyFilter nodelet folded in (lb_voxel_set_body_filter)
  char pass_field[32] = "";     // pcl/PassThrough nodelet folded in (lb_voxel_set_input_passthrough)
  double pass_min = -FLT_MAX, pass_max = FLT_MAX;
  int pass_negative = 0;
  DBuf<uint8_t> d_in, d_out;
  DBuf<int32_t> d_vidx;
  DBuf<uint32_t> keys, seg_status;
  DBuf<float4> rec;
  VoxState* d_st = nullptr;     // device
  VoxState* h_st = nullptr;     // pinned, written by vg_segment_kernel
  int bits_hint = 32;           // sort passes to enqueue: the key width of the previous call, rounded up to whole passes
  SortWork sort;
  FeatWork* feat = nullptr;     // created by the first lb_voxel_extract_features
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float t_last_ms = 0.f;
  double t_sum_ms = 0.0;        // since the last lb_voxel_kernel_time_avg(reset)
  uint64_t t_calls = 0;
};

static int voxel_create_impl(int device, void* stream, bool ext, lb_voxel** out) {
  if (!out) { set_error("lb_voxel_create: null handle pointer"); return LB_ERR_INVALID_ARG; }
  lb_voxel* h = new lb_voxel;
  int s = ctx_init(h->c, device, stream, ext);
  if (s != LB_OK) { delete h; return s; }
  if (cudaMalloc((void**)&h->d_st, sizeof(VoxState)) != cudaSuccess ||
      cudaMallocHost((void**)&h->h_st, sizeof(VoxState)) != cudaSuccess ||
      cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess) {
    set_error("lb_voxel_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    delete h;
    return LB_ERR_CUDA;
  }
  vg_state_init_kernel<<<1, 32, 0, h->c.stream>>>(h->d_st);
  cudaStreamSynchronize(h->c.stream);
  *out = h;
  return LB_OK;
}

namespace lb {
// Size the filter's scratch for raw scans of up to n_pts points of up to max_step bytes (host staging, keys, records,
// look-back words, sort buffers), so that no later call on such scans allocates.  The lidar pipelines call it at
// creation: their raw scan can grow mid-stream (a lidar comes back), and a cudaMalloc there would synchronise the
// whole device.  Results do not depend on the capacities.
int voxel_reserve(lb_voxel* h, size_t n_pts, uint32_t max_step) {
  if (!h || n_pts == 0 || n_pts > 0x7ffffff0ull) { set_error("voxel_reserve: bad argument"); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  LB_TRY(h->d_in.ensure(n_pts * max_step));
  LB_TRY(h->keys.ensure(n_pts)); LB_TRY(h->seg_status.ensure((size_t)cdiv((long long)n_pts, VG_SEG_TILE)));
  LB_TRY(h->rec.ensure(n_pts));
  return radix_sort_reserve(h->c, h->sort, n_pts);
}
}  // namespace lb

extern "C" {

int lb_voxel_create(int device, lb_voxel** h) { return voxel_create_impl(device, nullptr, false, h); }
int lb_voxel_create_on_stream(int device, void* stream, lb_voxel** h) { return voxel_create_impl(device, stream, true, h); }

int lb_voxel_destroy(lb_voxel* h) {
  if (!h) return LB_OK;
  cudaSetDevice(h->c.device);
  cudaStreamSynchronize(h->c.stream);
  h->d_in.release(); h->d_out.release(); h->d_vidx.release(); h->keys.release(); h->seg_status.release(); h->rec.release();
  h->sort.ka.release(); h->sort.kb.release(); h->sort.va.release(); h->sort.vb.release(); h->sort.state.release();
  feat_work_free(h->feat);
  if (h->d_st) cudaFree(h->d_st);
  if (h->h_st) cudaFreeHost(h->h_st);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  ctx_destroy(h->c);
  delete h;
  return LB_OK;
}

int lb_voxel_set_leaf_size(lb_voxel* h, float lx, float ly, float lz) {
  if (!h || !(lx > 0.f) || !(ly > 0.f) || !(lz > 0.f)) { set_error("lb_voxel_set_leaf_size: leaf must be > 0"); return LB_ERR_INVALID_ARG; }
  h->leaf[0] = lx; h->leaf[1] = ly; h->leaf[2] = lz;
  return LB_OK;
}
int lb_voxel_get_leaf_size(lb_voxel* h, float* leaf3) {
  if (!h || !leaf3) return LB_ERR_INVALID_ARG;
  leaf3[0] = h->leaf[0]; leaf3[1] = h->leaf[1]; leaf3[2] = h->leaf[2];
  return LB_OK;
}
int lb_voxel_set_filter_limits(lb_voxel* h, const char* field_name, double limit_min, double limit_max, int negative) {
  if (!h) return LB_ERR_INVALID_ARG;
  h->filter_field[0] = 0;
  if (field_name) { strncpy(h->filter_field, field_name, sizeof(h->filter_field) - 1); h->filter_field[sizeof(h->filter_field) - 1] = 0; }
  h->lim_min = limit_min; h->lim_max = limit_max; h->negative = negative ? 1 : 0;
  return LB_OK;
}
int lb_voxel_set_body_filter(lb_voxel* h, int enabled, const float* min3, const float* max3, float rotation_z) {
  if (!h || (enabled && (!min3 || !max3))) { set_error("lb_voxel_set_body_filter: null argument"); return LB_ERR_INVALID_ARG; }
  h->body.enabled = enabled ? 1 : 0;
  if (enabled) {
    // inverse of PCL's getTransformation(0,0,0, 0,0,rz) taken the way Eigen inverts a 3x3: adjugate / determinant
    float A = cosf(rotation_z), B = sinf(rotation_z);
    float det = A * A + B * B;
    h->body.ia = A / det; h->body.ib = B / det;
    for (int d = 0; d < 3; d++) { h->body.mn[d] = min3[d]; h->body.mx[d] = max3[d]; }
  }
  return LB_OK;
}
int lb_voxel_set_min_points_per_voxel(lb_voxel* h, int m) { if (!h) return LB_ERR_INVALID_ARG; h->min_points = m; return LB_OK; }
int lb_voxel_set_downsample_all_data(lb_voxel* h, int all) { if (!h) return LB_ERR_INVALID_ARG; h->downsample_all = all ? 1 : 0; return LB_OK; }
int lb_voxel_launch_count(lb_voxel* h, uint64_t* n) { if (!h || !n) return LB_ERR_INVALID_ARG; *n = h->c.launches; return LB_OK; }
int lb_voxel_kernel_time(lb_voxel* h, float* ms) { if (!h || !ms) return LB_ERR_INVALID_ARG; *ms = h->t_last_ms; return LB_OK; }
int lb_voxel_kernel_time_avg(lb_voxel* h, float* ms_avg, uint64_t* calls, int reset) {
  if (!h || !ms_avg) return LB_ERR_INVALID_ARG;
  *ms_avg = h->t_calls ? (float)(h->t_sum_ms / (double)h->t_calls) : 0.f;
  if (calls) *calls = h->t_calls;
  if (reset) { h->t_sum_ms = 0.0; h->t_calls = 0; }
  return LB_OK;
}

int lb_features_default_params(lb_features_params* p) {
  if (!p) return LB_ERR_INVALID_ARG;
  p->n_rings = 16; p->lower_deg = -15.f; p->upper_deg = 15.f; p->scan_period = 0.1f;
  p->curvature_region = 5; p->n_feature_regions = 6;
  p->max_corner_sharp = 2; p->max_corner_less_sharp = 20; p->max_surface_flat = 4;
  p->curvature_threshold = 0.1f; p->less_flat_leaf = 0.2f;
  return LB_OK;
}

int lb_voxel_extract_features(lb_voxel* h, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem_in,
                              const lb_features_params* p, float* out4, size_t out_capacity, lb_features_result* r,
                              int mem_out) {
  if (!h) { set_error("lb_voxel_extract_features: null handle"); return LB_ERR_INVALID_ARG; }
  if (!h->feat) h->feat = feat_work_new();
  return feat_extract(h->c, h->feat, pts, n, stride, xyz_off, mem_in, p, out4, out_capacity, r, mem_out);
}

int lb_voxel_set_input_passthrough(lb_voxel* h, const char* field_name, double limit_min, double limit_max, int negative) {
  if (!h) return LB_ERR_INVALID_ARG;
  h->pass_field[0] = 0;
  if (field_name) { strncpy(h->pass_field, field_name, sizeof(h->pass_field) - 1); h->pass_field[sizeof(h->pass_field) - 1] = 0; }
  h->pass_min = limit_min; h->pass_max = limit_max; h->pass_negative = negative ? 1 : 0;
  return LB_OK;
}

static int voxel_filter_impl(lb_voxel* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step, const lb_field* fields,
                             int n_fields, uint8_t* out, size_t out_capacity_pts, size_t* n_out, int32_t* out_voxel_idx,
                             int mem_in, int mem_out);

int lb_voxel_filter(lb_voxel* h, const uint8_t* data, size_t n_pts, uint32_t point_step, const lb_field* fields,
                    int n_fields, const int32_t* indices, size_t n_indices, uint8_t* out, size_t out_capacity_pts,
                    size_t* n_out, int32_t* out_voxel_idx, int mem_in, int mem_out) {
  (void)indices; (void)n_indices;  // pcl::VoxelGrid<PCLPointCloud2> ignores indices_ too
  lb_voxel_input in;
  in.data = data; in.n_pts = n_pts; in.transform = nullptr;
  return voxel_filter_impl(h, &in, 1, point_step, fields, n_fields, out, out_capacity_pts, n_out, out_voxel_idx, mem_in, mem_out);
}

int lb_voxel_filter_merged(lb_voxel* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step, const lb_field* fields,
                           int n_fields, uint8_t* out, size_t out_capacity_pts, size_t* n_out, int32_t* out_voxel_idx,
                           int mem_in, int mem_out) {
  if (!inputs || n_inputs < 1 || n_inputs > VG_MAX_INPUTS) { set_error("lb_voxel_filter_merged: 1 to %d input clouds", VG_MAX_INPUTS); return LB_ERR_INVALID_ARG; }
  return voxel_filter_impl(h, inputs, n_inputs, point_step, fields, n_fields, out, out_capacity_pts, n_out, out_voxel_idx, mem_in, mem_out);
}

static int voxel_filter_impl(lb_voxel* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step, const lb_field* fields,
                             int n_fields, uint8_t* out, size_t out_capacity_pts, size_t* n_out, int32_t* out_voxel_idx,
                             int mem_in, int mem_out) {
  if (!h || !n_out) { set_error("lb_voxel_filter: null handle / n_out"); return LB_ERR_INVALID_ARG; }
  *n_out = 0;
  size_t n_pts = 0;
  bool any_T = false;
  for (int i = 0; i < n_inputs; i++) {
    if (inputs[i].n_pts && !inputs[i].data) { set_error("lb_voxel_filter: null input cloud %d", i); return LB_ERR_INVALID_ARG; }
    n_pts += inputs[i].n_pts;
    any_T = any_T || inputs[i].transform != nullptr;
  }
  if (n_pts == 0) return LB_OK;
  if (!out || !fields || n_fields <= 0) { set_error("lb_voxel_filter: null data/out/fields"); return LB_ERR_INVALID_ARG; }
  if (point_step < 12 || (point_step & 3u)) { set_error("lb_voxel_filter: point_step must be a multiple of 4 and >= 12"); return LB_ERR_INVALID_ARG; }
  if (n_pts > 0x7ffffff0ull) { set_error("lb_voxel_filter: too many points"); return LB_ERR_INVALID_ARG; }
  if (!(h->leaf[0] > 0.f)) { set_error("lb_voxel_filter: leaf size not set"); return LB_ERR_INVALID_ARG; }
  int xo = -1, yo = -1, zo = -1, ffo = -1, pfo = -1;
  VoxelFieldsDev F; F.n_ff = 0;
  for (int f = 0; f < n_fields; f++) {
    const lb_field& fd = fields[f];
    bool is_f32 = fd.datatype == LB_FLOAT32;
    if (!strcmp(fd.name, "x") && is_f32) xo = (int)fd.offset;
    if (!strcmp(fd.name, "y") && is_f32) yo = (int)fd.offset;
    if (!strcmp(fd.name, "z") && is_f32) zo = (int)fd.offset;
    if (h->filter_field[0] && !strcmp(fd.name, h->filter_field)) {
      if (!is_f32) { set_error("lb_voxel_filter: distance filtering requires a FLOAT32 field"); return LB_ERR_UNSUPPORTED; }
      ffo = (int)fd.offset;
    }
    if (h->pass_field[0] && !strcmp(fd.name, h->pass_field)) {
      if (!is_f32) { set_error("lb_voxel_filter: PassThrough requires a FLOAT32 field"); return LB_ERR_UNSUPPORTED; }
      pfo = (int)fd.offset;
    }
    if (fd.offset + 4 > point_step || (fd.offset & 3u)) {
      if (is_f32) { set_error("lb_voxel_filter: field '%s' misaligned / out of range", fd.name); return LB_ERR_INVALID_ARG; }
    }
  }
  if (h->pass_field[0] && pfo < 0) { set_error("lb_voxel_filter: PassThrough field '%s' not found", h->pass_field); return LB_ERR_INVALID_ARG; }
  if (xo < 0 || yo < 0 || zo < 0) { set_error("lb_voxel_filter: x/y/z FLOAT32 fields required"); return LB_ERR_INVALID_ARG; }
  if (h->filter_field[0] && ffo < 0) { set_error("lb_voxel_filter: filter field '%s' not found", h->filter_field); return LB_ERR_INVALID_ARG; }
  if (h->downsample_all) {
    for (int f = 0; f < n_fields; f++) {
      if (fields[f].datatype != LB_FLOAT32) continue;
      uint32_t cnt = fields[f].count ? fields[f].count : 1;
      for (uint32_t c = 0; c < cnt; c++) {
        if (F.n_ff >= VG_MAX_FIELDS) { set_error("lb_voxel_filter: more than %d float fields", VG_MAX_FIELDS); return LB_ERR_UNSUPPORTED; }
        F.ff_off[F.n_ff++] = fields[f].offset + 4 * c;
      }
    }
  } else {
    F.n_ff = 3; F.ff_off[0] = xo; F.ff_off[1] = yo; F.ff_off[2] = zo;
  }

  // x,y,z must be contiguous (true for every PCL point type): the kernels read them as three consecutive floats
  if (yo != xo + 4 || zo != xo + 8) { set_error("lb_voxel_filter: x,y,z must be consecutive FLOAT32 fields"); return LB_ERR_UNSUPPORTED; }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t n = (uint32_t)n_pts;
  const size_t bytes = (size_t)n * point_step;
  LB_CUDA(cudaEventRecord(h->ev0, c.stream));
  VoxInputs vin;
  memset(&vin, 0, sizeof(vin));
  vin.n = n_inputs;
  vin.pass.ff_off = pfo; vin.pass.fmin = (float)h->pass_min; vin.pass.fmax = (float)h->pass_max;
  vin.pass.dmin = h->pass_min; vin.pass.dmax = h->pass_max; vin.pass.negative = h->pass_negative;
  if (mem_in == LB_MEM_HOST) LB_TRY(h->d_in.ensure(bytes));
  {
    size_t at = 0;
    for (int i = 0; i < VG_MAX_INPUTS; i++) {
      const bool have = i < n_inputs;
      vin.start[i] = (uint32_t)at;
      vin.base[i] = nullptr;
      if (have) {
        vin.base[i] = inputs[i].data;
        if (mem_in == LB_MEM_HOST) {          // the clouds are staged back to back: one device cloud
          if (inputs[i].n_pts)
            LB_CUDA(cudaMemcpyAsync(h->d_in.p + at * point_step, inputs[i].data, inputs[i].n_pts * point_step, cudaMemcpyHostToDevice, c.stream));
          vin.base[i] = h->d_in.p + at * point_step;
        }
        vin.has_T[i] = inputs[i].transform ? 1 : 0;
        if (inputs[i].transform) for (int e = 0; e < 12; e++) vin.T[i][e] = inputs[i].transform[e];
        at += inputs[i].n_pts;
      }
    }
    vin.start[VG_MAX_INPUTS] = (uint32_t)at;
    for (int i = n_inputs; i < VG_MAX_INPUTS; i++) vin.start[i] = (uint32_t)at;
  }
  uint8_t* d_out = out; int32_t* d_vidx = out_voxel_idx;
  uint32_t capacity = (uint32_t)(out_capacity_pts < n ? out_capacity_pts : n);
  if (mem_out == LB_MEM_HOST) {
    LB_TRY(h->d_out.ensure(bytes));
    d_out = h->d_out.p; capacity = n;
    if (out_voxel_idx) { LB_TRY(h->d_vidx.ensure(n)); d_vidx = h->d_vidx.p; }
  }
  const uint32_t seg_tiles = (uint32_t)cdiv(n, VG_SEG_TILE);
  LB_TRY(h->keys.ensure(n)); LB_TRY(h->seg_status.ensure(seg_tiles));
  LB_TRY(radix_sort_reserve(c, h->sort, n));
  const bool four = F.n_ff == 4;
  if (four) LB_TRY(h->rec.ensure(n));
  if (!four && (n_inputs > 1 || any_T)) {
    set_error("lb_voxel_filter_merged: merging / transforming inputs needs the x, y, z, intensity layout (4 averaged FLOAT32 fields)");
    return LB_ERR_UNSUPPORTED;
  }
  if (four && any_T && !(F.ff_off[0] == (uint32_t)xo && F.ff_off[1] == (uint32_t)yo && F.ff_off[2] == (uint32_t)zo)) {
    set_error("lb_voxel_filter_merged: x, y, z must be the first three FLOAT32 fields when inputs are transformed");
    return LB_ERR_UNSUPPORTED;
  }
  // 32-byte records on 16-byte aligned bases: two 16-byte loads per point instead of 4-byte strided ones
  int vec32 = point_step == 32 ? 1 : 0;
  for (int i = 0; i < n_inputs; i++) if (reinterpret_cast<uintptr_t>(vin.base[i]) & 15u) vec32 = 0;
  VoxLimits lim;
  lim.ff_off = ffo; lim.fmin = (float)h->lim_min; lim.fmax = (float)h->lim_max; lim.dmin = h->lim_min; lim.dmax = h->lim_max;
  lim.negative = h->negative;
  const float inv0 = 1.0f / h->leaf[0], inv1 = 1.0f / h->leaf[1], inv2 = 1.0f / h->leaf[2];
  // ---- one stream-ordered chain, no host round trip until the end.  The sort's key width follows from the bounding
  // box, i.e. it is known on the device only; passes are enqueued for the width the previous call needed (consecutive
  // scans of a stream have the same extent), passes beyond the actual width return at once, and in the rare case that
  // this call needs MORE passes than were enqueued the chain is simply run again with all four.
  for (int attempt = 0; attempt < 2; attempt++) {
    const int launched_bits = attempt == 0 ? h->bits_hint : 32;
    const int bb_blocks = min(cdiv(n, 256), c.sm_count * 4);
    vg_bbox_kernel<<<bb_blocks, 256, 0, c.stream>>>(vin, n, point_step, (uint32_t)xo, lim, h->body, inv0, inv1, inv2, vec32, h->d_st);
    vg_keys_kernel<<<cdiv(n, 256 * VG_KEYS_ITEMS), 256, 0, c.stream>>>(vin, n, point_step, (uint32_t)xo, lim, h->body, inv0, inv1, inv2,
                                                                        vec32, F, h->d_st, h->keys.p, four ? h->rec.p : nullptr,
                                                                        h->sort.dev(), h->sort.status(), rs_tiles(n),
                                                                        h->seg_status.p, seg_tiles);
    c.launches += 2;
    LB_TRY(radix_sort_pairs_devbits(c, h->sort, h->keys.p, n, launched_bits, &h->d_st->key_bits));
    const uint32_t *ka = h->sort.ka.p, *kb = h->sort.kb.p, *va = h->sort.va.p, *vb = h->sort.vb.p;
    if (four)
      vg_segment_kernel<true><<<seg_tiles, 256, 0, c.stream>>>(vin, point_step, ka, kb, va, vb, h->rec.p, h->d_st, h->h_st, h->seg_status.p,
                                                              n, h->min_points, F, capacity, vec32, d_out, d_vidx);
    else
      vg_segment_kernel<false><<<seg_tiles, 256, 0, c.stream>>>(vin, point_step, ka, kb, va, vb, nullptr, h->d_st, h->h_st, h->seg_status.p,
                                                               n, h->min_points, F, capacity, vec32, d_out, d_vidx);
    c.launches++;
    LB_CUDA(cudaGetLastError());
    if (mem_out != LB_MEM_HOST) LB_CUDA(cudaEventRecord(h->ev1, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));        // the one synchronisation of a device-to-device call
    if (h->h_st->key_bits <= launched_bits) break;   // every pass the key needs was enqueued
  }
  if (h->h_st->key_bits > 0) h->bits_hint = ((h->h_st->key_bits + 7) / 8) * 8;
  if (h->h_st->status != LB_OK) {
    set_error("lb_voxel_filter: leaf size too small for the input dataset, integer indices would overflow");
    return LB_ERR_VOXEL_OVERFLOW;
  }
  size_t m = h->h_st->key_bits ? h->h_st->n_final : 0;
  if (m > out_capacity_pts) {
    set_error("lb_voxel_filter: output capacity %zu < %zu voxels", out_capacity_pts, m);
    return LB_ERR_CAPACITY;
  }
  if (mem_out == LB_MEM_HOST) {
    if (m > 0) {
      LB_CUDA(cudaMemcpyAsync(out, d_out, m * point_step, cudaMemcpyDeviceToHost, c.stream));
      if (out_voxel_idx) LB_CUDA(cudaMemcpyAsync(out_voxel_idx, d_vidx, m * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    }
    LB_CUDA(cudaEventRecord(h->ev1, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  cudaEventElapsedTime(&h->t_last_ms, h->ev0, h->ev1);
  h->t_sum_ms += h->t_last_ms; h->t_calls++;
  *n_out = m;
  return LB_OK;
}

}  // extern "C"
