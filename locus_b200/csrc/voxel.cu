// voxel.cu -- VoxelGrid front-end (kernel K1): hash-and-centroid reduce.
//
// Replaces pcl::VoxelGrid<pcl::PCLPointCloud2>::applyFilter as driven by
// point_cloud_filter/src/custom_voxel_grid.cc:76-87 (index arithmetic cross-
// checked with multithreaded_ndt/voxel_grid_covariance_omp_impl.hpp:67-164).
//
// One call = one stream-ordered chain of kernels with NO host round trip in between: everything a later kernel needs
// from an earlier one (bounding box -> min_b / div_b / key width, voxel count) stays in a small device-resident state
// block; the host synchronises once, at the end, to learn the voxel count and the status.
//   vg_bbox_kernel     finite + filter-limit + body-box predicate, min/max reduce (two 16-byte loads per 32-byte
//                      record); the last CTA derives min_b, div_b, the overflow guard and the key width
//   vg_keys_kernel     int32 PCL leaf index per point (bit-exact float32 math) + a packed float4 record of the four
//                      averaged fields, so that no later kernel touches the raw cloud's strided layout again
//   radix sort         stable LSD sort of (leaf index, point#); passes beyond the key width return at once
//   vg_tile_heads_kernel + vg_segstart_kernel    voxel segments (per-tile head counts, then prefix + local scan)
//   vg_centroid4_kernel   a warp owns 32 consecutive voxels: float32 sum in ascending point order, / count
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

// device-resident state of one lb_voxel_filter call (written by the kernels, read back once at the end)
struct VoxState {
  BBoxAcc acc;                 // bounding box of the surviving points; reset by the CTA that consumes it
  unsigned ticket;             // last-CTA detection of vg_bbox_kernel
  int status;                  // LB_OK or LB_ERR_VOXEL_OVERFLOW
  int min_b[3], div_b[3];
  uint32_t sentinel;           // number of cells of the grid = key of a dropped point (sorts last)
  int key_bits;                // width of the sort key; 0: nothing to do (empty input / overflow)
  uint32_t count;              // surviving points
  uint32_t n_seg;              // occupied voxels
  uint32_t n_final;            // output points (after min_points_per_voxel)
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
  st->n_seg = 0; st->n_final = 0;
  bbox_reset(&st->acc);            // consumed: clean for the next call
  st->ticket = 0;
}

__global__ void __launch_bounds__(256)
vg_keys_kernel(const __grid_constant__ VoxInputs in, uint32_t n, uint32_t stride, uint32_t xyz_off, VoxLimits lim, BodyBox body,
               float inv0, float inv1, float inv2, int vec32, VoxelFieldsDev F, const VoxState* __restrict__ st,
               uint32_t* __restrict__ keys, float4* __restrict__ rec /*nullable: only for 4 averaged fields*/) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const int key_bits = st->key_bits;
  if (key_bits == 0 || i >= n) return;              // empty input or overflow: nothing is sorted
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
  keys[i] = key;
  if (rec) rec[i] = r4;
}

// which ping-pong buffer holds the sorted pairs: A after an odd number of executed passes, B after an even number
__device__ __forceinline__ bool vg_sorted_in_a(int key_bits) { return (((key_bits + 7) >> 3) & 1) != 0; }

constexpr int VG_TILE = 2048;      // sorted positions per CTA of the two segment kernels (256 threads x 8)

__device__ __forceinline__ uint32_t vg_head_flags8(const uint32_t* __restrict__ keys, uint32_t base, uint32_t n, uint32_t sentinel,
                                                   uint32_t* cnt) {
  // 8 consecutive sorted positions per thread; bit j: position base + j starts a voxel
  uint32_t bits = 0, c = 0;
  uint32_t prev = (base > 0 && base <= n) ? keys[base - 1] : 0xffffffffu;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint32_t i = base + j;
    if (i < n) {
      const uint32_t k = keys[i];
      if (k < sentinel && (i == 0 || k != prev)) { bits |= 1u << j; c++; }
      prev = k;
    }
  }
  *cnt = c;
  return bits;
}

__global__ void __launch_bounds__(256)
vg_tile_heads_kernel(const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb, const VoxState* __restrict__ st, uint32_t n,
                     uint32_t* __restrict__ tile_cnt) {
  __shared__ uint32_t sm[256 / 32 + 1];
  const int key_bits = st->key_bits;
  if (key_bits == 0) { if (threadIdx.x == 0) tile_cnt[blockIdx.x] = 0; return; }
  const uint32_t* keys = vg_sorted_in_a(key_bits) ? ka : kb;
  uint32_t c;
  vg_head_flags8(keys, blockIdx.x * VG_TILE + threadIdx.x * 8, n, st->sentinel, &c);
  uint32_t tot;
  block_excl_scan<256>(c, &tot, sm);
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = tot;
}

// seg_start[s] = sorted position where voxel s begins; the last CTA publishes the voxel count
__global__ void __launch_bounds__(256)
vg_segstart_kernel(const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb, VoxState* __restrict__ st, uint32_t n,
                   const uint32_t* __restrict__ tile_cnt, uint32_t* __restrict__ seg_start) {
  __shared__ uint32_t sm[256 / 32 + 1];
  __shared__ uint32_t pre_s;
  const int key_bits = st->key_bits;
  if (key_bits == 0) return;
  const uint32_t* keys = vg_sorted_in_a(key_bits) ? ka : kb;
  // voxels that start in earlier tiles
  uint32_t part = 0;
  for (uint32_t b = threadIdx.x; b < blockIdx.x; b += 256) part += tile_cnt[b];
  uint32_t pre;
  block_excl_scan<256>(part, &pre, sm);
  if (threadIdx.x == 0) pre_s = pre;
  uint32_t c;
  const uint32_t base = blockIdx.x * VG_TILE + threadIdx.x * 8;
  const uint32_t bits = vg_head_flags8(keys, base, n, st->sentinel, &c);
  uint32_t tot;
  uint32_t s = block_excl_scan<256>(c, &tot, sm) + pre_s;
#pragma unroll
  for (int j = 0; j < 8; j++)
    if (bits & (1u << j)) seg_start[s++] = base + j;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) { st->n_seg = pre_s + tot; st->n_final = pre_s + tot; }
}

// keep[s] = 1 iff voxel s holds >= min_points points
__global__ void __launch_bounds__(256)
vg_keep_kernel(const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb, const uint32_t* __restrict__ seg_start,
               const VoxState* __restrict__ st, uint32_t n, int min_points, uint32_t* __restrict__ keep) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t* keys = vg_sorted_in_a(st->key_bits) ? ka : kb;
  uint32_t n_seg = st->n_seg;
  if (s >= n_seg) { if (s < n) keep[s] = 0; return; }
  uint32_t a = seg_start[s];
  uint32_t k = keys[a];
  uint32_t e = a + 1;
  while (e < n && keys[e] == k) e++;
  keep[s] = ((int)(e - a) >= min_points) ? 1u : 0u;
}

// The common record layout (x, y, z, intensity averaged: 16-byte records).  A warp owns 32 consecutive voxels, i.e.
// ONE contiguous range of sorted positions: the warp stages the records of that range in shared memory (the packed
// float4 records written by vg_keys_kernel, fetched through the sorted point numbers: 16-byte gathers from an
// L2-resident array), and every lane then adds up its own voxel's records from shared memory in ascending input order
// (the order defines the float32 rounding) -- no per-lane chains of dependent global loads.
constexpr int VG4_TILE = 256;       // records per warp tile (4 KB)
__global__ void __launch_bounds__(128)
vg_centroid4_kernel(const __grid_constant__ VoxInputs in, uint32_t stride, const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb,
                    const uint32_t* __restrict__ va, const uint32_t* __restrict__ vb, const float4* __restrict__ rec,
                    const uint32_t* __restrict__ seg_start, const VoxState* __restrict__ st,
                    const uint32_t* __restrict__ slot /*nullable*/, const uint32_t* __restrict__ keep /*nullable*/,
                    uint32_t n, VoxelFieldsDev F, uint32_t capacity, int vec32, uint8_t* __restrict__ out,
                    int32_t* __restrict__ out_voxel_idx) {
  __shared__ float4 tile[4][VG4_TILE];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t n_seg = st->n_seg;
  const uint32_t s0 = (blockIdx.x * 4 + wib) * 32;
  if (s0 >= n_seg) return;                                  // whole warp
  const bool in_a = vg_sorted_in_a(st->key_bits);
  const uint32_t* keys = in_a ? ka : kb;
  const uint32_t* vals = in_a ? va : vb;
  const uint32_t s = s0 + lane;
  const bool seg = s < n_seg;
  uint32_t a = 0, e = 0, k = 0;
  if (seg) {
    a = seg_start[s];
    k = keys[a];
    // segment end: next segment's start, or the first sentinel key after the last voxel
    if (s + 1 < n_seg) e = seg_start[s + 1];
    else { e = a + 1; while (e < n && keys[e] == k) e++; }
  }
  const uint32_t n_act = min(32u, n_seg - s0);
  const uint32_t r0 = __shfl_sync(0xffffffffu, a, 0);
  const uint32_t r1 = __shfl_sync(0xffffffffu, e, (int)n_act - 1);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (uint32_t t0 = r0; t0 < r1; t0 += VG4_TILE) {
    const uint32_t t1 = min(r1, t0 + (uint32_t)VG4_TILE);
    // a tile is 8 records per lane: all 8 point numbers, then all 8 records, are in flight at once (a loop of
    // load -> store pairs would expose one memory latency per record)
    {
      uint32_t pv[VG4_TILE / 32];
      float4 rv[VG4_TILE / 32];
#pragma unroll
      for (int u = 0; u < VG4_TILE / 32; u++) {
        const uint32_t i = t0 + lane + 32u * u;
        pv[u] = (i < t1) ? vals[i] : 0xffffffffu;
      }
#pragma unroll
      for (int u = 0; u < VG4_TILE / 32; u++) rv[u] = (pv[u] != 0xffffffffu) ? rec[pv[u]] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < VG4_TILE / 32; u++) tile[wib][lane + 32 * u] = rv[u];
    }
    __syncwarp();
    if (seg) {
      uint32_t lo = max(a, t0), hi = min(e, t1);
      if (lo < hi && lo == a) { acc = tile[wib][lo - t0]; lo++; }      // the sum starts from the first record itself
      for (; lo + 4 <= hi; lo += 4) {
        const float4 v0 = tile[wib][lo - t0], v1 = tile[wib][lo + 1 - t0], v2 = tile[wib][lo + 2 - t0], v3 = tile[wib][lo + 3 - t0];
        acc.x = acc.x + v0.x; acc.y = acc.y + v0.y; acc.z = acc.z + v0.z; acc.w = acc.w + v0.w;
        acc.x = acc.x + v1.x; acc.y = acc.y + v1.y; acc.z = acc.z + v1.z; acc.w = acc.w + v1.w;
        acc.x = acc.x + v2.x; acc.y = acc.y + v2.y; acc.z = acc.z + v2.z; acc.w = acc.w + v2.w;
        acc.x = acc.x + v3.x; acc.y = acc.y + v3.y; acc.z = acc.z + v3.z; acc.w = acc.w + v3.w;
      }
      for (; lo < hi; lo++) {
        const float4 v = tile[wib][lo - t0];
        acc.x = acc.x + v.x; acc.y = acc.y + v.y; acc.z = acc.z + v.z; acc.w = acc.w + v.w;
      }
    }
    __syncwarp();
  }
  if (!seg) return;
  if (keep && !keep[s]) return;
  const uint32_t o = slot ? slot[s] : s;
  if (o >= capacity) return;
  const float cnt = (float)(e - a);
  int cfirst;
  const uint8_t* first = vg_point(in, vals[a], stride, cfirst);
  uint8_t* dst = out + (size_t)o * stride;
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
  if (out_voxel_idx) out_voxel_idx[o] = (int32_t)k;
}

// Any other set of averaged fields: one thread per voxel, float32 sum of its points in ascending input order (the order
// the stable sort produced), read straight from the caller's layout through the sorted point numbers; divide by the
// count (centroid /= float(n), PCL), write the output point.
__global__ void __launch_bounds__(128)
vg_centroid_kernel(const uint8_t* __restrict__ in, uint32_t stride, const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb,
                   const uint32_t* __restrict__ va, const uint32_t* __restrict__ vb,
                   const uint32_t* __restrict__ seg_start, const VoxState* __restrict__ st,
                   const uint32_t* __restrict__ slot /*nullable*/, const uint32_t* __restrict__ keep /*nullable*/,
                   uint32_t n, VoxelFieldsDev F, uint32_t capacity, uint8_t* __restrict__ out,
                   int32_t* __restrict__ out_voxel_idx) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n_seg = st->n_seg;
  if (s >= n_seg) return;
  if (keep && !keep[s]) return;
  uint32_t o = slot ? slot[s] : s;
  if (o >= capacity) return;
  const bool in_a = vg_sorted_in_a(st->key_bits);
  const uint32_t* keys = in_a ? ka : kb;
  const uint32_t* vals = in_a ? va : vb;
  uint32_t a = seg_start[s];
  uint32_t k = keys[a];
  // segment end: next segment's start, or the first sentinel key after the last voxel
  uint32_t e;
  if (s + 1 < n_seg) e = seg_start[s + 1];
  else { e = a + 1; while (e < n && keys[e] == k) e++; }
  float acc[VG_MAX_FIELDS];
  const int nf = F.n_ff;
  const uint8_t* first = in + (size_t)vals[a] * stride;
#pragma unroll
  for (int f = 0; f < VG_MAX_FIELDS; f++) acc[f] = (f < nf) ? *reinterpret_cast<const float*>(first + F.ff_off[f]) : 0.f;
  for (uint32_t j = a + 1; j < e; j++) {
    const uint8_t* p = in + (size_t)vals[j] * stride;
#pragma unroll
    for (int f = 0; f < VG_MAX_FIELDS; f++)
      if (f < nf) acc[f] = acc[f] + *reinterpret_cast<const float*>(p + F.ff_off[f]);
  }
  float cnt = (float)(e - a);
  uint8_t* dst = out + (size_t)o * stride;
  // bytes not covered by an averaged field come from the voxel's first point
  for (uint32_t w = 0; w < stride / 4; w++)
    reinterpret_cast<uint32_t*>(dst)[w] = reinterpret_cast<const uint32_t*>(first)[w];
#pragma unroll
  for (int f = 0; f < VG_MAX_FIELDS; f++)
    if (f < nf) *reinterpret_cast<float*>(dst + F.ff_off[f]) = acc[f] / cnt;
  if (out_voxel_idx) out_voxel_idx[o] = (int32_t)k;
}

__global__ void vg_state_init_kernel(VoxState* st) {
  if (threadIdx.x == 0) {
    bbox_reset(&st->acc);
    st->ticket = 0; st->status = 0; st->sentinel = 0; st->key_bits = 0; st->count = 0; st->n_seg = 0; st->n_final = 0;
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
  DBuf<uint32_t> keys, tile_cnt, seg_start, keep, slot;
  DBuf<float4> rec;
  VoxState* d_st = nullptr;     // device
  VoxState* h_st = nullptr;     // pinned
  int bits_hint = 32;           // sort passes to enqueue: the key width of the previous call, rounded up to whole passes
  SortWork sort;
  ScanWork scan;
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

extern "C" {

int lb_voxel_create(int device, lb_voxel** h) { return voxel_create_impl(device, nullptr, false, h); }
int lb_voxel_create_on_stream(int device, void* stream, lb_voxel** h) { return voxel_create_impl(device, stream, true, h); }

int lb_voxel_destroy(lb_voxel* h) {
  if (!h) return LB_OK;
  cudaSetDevice(h->c.device);
  cudaStreamSynchronize(h->c.stream);
  h->d_in.release(); h->d_out.release(); h->d_vidx.release(); h->keys.release(); h->tile_cnt.release();
  h->seg_start.release(); h->keep.release(); h->slot.release(); h->rec.release();
  h->sort.ka.release(); h->sort.kb.release(); h->sort.va.release(); h->sort.vb.release(); h->sort.hist.release();
  h->sort.scan.sums.release(); h->scan.sums.release();
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
  const uint32_t ntiles = (uint32_t)cdiv(n, VG_TILE);
  LB_TRY(h->keys.ensure(n)); LB_TRY(h->seg_start.ensure(n)); LB_TRY(h->tile_cnt.ensure(ntiles));
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
  const uint8_t* d_in = vin.base[0];
  VoxLimits lim;
  lim.ff_off = ffo; lim.fmin = (float)h->lim_min; lim.fmax = (float)h->lim_max; lim.dmin = h->lim_min; lim.dmax = h->lim_max;
  lim.negative = h->negative;
  const float inv0 = 1.0f / h->leaf[0], inv1 = 1.0f / h->leaf[1], inv2 = 1.0f / h->leaf[2];
  // ---- one stream-ordered chain, no host round trip until the end.  The sort's key width follows from the bounding
  // box, i.e. it is known on the device only; passes are enqueued for the width the previous call needed (consecutive
  // scans of a stream have the same extent), passes beyond the actual width return at once, and in the rare case that
  // this call needs MORE passes than were enqueued the chain is simply run again with all four.
  const uint32_t *ka = nullptr, *kb = nullptr, *va = nullptr, *vb = nullptr;
  for (int attempt = 0; attempt < 2; attempt++) {
    const int launched_bits = attempt == 0 ? h->bits_hint : 32;
    const int bb_blocks = min(cdiv(n, 256), c.sm_count * 4);
    vg_bbox_kernel<<<bb_blocks, 256, 0, c.stream>>>(vin, n, point_step, (uint32_t)xo, lim, h->body, inv0, inv1, inv2, vec32, h->d_st);
    vg_keys_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(vin, n, point_step, (uint32_t)xo, lim, h->body, inv0, inv1, inv2, vec32, F,
                                                       h->d_st, h->keys.p, four ? h->rec.p : nullptr);
    c.launches += 2;
    LB_TRY(radix_sort_pairs_devbits(c, h->sort, h->keys.p, n, launched_bits, &h->d_st->key_bits));
    ka = h->sort.ka.p; kb = h->sort.kb.p; va = h->sort.va.p; vb = h->sort.vb.p;
    vg_tile_heads_kernel<<<ntiles, 256, 0, c.stream>>>(ka, kb, h->d_st, n, h->tile_cnt.p);
    vg_segstart_kernel<<<ntiles, 256, 0, c.stream>>>(ka, kb, h->d_st, n, h->tile_cnt.p, h->seg_start.p);
    c.launches += 2;
    const uint32_t* slot = nullptr; const uint32_t* keep = nullptr;
    if (h->min_points > 1) {
      LB_TRY(h->keep.ensure(n)); LB_TRY(h->slot.ensure(n));
      vg_keep_kernel<<<cdiv(n, 256), 256, 0, c.stream>>>(ka, kb, h->seg_start.p, h->d_st, n, h->min_points, h->keep.p);
      c.launches++;
      LB_TRY(exclusive_scan_u32(c, h->scan, h->keep.p, h->slot.p, n, &h->d_st->n_final));
      slot = h->slot.p; keep = h->keep.p;
    }
    if (four)
      vg_centroid4_kernel<<<cdiv(n, 128), 128, 0, c.stream>>>(vin, point_step, ka, kb, va, vb, h->rec.p, h->seg_start.p, h->d_st,
                                                               slot, keep, n, F, capacity, vec32, d_out, d_vidx);
    else
      vg_centroid_kernel<<<cdiv(n, 128), 128, 0, c.stream>>>(d_in, point_step, ka, kb, va, vb, h->seg_start.p, h->d_st, slot, keep,
                                                              n, F, capacity, d_out, d_vidx);
    c.launches++;
    LB_CUDA(cudaGetLastError());
    LB_CUDA(cudaMemcpyAsync(h->h_st, h->d_st, sizeof(VoxState), cudaMemcpyDeviceToHost, c.stream));
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
