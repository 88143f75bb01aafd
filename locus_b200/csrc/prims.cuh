// prims.cuh -- device-wide primitives shared by the VoxelGrid and GICP paths:
// stream context + growable device buffers, bounding-box reduction, stable LSD
// radix sort of (key, value) pairs, exclusive scan.  All hand-written for
// sm_90a; no CUB/Thrust on the product path.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/locus_b200.h"
#include "hd.h"

namespace lb {

// ------------------------------------------------------------------ errors
void set_error(const char* fmt, ...);

#define LB_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      lb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return LB_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

#define LB_TRY(call)            \
  do {                          \
    int s__ = (call);           \
    if (s__ != LB_OK) return s__; \
  } while (0)

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint64_t launches = 0;
  int sm_count = 132;
};

int ctx_init(Ctx& c, int device, void* external_stream, bool use_external);
void ctx_destroy(Ctx& c);

// device allocations made by DBuf::ensure since the library was loaded (a steady-state call path must not add any)
unsigned long long& dbuf_alloc_count();

template <class T>
struct DBuf {
  T* p = nullptr;
  size_t cap = 0;
  int ensure(size_t n) {
    if (n <= cap) return LB_OK;
    dbuf_alloc_count()++;
    static const bool trace = getenv("LB_ALLOC_TRACE") != nullptr;      // tuning aid: which buffer still grows in steady state
    if (trace) fprintf(stderr, "[lb alloc] %zu x %zu bytes requested (capacity was %zu)\n", n, sizeof(T), cap);
    size_t nc = cap ? cap : 1024;
    while (nc < n) nc = nc + nc / 2 + 1024;
    if (p) LB_CUDA(cudaFree(p));
    p = nullptr; cap = 0;
    LB_CUDA(cudaMalloc((void**)&p, nc * sizeof(T)));
    cap = nc;
    return LB_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------ bbox
// ordered-uint encoding of float so that unsigned min/max == float min/max
__device__ __forceinline__ uint32_t f2ord(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float f; memcpy(&f, &b, 4); return f;
#endif
}

struct BBoxAcc {          // device-resident accumulator, 8 words
  uint32_t mn[3], mx[3];
  uint32_t count, pad;
};

__global__ void bbox_init_kernel(BBoxAcc* acc);

// accumulate one point into warp-level then global bounding box (call with all 32 lanes; valid = lane has a point)
__device__ __forceinline__ void bbox_warp_accumulate(bool valid, float x, float y, float z, BBoxAcc* acc) {
  uint32_t mn0 = 0xffffffffu, mn1 = 0xffffffffu, mn2 = 0xffffffffu, mx0 = 0, mx1 = 0, mx2 = 0, cnt = 0;
  if (valid) { mn0 = mx0 = f2ord(x); mn1 = mx1 = f2ord(y); mn2 = mx2 = f2ord(z); cnt = 1; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, o));
    mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, o));
    mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
    mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt > 0) {
    atomicMin(&acc->mn[0], mn0); atomicMin(&acc->mn[1], mn1); atomicMin(&acc->mn[2], mn2);
    atomicMax(&acc->mx[0], mx0); atomicMax(&acc->mx[1], mx1); atomicMax(&acc->mx[2], mx2);
    atomicAdd(&acc->count, cnt);
  }
}
__device__ __forceinline__ void bbox_reset(BBoxAcc* acc) {
  acc->mn[0] = acc->mn[1] = acc->mn[2] = 0xffffffffu;
  acc->mx[0] = acc->mx[1] = acc->mx[2] = 0u;
  acc->count = 0; acc->pad = 0;
}

// Finite-point bounding box of a strided cloud (x,y,z float32 at xyz_off).
// Optional limit filter (VoxelGrid getMinMax3D): field value v at ff_off is
// dropped if  negative ? (v < fmax && v > fmin) : (v > fmax || v < fmin), float compare.
__global__ void bbox_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off,
                            int ff_off, float fmin, float fmax, int negative, BodyBox body, BBoxAcc* acc);

// ------------------------------------------------------------------ scan
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) >= o) v += t;
  }
  return v;
}

// exclusive scan of one value per thread across the block; returns exclusive prefix, total in *total
template <int T>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total, uint32_t* smem /*T/32+1*/) {
  uint32_t incl = warp_incl_scan(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 31) smem[w] = incl;
  __syncthreads();
  if (w == 0) {
    uint32_t s = (l < T / 32) ? smem[l] : 0;
    uint32_t si = warp_incl_scan(s);
    if (l < T / 32) smem[l] = si - s;
    if (l == T / 32 - 1) smem[T / 32] = si;
  }
  __syncthreads();
  uint32_t r = smem[w] + incl - v;
  *total = smem[T / 32];
  __syncthreads();
  return r;
}

// Exclusive scan of n uint32 (in may alias out).  total (nullable, device) receives the grand total.
struct ScanWork { DBuf<uint32_t> sums; };
int exclusive_scan_u32(Ctx& c, ScanWork& w, const uint32_t* in, uint32_t* out, size_t n, uint32_t* total_dev);

// ------------------------------------------------------------------ decoupled look-back
// A tile status word: LB_NOT_READY, or a count of the tile alone (bit 31 clear) or the inclusive prefix over the tile
// and every tile before it (bit 31 set).  Counts stay below 2^31 - 1, so no published word equals LB_NOT_READY.
constexpr uint32_t LB_NOT_READY = 0xffffffffu, LB_PREFIX = 0x80000000u;

__device__ __forceinline__ void lookback_publish(uint32_t* w, uint32_t v) { *reinterpret_cast<volatile uint32_t*>(w) = v; }

// Exclusive prefix of tile `tile` from the status words of the tiles before it (word of tile j at status[j * stride]).
// Tile ids come from an atomic ticket taken at CTA start, so every tile waited on has started and publishes its own
// count without waiting on anyone: the walk always ends.
__device__ __forceinline__ uint32_t lookback_prefix(const uint32_t* status, size_t stride, uint32_t tile) {
  uint32_t excl = 0;
  for (int64_t j = (int64_t)tile - 1; j >= 0;) {
    const uint32_t s = *reinterpret_cast<const volatile uint32_t*>(status + (size_t)j * stride);
    if (s == LB_NOT_READY) continue;
    excl += s & ~LB_PREFIX;
    if (s & LB_PREFIX) break;
    j--;
  }
  return excl;
}

// ------------------------------------------------------------------ sort
// Stable LSD radix sort of (key, val) pairs on the low `key_bits` bits, 8-bit digits, one sweep per pass: one read of
// the keys fills every pass's digit histogram, then each pass is ONE scatter kernel whose tiles find their global digit
// offsets by decoupled look-back over per-tile, per-digit status words.
// vals_in == nullptr means val = element index.  Result ends in *keys_out/*vals_out
// (pointers into the ping-pong buffers a/b).
constexpr int RS_PASSES_MAX = 4;
constexpr int RS_TILE = 2048;              // keys per scatter tile (256 threads x 8)

// Device state of one SortWork, followed in memory by the tile status words (RS_PASSES_MAX x tiles x 256).
// Invariant between sorts: `acc` and `hist_ticket` are zero.  The histogram's last CTA turns `acc` into `base` and
// zeroes it; the kernel that fills the histogram also resets the status words and `tile_ticket` of the passes after it.
struct RsDev {
  uint32_t acc[RS_PASSES_MAX][256];        // digit counts of every pass (atomics of the histogram CTAs)
  uint32_t base[RS_PASSES_MAX][256];       // exclusive digit offsets of every pass (read by the scatters)
  uint32_t hist_ticket;                    // last-CTA detection of the histogram
  uint32_t tile_ticket[RS_PASSES_MAX];     // tile ids of the scatter passes
  uint32_t pad[3];
};
constexpr size_t RS_DEV_WORDS = sizeof(RsDev) / 4;

struct SortWork {
  DBuf<uint32_t> ka, kb, va, vb;
  DBuf<uint32_t> state;                    // RsDev + status words
  uint32_t tiles_cap = 0;                  // tiles the status words are sized for
  RsDev* dev() const { return reinterpret_cast<RsDev*>(state.p); }
  uint32_t* status() const { return state.p + RS_DEV_WORDS; }
};
static inline uint32_t rs_tiles(size_t n) { uint32_t t = (uint32_t)((n + RS_TILE - 1) / RS_TILE); return t ? t : 1; }

// Buffers for n keys (grown, never shrunk; a fresh state block is zeroed once, on the stream).
int radix_sort_reserve(Ctx& c, SortWork& w, size_t n);

// ---- the histogram, for kernels that already touch every key (256-thread CTAs)
// sh: __shared__ uint32_t[RS_PASSES_MAX][256], zeroed and synchronised by the caller.  All 32 lanes call it.
__device__ __forceinline__ void rs_hist_warp_add(uint32_t (*sh)[256], uint32_t key, bool valid, int passes) {
#pragma unroll
  for (int p = 0; p < RS_PASSES_MAX; p++) {
    if (p >= passes) break;
    const uint32_t d = valid ? ((key >> (8 * p)) & 255u) : 256u;
    const uint32_t m = __match_any_sync(0xffffffffu, d);
    if (d < 256u && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&sh[p][d], (uint32_t)__popc(m));
  }
}
// After the CTA's keys are in `sh`: one global atomic per non-zero digit, then the last CTA of the grid turns the
// totals into exclusive digit offsets and restores the zero invariant.  Call with the whole CTA (256 threads).
__device__ __forceinline__ void rs_hist_flush(uint32_t (*sh)[256], RsDev* rs, int passes, uint32_t* scan_sm /*9*/, bool* last_sm) {
  __syncthreads();
  const uint32_t d = threadIdx.x;
  for (int p = 0; p < passes; p++)
    if (sh[p][d]) atomicAdd(&rs->acc[p][d], sh[p][d]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *last_sm = atomicAdd(&rs->hist_ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!*last_sm) return;
  __threadfence();
  for (int p = 0; p < passes; p++) {
    const uint32_t v = atomicExch(&rs->acc[p][d], 0u);
    uint32_t tot;
    rs->base[p][d] = block_excl_scan<256>(v, &tot, scan_sm);
  }
  if (threadIdx.x == 0) rs->hist_ticket = 0;
}
// Status words and tile tickets of the scatters that follow (grid-stride; any grid that runs before them).
__device__ __forceinline__ void rs_reset_lookback(RsDev* rs, uint32_t* status, uint32_t tiles) {
  const size_t words = (size_t)RS_PASSES_MAX * tiles * 256;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x)
    status[i] = LB_NOT_READY;
  if (blockIdx.x == 0 && threadIdx.x < RS_PASSES_MAX) rs->tile_ticket[threadIdx.x] = 0;
}

int radix_sort_pairs(Ctx& c, SortWork& w, const uint32_t* keys_in, const uint32_t* vals_in, size_t n, int key_bits,
                     uint32_t** keys_out, uint32_t** vals_out);
// The scatter passes only (val = element index), for a caller whose own key kernel filled the histogram
// (rs_hist_warp_add / rs_hist_flush) and reset the look-back (rs_reset_lookback) after radix_sort_reserve.
int radix_sort_scatter(Ctx& c, SortWork& w, const uint32_t* keys_in, size_t n, int key_bits, uint32_t** keys_out, uint32_t** vals_out);
// The same when the key width is only known on the device: passes for max_key_bits are launched, those beyond *key_bits_dev return at once.
// Result: buffers w.ka / w.va after an odd number of executed passes ((*key_bits_dev + 7) / 8), w.kb / w.vb after an
// even number; consumers pick on the device.
int radix_sort_pairs_devbits(Ctx& c, SortWork& w, const uint32_t* keys_in, size_t n, int max_key_bits, const int* key_bits_dev);

}  // namespace lb
