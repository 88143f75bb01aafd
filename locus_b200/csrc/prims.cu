// prims.cu -- implementations of the device-wide primitives (see prims.cuh).
#include <stdarg.h>

#include "prims.cuh"

namespace lb {

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }
unsigned long long& dbuf_alloc_count() { static unsigned long long n = 0; return n; }

int ctx_init(Ctx& c, int device, void* external_stream, bool use_external) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    set_error("no CUDA device available (%s): the product path has no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return LB_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= n) { set_error("device %d out of range (%d devices)", device, n); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(device));
  c.device = device;
  if (use_external) {
    c.stream = (cudaStream_t)external_stream;
    c.own_stream = false;
  } else {
    LB_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    c.own_stream = true;
  }
  cudaDeviceProp prop;
  LB_CUDA(cudaGetDeviceProperties(&prop, device));
  c.sm_count = prop.multiProcessorCount;
  c.launches = 0;
  return LB_OK;
}

void ctx_destroy(Ctx& c) {
  if (c.own_stream && c.stream) cudaStreamDestroy(c.stream);
  c.stream = nullptr;
}

// ------------------------------------------------------------------ bbox
__global__ void bbox_init_kernel(BBoxAcc* acc) {
  if (threadIdx.x < 3) { acc->mn[threadIdx.x] = 0xffffffffu; acc->mx[threadIdx.x] = 0u; }
  if (threadIdx.x == 3) { acc->count = 0; acc->pad = 0; }
}

__global__ void __launch_bounds__(256)
bbox_kernel(const uint8_t* __restrict__ base, uint32_t n, uint32_t stride, uint32_t xyz_off,
            int ff_off, float fmin, float fmax, int negative, BodyBox body, BBoxAcc* acc) {
  uint32_t mn0 = 0xffffffffu, mn1 = 0xffffffffu, mn2 = 0xffffffffu, mx0 = 0, mx1 = 0, mx2 = 0, cnt = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint8_t* p = base + (size_t)i * stride;
    if (ff_off >= 0) {
      float v = *reinterpret_cast<const float*>(p + ff_off);
      bool drop = negative ? (v < fmax && v > fmin) : (v > fmax || v < fmin);
      if (drop) continue;
    }
    const float* q = reinterpret_cast<const float*>(p + xyz_off);
    float x = q[0], y = q[1], z = q[2];
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) continue;
    if (body_box_drops(body, x, y, z)) continue;
    uint32_t ox = f2ord(x), oy = f2ord(y), oz = f2ord(z);
    mn0 = min(mn0, ox); mn1 = min(mn1, oy); mn2 = min(mn2, oz);
    mx0 = max(mx0, ox); mx1 = max(mx1, oy); mx2 = max(mx2, oz);
    cnt++;
  }
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
  // one set of atomics per CTA (same-address atomics serialise in L2)
  __shared__ uint32_t sm[8][7];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sm[w][0] = mn0; sm[w][1] = mn1; sm[w][2] = mn2; sm[w][3] = mx0; sm[w][4] = mx1; sm[w][5] = mx2; sm[w][6] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; i++) {
      mn0 = min(mn0, sm[i][0]); mn1 = min(mn1, sm[i][1]); mn2 = min(mn2, sm[i][2]);
      mx0 = max(mx0, sm[i][3]); mx1 = max(mx1, sm[i][4]); mx2 = max(mx2, sm[i][5]);
      cnt += sm[i][6];
    }
    if (cnt > 0) {
      atomicMin(&acc->mn[0], mn0); atomicMin(&acc->mn[1], mn1); atomicMin(&acc->mn[2], mn2);
      atomicMax(&acc->mx[0], mx0); atomicMax(&acc->mx[1], mx1); atomicMax(&acc->mx[2], mx2);
      atomicAdd(&acc->count, cnt);
    }
  }
}

// ------------------------------------------------------------------ scan
constexpr int SC_T = 256, SC_I = 8, SC_TILE = SC_T * SC_I;

__global__ void __launch_bounds__(SC_T) scan_reduce_kernel(const uint32_t* __restrict__ in, size_t n, uint32_t* sums) {
  __shared__ uint32_t sm[SC_T / 32 + 1];
  size_t base = (size_t)blockIdx.x * SC_TILE + (size_t)threadIdx.x * SC_I;
  uint32_t s = 0;
#pragma unroll
  for (int j = 0; j < SC_I; j++) if (base + j < n) s += in[base + j];
  uint32_t tot;
  block_excl_scan<SC_T>(s, &tot, sm);
  if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(1024) scan_spine_kernel(uint32_t* sums, size_t nb, uint32_t* total) {
  __shared__ uint32_t sm[1024 / 32 + 1];
  uint32_t carry = 0;
  for (size_t start = 0; start < nb; start += 1024 * 8) {
    size_t base = start + (size_t)threadIdx.x * 8;
    uint32_t v[8]; uint32_t s = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { v[j] = (base + j < nb) ? sums[base + j] : 0; s += v[j]; }
    uint32_t tot;
    uint32_t ex = block_excl_scan<1024>(s, &tot, sm) + carry;
#pragma unroll
    for (int j = 0; j < 8; j++) { if (base + j < nb) sums[base + j] = ex; ex += v[j]; }
    carry += tot;
  }
  if (threadIdx.x == 0 && total) *total = carry;
}

__global__ void __launch_bounds__(SC_T)
scan_down_kernel(const uint32_t* in, uint32_t* out, size_t n, const uint32_t* __restrict__ sums) {
  __shared__ uint32_t sm[SC_T / 32 + 1];
  size_t base = (size_t)blockIdx.x * SC_TILE + (size_t)threadIdx.x * SC_I;
  uint32_t v[SC_I]; uint32_t s = 0;
#pragma unroll
  for (int j = 0; j < SC_I; j++) { v[j] = (base + j < n) ? in[base + j] : 0; s += v[j]; }
  uint32_t tot;
  uint32_t ex = block_excl_scan<SC_T>(s, &tot, sm) + sums[blockIdx.x];
#pragma unroll
  for (int j = 0; j < SC_I; j++) { if (base + j < n) out[base + j] = ex; ex += v[j]; }
}

// whole scan in one CTA (n up to a few 10^4: launch latency, not bandwidth, is what matters there)
__global__ void __launch_bounds__(1024) scan_single_kernel(const uint32_t* in, uint32_t* out, size_t n, uint32_t* total) {
  __shared__ uint32_t sm[1024 / 32 + 1];
  uint32_t carry = 0;
  for (size_t start = 0; start < n; start += 1024 * 8) {
    size_t base = start + (size_t)threadIdx.x * 8;
    uint32_t v[8]; uint32_t s = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { v[j] = (base + j < n) ? in[base + j] : 0; s += v[j]; }
    uint32_t tot;
    uint32_t ex = block_excl_scan<1024>(s, &tot, sm) + carry;
#pragma unroll
    for (int j = 0; j < 8; j++) { if (base + j < n) out[base + j] = ex; ex += v[j]; }
    carry += tot;
  }
  if (threadIdx.x == 0 && total) *total = carry;
}

int exclusive_scan_u32(Ctx& c, ScanWork& w, const uint32_t* in, uint32_t* out, size_t n, uint32_t* total_dev) {
  if (n == 0) {
    if (total_dev) LB_CUDA(cudaMemsetAsync(total_dev, 0, sizeof(uint32_t), c.stream));
    return LB_OK;
  }
  if (n <= 8192) {
    scan_single_kernel<<<1, 1024, 0, c.stream>>>(in, out, n, total_dev);
    c.launches += 1;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
  }
  size_t nb = (n + SC_TILE - 1) / SC_TILE;
  LB_TRY(w.sums.ensure(nb > 16384 ? nb : 16384));      // never regrown for a slightly larger input (a regrow = cudaFree + cudaMalloc = device-wide sync)
  scan_reduce_kernel<<<(unsigned)nb, SC_T, 0, c.stream>>>(in, n, w.sums.p);
  scan_spine_kernel<<<1, 1024, 0, c.stream>>>(w.sums.p, nb, total_dev);
  scan_down_kernel<<<(unsigned)nb, SC_T, 0, c.stream>>>(in, out, n, w.sums.p);
  c.launches += 3;
  LB_CUDA(cudaGetLastError());
  return LB_OK;
}

// ------------------------------------------------------------------ radix sort
constexpr int RS_WARPS = 8, RS_ITEMS = 8;
static_assert(RS_WARPS * 32 * RS_ITEMS == RS_TILE, "a scatter tile is 256 threads x RS_ITEMS keys");
static_assert(RS_WARPS * 32 == 256, "one thread per digit");

int radix_sort_reserve(Ctx& c, SortWork& w, size_t n) {
  if (n > 0x7ffffff0ull) { set_error("radix_sort_pairs: n too large"); return LB_ERR_INVALID_ARG; }
  LB_TRY(w.ka.ensure(n ? n : 1)); LB_TRY(w.kb.ensure(n ? n : 1));
  LB_TRY(w.va.ensure(n ? n : 1)); LB_TRY(w.vb.ensure(n ? n : 1));
  const uint32_t tiles = rs_tiles(w.ka.cap);     // sized by the CAPACITY of the key buffers: grows only together with them
  if (!w.state.p || tiles > w.tiles_cap) {
    LB_TRY(w.state.ensure(RS_DEV_WORDS + (size_t)RS_PASSES_MAX * tiles * 256));
    w.tiles_cap = tiles;
    LB_CUDA(cudaMemsetAsync(w.state.p, 0, sizeof(RsDev), c.stream));      // the zero invariant of a fresh block
  }
  return LB_OK;
}

// Every pass's digit histogram in one read of the keys (for callers whose key kernel does not fill it); also resets
// the look-back state of the scatters that follow.
__global__ void __launch_bounds__(256)
rs_upsweep_kernel(const uint32_t* __restrict__ keys, uint32_t n, int passes, RsDev* __restrict__ rs, uint32_t* __restrict__ status,
                  uint32_t tiles) {
  __shared__ uint32_t sh[RS_PASSES_MAX][256];
  __shared__ uint32_t scan_sm[256 / 32 + 1];
  __shared__ bool last;
  for (int t = threadIdx.x; t < RS_PASSES_MAX * 256; t += 256) (&sh[0][0])[t] = 0;
  rs_reset_lookback(rs, status, tiles);
  __syncthreads();
  for (uint32_t b = blockIdx.x * 256u; b < n; b += gridDim.x * 256u) {      // uniform per CTA: all lanes rank together
    const uint32_t i = b + threadIdx.x;
    const bool v = i < n;
    rs_hist_warp_add(sh, v ? keys[i] : 0u, v, passes);
  }
  rs_hist_flush(sh, rs, passes, scan_sm, &last);
}

// One pass: a tile of RS_TILE keys, taken in ticket order, ranked per warp (__match_any_sync, stable), then its global
// position per digit = the pass's digit offset + the same digit's count in all earlier tiles, found by decoupled
// look-back (thread d walks back over digit d's status words).
__global__ void __launch_bounds__(RS_WARPS * 32)
rs_onesweep_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                   uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, uint32_t n, int pass,
                   RsDev* __restrict__ rs, uint32_t* __restrict__ status /*this pass: [tiles][256]*/,
                   const int* __restrict__ key_bits_dev) {
  __shared__ uint32_t whist[RS_WARPS][256];
  __shared__ uint32_t tile_sm;
  const int shift = 8 * pass;
  if (key_bits_dev && shift >= *key_bits_dev) return;     // pass not needed for this key width (known on the device only)
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_WARPS * 32) (&whist[0][0])[i] = 0;
  if (threadIdx.x == 0) tile_sm = atomicAdd(&rs->tile_ticket[pass], 1u);
  __syncthreads();
  const uint32_t tile = tile_sm;
  const uint32_t warp_base = tile * RS_TILE + w * (32 * RS_ITEMS);
  uint32_t key[RS_ITEMS], val[RS_ITEMS], rank[RS_ITEMS];
  const uint32_t lt_mask = (1u << l) - 1u;
#pragma unroll
  for (int j = 0; j < RS_ITEMS; j++) {
    uint32_t i = warp_base + j * 32 + l;
    bool valid = i < n;
    key[j] = valid ? keys_in[i] : 0xffffffffu;
    val[j] = valid ? (vals_in ? vals_in[i] : i) : 0u;
    uint32_t d = valid ? ((key[j] >> shift) & 255u) : 256u;
    uint32_t mask = __match_any_sync(0xffffffffu, d);
    int leader = __ffs(mask) - 1;
    uint32_t old = 0;
    if (l == leader && d < 256u) {
      old = whist[w][d];
      whist[w][d] = old + __popc(mask);
    }
    old = __shfl_sync(0xffffffffu, old, leader);
    rank[j] = old + __popc(mask & lt_mask);
    __syncwarp();
  }
  __syncthreads();
  {
    const uint32_t d = threadIdx.x;
    uint32_t cnt = 0;                     // digit d in this tile; whist becomes each warp's offset within the tile
#pragma unroll
    for (int ww = 0; ww < RS_WARPS; ww++) {
      const uint32_t c = whist[ww][d];
      whist[ww][d] = cnt;
      cnt += c;
    }
    uint32_t* mine = status + (size_t)tile * 256 + d;
    uint32_t excl = 0;
    if (tile == 0) {
      lookback_publish(mine, LB_PREFIX | cnt);
    } else {
      lookback_publish(mine, cnt);
      excl = lookback_prefix(status + d, 256, tile);
      lookback_publish(mine, LB_PREFIX | (excl + cnt));
    }
    const uint32_t off = rs->base[pass][d] + excl;
#pragma unroll
    for (int ww = 0; ww < RS_WARPS; ww++) whist[ww][d] += off;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < RS_ITEMS; j++) {
    uint32_t i = warp_base + j * 32 + l;
    if (i < n) {
      uint32_t d = (key[j] >> shift) & 255u;
      uint32_t pos = whist[w][d] + rank[j];
      keys_out[pos] = key[j];
      vals_out[pos] = val[j];
    }
  }
}

// key_bits_dev != nullptr: the key width is only known on the device (lb_voxel_filter: it follows from the bounding box
// of the call's own input).  `key_bits` is then the host's upper bound: that many bits' worth of passes are LAUNCHED,
// and a pass whose digit lies beyond *key_bits_dev returns at once -- the executed passes are a prefix, so the result
// sits in buffer A (w.ka / w.va) after an odd number of executed passes and in B after an even number (> 0).
static int radix_sort_impl(Ctx& c, SortWork& w, const uint32_t* keys_in, const uint32_t* vals_in, size_t n, int key_bits,
                           const int* key_bits_dev, bool histogram, uint32_t** keys_out, uint32_t** vals_out) {
  LB_TRY(radix_sort_reserve(c, w, n));
  const uint32_t tiles = rs_tiles(n);
  int passes = (key_bits + 7) / 8;
  if (passes < 1) passes = 1;
  if (passes > RS_PASSES_MAX) passes = RS_PASSES_MAX;
  if (histogram) {
    const uint32_t grid = tiles < (uint32_t)(2 * c.sm_count) ? tiles : (uint32_t)(2 * c.sm_count);
    rs_upsweep_kernel<<<grid, 256, 0, c.stream>>>(keys_in, (uint32_t)n, passes, w.dev(), w.status(), tiles);
    c.launches++;
  }
  const uint32_t* kin = keys_in; const uint32_t* vin = vals_in;
  uint32_t* kout = w.ka.p; uint32_t* vout = w.va.p;
  for (int p = 0; p < passes; p++) {
    rs_onesweep_kernel<<<tiles, RS_WARPS * 32, 0, c.stream>>>(kin, vin, kout, vout, (uint32_t)n, p, w.dev(),
                                                               w.status() + (size_t)p * tiles * 256, key_bits_dev);
    c.launches++;
    kin = kout; vin = vout;
    if (kout == w.ka.p) { kout = w.kb.p; vout = w.vb.p; } else { kout = w.ka.p; vout = w.va.p; }
  }
  LB_CUDA(cudaGetLastError());
  if (keys_out) *keys_out = const_cast<uint32_t*>(kin);
  if (vals_out) *vals_out = const_cast<uint32_t*>(vin);
  return LB_OK;
}

int radix_sort_pairs(Ctx& c, SortWork& w, const uint32_t* keys_in, const uint32_t* vals_in, size_t n, int key_bits,
                     uint32_t** keys_out, uint32_t** vals_out) {
  return radix_sort_impl(c, w, keys_in, vals_in, n, key_bits, nullptr, true, keys_out, vals_out);
}

int radix_sort_scatter(Ctx& c, SortWork& w, const uint32_t* keys_in, size_t n, int key_bits, uint32_t** keys_out, uint32_t** vals_out) {
  return radix_sort_impl(c, w, keys_in, nullptr, n, key_bits, nullptr, false, keys_out, vals_out);
}

int radix_sort_pairs_devbits(Ctx& c, SortWork& w, const uint32_t* keys_in, size_t n, int max_key_bits, const int* key_bits_dev) {
  return radix_sort_impl(c, w, keys_in, nullptr, n, max_key_bits, key_bits_dev, false, nullptr, nullptr);
}

}  // namespace lb
