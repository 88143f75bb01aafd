// gicp.cu -- host side of the GICP scan matcher and its C ABI.
//
// One lb_gicp handle = one CUDA stream + the device-resident state of a
// registration object (the role pcl::Registration<PointF,PointF>::Ptr icp_
// plays in PointCloudOdometry.h:154 / PointCloudLocalization.h:228):
//   source / target clouds as cell-sorted float4 + voxel-hash CSR + covariances,
//   correspondence arrays, reduction scratch, last result.
// All compute runs in the kernels of gicp_kernels.cuh; the host only sequences
// launches (host-driven mode) or launches ONE cooperative kernel per align()
// (persistent mode).  There is no CPU compute path: without a CUDA device every
// entry point fails with LB_ERR_NO_DEVICE.
#include <math.h>
#include <stdlib.h>

#include <string>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <deque>
#include <vector>

#include "align_cluster.cuh"
#include "gicp_kernels.cuh"
#include "icp_cov.h"

namespace lb {
const char* last_error();
// submap.cuh: the normal buffer of a submap whose points a target cloud indexes (nullptr: no point has one);
// LB_ERR_INVALID_ARG when the map changed since that cloud was built from it
int submap_target_normals(const lb_submap* m, uint64_t generation, const f4** nrm);

struct Cloud {
  size_t n = 0;
  bool valid = false;
  bool has_normals = false;
  bool cov_valid = false;
  DBuf<f4> raw;                // original order (x,y,z,1)
  DBuf<f4> nrm;                // original order normals
  DBuf<f4> pts;                // cell-sorted, w = original index
  DBuf<uint32_t> cell_start;   // ncells + 1
  DBuf<double> cov;            // sorted order, 6 per point
  GridGeom geom{};
  size_t ncells = 0;
  uint64_t generation = 0;
  bool index_dirty = false;    // uploaded + geometry chosen, CSR index not built yet (built lazily in align)
  int keys_slot = -1;          // >= 0: that slot's scratch holds this cloud's cell keys, occupancy marks and sort histograms for `geom`
                               // (left there by the accepted round of the occupancy probe)
  uint64_t dense_generation = 0;   // generation for which dense_fraction was measured (lb_gicp_nn_target picks its kernel by it)
  double dense_fraction = 0.0;     // share of the points that sit in cells with more than 32 points
  // the submap whose points this cloud indexes (its normals live there), and the map generation it was built from
  const lb_submap* map = nullptr;
  uint64_t map_generation = 0;

  GridView view() const {
    GridView v;
    v.pts = pts.p; v.cell_start = cell_start.p;
    v.ox = geom.ox; v.oy = geom.oy; v.oz = geom.oz; v.inv_h = geom.inv_h; v.h = geom.h;
    v.nx = geom.nx; v.ny = geom.ny; v.nz = geom.nz; v.n = (int)n;
    return v;
  }
  // set by lb_gicp_prepare_source: index + covariances are enqueued up to this event (another handle that adopts the
  // cloud as its target waits for it on its own stream)
  cudaEvent_t ready = nullptr;
  int device = 0;
  const void* owner = nullptr;   // the handle that created the object (only the owner recycles it)
  void release() { raw.release(); nrm.release(); pts.release(); cell_start.release(); cov.release(); }
  ~Cloud() {
    cudaSetDevice(device);
    release();
    if (ready) cudaEventDestroy(ready);
  }
};

// per-slot scratch so that the source and target pipelines can run concurrently on two streams
struct Scratch {
  Ctx c;                         // copy of the handle context with this slot's stream
  DBuf<uint8_t> stage;           // H2D staging of the caller cloud
  DBuf<uint32_t> keys, cell_cnt, worklist;   // worklist: queries the quad k-NN kernel hands to the tail kernel
  SortWork sort;
  ScanWork scan;
  IndexState* d_st = nullptr; IndexState* h_st = nullptr;   // state of the index build and its pinned host copy
  uint32_t* d_u32 = nullptr; uint32_t* h_u32 = nullptr;
  bool marks_zero = false;       // every word of cell_cnt (the occupancy marks) is zero
  bool wl_zero = false;          // d_st->wl is zero
  // the occupancy marks for a grid of `cells` cells, all zero (a probe round that was accepted is cleared by
  // grid_reorder_kernel; anything else -- a rejected round, a grown buffer -- costs a memset here)
  int ensure_marks(size_t cells) {
    const size_t cap = cell_cnt.cap;
    LB_TRY(cell_cnt.ensure(cells));
    if (cell_cnt.cap != cap) marks_zero = false;
    if (!marks_zero && cell_cnt.cap) LB_CUDA(cudaMemsetAsync(cell_cnt.p, 0, cell_cnt.cap * sizeof(uint32_t), c.stream));
    marks_zero = true;
    return LB_OK;
  }
  void release() {
    stage.release(); keys.release(); cell_cnt.release(); worklist.release();
    sort.ka.release(); sort.kb.release(); sort.va.release(); sort.vb.release(); sort.state.release();
    scan.sums.release();
    if (d_st) cudaFree(d_st);
    if (h_st) cudaFreeHost(h_st);
    if (d_u32) cudaFree(d_u32);
    if (h_u32) cudaFreeHost(h_u32);
  }
};

struct KTimer {          // CUDA-event timing of one kernel class
  std::string name;
  std::vector<cudaEvent_t> ev;   // pairs
  size_t used = 0;
  double total_ms = 0;
  uint64_t launches = 0;
};

// The per-device align budget (SmBudget below) counts half SMs: a CTA of the persistent and cluster kernels holds a
// whole SM, a CTA of the 160-thread loop_solve_kernel half of one when two of them fit on an SM.
constexpr int SM_SLOTS = 2;

}  // namespace lb

using namespace lb;

struct lb_gicp {
  Ctx c;
  lb_gicp_params P;
  // Clouds are shared objects: a prepared source (index + covariances) can be adopted by another handle as its
  // target (lb_gicp_share_source / lb_gicp_set_target_cloud).  A handle never writes into a cloud somebody else
  // still holds: set_source / set_target switch to a fresh (or recycled) object first.
  std::shared_ptr<Cloud> src, tgt;
  std::vector<std::shared_ptr<Cloud>> pool;     // objects this handle gave away earlier, recycled once they are unshared
  uint64_t gen_counter = 0;
  // staging / scratch: slot 0 = source pipeline (handle stream), slot 1 = target pipeline (second stream)
  Scratch sc[2];
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // align state
  DBuf<f4> src_work, corr;
  DBuf<double> M;
  DBuf<SlotWord> slots;
  unsigned long long epoch_base = 1ull << 20;
  long long* d_debug = nullptr; long long* h_debug = nullptr;
  DBuf<long long> nnprof;          // tuning aid (LB_NNPROF)
  std::shared_ptr<Cloud> last_src;  // the source before the current one (a target equal to it adopts it)
  size_t max_points_seen[2] = {0, 0}, max_cells_seen[2] = {0, 0};   // per role (source / target): capacity the role's cloud objects are grown to
  uint64_t adopted_targets = 0;
  bool adopt_previous_source = getenv("LB_NO_ADOPT") == nullptr;
  DBuf<NnsFarItem> far_items;      // staged correspondence search: queue of the undecided queries of a step
  DBuf<int> far_count;             // its two counters
  DBuf<SlotWord> cslots;           // cluster kernel: [CL_MAX_CTAS] hit-count words + [CL_CMD_WORDS] command words
  bool cluster_ok = false;
  int cluster_count = 0;           // clusters per launch (solver cluster + helpers)
  unsigned* d_barrier = nullptr;      // [2]: (unused), ticket of the host-driven objective kernel
  int* d_m = nullptr;
  double* h_sums = nullptr; double* d_sums = nullptr;        // mapped pinned [32]
  int* h_m = nullptr;                                         // pinned
  OuterResult* d_result = nullptr; OuterResult* h_result = nullptr;
  LoopState* d_loop = nullptr; LoopState* h_loop = nullptr;    // stream-ordered execution: the outer loop's state
  int align_blocks = 0;
  int wide_solve_slots = SM_SLOTS;   // budget slots one CTA of loop_solve_kernel<2 * AL_PPL, AL_SOLVE_THREADS> takes
  int knn_resident_blocks = 0;    // CTAs of knn_cov_quadreg_kernel that are resident at once on this device
  bool have_result = false;
  float final_T[16];
  DBuf<uint8_t> io;              // transform/nn output staging
  DBuf<int32_t> io_idx; DBuf<float> io_d2;
  std::vector<uint8_t> h_io;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  bool timing = false;          // event timers of every kernel class + the align kernel's cycle counters
  bool timing_light = false;    // only the CUDA-event pair around the align kernel (what a throughput run can afford)
  std::deque<KTimer> timers;       // deque: a ScopedKernelTime keeps a pointer to its timer while nested scopes may add timers
  uint64_t probe_rounds = 0;       // occupancy-probe rounds since creation (diagnostic)
};

namespace {

// The CTAs of one align() kernel spin on each other, so the cooperative grids of concurrently used handles
// (lb_odometry workers, or a caller's own threads) must fit on the device TOGETHER: more CTAs than fit would leave a
// cooperative grid waiting for SMs held by other spinning grids.  A persistent or cluster CTA occupies a whole SM
// (255 registers x 256 threads = the whole register file), and so does a 256-thread loop_solve_kernel CTA; a
// 160-thread loop_solve_kernel CTA (168 registers) half of one.  Per device, launches take their share in half SMs (SM_SLOTS per SM) from this budget and give it
// back after the stream sync; a few SMs stay reserved for the short kernels (VoxelGrid, index, k-NN) of the other
// pipeline stages.  A lone align always runs.
constexpr int LB_MAX_DEVICES = 64;
struct SmBudget {
  std::mutex mu;
  std::condition_variable cv;
  int in_use = 0;
};
SmBudget g_sm_budget[LB_MAX_DEVICES];

struct SmLease {
  SmBudget* b = nullptr; int n = 0;
  void acquire(int device, int ctas, int capacity) {
    if (device < 0 || device >= LB_MAX_DEVICES) return;
    b = &g_sm_budget[device]; n = ctas;
    std::unique_lock<std::mutex> lk(b->mu);
    b->cv.wait(lk, [&] { return b->in_use == 0 || b->in_use + n <= capacity; });
    b->in_use += n;
  }
  ~SmLease() {
    if (!b) return;
    { std::lock_guard<std::mutex> lk(b->mu); b->in_use -= n; }
    b->cv.notify_all();
  }
};

KTimer* timer_for(lb_gicp* h, const char* name) {
  for (auto& t : h->timers) if (t.name == name) return &t;
  h->timers.push_back(KTimer());
  h->timers.back().name = name;
  return &h->timers.back();
}

struct ScopedKernelTime {
  lb_gicp* h; KTimer* t; size_t slot;
  ScopedKernelTime(lb_gicp* h_, const char* name) : h(h_), t(nullptr), slot(0) {
    if (!h->timing && !(h->timing_light && !strcmp(name, "align_persistent"))) return;
    t = timer_for(h, name);
    if (t->used + 2 > t->ev.size()) {
      cudaEvent_t a, b;
      cudaEventCreate(&a); cudaEventCreate(&b);
      t->ev.push_back(a); t->ev.push_back(b);
    }
    slot = t->used; t->used += 2;
    cudaEventRecord(t->ev[slot], h->c.stream);
  }
  ~ScopedKernelTime() {
    if (!t) return;
    cudaEventRecord(t->ev[slot + 1], h->c.stream);
    t->launches++;
  }
};

void timers_collect(lb_gicp* h) {   // call after a stream sync
  for (auto& t : h->timers) {
    for (size_t i = 0; i + 1 < t.used; i += 2) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, t.ev[i], t.ev[i + 1]) == cudaSuccess) t.total_ms += ms;
    }
    t.used = 0;
  }
}

void mat16_to_34(const float* T16, Mat34& m) { for (int i = 0; i < 12; i++) m.m[i] = T16[i]; }

// smallest float g with (d2 < g) <=> ((double)d2 < D) for every float d2
float float_gate(double D) {
  float g = (float)D;
  if ((double)g < D) g = nextafterf(g, INFINITY);
  return g;
}

// largest float t with (d2 <= t) <=> ((double)d2 <= D) for every float d2
float float_floor(double D) {
  float t = (float)D;
  if ((double)t > D) t = nextafterf(t, -INFINITY);
  return t;
}

// dynamic shared memory of a kernel that runs the staged correspondence search with `threads` threads per CTA
static inline size_t nn_stage_bytes(const CorrArgs& ca, int threads) {
  return ca.nn_mode ? (size_t)(threads / 32) * ((size_t)ca.nn_cap * sizeof(f4) + 16) : 0;
}
// Search of the correspondence step: 0 = every thread on its own (nn1_pruned), 1 = staged through shared memory with
// cp.async, 2 = staged with TMA bulk copies (nn_staged.cuh).  The staged
// search wins where the step is its own full-occupancy kernels (stream-ordered and host-driven execution) and
// loses inside the persistent kernels (8 warps per SM and two more grid-wide exchanges per step), so that is the
// default; LB_NN_MODE forces one mode everywhere (A/B aid).  All modes give identical bits.
static inline void nn_stage_config(int execution, int& mode, int& cap) {
  static const int forced = [] { const char* e = getenv("LB_NN_MODE"); return e ? atoi(e) : -1; }();
  static const int c = [] { const char* e = getenv("LB_NN_CAP"); int v = e ? atoi(e) : 1024; return v < 64 ? 64 : (v > 1536 ? 1536 : v); }();
  mode = forced >= 0 ? forced : ((execution == LB_EXEC_STREAM_ORDERED || execution == LB_EXEC_HOST_DRIVEN) ? 2 : 0);
  cap = c;
}

int gicp_create_impl(int device, void* stream, bool ext, lb_gicp** out) {
  if (!out) { set_error("lb_gicp_create: null handle pointer"); return LB_ERR_INVALID_ARG; }
  lb_gicp* h = new lb_gicp;
  h->src = std::make_shared<Cloud>(); h->tgt = std::make_shared<Cloud>();
  int s = ctx_init(h->c, device, stream, ext);
  if (s != LB_OK) { delete h; return s; }
  h->src->device = h->tgt->device = device;
  h->src->owner = h->tgt->owner = h;
  lb_gicp_default_params(&h->P);
  bool ok = cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) == cudaSuccess;
  for (int k = 0; ok && k < 2; k++) {
    Scratch& S = h->sc[k];
    S.c = h->c; S.c.own_stream = false; S.c.launches = 0;
    if (k == 1) S.c.stream = h->stream2;
    ok = cudaMalloc((void**)&S.d_st, sizeof(IndexState)) == cudaSuccess &&
         cudaMemset(S.d_st, 0, sizeof(IndexState)) == cudaSuccess &&
         cudaMallocHost((void**)&S.h_st, sizeof(IndexState)) == cudaSuccess &&
         cudaMalloc((void**)&S.d_u32, 8 * sizeof(uint32_t)) == cudaSuccess &&
         cudaMallocHost((void**)&S.h_u32, 8 * sizeof(uint32_t)) == cudaSuccess;
  }
  ok = ok && cudaMalloc((void**)&h->d_barrier, 2 * sizeof(unsigned)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_m, sizeof(int)) == cudaSuccess &&
            cudaHostAlloc((void**)&h->h_sums, 32 * sizeof(double), cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer((void**)&h->d_sums, h->h_sums, 0) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_m, sizeof(int)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_result, sizeof(OuterResult)) == cudaSuccess &&
            cudaMalloc((void**)&h->d_loop, sizeof(LoopState)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_loop, sizeof(LoopState)) == cudaSuccess &&
            cudaMallocHost((void**)&h->h_result, sizeof(OuterResult)) == cudaSuccess;
  for (int i = 0; ok && i < 4; i++) ok = cudaEventCreate(&h->ev[i]) == cudaSuccess;
  if (ok) ok = cudaMemset(h->d_barrier, 0, 2 * sizeof(unsigned)) == cudaSuccess;
  if (ok) {
    for (int k = 0; k < 2; k++) bbox_init_kernel<<<1, 32, 0, h->c.stream>>>(&h->sc[k].d_st->acc);
    ok = cudaStreamSynchronize(h->c.stream) == cudaSuccess;
  }
  if (!ok) {
    set_error("lb_gicp_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    delete h;
    return LB_ERR_CUDA;
  }
  // persistent kernel: one CTA per SM, co-resident (cooperative launch)
  int per_sm = 0;
  {
    // the staged correspondence search keeps one candidate stage per warp in dynamic shared memory
    CorrArgs probe; nn_stage_config(LB_EXEC_STREAM_ORDERED, probe.nn_mode, probe.nn_cap); probe.nn_mode = 2;   // sizes only
    const int big = (int)nn_stage_bytes(probe, AL_THREADS), small = (int)nn_stage_bytes(probe, 128);
    if (cudaFuncSetAttribute(align_persistent_kernel<AL_PPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess ||
        cudaFuncSetAttribute(align_persistent_kernel<2 * AL_PPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess ||
        cudaFuncSetAttribute(nn_corr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, small) != cudaSuccess ||
        cudaFuncSetAttribute(loop_nn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, small) != cudaSuccess ||
        cudaFuncSetAttribute(nn_query_staged_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, small) != cudaSuccess ||
        cudaFuncSetAttribute(nn_query_staged_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, small) != cudaSuccess) {
      set_error("lb_gicp_create: shared-memory configuration refused: %s", cudaGetErrorString(cudaGetLastError()));
      delete h;
      return LB_ERR_CUDA;
    }
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, align_persistent_kernel<AL_PPL>, AL_THREADS, big);
    // the stream-ordered solve at 8 points per lane: correspondences in dynamic shared memory, the carveout at its
    // maximum so that two CTAs (2 x ~110 KB) fit on one SM
    int solve_per_sm = 0;
    const int solve_bytes = (int)SmemCacheT<2 * AL_PPL>::kBytes;
    if (cudaFuncSetAttribute(loop_solve_kernel<2 * AL_PPL, AL_SOLVE_THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, solve_bytes) != cudaSuccess ||
        cudaFuncSetAttribute(loop_solve_kernel<2 * AL_PPL, AL_SOLVE_THREADS>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&solve_per_sm, loop_solve_kernel<2 * AL_PPL, AL_SOLVE_THREADS>, AL_SOLVE_THREADS, solve_bytes) != cudaSuccess) {
      set_error("lb_gicp_create: solve kernel configuration refused: %s", cudaGetErrorString(cudaGetLastError()));
      delete h;
      return LB_ERR_CUDA;
    }
    h->wide_solve_slots = solve_per_sm >= SM_SLOTS ? 1 : SM_SLOTS;
  }
  {
    int knn_per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&knn_per_sm, knn_cov_quadreg_kernel<20, CovFin>, KQ_THREADS, 0);
    h->knn_resident_blocks = h->c.sm_count * (knn_per_sm > 0 ? knn_per_sm : 1);
  }
  h->align_blocks = h->c.sm_count * (per_sm >= 1 ? 1 : 0);
  if (h->align_blocks <= 0) h->align_blocks = h->c.sm_count;
  if (h->slots.ensure((size_t)2 * h->c.sm_count * AL_PSTRIDE) != LB_OK ||
      cudaMemset(h->slots.p, 0, (size_t)2 * h->c.sm_count * AL_PSTRIDE * sizeof(SlotWord)) != cudaSuccess ||
      cudaMalloc((void**)&h->d_debug, (16 + 2 * AL_MAXCTA) * sizeof(long long)) != cudaSuccess ||
      cudaMallocHost((void**)&h->h_debug, (16 + 2 * AL_MAXCTA) * sizeof(long long)) != cudaSuccess) {
    set_error("lb_gicp_create: allocation failed");
    delete h;
    return LB_ERR_CUDA;
  }
  memset(h->h_debug, 0, (16 + 2 * AL_MAXCTA) * sizeof(long long));
  cudaMemset(h->d_debug, 0, (16 + 2 * AL_MAXCTA) * sizeof(long long));
  // thread-block-cluster variant of the persistent kernel: needs a non-portable cluster of 16 CTAs with
  // 147 KB of dynamic shared memory each; fall back to the all-SM kernel when the device cannot host it
  {
    bool okc = cudaFuncSetAttribute(align_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess &&
               cudaFuncSetAttribute(align_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ClusterCache)) == cudaSuccess;
    int ncl = 0;
    if (okc) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(CL_SIZE * 8); cfg.blockDim = dim3(AL_THREADS); cfg.dynamicSmemBytes = sizeof(ClusterCache);
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = CL_SIZE; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      okc = cudaOccupancyMaxActiveClusters(&ncl, align_cluster_kernel, &cfg) == cudaSuccess && ncl >= 1;
    }
    cudaGetLastError();
    const char* e = getenv("LB_CLUSTER");
    if (e && atoi(e) == 0) okc = false;
    h->cluster_ok = okc;
    h->cluster_count = okc ? (ncl > 9 ? 9 : ncl) : 0;
    if (okc && (h->cslots.ensure(CL_MAX_CTAS + CL_CMD_WORDS) != LB_OK ||
                cudaMemset(h->cslots.p, 0, (CL_MAX_CTAS + CL_CMD_WORDS) * sizeof(SlotWord)) != cudaSuccess))
      h->cluster_ok = false;
  }
  for (int i = 0; i < 16; i++) h->final_T[i] = (i % 5 == 0) ? 1.f : 0.f;
  *out = h;
  return LB_OK;
}

// hand an object of this handle back for recycling (once): spare_cloud() reuses it when nobody else holds it any more
void pool_release(lb_gicp* h, const std::shared_ptr<Cloud>& c) {
  if (!c || c->owner != h) return;
  for (auto& p : h->pool) if (p.get() == c.get()) return;
  h->pool.push_back(c);
}

// Before a handle writes into one of its clouds: if another holder still references the object (it was shared with
// lb_gicp_share_source), switch to an object nobody else holds -- one of the earlier give-aways that has come back,
// or a new one.  A reference is only dropped after the holder's own GPU work on the cloud has been synchronised.
void make_private(lb_gicp* h, std::shared_ptr<Cloud>& c) {
  if (c.use_count() == 1 && c->owner == h) return;
  pool_release(h, c);                           // my own give-away: comes back when the other holders drop it
  // (an adopted cloud of another handle is simply let go)
  for (size_t i = 0; i < h->pool.size(); i++) {
    if (h->pool[i].use_count() == 1) {          // only the pool holds it: free to recycle (buffers are kept)
      c = h->pool[i];
      h->pool.erase(h->pool.begin() + (long)i);
      return;
    }
  }
  c = std::make_shared<Cloud>();
  c->device = h->c.device;
  c->owner = h;
}

// A cloud object nobody else holds, for the next upload: one of this handle's earlier objects that has come back
// (its buffers are kept), or a new one.
std::shared_ptr<Cloud> spare_cloud(lb_gicp* h) {
  for (size_t i = 0; i < h->pool.size(); i++) {
    if (h->pool[i].use_count() == 1) {
      std::shared_ptr<Cloud> c = h->pool[i];
      h->pool.erase(h->pool.begin() + (long)i);
      return c;
    }
  }
  std::shared_ptr<Cloud> c = std::make_shared<Cloud>();
  c->device = h->c.device;
  c->owner = h;
  return c;
}

// Phase 1 (inside set_source / set_target, synchronous because the caller's buffer is only borrowed for the
// duration of the call): upload, gather into packed float4 + bounding box in one kernel, choose the grid.
// same_as (nullable): a prepared cloud of this handle.  When the uploaded points (and normals) equal it bit for bit, the
// call stops after the gather and returns LB_SAME_CLOUD: the caller adopts that object instead of building another index
// and another set of covariances for the same data.
constexpr int LB_SAME_CLOUD = 1;
int upload_cloud(lb_gicp* h, Cloud& cl, int slot, const void* pts, size_t n, size_t stride, size_t xyz_off,
                 ptrdiff_t normal_off, int mem, const char* what, const Cloud* same_as = nullptr) {
  Scratch& S = h->sc[slot];
  Ctx& c = S.c;
  if (!pts) { set_error("%s: null cloud", what); return LB_ERR_INVALID_ARG; }
  if (n > 0x7ffffff0ull) { set_error("%s: too many points", what); return LB_ERR_INVALID_ARG; }
  if ((stride & 3u) || (xyz_off & 3u) || xyz_off + 12 > stride || (normal_off >= 0 && ((normal_off & 3) || (size_t)normal_off + 12 > stride))) {
    set_error("%s: stride/offsets must be 4-byte aligned and inside the point", what);
    return LB_ERR_INVALID_ARG;
  }
  LB_CUDA(cudaSetDevice(c.device));
  ScopedKernelTime kt(h, "index_build");
  const uint32_t N = (uint32_t)n;
  cl.valid = false; cl.cov_valid = false; cl.index_dirty = false; cl.keys_slot = -1;
  const uint8_t* d_src = (const uint8_t*)pts;
  if (mem == LB_MEM_HOST) {
    LB_TRY(S.stage.ensure(n * stride));
    LB_CUDA(cudaMemcpyAsync(S.stage.p, pts, n * stride, cudaMemcpyHostToDevice, c.stream));
    d_src = S.stage.p;
  }
  // A cloud object is sized for the largest cloud (and grid) its role (source / target) has seen on this handle, not just
  // for the one it receives now: the objects rotate (source, previous source, spares), and an object that had to grow
  // when it met a bigger cloud would mean a cudaFree + cudaMalloc -- a device-wide synchronisation -- in steady state.
  size_t& maxn = h->max_points_seen[slot];
  if (n > maxn) maxn = n;                 // (DBuf::ensure itself grows geometrically)
  LB_TRY(cl.raw.ensure(maxn)); LB_TRY(cl.pts.ensure(maxn));
  if (normal_off >= 0) LB_TRY(cl.nrm.ensure(maxn));
  if (same_as && !(same_as->valid && same_as->n == n && same_as->has_normals == (normal_off >= 0))) same_as = nullptr;
  const bool auto_cell = !(h->P.index_cell_size > 0.f);
  if (auto_cell) {
    LB_TRY(S.keys.ensure(n));
    LB_TRY(radix_sort_reserve(c, S.sort, n));
    LB_TRY(S.ensure_marks(0));
  }
  gather_cloud_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_src, N, (uint32_t)stride, (uint32_t)xyz_off, (int)normal_off,
                                                          cl.raw.p, normal_off >= 0 ? cl.nrm.p : nullptr, S.d_st,
                                                          same_as ? same_as->raw.p : nullptr,
                                                          same_as && normal_off >= 0 ? same_as->nrm.p : nullptr);
  c.launches += 1;
  // Automatic cell size: the first occupancy-probe round follows at once, on the grid the gather's last CTA chose.
  // The cell size is a pure function of the cloud (no memory of earlier clouds): the same cloud gives the same
  // grid, hence the same summation order in the align kernel and bit-identical poses, whichever handle or
  // pipeline worker sees it.  The accepted round's keys and sort histograms are what finish_index needs.
  if (auto_cell && S.cell_cnt.cap) {
    grid_index_keys_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(cl.raw.p, N, GridGeom(), true, S.d_st, S.keys.p, S.cell_cnt.p, S.cell_cnt.cap,
                                                               S.sort.dev(), S.sort.status(), rs_tiles(n));
    c.launches += 1;
    S.marks_zero = false;
  }
  // the one round trip of an upload: bounding box, finite count, "same cloud" flag, the device's grid and its occupancy
  LB_CUDA(cudaMemcpyAsync(S.h_st, S.d_st, sizeof(IndexState), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const IndexState& st = *S.h_st;
  if (auto_cell && S.cell_cnt.cap && !st.probed) S.marks_zero = true;     // the key kernel stood aside: nothing was marked
  if (st.count != N) {
    set_error("%s: cloud holds %u non-finite points; GICP inputs must be dense (PCL kd-tree precondition)", what, N - st.count);
    return LB_ERR_INVALID_ARG;
  }
  if (same_as && st.differs == 0) return LB_SAME_CLOUD;
  float mn[3], mx[3];
  for (int d = 0; d < 3; d++) { mn[d] = ord2f(st.mn[d]); mx[d] = ord2f(st.mx[d]); }
  const float ext[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};

  GridGeom g;
  if (!auto_cell) {
    g = grid_make_geom(mn, ext, h->P.index_cell_size);
  } else {
    float cell = grid_auto_cell(ext, N);
    g = grid_make_geom(mn, ext, cell);
    int round = 0;
    bool accepted = false;
    // the device's round counts when it ran on exactly this grid; otherwise (no room for the marks yet, on a handle's
    // first clouds) the rounds below start from the beginning
    if (st.probed && !memcmp(&g, &st.geom, sizeof(GridGeom))) {
      h->probe_rounds++;
      accepted = grid_probe_accept(N, st.n_occ, g.h, &cell);
      round = 1;
    }
    for (; !accepted && round < GRID_PROBE_ROUNDS; round++) {
      g = grid_make_geom(mn, ext, cell);
      LB_TRY(S.ensure_marks((size_t)g.nx * g.ny * g.nz + 1));
      LB_CUDA(cudaMemsetAsync(&S.d_st->n_occ, 0, sizeof(uint32_t), c.stream));
      grid_index_keys_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(cl.raw.p, N, g, false, S.d_st, S.keys.p, S.cell_cnt.p, S.cell_cnt.cap,
                                                                 S.sort.dev(), S.sort.status(), rs_tiles(n));
      c.launches += 1;
      S.marks_zero = false;
      LB_CUDA(cudaMemcpyAsync(&S.h_st->n_occ, &S.d_st->n_occ, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
      LB_CUDA(cudaStreamSynchronize(c.stream));
      h->probe_rounds++;
      accepted = grid_probe_accept(N, st.n_occ, g.h, &cell);
    }
    cl.keys_slot = slot;
  }
  cl.geom = g;
  cl.ncells = (size_t)g.nx * g.ny * g.nz;
  cl.n = n;
  cl.valid = true;
  cl.has_normals = normal_off >= 0;
  cl.cov_valid = false;
  cl.index_dirty = true;
  cl.generation = ++h->gen_counter;
  cl.map = nullptr;
  return LB_OK;
}

// set_source / set_target: the new cloud is uploaded into a SPARE object and only swapped in when the upload
// succeeded -- on any error (non-finite points, bad stride, out of memory) the handle keeps its previous cloud, which is
// the header's contract and what the reference does (gicp.h:164-171: "invalid or empty dataset" -> return, input kept).
int replace_cloud(lb_gicp* h, std::shared_ptr<Cloud>& dst, int slot, const void* pts, size_t n, size_t stride, size_t xyz_off,
                  ptrdiff_t normal_off, int mem, const char* what) {
  std::shared_ptr<Cloud> fresh = spare_cloud(h);
  // A new target that IS the previous source (what LOCUS's scan-to-scan odometry passes: reference_ is a copy of the last
  // query_, PointCloudOdometry.cc:252-262) adopts that cloud with its index and covariances -- when source and target
  // covariances are computed the same way, which is the reference's only configuration (one recompute_covariances flag).
  const Cloud* same_as = nullptr;
  if (slot == 1 && h->last_src && h->last_src.get() != h->src.get() && h->last_src.get() != dst.get() &&
      h->P.recompute_source_covariance == h->P.recompute_target_covariance && h->adopt_previous_source)
    same_as = h->last_src.get();
  int s = upload_cloud(h, *fresh, slot, pts, n, stride, xyz_off, normal_off, mem, what, same_as);
  if (dst->keys_slot == slot) dst->keys_slot = -1;     // the slot's scratch (cell keys of the occupancy probe) was reused
  if (s != LB_OK && s != LB_SAME_CLOUD) {
    fresh->valid = false;
    pool_release(h, fresh);                             // keeps its buffers for the next upload
    return s;
  }
  // the previous object may still be referenced by other handles (shared prepared cloud), or be an adopted cloud of
  // another handle: only this handle's own objects are recycled, and only once nobody else holds them
  if (slot == 0) h->last_src = dst;                     // stays alive (not recycled) until the next source replaces it
  pool_release(h, dst);
  if (s == LB_SAME_CLOUD) {
    fresh->valid = false;
    pool_release(h, fresh);
    dst = h->last_src;
    h->adopted_targets++;
    return LB_OK;
  }
  dst = fresh;
  return LB_OK;
}

// Phase 2 (asynchronous, on the slot's stream): cell keys, stable sort, cell-contiguous copy, CSR offsets.
int finish_index(lb_gicp* h, Cloud& cl, int slot) {
  if (!cl.index_dirty) return LB_OK;
  Scratch& S = h->sc[slot];
  Ctx& c = S.c;
  const uint32_t N = (uint32_t)cl.n;
  const int key_bits = grid_key_bits(cl.ncells);
  const bool have_keys = cl.keys_slot == slot;     // the occupancy probe left keys, marks and the sort histograms in this slot
  cl.keys_slot = -1;
  size_t& maxc = h->max_cells_seen[slot];
  if (cl.ncells + 1 > maxc) maxc = cl.ncells + 1;
  LB_TRY(cl.cell_start.ensure(maxc));
  if (!have_keys) {
    LB_TRY(S.keys.ensure(cl.n));
    LB_TRY(radix_sort_reserve(c, S.sort, cl.n));
    grid_index_keys_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(cl.raw.p, N, cl.geom, false, S.d_st, S.keys.p, nullptr, 0,
                                                               S.sort.dev(), S.sort.status(), rs_tiles(cl.n));
    c.launches++;
  }
  uint32_t *sk = nullptr, *sv = nullptr;
  LB_TRY(radix_sort_scatter(c, S.sort, S.keys.p, cl.n, key_bits, &sk, &sv));
  grid_reorder_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(cl.raw.p, sk, sv, N, (uint32_t)cl.ncells, cl.pts.p, cl.cell_start.p,
                                                          have_keys ? S.cell_cnt.p : nullptr, S.d_st->wl);
  c.launches++;
  if (have_keys) S.marks_zero = true;
  S.wl_zero = true;
  LB_CUDA(cudaGetLastError());
  cl.index_dirty = false;
  return LB_OK;
}

// Build whatever is missing (indices, covariances) for both clouds: the target pipeline runs on the second
// stream, concurrently with the source pipeline on the handle's stream (fork / join with events).
int prepare_clouds(lb_gicp* h, bool need_cov, bool src_knn, bool tgt_knn);

int compute_covariances(lb_gicp* h, Cloud& cl, int slot, bool recompute) {
  Ctx& c = h->sc[slot].c;
  const uint32_t N = (uint32_t)cl.n;
  LB_TRY(cl.cov.ensure(6 * (cl.n > h->max_points_seen[slot] ? cl.n : h->max_points_seen[slot])));
  if (!recompute && cl.has_normals) {
    normal_cov_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(cl.pts.p, cl.nrm.p, N, h->P.gicp_epsilon, cl.cov.p);
  } else {
    int k = h->P.k_correspondences;
    GridView v = cl.view();
    // tuning aid: LB_KNN=quadlocal selects the quad kernel with local-memory lists (default: quad-per-query with
    // register-resident lists; a warp-per-query and a thread-per-query kernel were tried in round 1 and removed:
    // issue-bound at 5x the instructions, resp. 10/32 active lanes)
    static const int variant = [] { const char* e = getenv("LB_KNN"); return (e && !strcmp(e, "quadlocal")) ? 2 : 0; }();
    {
      const int no_cap = 1 << 30;
      struct QuadTune { int split_from, lazy_merge, qthreads; };   // tuning aids; magic static: initialised once, thread-safe
      static const QuadTune qt = [] {
        QuadTune t;
        const char* e = getenv("LB_QSPLIT"); t.split_from = e ? atoi(e) : 99;
        e = getenv("LB_QMERGE"); t.lazy_merge = e ? atoi(e) : 1;
        e = getenv("LB_QTHREADS"); t.qthreads = e ? atoi(e) : 128;
        return t;
      }();
      const int split_from = qt.split_from, lazy_merge = qt.lazy_merge, qthreads = qt.qthreads;
      if (k <= 20 && variant == 0) {
        static const int ring_cap = [] { const char* e = getenv("LB_RING_CAP"); return e ? atoi(e) : 6; }();   // tuning aid; 6 was chosen on an earlier GPU, not re-tuned for the H100
        Scratch& S = h->sc[slot];
        LB_TRY(S.worklist.ensure(N));
        uint32_t* d_wl = S.d_st->wl;       // [0] worklist count, [1] next query batch: left at zero by the index build
        if (!S.wl_zero) LB_CUDA(cudaMemsetAsync(d_wl, 0, 2 * sizeof(uint32_t), c.stream));     // covariances again on an index built earlier
        S.wl_zero = false;
        // tuning aid LB_KNN_DYN=1: a resident grid pulls 8-query batches from a counter (slower than the static
        // grid at 30 k and 500 k points, so off by default)
        static const int dyn = [] { const char* e = getenv("LB_KNN_DYN"); return e ? atoi(e) : 0; }();
        int blocks = cdiv(4ll * N, KQ_THREADS);
        const bool use_dyn = dyn && h->knn_resident_blocks > 0 && blocks > h->knn_resident_blocks;    // more than one wave
        if (use_dyn) blocks = h->knn_resident_blocks;
        CovFin fin;
        fin.eps = h->P.gicp_epsilon; fin.cov = cl.cov.p;
        knn_cov_quadreg_kernel<20, CovFin><<<blocks, KQ_THREADS, 0, c.stream>>>(v, cl.raw.p, k, fin, split_from, ring_cap, S.worklist.p,
                                                                              d_wl, use_dyn ? d_wl + 1 : nullptr);
        // queries of sparse neighbourhoods (count read on the device: no host sync; a few resident warps when empty)
        knn_cov_tail_kernel<20, CovFin><<<c.sm_count * 2, 128, 0, c.stream>>>(v, k, fin, S.worklist.p, d_wl);
        c.launches++;
      }
      else if (k <= 20) knn_cov_quad_kernel<20><<<cdiv(4ll * N, qthreads), qthreads, 0, c.stream>>>(v, k, h->P.gicp_epsilon, cl.cov.p, no_cap, nullptr, nullptr, split_from, lazy_merge);
      else knn_cov_quad_kernel<32><<<cdiv(4ll * N, qthreads), qthreads, 0, c.stream>>>(v, k, h->P.gicp_epsilon, cl.cov.p, no_cap, nullptr, nullptr, split_from, lazy_merge);
    }
  }
  c.launches++;
  LB_CUDA(cudaGetLastError());
  cl.cov_valid = true;
  return LB_OK;
}

int prepare_clouds(lb_gicp* h, bool need_cov, bool src_knn, bool tgt_knn) {
  Ctx& c = h->c;
  bool tgt_work = h->tgt->valid && (h->tgt->index_dirty || (need_cov && !h->tgt->cov_valid));
  bool src_work = h->src->valid && (h->src->index_dirty || (need_cov && !h->src->cov_valid));
  if (!tgt_work && !src_work) return LB_OK;
  ScopedKernelTime kt(h, "knn_cov");
  if (tgt_work) {
    LB_CUDA(cudaEventRecord(h->ev_fork, c.stream));
    LB_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
    LB_TRY(finish_index(h, *h->tgt, 1));
    if (need_cov && !h->tgt->cov_valid) LB_TRY(compute_covariances(h, *h->tgt, 1, tgt_knn));   // target first, gicp.hpp:420-432
  }
  if (src_work) {
    LB_TRY(finish_index(h, *h->src, 0));
    if (need_cov && !h->src->cov_valid) LB_TRY(compute_covariances(h, *h->src, 0, src_knn));
  }
  if (tgt_work) {
    LB_CUDA(cudaEventRecord(h->ev_join, h->stream2));
    LB_CUDA(cudaStreamWaitEvent(c.stream, h->ev_join, 0));
  }
  return LB_OK;
}

// CTAs of the align kernels: one thread per source point, at least 8 and at most one CTA per SM.
// Both execution modes use the same grid so their reductions have the same shape (identical bits).
int grid_for(lb_gicp* h, int n_src) {
  static const int env_ppc = [] { const char* e = getenv("LB_PPC"); return e ? atoi(e) : 0; }();   // tuning aid
  int ppc = h->P.align_points_per_cta > 0 ? h->P.align_points_per_cta : (env_ppc > 0 ? env_ppc : AL_PPC);
  if (ppc < AL_ACC) ppc = AL_ACC;
  int g = cdiv(n_src, ppc);
  if (g < 8) g = 8;
  if (g > h->align_blocks) g = h->align_blocks;
  if (g > AL_MAXCTA) g = AL_MAXCTA;
  return g;
}

// ---- host-driven backend: the Backend concept of bfgs.h implemented with kernel launches ----
struct HostBackend {
  lb_gicp* h;
  CorrArgs ca;
  int m = 0;
  int status = LB_OK;
  int corr_calls = 0;        // correspondence steps of this align(): from the second on, ca.corr bounds the search

  int correspond(const float* T, const double* R) {
    Ctx& c = h->c;
    Mat34 t; Mat33d r;
    for (int i = 0; i < 12; i++) t.m[i] = T[i];
    for (int i = 0; i < 9; i++) r.m[i] = R[i];
    cudaMemsetAsync(h->d_m, 0, sizeof(int), c.stream);
    {
      ScopedKernelTime kt(h, "nn_corr");
      if (ca.nn_mode) cudaMemsetAsync(ca.far_count, 0, sizeof(int), c.stream);
      nn_corr_kernel<<<cdiv(ca.n_src, 128), 128, nn_stage_bytes(ca, 128), c.stream>>>(ca, t, r, corr_calls > 0, h->d_m);
      corr_calls++;
      c.launches++;
      if (ca.nn_mode) { nn_far_kernel<<<4 * h->c.sm_count, NN_FAR_THREADS, 0, c.stream>>>(ca, t, r, h->d_m); c.launches++; }
    }
    cudaMemcpyAsync(h->h_m, h->d_m, sizeof(int), cudaMemcpyDeviceToHost, c.stream);
    if (cudaStreamSynchronize(c.stream) != cudaSuccess) { status = LB_ERR_CUDA; return 0; }
    m = *h->h_m;
    return m;
  }
  template <int NV>
  bool run_objective(const double* x) {
    Ctx& c = h->c;
    ObjArgs oa{ca.src, ca.corr, ca.M, ca.n_src};
    Vec6d xv;
    for (int i = 0; i < 6; i++) xv.v[i] = x[i];
    {
      ScopedKernelTime kt(h, "objective");
      objective_kernel<NV><<<grid_for(h, ca.n_src), AL_THREADS, 0, c.stream>>>(oa, xv, h->slots.p, h->d_barrier + 1, h->d_sums);
      c.launches++;
    }
    if (cudaStreamSynchronize(c.stream) != cudaSuccess) { status = LB_ERR_CUDA; return false; }
    return true;
  }
  void fdf(const double* x, double* f, double* g) {
    if (!run_objective<13>(x)) { *f = 0; for (int i = 0; i < 6; i++) g[i] = 0; return; }
    objective_finish(h->h_sums, m, x, f, g);
  }
  int gn(const double* x, double* f, double* b, double* H) {
    if (!run_objective<28>(x)) return -1;
    *f = h->h_sums[0] / (double)m;
    for (int e = 0; e < 6; e++) b[e] = h->h_sums[1 + e];
    for (int e = 0; e < 21; e++) H[e] = h->h_sums[7 + e];
    return 0;
  }
};

}  // namespace

extern "C" {

int lb_version(void) { return LB_VERSION; }
const char* lb_last_error_string(void) { return lb::last_error(); }
const char* lb_status_string(int s) {
  switch (s) {
    case LB_OK: return "ok";
    case LB_ERR_INVALID_ARG: return "invalid argument";
    case LB_ERR_CUDA: return "CUDA error";
    case LB_ERR_NO_DEVICE: return "no CUDA device (the product path has no CPU fallback)";
    case LB_ERR_EMPTY_SOURCE: return "empty source cloud";
    case LB_ERR_NO_TARGET: return "no target cloud";
    case LB_ERR_TOO_FEW_POINTS: return "fewer points than k_correspondences";
    case LB_ERR_VOXEL_OVERFLOW: return "voxel index overflow (leaf too small)";
    case LB_ERR_CAPACITY: return "output capacity too small";
    case LB_ERR_UNSUPPORTED: return "unsupported";
    case LB_ERR_NO_ALIGN: return "no align() result yet";
    default: return "unknown status";
  }
}
int lb_device_count(int* n) {
  if (!n) return LB_ERR_INVALID_ARG;
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) { *n = 0; cudaGetLastError(); return LB_OK; }
  *n = c;
  return LB_OK;
}

int lb_gicp_default_params(lb_gicp_params* p) {
  if (!p) return LB_ERR_INVALID_ARG;
  memset(p, 0, sizeof(*p));
  p->k_correspondences = 20;              // gicp.h:112
  p->gicp_epsilon = 0.001;                // gicp.h:118
  p->rotation_epsilon = 2e-3;             // gicp.h:119
  p->transformation_epsilon = 5e-4;       // gicp.h:126
  p->max_correspondence_distance = 5.0;   // gicp.h:127
  p->max_iterations = 200;                // gicp.h:125
  p->max_optimizer_iterations = 20;       // gicp.h:121
  p->recompute_source_covariance = 1;
  p->recompute_target_covariance = 1;
  p->optimizer = LB_OPT_BFGS;
  p->execution = LB_EXEC_STREAM_ORDERED;
  p->euclidean_fitness_epsilon = 0.0;
  p->ransac_iterations = 0;
  p->num_threads = 1;
  p->enable_timing_output = 0;
  p->index_cell_size = 0.f;
  p->align_points_per_cta = 0;
  return LB_OK;
}

int lb_gicp_create(int device, lb_gicp** h) { return gicp_create_impl(device, nullptr, false, h); }
int lb_gicp_create_on_stream(int device, void* stream, lb_gicp** h) { return gicp_create_impl(device, stream, true, h); }

int lb_gicp_destroy(lb_gicp* h) {
  if (!h) return LB_OK;
  cudaSetDevice(h->c.device);
  cudaStreamSynchronize(h->c.stream);
  h->src.reset(); h->tgt.reset(); h->pool.clear();
  cudaStreamSynchronize(h->stream2);
  h->sc[0].release(); h->sc[1].release();
  if (h->stream2) cudaStreamDestroy(h->stream2);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  h->src_work.release(); h->corr.release(); h->M.release(); h->slots.release(); h->cslots.release();
  h->far_items.release(); h->far_count.release(); h->nnprof.release();
  h->io.release(); h->io_idx.release(); h->io_d2.release();
  if (h->d_barrier) cudaFree(h->d_barrier);
  if (h->d_debug) cudaFree(h->d_debug);
  if (h->h_debug) cudaFreeHost(h->h_debug);
  if (h->d_m) cudaFree(h->d_m);
  if (h->h_sums) cudaFreeHost(h->h_sums);
  if (h->h_m) cudaFreeHost(h->h_m);
  if (h->d_result) cudaFree(h->d_result);
  if (h->d_loop) cudaFree(h->d_loop);
  if (h->h_loop) cudaFreeHost(h->h_loop);
  if (h->h_result) cudaFreeHost(h->h_result);
  for (int i = 0; i < 4; i++) if (h->ev[i]) cudaEventDestroy(h->ev[i]);
  for (auto& t : h->timers) for (auto e : t.ev) cudaEventDestroy(e);
  ctx_destroy(h->c);
  delete h;
  return LB_OK;
}

int lb_gicp_set_params(lb_gicp* h, const lb_gicp_params* p) {
  if (!h || !p) { set_error("lb_gicp_set_params: null argument"); return LB_ERR_INVALID_ARG; }
  if (p->k_correspondences < 1 || p->k_correspondences > 32) { set_error("k_correspondences must be in [1, 32]"); return LB_ERR_UNSUPPORTED; }
  if (!(p->gicp_epsilon > 0) || !(p->rotation_epsilon > 0) || !(p->transformation_epsilon > 0) ||
      !(p->max_correspondence_distance > 0) || p->max_iterations < 1 || p->max_optimizer_iterations < 1) {
    set_error("lb_gicp_set_params: epsilons / distance / iteration caps must be positive");
    return LB_ERR_INVALID_ARG;
  }
  bool cov_change = p->k_correspondences != h->P.k_correspondences || p->gicp_epsilon != h->P.gicp_epsilon ||
                    p->recompute_source_covariance != h->P.recompute_source_covariance ||
                    p->recompute_target_covariance != h->P.recompute_target_covariance;
  h->P = *p;
  if (cov_change) {
    // covariances of a cloud shared with other handles are theirs too: let go of it instead of invalidating it
    for (std::shared_ptr<Cloud>* c : {&h->src, &h->tgt}) {
      const bool shared = c->use_count() > 1 || (*c)->owner != h;
      if (shared) { make_private(h, *c); (*c)->valid = false; (*c)->n = 0; }
      (*c)->cov_valid = false;
    }
  }
  return LB_OK;
}
int lb_gicp_get_params(lb_gicp* h, lb_gicp_params* p) { if (!h || !p) return LB_ERR_INVALID_ARG; *p = h->P; return LB_OK; }

int lb_gicp_set_source(lb_gicp* h, const void* pts, size_t n, size_t stride, size_t xyz_off, ptrdiff_t normal_off, int mem) {
  if (!h) { set_error("lb_gicp_set_source: null handle"); return LB_ERR_INVALID_ARG; }
  if (n == 0) {
    // gicp.h:164-171: "Invalid or empty point cloud dataset given!" -> return, previous input kept
    set_error("lb_gicp_set_source: invalid or empty point cloud dataset given");
    return LB_ERR_EMPTY_SOURCE;
  }
  return replace_cloud(h, h->src, 0, pts, n, stride, xyz_off, normal_off, mem, "lb_gicp_set_source");
}

int lb_gicp_set_target(lb_gicp* h, const void* pts, size_t n, size_t stride, size_t xyz_off, ptrdiff_t normal_off, int mem,
                       uint64_t* generation) {
  if (!h) { set_error("lb_gicp_set_target: null handle"); return LB_ERR_INVALID_ARG; }
  if (n == 0) { set_error("lb_gicp_set_target: empty target cloud"); return LB_ERR_NO_TARGET; }
  int s = replace_cloud(h, h->tgt, 1, pts, n, stride, xyz_off, normal_off, mem, "lb_gicp_set_target");
  if (s == LB_OK && generation) *generation = h->tgt->generation;
  return s;
}

// Pre-size the handle's cloud objects (current source / target and `spare_clouds` spares) for clouds of up to max_points
// points, so that the steady state of a stream performs no device allocation (cudaMalloc / cudaFree synchronise the
// whole device: with several handles working concurrently -- lb_odometry's workers -- one allocation stalls all of them).
int lb_gicp_reserve(lb_gicp* h, size_t max_points, int spare_clouds) {
  if (!h || max_points == 0 || spare_clouds < 0 || spare_clouds > 64) { set_error("lb_gicp_reserve: bad argument"); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  const size_t cells = 8 * max_points + 1024;          // the automatic cell size keeps 3-12 points per occupied cell
  auto size_cloud = [&](Cloud& cl) -> int {
    LB_TRY(cl.raw.ensure(max_points)); LB_TRY(cl.pts.ensure(max_points));
    LB_TRY(cl.cov.ensure(6 * max_points)); LB_TRY(cl.cell_start.ensure(cells + 1));
    return LB_OK;
  };
  if (h->src.use_count() == 1 && h->src->owner == h) LB_TRY(size_cloud(*h->src));
  if (h->tgt.use_count() == 1 && h->tgt->owner == h) LB_TRY(size_cloud(*h->tgt));
  int have = 0;
  for (auto& c : h->pool) if (c.use_count() == 1) { LB_TRY(size_cloud(*c)); have++; }
  for (; have < spare_clouds; have++) {
    std::shared_ptr<Cloud> c = std::make_shared<Cloud>();
    c->device = h->c.device; c->owner = h;
    LB_TRY(size_cloud(*c));
    h->pool.push_back(c);
  }
  for (int k = 0; k < 2; k++) {
    Scratch& S = h->sc[k];
    LB_TRY(S.keys.ensure(max_points)); LB_TRY(S.ensure_marks(cells + 1)); LB_TRY(S.worklist.ensure(max_points));
    LB_TRY(S.sort.ka.ensure(max_points)); LB_TRY(S.sort.kb.ensure(max_points));
    LB_TRY(S.sort.va.ensure(max_points)); LB_TRY(S.sort.vb.ensure(max_points));
  }
  LB_TRY(h->src_work.ensure(max_points)); LB_TRY(h->corr.ensure(max_points)); LB_TRY(h->M.ensure(6 * max_points));
  LB_TRY(h->far_items.ensure(max_points)); LB_TRY(h->far_count.ensure(2));
  return LB_OK;
}

int lb_gicp_promote_source_to_target(lb_gicp* h) {
  if (!h) return LB_ERR_INVALID_ARG;
  if (!h->src->valid) { set_error("lb_gicp_promote_source_to_target: no source set"); return LB_ERR_EMPTY_SOURCE; }
  std::swap(h->src, h->tgt);
  make_private(h, h->src);            // the old target may be a cloud shared with other handles: never write into it
  h->src->valid = false; h->src->cov_valid = false; h->src->n = 0;
  h->tgt->generation = ++h->gen_counter;
  return LB_OK;
}

// ---- shared, prepared clouds (each scan's index + covariances computed once, used by two registrations)
struct lb_cloud { std::shared_ptr<Cloud> c; };

int lb_gicp_prepare_source(lb_gicp* h) {
  if (!h) { set_error("lb_gicp_prepare_source: null handle"); return LB_ERR_INVALID_ARG; }
  if (!h->src->valid) { set_error("lb_gicp_prepare_source: no source cloud"); return LB_ERR_EMPTY_SOURCE; }
  if ((size_t)h->P.k_correspondences > h->src->n) {
    set_error("lb_gicp_prepare_source: number of points in cloud (%zu) is less than k_correspondences (%d)", h->src->n, h->P.k_correspondences);
    return LB_ERR_TOO_FEW_POINTS;
  }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  Cloud& cl = *h->src;
  const bool knn = h->P.recompute_source_covariance || !cl.has_normals;
  {
    ScopedKernelTime kt(h, "knn_cov");
    LB_TRY(finish_index(h, cl, 0));
    if (!cl.cov_valid) LB_TRY(compute_covariances(h, cl, 0, knn));
  }
  if (!cl.ready) LB_CUDA(cudaEventCreateWithFlags(&cl.ready, cudaEventDisableTiming));
  LB_CUDA(cudaEventRecord(cl.ready, c.stream));
  return LB_OK;
}

int lb_gicp_share_source(lb_gicp* h, lb_cloud** out) {
  if (!h || !out) { set_error("lb_gicp_share_source: null argument"); return LB_ERR_INVALID_ARG; }
  Cloud& cl = *h->src;
  if (!cl.valid || cl.index_dirty || !cl.cov_valid || !cl.ready) {
    set_error("lb_gicp_share_source: the source is not prepared (call lb_gicp_prepare_source or lb_gicp_align first)");
    return LB_ERR_INVALID_ARG;
  }
  *out = new lb_cloud{h->src};
  return LB_OK;
}

int lb_cloud_release(lb_cloud* c) {
  delete c;          // drops one reference; the buffers go back to the owning handle's pool (or are freed with the last one)
  return LB_OK;
}

int lb_gicp_set_target_cloud(lb_gicp* h, lb_cloud* c) {
  if (!h || !c || !c->c) { set_error("lb_gicp_set_target_cloud: null argument"); return LB_ERR_INVALID_ARG; }
  if (c->c->device != h->c.device) { set_error("lb_gicp_set_target_cloud: cloud lives on device %d, handle on %d", c->c->device, h->c.device); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  if (h->tgt.use_count() > 1 && h->tgt != c->c) pool_release(h, h->tgt);   // my give-away stays recyclable
  h->tgt = c->c;
  // everything this handle launches from now on (on its main stream) comes after the cloud's preparation
  LB_CUDA(cudaStreamWaitEvent(h->c.stream, h->tgt->ready, 0));
  return LB_OK;
}

// The source counterpart.  Nothing on the align, transform_source, nn_target or fitness paths writes into the source
// object once it is prepared: prepare_clouds only builds what index_dirty / cov_valid say is missing, and the align
// kernels transform a copy (src_work).  The next set_source / promote switches this handle to a private object first.
int lb_gicp_set_source_cloud(lb_gicp* h, lb_cloud* c) {
  if (!h || !c || !c->c) { set_error("lb_gicp_set_source_cloud: null argument"); return LB_ERR_INVALID_ARG; }
  if (c->c->device != h->c.device) { set_error("lb_gicp_set_source_cloud: cloud lives on device %d, handle on %d", c->c->device, h->c.device); return LB_ERR_INVALID_ARG; }
  LB_CUDA(cudaSetDevice(h->c.device));
  if (h->src.use_count() > 1 && h->src != c->c) pool_release(h, h->src);   // my give-away stays recyclable
  h->src = c->c;
  LB_CUDA(cudaStreamWaitEvent(h->c.stream, h->src->ready, 0));
  return LB_OK;
}

int lb_gicp_align(lb_gicp* h, const float* guess_in, lb_gicp_result* out) {
  if (!h || !out) { set_error("lb_gicp_align: null argument"); return LB_ERR_INVALID_ARG; }
  memset(out, 0, sizeof(*out));
  for (int i = 0; i < 16; i++) out->final_transformation[i] = out->transformation[i] = (i % 5 == 0) ? 1.f : 0.f;
  if (!h->src->valid || h->src->n == 0) { set_error("lb_gicp_align: no source cloud"); out->status = LB_ERR_EMPTY_SOURCE; return LB_ERR_EMPTY_SOURCE; }
  if (!h->tgt->valid || h->tgt->n == 0) { set_error("lb_gicp_align: no target cloud"); out->status = LB_ERR_NO_TARGET; return LB_ERR_NO_TARGET; }
  const int k = h->P.k_correspondences;
  bool src_knn = h->P.recompute_source_covariance || !h->src->has_normals;
  bool tgt_knn = h->P.recompute_target_covariance || !h->tgt->has_normals;
  // gicp.hpp:72-79 applies the k > size check in both covariance modes
  if ((size_t)k > h->src->n || (size_t)k > h->tgt->n) {
    set_error("lb_gicp_align: number of points in cloud (%zu / %zu) is less than k_correspondences (%d)", h->src->n, h->tgt->n, k);
    out->status = LB_ERR_TOO_FEW_POINTS;
    return LB_ERR_TOO_FEW_POINTS;
  }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  float guess[16];
  for (int i = 0; i < 16; i++) guess[i] = guess_in ? guess_in[i] : ((i % 5 == 0) ? 1.f : 0.f);

  LB_CUDA(cudaEventRecord(h->ev[0], c.stream));
  LB_TRY(prepare_clouds(h, true, src_knn, tgt_knn));
  LB_CUDA(cudaEventRecord(h->ev[1], c.stream));

  const uint32_t N = (uint32_t)h->src->n;
  LB_TRY(h->src_work.ensure(N)); LB_TRY(h->corr.ensure(N)); LB_TRY(h->M.ensure(6 * (size_t)N));
  Mat34 G; mat16_to_34(guess, G);
  prep_source_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(h->src->pts.p, N, G, h->src_work.p);   // gicp.hpp:440
  c.launches++;

  CorrArgs ca;
  ca.tgt = h->tgt->view(); ca.tgt_cov = h->tgt->cov.p; ca.src = h->src_work.p; ca.src_cov = h->src->cov.p;
  ca.n_src = (int)N; ca.max_d2 = float_gate(h->P.max_correspondence_distance * h->P.max_correspondence_distance);
  ca.corr = h->corr.p; ca.M = h->M.p;
  static const int exec_override = [] { const char* e = getenv("LB_EXEC_OVERRIDE"); return e ? atoi(e) : -1; }();   // tuning aid
  const int execution = exec_override >= 0 ? exec_override : h->P.execution;
  nn_stage_config(execution, ca.nn_mode, ca.nn_cap);
  static const float nn_r0 = [] { const char* e = getenv("LB_NN_R0"); float v = e ? (float)atof(e) : NNS_R0; return (v > 0.05f && v <= 1.0f) ? v : NNS_R0; }();
  ca.nn_r0 = nn_r0;
  ca.far_items = nullptr; ca.far_count = nullptr;
  if (ca.nn_mode) {
    LB_TRY(h->far_items.ensure(N)); LB_TRY(h->far_count.ensure(2));
    LB_CUDA(cudaMemsetAsync(h->far_count.p, 0, 2 * sizeof(int), c.stream));
    ca.far_items = h->far_items.p; ca.far_count = h->far_count.p;
  }
  ca.prof = nullptr;
  static const bool nnprof = getenv("LB_NNPROF") != nullptr;
  if (nnprof && ca.nn_mode) {
    LB_TRY(h->nnprof.ensure(8 * (N / 32 + 2)));
    LB_CUDA(cudaMemsetAsync(h->nnprof.p, 0, 8 * (N / 32 + 2) * sizeof(long long), c.stream));
    ca.prof = h->nnprof.p;
  }
  OuterParams OP;
  OP.rotation_epsilon = h->P.rotation_epsilon; OP.transformation_epsilon = h->P.transformation_epsilon;
  OP.max_iterations = h->P.max_iterations; OP.max_inner_iterations = h->P.max_optimizer_iterations;
  OP.optimizer = h->P.optimizer == LB_OPT_GAUSS_NEWTON ? 1 : 0;

  OuterResult R;
  if (execution == LB_EXEC_HOST_DRIVEN) {
    HostBackend be; be.h = h; be.ca = ca;
    gicp_outer_loop(be, OP, guess, R);
    if (be.status != LB_OK) { set_error("lb_gicp_align: CUDA failure in host-driven loop: %s", cudaGetErrorString(cudaGetLastError())); out->status = be.status; return be.status; }
  } else if (execution == LB_EXEC_STREAM_ORDERED) {
    // per launch of the solve kernel: one epoch per objective evaluation of ONE inner solve
    const unsigned long long need = 16ull + (unsigned long long)h->P.max_optimizer_iterations * 402ull;
    if (need * LOOP_K >= (1ull << 31)) { set_error("lb_gicp_align: max_optimizer_iterations too large"); out->status = LB_ERR_UNSUPPORTED; return LB_ERR_UNSUPPORTED; }
    unsigned long long stride = 1ull << 12;
    while (stride < need) stride <<= 1;
    // loop state: transformation_ = I, R = rot(guess), nothing found yet
    LoopState& L0 = *h->h_loop;
    memset(&L0, 0, sizeof(L0));
    outer_init(L0.s);
    outer_rotation(L0.s, guess, L0.R);
    LB_CUDA(cudaMemcpyAsync(h->d_loop, h->h_loop, sizeof(LoopState), cudaMemcpyHostToDevice, c.stream));
    AlignArgs aa;
    aa.c = ca; aa.slots = h->slots.p; aa.P = OP; aa.result = h->d_result;
    static int poll_delay_s = -1;
    if (poll_delay_s < 0) { const char* e = getenv("LB_POLL_DELAY"); poll_delay_s = e ? atoi(e) : (int)AL_POLL_DELAY; }
    aa.poll_delay = poll_delay_s;
    aa.debug = nullptr;
    for (int i = 0; i < 16; i++) aa.guess[i] = guess[i];
    const int grid = grid_for(h, ca.n_src);
    static const int reserve_s = [] { const char* e = getenv("LB_SM_RESERVE"); return e ? atoi(e) : 16; }();
    const int chunk = cdiv(ca.n_src, grid);
    // up to 512 points per CTA: the one-per-SM shape (lowest latency); beyond: the two-per-SM shape (throughput)
    const bool wide = chunk > AL_PPC;
    void* kfn = wide ? (void*)loop_solve_kernel<2 * AL_PPL, AL_SOLVE_THREADS> : (void*)loop_solve_kernel<AL_PPL, AL_THREADS>;
    const int solve_threads = wide ? AL_SOLVE_THREADS : AL_THREADS;
    const size_t solve_bytes = wide ? SmemCacheT<2 * AL_PPL>::kBytes : 0;
    SmLease lease;
    lease.acquire(c.device, grid * (wide ? h->wide_solve_slots : SM_SLOTS), SM_SLOTS * (h->align_blocks - reserve_s));
    {
      ScopedKernelTime kt(h, "align_persistent");
      for (int done = 0; !done;) {
        for (int k = 0; k < LOOP_K; k++) {
          // the slot tags are the low 32 bits of the epoch: clear the slots whenever the base wraps them
          if ((h->epoch_base >> 32) != ((h->epoch_base + stride) >> 32) || (h->epoch_base & 0xffffffffull) == 0) {
            LB_CUDA(cudaMemsetAsync(h->slots.p, 0, (size_t)2 * h->c.sm_count * AL_PSTRIDE * sizeof(SlotWord), c.stream));
            h->epoch_base = ((h->epoch_base >> 32) + 1) << 32 | (1ull << 20);
          }
          aa.epoch_base = h->epoch_base;
          h->epoch_base += stride;
          {
            ScopedKernelTime kn(h, "loop_nn");
            loop_nn_kernel<<<cdiv(ca.n_src, 128), 128, nn_stage_bytes(ca, 128), c.stream>>>(ca, h->d_loop, k);
            if (ca.nn_mode) { loop_far_kernel<<<4 * h->c.sm_count, NN_FAR_THREADS, 0, c.stream>>>(ca, h->d_loop, k); c.launches++; }
          }
          LoopState* dl = h->d_loop;
          int kk = k;
          void* args[] = {&aa, &dl, &kk};
          ScopedKernelTime ks(h, "loop_solve");
          LB_CUDA(cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(solve_threads), args, solve_bytes, c.stream));
          c.launches += 2;
        }
        LB_CUDA(cudaMemcpyAsync(h->h_loop, h->d_loop, sizeof(LoopState), cudaMemcpyDeviceToHost, c.stream));
        LB_CUDA(cudaStreamSynchronize(c.stream));
        done = h->h_loop->s.done;
      }
    }
    R = h->h_loop->result;
  } else {
    // the slot tags are the low 32 bits of the epoch: clear the slots whenever the base wraps them
    // One launch consumes a range of collective epochs (the slot tags): at most one per correspondence step plus one
    // per objective evaluation.  The range reserved per launch covers the caller's iteration caps (pcl::BFGS: <= 100
    // bracketing + 100 sectioning steps of <= 2 evaluations per inner iteration), so a launch can never run into the
    // tags of the next one.
    const unsigned long long need = (unsigned long long)h->P.max_iterations * (2ull + (unsigned long long)h->P.max_optimizer_iterations * 402ull) + 16ull;
    if (need >= (1ull << 31)) {
      set_error("lb_gicp_align: max_iterations x max_optimizer_iterations too large for the persistent kernel's epoch range; use LB_EXEC_HOST_DRIVEN");
      out->status = LB_ERR_UNSUPPORTED;
      return LB_ERR_UNSUPPORTED;
    }
    unsigned long long stride = 1ull << 20;
    while (stride < need) stride <<= 1;
    // the slot tags are the low 32 bits of the epoch: clear the slots whenever the base wraps them
    if ((h->epoch_base >> 32) != ((h->epoch_base + stride) >> 32) || (h->epoch_base & 0xffffffffull) == 0) {
      LB_CUDA(cudaMemsetAsync(h->slots.p, 0, (size_t)2 * h->c.sm_count * AL_PSTRIDE * sizeof(SlotWord), c.stream));
      if (h->cslots.p) LB_CUDA(cudaMemsetAsync(h->cslots.p, 0, (CL_MAX_CTAS + CL_CMD_WORDS) * sizeof(SlotWord), c.stream));
      h->epoch_base = ((h->epoch_base >> 32) + 1) << 32 | (1ull << 20);
    }
    const unsigned long long epoch_base = h->epoch_base;
    h->epoch_base += stride;
    bool use_cluster = h->cluster_ok && execution == LB_EXEC_PERSISTENT_CLUSTER && N <= (uint32_t)(CL_SIZE * CL_CAP);
    bool launched = false;
    SmLease lease;     // released when this block ends, i.e. after the stream sync below
    if (use_cluster) {
      ClusterArgs ka;
      ka.c = ca; ka.gslots = h->cslots.p; ka.gcmd = h->cslots.p + CL_MAX_CTAS; ka.epoch_base = epoch_base;
      ka.P = OP; ka.result = h->d_result; ka.debug = h->timing ? h->d_debug : nullptr;
      for (int i = 0; i < 16; i++) ka.guess[i] = guess[i];
      // helpers only pay off when there is enough NN work for them
      int clusters = cdiv(N, CL_SIZE * 256);
      if (clusters < 1) clusters = 1;
      if (clusters > h->cluster_count) clusters = h->cluster_count;
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(CL_SIZE * clusters); cfg.blockDim = dim3(AL_THREADS);
      cfg.dynamicSmemBytes = sizeof(ClusterCache); cfg.stream = c.stream;
      cudaLaunchAttribute at[2];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = CL_SIZE; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      at[1].id = cudaLaunchAttributeCooperative; at[1].val.cooperative = 1;
      cfg.attrs = at; cfg.numAttrs = 2;
      // the solver cluster and its helpers spin on each other like the all-SM grid does: same per-device SM budget
      static const int reserve_c = [] { const char* ev = getenv("LB_SM_RESERVE"); return ev ? atoi(ev) : 16; }();
      lease.acquire(c.device, SM_SLOTS * CL_SIZE * clusters, SM_SLOTS * (h->align_blocks - reserve_c));
      ScopedKernelTime kt(h, "align_persistent");
      cudaError_t e = cudaLaunchKernelEx(&cfg, align_cluster_kernel, ka);
      if (e == cudaSuccess) { launched = true; c.launches++; }
      else { cudaGetLastError(); h->cluster_ok = false; }   // e.g. cooperative + cluster launch refused: use the all-SM kernel from now on
    }
    if (!launched) {
      AlignArgs aa;
      aa.c = ca; aa.slots = h->slots.p; aa.P = OP; aa.result = h->d_result;
      aa.epoch_base = epoch_base;
      static int poll_delay = -1;   // tuning aid
      if (poll_delay < 0) { const char* e = getenv("LB_POLL_DELAY"); poll_delay = e ? atoi(e) : (int)AL_POLL_DELAY; }
      aa.poll_delay = poll_delay;
      aa.debug = h->timing ? h->d_debug : nullptr;
      for (int i = 0; i < 16; i++) aa.guess[i] = guess[i];
      void* args[] = {&aa};
      const int grid = grid_for(h, ca.n_src);
      static const int reserve = [] { const char* e = getenv("LB_SM_RESERVE"); return e ? atoi(e) : 16; }();
      lease.acquire(c.device, SM_SLOTS * grid, SM_SLOTS * (h->align_blocks - reserve));
      ScopedKernelTime kt(h, "align_persistent");
      // points per CTA up to 512: 4 per accumulating lane in registers; up to 1024: 8 (beyond: read back from L2)
      const int chunk = cdiv(ca.n_src, grid);
      void* kfn = chunk <= AL_PPC ? (void*)align_persistent_kernel<AL_PPL> : (void*)align_persistent_kernel<2 * AL_PPL>;
      LB_CUDA(cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(AL_THREADS), args, nn_stage_bytes(ca, AL_THREADS), c.stream));
      c.launches++;
    }
    if (h->timing) LB_CUDA(cudaMemcpyAsync(h->h_debug, h->d_debug, (16 + 2 * AL_MAXCTA) * sizeof(long long), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaMemcpyAsync(h->h_result, h->d_result, sizeof(OuterResult), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
    R = *h->h_result;
  }
  LB_CUDA(cudaEventRecord(h->ev[2], c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  if (ca.prof) {   // tuning aid: what the warps of the LAST correspondence step spent where
    const size_t nw = (N + 31) / 32;
    std::vector<long long> hp(8 * nw);
    cudaMemcpy(hp.data(), ca.prof, hp.size() * sizeof(long long), cudaMemcpyDeviceToHost);
    long long sum[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, mx[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int hist[5] = {0, 0, 0, 0, 0};
    for (size_t i = 0; i < nw; i++) {
      const long long chunks = hp[8 * i + 7] >> 40; hp[8 * i + 7] &= (1ll << 40) - 1;
      sum[8] += chunks; if (chunks > mx[8]) mx[8] = chunks;
      for (int k = 0; k < 8; k++) { sum[k] += hp[8 * i + k]; if (hp[8 * i + k] > mx[k]) mx[k] = hp[8 * i + k]; }
      const long long f = hp[8 * i + 2];
      hist[f == 0 ? 0 : f <= 2 ? 1 : f <= 8 ? 2 : f <= 16 ? 3 : 4]++;
    }
    fprintf(stderr, "[nnprof] warps %zu iters %d | staged pass cycles mean %.0f max %lld | far pass mean %.0f max %lld | far lanes mean %.2f max %lld "
            "hist(0,1-2,3-8,9-16,17+) %d %d %d %d %d | finish mean %.0f max %lld | staged lanes mean %.1f | candidates per warp mean %.0f max %lld\n",
            nw, R.nr_iterations, (double)sum[0] / nw, mx[0], (double)sum[1] / nw, mx[1], (double)sum[2] / nw, mx[2], hist[0], hist[1], hist[2], hist[3],
            hist[4], (double)sum[3] / nw, mx[3], (double)sum[4] / nw, (double)sum[5] / nw, mx[5]);
    fprintf(stderr, "[nnprof]   rows+csr mean %.0f max %lld | copy+wait mean %.0f max %lld | scan mean %.0f max %lld | chunks mean %.2f max %lld\n",
            (double)sum[4] / nw, mx[4], (double)sum[6] / nw, mx[6], (double)sum[7] / nw, mx[7], (double)sum[8] / nw, mx[8]);
  }
  timers_collect(h);
  for (int i = 0; i < 16; i++) { out->final_transformation[i] = R.final_T[i]; h->final_T[i] = R.final_T[i]; out->transformation[i] = R.prev_T[i]; }
  h->have_result = true;
  out->converged = R.converged;
  out->iterations = R.nr_iterations;
  out->n_correspondences = R.n_corr;
  out->delta = R.delta;
  out->n_objective_evals = R.st.n_evals;
  out->n_inner_iterations = R.st.n_inner;
  cudaEventElapsedTime(&out->t_covariances_ms, h->ev[0], h->ev[1]);
  cudaEventElapsedTime(&out->t_iterations_ms, h->ev[1], h->ev[2]);
  cudaEventElapsedTime(&out->t_total_ms, h->ev[0], h->ev[2]);
  out->status = LB_OK;
  return LB_OK;
}

int lb_gicp_transform_source(lb_gicp* h, const float* T_in, void* out_pts, size_t stride, size_t xyz_off, ptrdiff_t normal_off, int mem) {
  if (!h || !out_pts) { set_error("lb_gicp_transform_source: null argument"); return LB_ERR_INVALID_ARG; }
  if (!h->src->valid) { set_error("lb_gicp_transform_source: no source cloud"); return LB_ERR_EMPTY_SOURCE; }
  if (!T_in && !h->have_result) { set_error("lb_gicp_transform_source: no align() result yet"); return LB_ERR_NO_ALIGN; }
  if ((stride & 3u) || (xyz_off & 3u) || xyz_off + 12 > stride) { set_error("lb_gicp_transform_source: bad stride/offset"); return LB_ERR_INVALID_ARG; }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)h->src->n;
  Mat34 T; mat16_to_34(T_in ? T_in : h->final_T, T);
  bool nrm = normal_off >= 0 && h->src->has_normals;
  if (mem == LB_MEM_DEVICE) {
    transform_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(h->src->raw.p, nrm ? h->src->nrm.p : nullptr, N, T, (uint8_t*)out_pts,
                                                         (uint32_t)stride, (uint32_t)xyz_off, nrm ? (int)normal_off : -1);
    c.launches++;
    LB_CUDA(cudaStreamSynchronize(c.stream));
    return LB_OK;
  }
  // host output: packed (xyz | normal) rows on the device, one D2H, scatter into the caller's layout
  const uint32_t row = nrm ? 24 : 12;
  LB_TRY(h->io.ensure((size_t)N * row));
  transform_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(h->src->raw.p, nrm ? h->src->nrm.p : nullptr, N, T, h->io.p, row, 0, nrm ? 12 : -1);
  c.launches++;
  h->h_io.resize((size_t)N * row);
  LB_CUDA(cudaMemcpyAsync(h->h_io.data(), h->io.p, (size_t)N * row, cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  uint8_t* o = (uint8_t*)out_pts;
  for (uint32_t i = 0; i < N; i++) {
    memcpy(o + (size_t)i * stride + xyz_off, h->h_io.data() + (size_t)i * row, 12);
    if (nrm) memcpy(o + (size_t)i * stride + normal_off, h->h_io.data() + (size_t)i * row + 12, 12);
  }
  return LB_OK;
}

// Exact 1-NN of N device queries (xyz at the start of each `stride`-byte row) in the prepared target, enqueued on the
// handle's stream: lb_gicp_nn_target and lb_gicp_icp_covariance.  The kernel is chosen per target by its density over the
// voxel hash, measured once per target cloud (that measurement synchronises).
static int nn_search(lb_gicp* h, const uint8_t* dq, uint32_t N, uint32_t stride, int32_t* di, float* dd) {
  Ctx& c = h->c;
  if (h->tgt->dense_generation != h->tgt->generation) {      // once per target cloud: how uneven it is over its voxel hash
    Cloud& t = *h->tgt;
    LB_CUDA(cudaMemsetAsync(h->d_debug + 6, 0, sizeof(long long), c.stream));
    cell_density_kernel<<<c.sm_count * 4, 256, 0, c.stream>>>(t.cell_start.p, t.ncells, 32u, (unsigned long long*)(h->d_debug + 6));
    long long dense = 0;
    LB_CUDA(cudaMemcpyAsync(&dense, h->d_debug + 6, sizeof(long long), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
    t.dense_fraction = t.n ? (double)dense / (double)t.n : 0.0;
    t.dense_generation = t.generation;
    c.launches++;
  }
  {
    ScopedKernelTime kt(h, "nn_query");
    // Default: 32 queries per warp through the staged search with TMA bulk copies, undecided queries queued and finished
    // one per warp by a second kernel (nn_staged.cuh).  LB_NN = warp | thread | staged selects the warp-per-query kernel,
    // the thread-per-query kernel, or the cp.async staging (A/B aid).
    static int nnv_env = -2;
    if (nnv_env == -2) { const char* e = getenv("LB_NN"); nnv_env = !e ? -1 : !strcmp(e, "thread") ? 0 : !strcmp(e, "warp") ? 1 : !strcmp(e, "staged") ? 2 : 3; }
    int nnv = nnv_env;
    if (nnv < 0) nnv = h->tgt->dense_fraction > 0.10 ? 1 : 3;       // locally very dense (raw) maps: the warp-per-query kernel
    CorrArgs probe; nn_stage_config(LB_EXEC_STREAM_ORDERED, probe.nn_mode, probe.nn_cap); probe.nn_mode = 2;
    if (nnv == 0) {
      nn_query_kernel<<<cdiv(N, 128), 128, 0, c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, di, dd, 3.0e38f);
    } else if (nnv >= 2) {
      LB_TRY(h->far_items.ensure(N)); LB_TRY(h->far_count.ensure(2));
      LB_CUDA(cudaMemsetAsync(h->far_count.p, 0, sizeof(int), c.stream));
      {
        ScopedKernelTime k1(h, "nn_query_first");
        if (nnv == 2) nn_query_staged_kernel<false><<<cdiv(N, 128), 128, nn_stage_bytes(probe, 128), c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, di, dd, 3.0e38f, probe.nn_cap, h->far_items.p, h->far_count.p, nullptr);
        else nn_query_staged_kernel<true><<<cdiv(N, 128), 128, nn_stage_bytes(probe, 128), c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, di, dd, 3.0e38f, probe.nn_cap, h->far_items.p, h->far_count.p, nullptr);
      }
      ScopedKernelTime k2(h, "nn_query_far");
      nn_query_far_kernel<<<c.sm_count * 8, 256, 0, c.stream>>>(h->tgt->view(), dq, (uint32_t)stride, di, dd, 3.0e38f, h->far_items.p, h->far_count.p);
      c.launches++;
    } else {
      int blocks = cdiv(N, 8);
      if (blocks > c.sm_count * 8) blocks = c.sm_count * 8;
      nn_query_warp_kernel<<<blocks, 256, 0, c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, di, dd, 3.0e38f);
    }
    c.launches++;
  }
  return LB_OK;
}

int lb_gicp_nn_target(lb_gicp* h, const void* xyz, size_t n, size_t stride, int32_t* idx, float* d2, int mem) {
  if (!h || !xyz || !idx || !d2) { set_error("lb_gicp_nn_target: null argument"); return LB_ERR_INVALID_ARG; }
  if (!h->tgt->valid) { set_error("lb_gicp_nn_target: no target cloud"); return LB_ERR_NO_TARGET; }
  if (n == 0) return LB_OK;
  if ((stride & 3u) || stride < 12) { set_error("lb_gicp_nn_target: bad stride"); return LB_ERR_INVALID_ARG; }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(prepare_clouds(h, false, false, false));
  const uint32_t N = (uint32_t)n;
  const uint8_t* dq = (const uint8_t*)xyz; int32_t* di = idx; float* dd = d2;
  if (mem == LB_MEM_HOST) {
    LB_TRY(h->io.ensure(n * stride)); LB_TRY(h->io_idx.ensure(n)); LB_TRY(h->io_d2.ensure(n));
    LB_CUDA(cudaMemcpyAsync(h->io.p, xyz, n * stride, cudaMemcpyHostToDevice, c.stream));
    dq = h->io.p; di = h->io_idx.p; dd = h->io_d2.p;
  }
  LB_TRY(nn_search(h, dq, N, (uint32_t)stride, di, dd));
  if (h->timing) {   // profiling aid: mean number of target points a query visits -> h_debug[4], h_debug[5]
    static int nnv2_env = -2;
    if (nnv2_env == -2) { const char* e = getenv("LB_NN"); nnv2_env = !e ? -1 : !strcmp(e, "thread") ? 0 : !strcmp(e, "warp") ? 1 : !strcmp(e, "staged") ? 2 : 3; }
    const int nnv2 = nnv2_env >= 0 ? nnv2_env : (h->tgt->dense_fraction > 0.10 ? 1 : 3);
    LB_CUDA(cudaMemsetAsync(h->d_debug + 4, 0, 2 * sizeof(long long), c.stream));
    if (nnv2 >= 2) {      // the staged search: candidates staged by the first look; h_debug[6] = queries left to the second kernel
      CorrArgs probe; nn_stage_config(LB_EXEC_STREAM_ORDERED, probe.nn_mode, probe.nn_cap); probe.nn_mode = 2;
      LB_CUDA(cudaMemsetAsync(h->far_count.p, 0, sizeof(int), c.stream));
      nn_query_staged_kernel<true><<<cdiv(N, 128), 128, nn_stage_bytes(probe, 128), c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, di, dd, 3.0e38f, probe.nn_cap, h->far_items.p, h->far_count.p, h->d_debug + 4);
      nn_query_far_kernel<<<c.sm_count * 8, 256, 0, c.stream>>>(h->tgt->view(), dq, (uint32_t)stride, di, dd, 3.0e38f, h->far_items.p, h->far_count.p);
      int nf = 0;
      LB_CUDA(cudaMemcpyAsync(&nf, h->far_count.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
      LB_CUDA(cudaStreamSynchronize(c.stream));
      h->h_debug[6] = nf;
    } else {
      nn_count_kernel<<<cdiv(N, 128), 128, 0, c.stream>>>(h->tgt->view(), dq, N, (uint32_t)stride, 3.0e38f,
                                                          (unsigned long long*)(h->d_debug + 4));
    }
    LB_CUDA(cudaMemcpyAsync(h->h_debug + 4, h->d_debug + 4, sizeof(long long), cudaMemcpyDeviceToHost, c.stream));
    h->h_debug[5] = (long long)N;
  }
  if (mem == LB_MEM_HOST) {
    LB_CUDA(cudaMemcpyAsync(idx, di, n * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaMemcpyAsync(d2, dd, n * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  }
  LB_CUDA(cudaStreamSynchronize(c.stream));
  LB_CUDA(cudaGetLastError());
  return LB_OK;
}

int lb_gicp_fitness(lb_gicp* h, const float* T_in, double max_range, double* score) {
  if (!h || !score) { set_error("lb_gicp_fitness: null argument"); return LB_ERR_INVALID_ARG; }
  if (!h->src->valid) { set_error("lb_gicp_fitness: no source cloud"); return LB_ERR_EMPTY_SOURCE; }
  if (!h->tgt->valid) { set_error("lb_gicp_fitness: no target cloud"); return LB_ERR_NO_TARGET; }
  if (!T_in && !h->have_result) { set_error("lb_gicp_fitness: no align() result yet"); return LB_ERR_NO_ALIGN; }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(prepare_clouds(h, false, false, false));
  const uint32_t N = (uint32_t)h->src->n;
  int nb = cdiv(N, 128);
  LB_TRY(h->io.ensure((size_t)nb * 2 * sizeof(double)));
  Mat34 T; mat16_to_34(T_in ? T_in : h->final_T, T);
  fitness_kernel<<<nb, 128, 0, c.stream>>>(h->tgt->view(), h->src->raw.p, N, T, max_range, (double*)h->io.p);
  c.launches++;
  std::vector<double> part((size_t)nb * 2);
  LB_CUDA(cudaMemcpyAsync(part.data(), h->io.p, part.size() * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  double sum = 0, cnt = 0;
  for (int b = 0; b < nb; b++) { sum += part[2 * (size_t)b]; cnt += part[2 * (size_t)b + 1]; }
  *score = cnt > 0 ? sum / cnt : 1.7976931348623157e308;   // PCL returns numeric_limits<double>::max()
  return LB_OK;
}

int lb_gicp_point2plane_information(lb_gicp* h, const void* query, size_t n, size_t q_stride, size_t q_xyz_off,
                                    const void* reference, size_t n_ref, size_t r_stride, size_t r_normal_off,
                                    const int32_t* correspondences, const float* T, int normalize, double* Ap36, int mem) {
  if (!h || !query || !reference || !correspondences || !Ap36) { set_error("lb_gicp_point2plane_information: null argument"); return LB_ERR_INVALID_ARG; }
  if ((q_stride & 3u) || (q_xyz_off & 3u) || q_xyz_off + 12 > q_stride || (r_stride & 3u) || (r_normal_off & 3u) || r_normal_off + 12 > r_stride) {
    set_error("lb_gicp_point2plane_information: bad stride/offset");
    return LB_ERR_INVALID_ARG;
  }
  for (int i = 0; i < 36; i++) Ap36[i] = 0.0;
  if (n == 0) return LB_OK;
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  const uint32_t N = (uint32_t)n;
  const uint8_t *dq = (const uint8_t*)query, *dr = (const uint8_t*)reference;
  const int32_t* dc = correspondences;
  if (mem == LB_MEM_HOST) {
    size_t bq = n * q_stride, br = n_ref * r_stride, bc = n * sizeof(int32_t);
    size_t o1 = (bq + 255) & ~(size_t)255, o2 = o1 + ((br + 255) & ~(size_t)255);
    LB_TRY(h->io.ensure(o2 + bc));
    LB_CUDA(cudaMemcpyAsync(h->io.p, query, bq, cudaMemcpyHostToDevice, c.stream));
    LB_CUDA(cudaMemcpyAsync(h->io.p + o1, reference, br, cudaMemcpyHostToDevice, c.stream));
    LB_CUDA(cudaMemcpyAsync(h->io.p + o2, correspondences, bc, cudaMemcpyHostToDevice, c.stream));
    dq = h->io.p; dr = h->io.p + o1; dc = (const int32_t*)(h->io.p + o2);
  }
  int nb = cdiv(N, 256);
  if (nb > c.sm_count * 4) nb = c.sm_count * 4;
  DBuf<double>& scratch = h->M;   // not in use outside align()
  LB_TRY(scratch.ensure((size_t)nb * 21 + 4));
  std::vector<double> part((size_t)nb * 21);
  float* d_norm = reinterpret_cast<float*>(scratch.p + (size_t)nb * 21);
  ApArgs a;
  a.q = dq; a.n = N; a.q_stride = (uint32_t)q_stride; a.q_xyz_off = (uint32_t)q_xyz_off;
  a.ref = dr; a.n_ref = (uint32_t)n_ref; a.r_stride = (uint32_t)r_stride; a.r_normal_off = (uint32_t)r_normal_off;
  a.corr = dc; a.norm = nullptr; a.use_R = T ? 1 : 0; a.use_Rf = 0; a.counters = nullptr;
  for (int i = 0; i < 9; i++) a.R[i] = T ? (double)T[(i / 3) * 4 + (i % 3)] : ((i % 4 == 0) ? 1.0 : 0.0);
  if (normalize) {
    // normalizePCloud's centroid and mean distance, float32 sums in point order like the reference; they stay on the
    // device (the accumulation kernel derives factor and offset from them): no host round trip
    ap_normalize_seq_kernel<<<1, 256, 0, c.stream>>>(dq, N, (uint32_t)q_stride, (uint32_t)q_xyz_off, d_norm);
    c.launches++;
    a.norm = d_norm;
  }
  ap_accumulate_kernel<<<nb, 256, 0, c.stream>>>(a, scratch.p);
  c.launches++;
  LB_CUDA(cudaMemcpyAsync(part.data(), scratch.p, (size_t)nb * 21 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  LB_CUDA(cudaGetLastError());
  double up[21] = {0};
  for (int b = 0; b < nb; b++) for (int e = 0; e < 21; e++) up[e] += part[21 * (size_t)b + e];
  int e = 0;
  for (int r = 0; r < 6; r++) for (int cc = r; cc < 6; cc++) { Ap36[r * 6 + cc] = up[e]; Ap36[cc * 6 + r] = up[e]; e++; }
  return LB_OK;
}

// SURVEY 8f row f1, completed: PointCloudLocalization.cc:325-336 + ComputePoint2PlaneICPCovariance (:469-541).  The
// per-point work is the transform, 1-NN, normalize and Ap kernels above, enqueued on the handle's stream into align
// scratch (src_work: aligned points; corr: indices and distances; M: partials, centroid, counters), then ONE copy-back;
// the 6x6 algebra runs on the host (icp_cov.h).
int lb_gicp_icp_covariance(lb_gicp* h, const float* T_in, const int32_t* correspondences, int mem, const float* normal_rotation,
                           double max_covariance, lb_icp_covariance* out) {
  if (!h || !out) { set_error("lb_gicp_icp_covariance: null argument"); return LB_ERR_INVALID_ARG; }
  if (!std::isfinite(max_covariance) || !(max_covariance > 0.0)) {
    set_error("lb_gicp_icp_covariance: max_covariance must be finite and > 0");
    return LB_ERR_INVALID_ARG;
  }
  if (!h->src->valid) { set_error("lb_gicp_icp_covariance: no source cloud"); return LB_ERR_EMPTY_SOURCE; }
  if (!h->tgt->valid) { set_error("lb_gicp_icp_covariance: no target cloud"); return LB_ERR_NO_TARGET; }
  if (!T_in && !correspondences && !h->have_result) { set_error("lb_gicp_icp_covariance: no align() result yet"); return LB_ERR_NO_ALIGN; }
  Ctx& c = h->c;
  LB_CUDA(cudaSetDevice(c.device));
  const Cloud& tg = *h->tgt;
  const f4* nrm = tg.has_normals ? tg.nrm.p : nullptr;
  if (tg.map) LB_TRY(submap_target_normals(tg.map, tg.map_generation, &nrm));
  const uint32_t N = (uint32_t)h->src->n;
  LB_TRY(h->src_work.ensure(N)); LB_TRY(h->corr.ensure(N));
  int nb = cdiv(N, 256);
  if (nb > c.sm_count * 4) nb = c.sm_count * 4;
  LB_TRY(h->M.ensure((size_t)nb * 21 + 3));
  float* d_norm = reinterpret_cast<float*>(h->M.p + (size_t)nb * 21);          // 4 floats
  unsigned* d_cnt = reinterpret_cast<unsigned*>(h->M.p + (size_t)nb * 21 + 2);  // rows used, bad index
  int32_t* d_corr = reinterpret_cast<int32_t*>(h->corr.p);
  const int32_t* dc = correspondences;
  if (!correspondences) {
    // 1-2: aligned = T q (transformPointCloudWithNormals' float association), exact 1-NN in the target
    LB_TRY(prepare_clouds(h, false, false, false));
    Mat34 T; mat16_to_34(T_in ? T_in : h->final_T, T);
    transform_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(h->src->raw.p, nullptr, N, T, reinterpret_cast<uint8_t*>(h->src_work.p),
                                                         (uint32_t)sizeof(f4), 0, -1);
    c.launches++;
    LB_TRY(nn_search(h, reinterpret_cast<const uint8_t*>(h->src_work.p), N, (uint32_t)sizeof(f4), d_corr,
                     reinterpret_cast<float*>(h->corr.p) + N));
    dc = d_corr;
  } else if (mem == LB_MEM_HOST) {
    LB_CUDA(cudaMemcpyAsync(d_corr, correspondences, (size_t)N * sizeof(int32_t), cudaMemcpyHostToDevice, c.stream));
    dc = d_corr;
  }
  LB_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned), c.stream));
  // 3: normalizePCloud(q)'s centroid and mean distance
  ap_normalize_seq_kernel<<<1, 256, 0, c.stream>>>(reinterpret_cast<const uint8_t*>(h->src->raw.p), N, (uint32_t)sizeof(f4), 0, d_norm);
  // 4: Ap from the target's own normal buffer, rotated in float
  ApArgs a;
  a.q = reinterpret_cast<const uint8_t*>(h->src->raw.p); a.n = N; a.q_stride = (uint32_t)sizeof(f4); a.q_xyz_off = 0;
  a.ref = reinterpret_cast<const uint8_t*>(nrm); a.n_ref = (uint32_t)tg.n; a.r_stride = (uint32_t)sizeof(f4); a.r_normal_off = 0;
  a.corr = dc; a.norm = d_norm; a.use_R = 0;
  for (int i = 0; i < 9; i++) { a.R[i] = 0.0; a.Rf[i] = normal_rotation ? normal_rotation[i] : 0.f; }
  a.use_Rf = normal_rotation ? 1 : 0;
  a.counters = d_cnt;
  ap_accumulate_kernel<<<nb, 256, 0, c.stream>>>(a, h->M.p);
  c.launches += 2;
  std::vector<double> part((size_t)nb * 21 + 3);
  LB_CUDA(cudaMemcpyAsync(part.data(), h->M.p, part.size() * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  LB_CUDA(cudaGetLastError());
  unsigned cnt[2];
  memcpy(cnt, &part[(size_t)nb * 21 + 2], sizeof(cnt));
  if (cnt[1]) { set_error("lb_gicp_icp_covariance: a correspondence is outside the target (%zu points)", tg.n); return LB_ERR_INVALID_ARG; }
  double up[21] = {0};
  for (int b = 0; b < nb; b++) for (int e = 0; e < 21; e++) up[e] += part[21 * (size_t)b + e];
  int e = 0;
  for (int r = 0; r < 6; r++) for (int cc = r; cc < 6; cc++) { out->Ap[r * 6 + cc] = up[e]; out->Ap[cc * 6 + r] = up[e]; e++; }
  // 5-9 on the host
  const icpcov::Result res = icpcov::compute(out->Ap, max_covariance);
  memcpy(out->covariance, res.cov, sizeof(res.cov));
  out->condition_number = res.condition_number;
  out->flags = res.flags;
  out->n_query = N;
  out->n_used = cnt[0];
  return LB_OK;
}

// SURVEY 8f row f2: point_cloud_filter::NormalComputation::filter in k-NN mode (normal_computation.cc:26-59).
int lb_gicp_compute_normals(lb_gicp* h, int which, int k, const float* viewpoint, float* out4, int mem) {
  if (!h || !out4 || (which != 0 && which != 1)) { set_error("lb_gicp_compute_normals: bad argument"); return LB_ERR_INVALID_ARG; }
  Cloud& cl = which == 0 ? *h->src : *h->tgt;
  if (!cl.valid) { set_error("lb_gicp_compute_normals: no %s cloud", which == 0 ? "source" : "target"); return which == 0 ? LB_ERR_EMPTY_SOURCE : LB_ERR_NO_TARGET; }
  if (k < 3 || k > 20) { set_error("lb_gicp_compute_normals: k must be in [3, 20] (PCL yields NaN normals below 3)"); return LB_ERR_UNSUPPORTED; }
  if ((size_t)k > cl.n) { set_error("lb_gicp_compute_normals: cloud has %zu points, fewer than k = %d", cl.n, k); return LB_ERR_TOO_FEW_POINTS; }
  Scratch& S = h->sc[which];
  Ctx& c = S.c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(finish_index(h, cl, which));
  const uint32_t N = (uint32_t)cl.n;
  f4* d_out = reinterpret_cast<f4*>(out4);
  if (mem == LB_MEM_HOST) { LB_TRY(h->io.ensure((size_t)N * sizeof(f4))); d_out = reinterpret_cast<f4*>(h->io.p); }
  LB_TRY(S.worklist.ensure(N));
  uint32_t* d_wl = S.d_u32 + 4;
  LB_CUDA(cudaMemsetAsync(d_wl, 0, 2 * sizeof(uint32_t), c.stream));
  NormalFin fin;
  fin.vp[0] = viewpoint ? viewpoint[0] : 0.f; fin.vp[1] = viewpoint ? viewpoint[1] : 0.f; fin.vp[2] = viewpoint ? viewpoint[2] : 0.f;
  fin.out = d_out;
  GridView v = cl.view();
  static const int ring_cap = [] { const char* e = getenv("LB_RING_CAP"); return e ? atoi(e) : 6; }();
  knn_cov_quadreg_kernel<20, NormalFin><<<cdiv(4ll * N, KQ_THREADS), KQ_THREADS, 0, c.stream>>>(v, cl.raw.p, k, fin, 99, ring_cap,
                                                                                        S.worklist.p, d_wl, nullptr);
  knn_cov_tail_kernel<20, NormalFin><<<c.sm_count * 2, 128, 0, c.stream>>>(v, k, fin, S.worklist.p, d_wl);
  c.launches += 2;
  LB_CUDA(cudaGetLastError());
  if (mem == LB_MEM_HOST) LB_CUDA(cudaMemcpyAsync(out4, d_out, (size_t)N * sizeof(f4), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  return LB_OK;
}

// The same kernels with the cloud's own normal buffer as output: NormalFin writes (nx, ny, nz, curvature) in original
// order, which is Cloud::nrm's layout (the covariance and transform kernels read x, y, z only).  Asynchronous: the
// source's consumers run on the handle's stream, the target's on stream2 (joined into the handle's stream here).
int lb_gicp_estimate_normals(lb_gicp* h, int which, int k, const float* viewpoint) {
  if (!h || (which != 0 && which != 1)) { set_error("lb_gicp_estimate_normals: bad argument"); return LB_ERR_INVALID_ARG; }
  std::shared_ptr<Cloud>& ref = which == 0 ? h->src : h->tgt;
  Cloud& cl = *ref;
  if (!cl.valid) { set_error("lb_gicp_estimate_normals: no %s cloud", which == 0 ? "source" : "target"); return which == 0 ? LB_ERR_EMPTY_SOURCE : LB_ERR_NO_TARGET; }
  if (k < 3 || k > 20) { set_error("lb_gicp_estimate_normals: k must be in [3, 20] (PCL yields NaN normals below 3)"); return LB_ERR_UNSUPPORTED; }
  if ((size_t)k > cl.n) { set_error("lb_gicp_estimate_normals: cloud has %zu points, fewer than k = %d", cl.n, k); return LB_ERR_TOO_FEW_POINTS; }
  // a target adopted from this handle's previous source is held twice by the handle itself; any other holder means the
  // cloud was shared (or adopted from another handle) and is immutable
  const long own_refs = 1 + (h->last_src == ref ? 1 : 0);
  if (ref->owner != h || ref.use_count() > own_refs) {
    set_error("lb_gicp_estimate_normals: the %s cloud is shared with another handle", which == 0 ? "source" : "target");
    return LB_ERR_INVALID_ARG;
  }
  Scratch& S = h->sc[which];
  Ctx& c = S.c;
  LB_CUDA(cudaSetDevice(c.device));
  const size_t cap = cl.n > h->max_points_seen[which] ? cl.n : h->max_points_seen[which];
  LB_TRY(cl.nrm.ensure(cap));
  LB_TRY(finish_index(h, cl, which));
  const uint32_t N = (uint32_t)cl.n;
  LB_TRY(S.worklist.ensure(N));
  uint32_t* d_wl = S.d_u32 + 4;
  LB_CUDA(cudaMemsetAsync(d_wl, 0, 2 * sizeof(uint32_t), c.stream));
  NormalFin fin;
  fin.vp[0] = viewpoint ? viewpoint[0] : 0.f; fin.vp[1] = viewpoint ? viewpoint[1] : 0.f; fin.vp[2] = viewpoint ? viewpoint[2] : 0.f;
  fin.out = cl.nrm.p;
  GridView v = cl.view();
  static const int ring_cap = [] { const char* e = getenv("LB_RING_CAP"); return e ? atoi(e) : 6; }();
  knn_cov_quadreg_kernel<20, NormalFin><<<cdiv(4ll * N, KQ_THREADS), KQ_THREADS, 0, c.stream>>>(v, cl.raw.p, k, fin, 99, ring_cap,
                                                                                        S.worklist.p, d_wl, nullptr);
  knn_cov_tail_kernel<20, NormalFin><<<c.sm_count * 2, 128, 0, c.stream>>>(v, k, fin, S.worklist.p, d_wl);
  c.launches += 2;
  LB_CUDA(cudaGetLastError());
  if (which == 1) {
    LB_CUDA(cudaEventRecord(h->ev_join, c.stream));
    LB_CUDA(cudaStreamWaitEvent(h->c.stream, h->ev_join, 0));
  }
  cl.has_normals = true;
  cl.cov_valid = false;
  return LB_OK;
}

// SURVEY 8f row f2, the nodelet's radius mode + NaN-normal removal (normal_computation.cc:53-57,73-77).
int lb_gicp_compute_normals_radius(lb_gicp* h, int which, double radius, const float* viewpoint, float* out4, int32_t* valid_idx,
                                   size_t* n_valid, int mem) {
  if (!h || !out4 || (which != 0 && which != 1)) { set_error("lb_gicp_compute_normals_radius: bad argument"); return LB_ERR_INVALID_ARG; }
  if (!(radius > 0.0)) { set_error("lb_gicp_compute_normals_radius: radius must be > 0"); return LB_ERR_INVALID_ARG; }
  Cloud& cl = which == 0 ? *h->src : *h->tgt;
  if (!cl.valid) { set_error("lb_gicp_compute_normals_radius: no %s cloud", which == 0 ? "source" : "target"); return which == 0 ? LB_ERR_EMPTY_SOURCE : LB_ERR_NO_TARGET; }
  if (n_valid) *n_valid = 0;
  Scratch& S = h->sc[which];
  Ctx& c = S.c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(finish_index(h, cl, which));
  const uint32_t N = (uint32_t)cl.n;
  static const bool attr_ok = [] {
    return cudaFuncSetAttribute(normals_radius_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)(NR_WARPS * NR_CAP * sizeof(unsigned long long))) == cudaSuccess;
  }();
  if (!attr_ok) { set_error("lb_gicp_compute_normals_radius: cannot reserve shared memory"); return LB_ERR_CUDA; }
  f4* d_out = reinterpret_cast<f4*>(out4);
  int32_t* d_vidx = valid_idx;
  if (mem == LB_MEM_HOST) {
    LB_TRY(h->io.ensure((size_t)N * sizeof(f4)));
    d_out = reinterpret_cast<f4*>(h->io.p);
    if (valid_idx) { LB_TRY(h->io_idx.ensure(N)); d_vidx = h->io_idx.p; }
  }
  LB_TRY(S.keys.ensure(N)); LB_TRY(S.worklist.ensure(N));
  uint32_t* d_flags = S.keys.p; uint32_t* d_pos = S.worklist.p;
  cl.keys_slot = -1;                               // the slot's key scratch is reused as the flag array
  uint32_t* d_tot = S.d_u32 + 6;                   // [6] number of valid normals, [7] overflow flag
  LB_CUDA(cudaMemsetAsync(d_tot, 0, 2 * sizeof(uint32_t), c.stream));
  int blocks = cdiv(N, NR_WARPS);
  if (blocks > c.sm_count * 8) blocks = c.sm_count * 8;
  normals_radius_kernel<<<blocks, NR_WARPS * 32, NR_WARPS * NR_CAP * sizeof(unsigned long long), c.stream>>>(
      cl.view(), cl.raw.p, (float)(radius * radius), viewpoint ? viewpoint[0] : 0.f, viewpoint ? viewpoint[1] : 0.f,
      viewpoint ? viewpoint[2] : 0.f, d_out, d_flags, reinterpret_cast<int*>(d_tot + 1));
  c.launches++;
  LB_TRY(exclusive_scan_u32(c, S.scan, d_flags, d_pos, N, d_tot));
  if (valid_idx) {
    compact_indices_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_flags, d_pos, N, d_vidx);
    c.launches++;
  }
  LB_CUDA(cudaGetLastError());
  LB_CUDA(cudaMemcpyAsync(S.h_u32 + 6, d_tot, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  if (mem == LB_MEM_HOST) LB_CUDA(cudaMemcpyAsync(out4, d_out, (size_t)N * sizeof(f4), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  if (S.h_u32[7]) {
    set_error("lb_gicp_compute_normals_radius: a neighbourhood holds more than %d points; use a smaller radius or the k-NN mode", NR_CAP);
    return LB_ERR_CAPACITY;
  }
  const size_t m = S.h_u32[6];
  if (valid_idx && mem == LB_MEM_HOST && m) {
    LB_CUDA(cudaMemcpyAsync(valid_idx, d_vidx, m * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  if (n_valid) *n_valid = m;
  return LB_OK;
}

namespace {
// flags (original order) -> ascending indices of the flagged points; the count lands in S.h_u32[6] after the stream sync
int compact_flags(Ctx& c, Scratch& S, const uint32_t* d_flags, uint32_t* d_pos, uint32_t N, int32_t* d_idx) {
  uint32_t* d_tot = S.d_u32 + 6;
  LB_TRY(exclusive_scan_u32(c, S.scan, d_flags, d_pos, N, d_tot));
  compact_indices_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_flags, d_pos, N, d_idx);
  c.launches++;
  LB_CUDA(cudaGetLastError());
  LB_CUDA(cudaMemcpyAsync(S.h_u32 + 6, d_tot, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  return LB_OK;
}
}  // namespace

// Row f5: pcl::StatisticalOutlierRemoval (PointCloudFilter.cc:126-133).
int lb_gicp_statistical_outlier_removal(lb_gicp* h, int which, int mean_k, double std_mul, int negative, int32_t* kept_idx,
                                        size_t* n_kept, float* mean_dist, double* stats3, int mem) {
  if (!h || !kept_idx || !n_kept || (which != 0 && which != 1)) { set_error("lb_gicp_statistical_outlier_removal: bad argument"); return LB_ERR_INVALID_ARG; }
  *n_kept = 0;
  Cloud& cl = which == 0 ? *h->src : *h->tgt;
  if (!cl.valid) { set_error("lb_gicp_statistical_outlier_removal: no %s cloud", which == 0 ? "source" : "target"); return which == 0 ? LB_ERR_EMPTY_SOURCE : LB_ERR_NO_TARGET; }
  if (mean_k < 1) { set_error("lb_gicp_statistical_outlier_removal: mean_k must be >= 1"); return LB_ERR_INVALID_ARG; }
  if (mean_k > 19) { set_error("lb_gicp_statistical_outlier_removal: mean_k must be <= 19 (20 neighbours with the point itself)"); return LB_ERR_UNSUPPORTED; }
  if (cl.n < (size_t)mean_k + 1) { set_error("lb_gicp_statistical_outlier_removal: cloud has %zu points, fewer than mean_k + 1 = %d", cl.n, mean_k + 1); return LB_ERR_TOO_FEW_POINTS; }
  Scratch& S = h->sc[which];
  Ctx& c = S.c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(finish_index(h, cl, which));
  const uint32_t N = (uint32_t)cl.n;
  float* d_dist = mean_dist;
  double* d_stats = stats3;
  int32_t* d_idx = kept_idx;
  if (mem == LB_MEM_HOST || !mean_dist) { LB_TRY(h->io_d2.ensure(N)); d_dist = h->io_d2.p; }
  if (mem == LB_MEM_HOST || !stats3) { LB_TRY(h->M.ensure(3)); d_stats = h->M.p; }    // M: not in use outside align()
  if (mem == LB_MEM_HOST) { LB_TRY(h->io_idx.ensure(N)); d_idx = h->io_idx.p; }
  LB_TRY(S.worklist.ensure(N)); LB_TRY(S.keys.ensure(N));
  cl.keys_slot = -1;                               // the slot's key scratch is reused as the flag array
  uint32_t* d_wl = S.d_u32 + 4;
  LB_CUDA(cudaMemsetAsync(d_wl, 0, 2 * sizeof(uint32_t), c.stream));
  MeanDistFin fin;
  fin.out = d_dist;
  GridView v = cl.view();
  static const int ring_cap = [] { const char* e = getenv("LB_RING_CAP"); return e ? atoi(e) : 6; }();
  knn_cov_quadreg_kernel<20, MeanDistFin><<<cdiv(4ll * N, KQ_THREADS), KQ_THREADS, 0, c.stream>>>(v, cl.raw.p, mean_k + 1, fin, 99,
                                                                                          ring_cap, S.worklist.p, d_wl, nullptr);
  knn_cov_tail_kernel<20, MeanDistFin><<<c.sm_count * 2, 128, 0, c.stream>>>(v, mean_k + 1, fin, S.worklist.p, d_wl);
  sor_stats_kernel<<<1, 256, 0, c.stream>>>(d_dist, N, std_mul, d_stats);
  sor_flags_kernel<<<cdiv(N, 256), 256, 0, c.stream>>>(d_dist, N, d_stats, negative, S.keys.p);
  c.launches += 4;
  LB_CUDA(cudaGetLastError());
  LB_TRY(compact_flags(c, S, S.keys.p, S.worklist.p, N, d_idx));
  if (mem == LB_MEM_HOST && mean_dist) LB_CUDA(cudaMemcpyAsync(mean_dist, d_dist, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost, c.stream));
  if (mem == LB_MEM_HOST && stats3) LB_CUDA(cudaMemcpyAsync(stats3, d_stats, 3 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const size_t m = S.h_u32[6];
  if (mem == LB_MEM_HOST && m) {
    LB_CUDA(cudaMemcpyAsync(kept_idx, d_idx, m * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  *n_kept = m;
  return LB_OK;
}

// Row f5: pcl::RadiusOutlierRemoval (PointCloudFilter.cc:135-143, PointCloudMerger.cc:112-117,139-144,169-174).
int lb_gicp_radius_outlier_removal(lb_gicp* h, int which, double radius, int min_neighbors, int dense, int negative,
                                   int32_t* kept_idx, size_t* n_kept, int mem) {
  if (!h || !kept_idx || !n_kept || (which != 0 && which != 1)) { set_error("lb_gicp_radius_outlier_removal: bad argument"); return LB_ERR_INVALID_ARG; }
  *n_kept = 0;
  if (!(radius > 0.0)) { set_error("lb_gicp_radius_outlier_removal: radius must be > 0"); return LB_ERR_INVALID_ARG; }
  if (min_neighbors < 0) { set_error("lb_gicp_radius_outlier_removal: min_neighbors must be >= 0"); return LB_ERR_INVALID_ARG; }
  Cloud& cl = which == 0 ? *h->src : *h->tgt;
  if (!cl.valid) { set_error("lb_gicp_radius_outlier_removal: no %s cloud", which == 0 ? "source" : "target"); return which == 0 ? LB_ERR_EMPTY_SOURCE : LB_ERR_NO_TARGET; }
  Scratch& S = h->sc[which];
  Ctx& c = S.c;
  LB_CUDA(cudaSetDevice(c.device));
  LB_TRY(finish_index(h, cl, which));
  const uint32_t N = (uint32_t)cl.n;
  int32_t* d_idx = kept_idx;
  if (mem == LB_MEM_HOST) { LB_TRY(h->io_idx.ensure(N)); d_idx = h->io_idx.p; }
  LB_TRY(S.worklist.ensure(N)); LB_TRY(S.keys.ensure(N));
  cl.keys_slot = -1;                               // the slot's key scratch is reused as the flag array
  // at most N points can pass the test: a larger count is never reached either way
  const int need = (size_t)min_neighbors + 1 > (size_t)N + 1 ? (int)N + 1 : min_neighbors + 1;
  const double r2 = radius * radius;
  if (dense) radius_count_kernel<false><<<cdiv(N, 256), 256, 0, c.stream>>>(cl.view(), float_floor(r2), need, negative, S.keys.p);
  else radius_count_kernel<true><<<cdiv(N, 256), 256, 0, c.stream>>>(cl.view(), (float)r2, need, negative, S.keys.p);
  c.launches++;
  LB_CUDA(cudaGetLastError());
  LB_TRY(compact_flags(c, S, S.keys.p, S.worklist.p, N, d_idx));
  LB_CUDA(cudaStreamSynchronize(c.stream));
  const size_t m = S.h_u32[6];
  if (mem == LB_MEM_HOST && m) {
    LB_CUDA(cudaMemcpyAsync(kept_idx, d_idx, m * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
    LB_CUDA(cudaStreamSynchronize(c.stream));
  }
  *n_kept = m;
  return LB_OK;
}

int lb_gicp_get_covariances(lb_gicp* h, int which, double* out9, size_t capacity_points) {
  if (!h || !out9) return LB_ERR_INVALID_ARG;
  Cloud& cl = which ? *h->tgt : *h->src;
  if (!cl.valid || !cl.cov_valid) { set_error("lb_gicp_get_covariances: covariances not computed (run align first)"); return LB_ERR_NO_ALIGN; }
  if (capacity_points < cl.n) { set_error("lb_gicp_get_covariances: capacity too small"); return LB_ERR_CAPACITY; }
  LB_CUDA(cudaSetDevice(h->c.device));
  std::vector<double> c6(6 * cl.n);
  std::vector<f4> pts(cl.n);
  LB_CUDA(cudaMemcpyAsync(c6.data(), cl.cov.p, c6.size() * sizeof(double), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaMemcpyAsync(pts.data(), cl.pts.p, pts.size() * sizeof(f4), cudaMemcpyDeviceToHost, h->c.stream));
  LB_CUDA(cudaStreamSynchronize(h->c.stream));
  for (size_t s = 0; s < cl.n; s++) {
    size_t i = (size_t)float_to_bits(pts[s].w);
    const double* m = &c6[6 * s];
    double* o = &out9[9 * i];
    o[0] = m[SXX]; o[1] = m[SXY]; o[2] = m[SXZ];
    o[3] = m[SXY]; o[4] = m[SYY]; o[5] = m[SYZ];
    o[6] = m[SXZ]; o[7] = m[SYZ]; o[8] = m[SZZ];
  }
  return LB_OK;
}

int lb_gicp_cloud_size(lb_gicp* h, int which, size_t* n) {
  if (!h || !n) return LB_ERR_INVALID_ARG;
  Cloud& cl = which ? *h->tgt : *h->src;
  *n = cl.valid ? cl.n : 0;
  return LB_OK;
}
int lb_gicp_launch_count(lb_gicp* h, uint64_t* n) {
  if (!h || !n) return LB_ERR_INVALID_ARG;
  *n = h->c.launches + h->sc[0].c.launches + h->sc[1].c.launches;
  return LB_OK;
}

int lb_gicp_kernel_time(lb_gicp* h, const char* name, float* ms_avg, uint64_t* launches) {
  if (!h || !name || !ms_avg) return LB_ERR_INVALID_ARG;
  *ms_avg = 0.f; if (launches) *launches = 0;
  cudaStreamSynchronize(h->c.stream);
  timers_collect(h);
  if (!strncmp(name, "debug", 5) && name[5] >= '0' && name[5] <= '9') {   // cycle counters of the last persistent align
    *ms_avg = (float)h->h_debug[name[5] - '0'];
    return LB_OK;
  }
  if (!strncmp(name, "dbg", 3) && name[3] >= '0' && name[3] <= '9') {   // "dbgNN": any of the 16 debug words
    const int i = atoi(name + 3);
    if (i < 0 || i >= 16) return LB_ERR_INVALID_ARG;
    *ms_avg = (float)h->h_debug[i];
    return LB_OK;
  }
  if (!strcmp(name, "probe_rounds")) { *ms_avg = (float)h->probe_rounds; return LB_OK; }
  if (!strcmp(name, "dbuf_allocs")) { *ms_avg = (float)dbuf_alloc_count(); return LB_OK; }   // device allocations so far (process-wide)
  if (!strcmp(name, "pool_clouds")) { *ms_avg = (float)h->pool.size(); return LB_OK; }
  if (!strcmp(name, "cell_src")) { *ms_avg = h->src->geom.h; return LB_OK; }      // cell size of the current index (m)
  if (!strcmp(name, "cell_tgt")) { *ms_avg = h->tgt->geom.h; return LB_OK; }
  if (!strcmp(name, "adopted_targets")) { *ms_avg = (float)h->adopted_targets; return LB_OK; }   // set_target calls that found the previous source
  if (!strcmp(name, "dense_tgt")) { *ms_avg = (float)h->tgt->dense_fraction; return LB_OK; }   // share of target points in cells with > 32 points
  if (!strncmp(name, "snap", 4)) {   // "snapP<i>" / "snapC<i>": publish / completion time (ns, relative) of CTA i at collective 100
    int i = atoi(name + 5);
    if (i < 0 || i >= AL_MAXCTA) return LB_ERR_INVALID_ARG;
    long long base = h->h_debug[16];
    *ms_avg = (float)(h->h_debug[16 + (name[4] == 'C' ? AL_MAXCTA : 0) + i] - base);
    return LB_OK;
  }
  for (auto& t : h->timers) {
    if (t.name == name) {
      if (t.launches) *ms_avg = (float)(t.total_ms / (double)t.launches);
      if (launches) *launches = t.launches;
    }
  }
  return LB_OK;
}
int lb_gicp_reset_kernel_times(lb_gicp* h, int enable) {
  if (!h) return LB_ERR_INVALID_ARG;
  cudaStreamSynchronize(h->c.stream);
  timers_collect(h);
  for (auto& t : h->timers) { t.total_ms = 0; t.launches = 0; t.used = 0; }
  h->timing = enable == 1;
  h->timing_light = enable == 2;
  return LB_OK;
}

}  // extern "C"

#include "submap.cuh"
