// Scan-to-scan odometry pipeline (lb_odometry_*): the per-scan chain of the reference's lidar callback
//   filtered scan -> PointCloudOdometry::SetLidar -> UpdateEstimate -> UpdateICP
//   (locus/src/Locus.cc:451-453, point_cloud_odometry/src/PointCloudOdometry.cc:221-274)
// as a two-stage host pipeline over the library's own C ABI:
//
//   stage V  one thread, one lb_voxel handle (own stream): VoxelGrid of scan k into slot k % R of a ring of
//            device-resident filtered clouds
//   stage G  `depth` threads, one lb_gicp handle each (own streams): set_source(ring[k]), set_target(ring[k-1]),
//            align -> result k; under LB_REG_NDT (lb_odometry_set_registration) the same three calls on the worker's
//            lb_ndt handle instead
//
// Nothing here touches a point: every byte of device work is done by voxel.cu / gicp.cu kernels.  The pipeline
// exists because one align() is a chain of latency-bound kernels on a fraction of the SMs: the rest of the GPU filters
// and indexes the following scans, and several aligns (each on its own CTAs) are in flight at once.  Results are
// those of the sequential calls: registration k reads only filtered clouds k and k-1 and its caller-given prior.
//
// lb_locus_* (end of this file) runs the same core with a third stage L behind stage G: one thread, one lb_gicp handle
// bound to the caller's lb_submap, localizing the scans strictly in order (pose semantics: lo_pose.h).  In that mode a
// ticket is done when stage L has finished it, so stages V and G run at most the usual in-flight bound ahead of it.
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

#if defined(LB_LOCUS_STUB)       // TEST-ONLY build without CUDA: tests/locus_harness.cpp supplies fake stages
#include "locus_stub.h"
#include "front_end_stub.h"
#include "icp_covariance_stub.h"
#include "merged_stub.h"
#include "ndt_stub.h"
#elif defined(LB_ODOMETRY_STUB)  // TEST-ONLY build without CUDA: tests/odometry_harness.cpp supplies fake stages
#include "odometry_stub.h"
#include "front_end_stub.h"
#include "merged_stub.h"
#include "ndt_stub.h"
#else
#include "prims.cuh"
namespace lb {
int voxel_reserve(lb_voxel* h, size_t n_pts, uint32_t max_step);   // voxel.cu
int ndt_reserve(lb_ndt* h, size_t max_points);                       // ndt.cu
int ndt_check_params(const lb_ndt_params* p, const char* who);      // ndt.cu
}
#endif
#include "lo_pose.h"

using namespace lb;

namespace {

constexpr int MAX_LIDARS = 3;      // lb_voxel_filter_merged's input limit

struct Job {
  uint64_t ticket = 0;
  const uint8_t* scan = nullptr;
  size_t n_pts = 0;
  // lb_odometry_submit_merged: n_inputs > 0 clouds in merge order (scan unused; n_pts = their sum), each with its
  // transform copied at submit (has_T[i] = 0: identity)
  int n_inputs = 0;
  const uint8_t* in_data[MAX_LIDARS] = {nullptr, nullptr, nullptr};
  size_t in_pts[MAX_LIDARS] = {0, 0, 0};
  bool has_T[MAX_LIDARS] = {false, false, false};
  float T[MAX_LIDARS][16];
  uint32_t point_step = 0;
  std::vector<lb_field> fields;
  int mem = LB_MEM_HOST;
  bool has_guess = false;
  float guess[16];
  uint8_t* filtered_out = nullptr;
  int mem_filtered = LB_MEM_HOST;
  int xyz_off = 0;
};

struct Slot {            // one filtered cloud of the ring
  uint8_t* d = nullptr;
  size_t n = 0;          // points; 0 = unusable (stage V failed)
  uint32_t point_step = 0;
  int xyz_off = 0;
  int status = LB_OK;
  char error[160] = "";
};

struct Prepared {        // cloud-sharing mode: scan t's prepared cloud, published by the worker of registration t
  uint64_t ticket = ~0ull;
  lb_cloud* cloud = nullptr;     // null when the preparation failed
  bool ready = false;
};

struct Entry {           // per in-flight ticket
  Job job;
  lb_odometry_result res;
  bool filtered = false; // stage V done
  bool aligned = false;  // stage G done (lb_locus only)
  float leaf = 0.f;      // lb_locus: the VoxelGrid x leaf the scan was filtered with
  bool done = false;     // result complete: stage G done, or stage L with lb_locus
  lb_cloud* loc_cloud = nullptr;   // lb_locus: stage L's reference to this scan's prepared cloud
  lb_locus_result loc;             // lb_locus: filled by stage L
};

}  // namespace

struct lb_odometry {
  int device = 0;
  int depth = 1;
  size_t max_points = 0;
  uint32_t max_step = 0;
  lb_voxel* vg = nullptr;
  std::vector<lb_gicp*> gicp;
  std::vector<Slot> ring;
  std::vector<Prepared> prep;          // same indexing as ring (ticket % R); used when share is on
  bool share = true;                   // lb_odometry_set_cloud_sharing (on by default)
  bool chain = false;                  // run by lb_locus: stage L completes the tickets
  int normals_k = 0;                   // lb_odometry_set_normals (0 = off)
  float normals_vp[3] = {0.f, 0.f, 0.f};
  int method = LB_REG_GICP;            // lb_odometry_set_registration
  std::vector<lb_ndt*> ndt;            // one per worker (own streams), created when NDT is first selected
  // lb_locus's adaptive input voxelization (Locus.cc:780-810), touched by stage V only (and by lb_locus_set_params
  // while nothing is in flight)
  bool adaptive = false;
  int points_to_process = 0;
  bool leaf_started = false;           // `leaf` holds the VoxelGrid's leaf as of the first scan
  double leaf = 0;                     // double_param.value
  int leaf_counter = 0;                // counter_voxel_
  cudaStream_t copy_stream = nullptr;
  cudaStream_t voxel_stream = nullptr;

  std::mutex mu;
  std::condition_variable cv;          // one condition variable for every state change (few threads, short waits)
  std::deque<Entry*> inflight;         // tickets [next_return, next_ticket), in order
  uint64_t next_ticket = 0;            // next submission number
  uint64_t next_filter = 0;            // next ticket stage V takes
  uint64_t next_align = 0;             // next ticket stage G hands to a worker
  uint64_t next_return = 0;            // next ticket lb_odometry_next returns
  uint64_t done_floor = 0;             // every ticket < done_floor has finished stage G
  bool stop = false;
  // stage accounting (seconds, host wall clock; mu held when updated): which stage bounds the throughput
  double t_voxel_busy = 0, t_voxel_wait = 0, t_worker_busy = 0, t_worker_wait = 0;
  uint64_t n_filtered = 0, n_registered = 0;
  std::thread vthread;
  std::vector<std::thread> gthreads;

  Entry* entry(uint64_t t) { return inflight[(size_t)(t - next_return)]; }   // mu held
};

namespace {

void copy_err(char* dst, size_t cap) {
  const char* e = lb_last_error_string();
  strncpy(dst, e ? e : "", cap - 1);
  dst[cap - 1] = 0;
}

// what lb_odometry_result.gicp (and lb_locus_result.odometry / .localization) carry under NDT: the pose, converged,
// iterations and status; every other field 0
void ndt_as_gicp(const lb_ndt_result& n, lb_gicp_result& g) {
  memset(&g, 0, sizeof(g));
  memcpy(g.final_transformation, n.final_transformation, sizeof(g.final_transformation));
  g.converged = n.converged;
  g.iterations = n.nr_iterations;
  g.status = LB_OK;
}

void advance_done_floor(lb_odometry* h) {   // mu held
  while (h->done_floor < h->next_ticket) {
    uint64_t t = h->done_floor;
    if (t < h->next_return) { h->done_floor++; continue; }
    if (!h->entry(t)->done) break;
    h->done_floor++;
  }
}

// Locus::ApplyAdaptiveInputVoxelization (Locus.cc:780-810) after a scan whose VoxelGrid kept n points.  The reference
// publishes the new leaf on a topic and the VoxelGrid nodelet applies it to whichever scan it filters next; here it
// applies to the next scan exactly (the same rule, deterministic timing).
void adapt_leaf(lb_odometry* h, size_t n) {
  double d = h->leaf * ((double)n / (double)h->points_to_process);
  if (d < 0.01) d = 0.01;
  if (d > 5.0) d = 5.0;
  const bool change = std::abs(h->leaf - d) > 0.01 || h->leaf_counter % 20 == 0;
  if (change) { h->leaf = d; h->leaf_counter = 0; }
  h->leaf_counter++;
  // CustomVoxelGrid::ChangeLeafSizeRostopic (custom_voxel_grid.cc:62-73): the double becomes a float leaf on every axis
  if (change) lb_voxel_set_leaf_size(h->vg, (float)h->leaf, (float)h->leaf, (float)h->leaf);
}

void voxel_stage(lb_odometry* h) {
  cudaSetDevice(h->device);
  const uint64_t R = h->ring.size();
  for (;;) {
    Entry* e = nullptr;
    uint64_t t = 0;
    const auto tw0 = std::chrono::steady_clock::now();
    {
      std::unique_lock<std::mutex> lk(h->mu);
      // slot t % R was last read by registrations t-R (source) and t-R+1 (target): both must have finished
      h->cv.wait(lk, [&] {
        return h->stop || (h->next_filter < h->next_ticket && (h->next_filter + 2 <= R + h->done_floor));
      });
      if (h->stop) return;
      t = h->next_filter;
      e = h->entry(t);
    }
    const auto tb0 = std::chrono::steady_clock::now();
    Slot& s = h->ring[t % R];
    const Job& j = e->job;
    size_t n_out = 0;
    float leaf3[3] = {0.f, 0.f, 0.f};
    if (h->chain) {
      lb_voxel_get_leaf_size(h->vg, leaf3);
      if (!h->leaf_started) { h->leaf = leaf3[0]; h->leaf_started = true; }
    }
    int st;
    if (j.n_inputs) {
      // the lidars of one scan merged, transformed and filtered by one stream-ordered VoxelGrid chain (row f4)
      lb_voxel_input in[MAX_LIDARS];
      for (int i = 0; i < j.n_inputs; i++) {
        in[i].data = j.in_data[i]; in[i].n_pts = j.in_pts[i]; in[i].transform = j.has_T[i] ? j.T[i] : nullptr;
      }
      st = lb_voxel_filter_merged(h->vg, in, j.n_inputs, j.point_step, j.fields.data(), (int)j.fields.size(), s.d,
                                  h->max_points, &n_out, nullptr, j.mem, LB_MEM_DEVICE);
    } else {
      st = lb_voxel_filter(h->vg, j.scan, j.n_pts, j.point_step, j.fields.data(), (int)j.fields.size(), nullptr, 0, s.d,
                           h->max_points, &n_out, nullptr, j.mem, LB_MEM_DEVICE);
    }
    s.status = st; s.n = (st == LB_OK) ? n_out : 0; s.point_step = j.point_step; s.xyz_off = j.xyz_off;
    if (st != LB_OK) copy_err(s.error, sizeof(s.error));
    if (st == LB_OK && h->adaptive) adapt_leaf(h, n_out);     // a failed VoxelGrid is a callback that never ran
    if (st == LB_OK && j.filtered_out && n_out) {
      cudaError_t ce = cudaMemcpyAsync(j.filtered_out, s.d, n_out * j.point_step,
                                       j.mem_filtered == LB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice,
                                       h->copy_stream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(h->copy_stream);
      if (ce != cudaSuccess) {
        s.status = LB_ERR_CUDA; s.n = 0;
        snprintf(s.error, sizeof(s.error), "lb_odometry: filtered cloud copy failed: %s", cudaGetErrorString(ce));
      }
    }
    {
      std::lock_guard<std::mutex> lk(h->mu);
      e->filtered = true;
      e->res.n_filtered = s.n;
      e->leaf = leaf3[0];
      h->next_filter = t + 1;
      h->t_voxel_wait += std::chrono::duration<double>(tb0 - tw0).count();
      h->t_voxel_busy += std::chrono::duration<double>(std::chrono::steady_clock::now() - tb0).count();
      h->n_filtered++;
    }
    h->cv.notify_all();
  }
}

void align_stage(lb_odometry* h, int w) {
  cudaSetDevice(h->device);
  lb_gicp* g = h->gicp[(size_t)w];
  const uint64_t R = h->ring.size();
  for (;;) {
    Entry* e = nullptr;
    uint64_t t = 0;
    const auto tw0 = std::chrono::steady_clock::now();
    {
      std::unique_lock<std::mutex> lk(h->mu);
      h->cv.wait(lk, [&] { return h->stop || h->next_align < h->next_filter; });
      if (h->stop) return;
      t = h->next_align++;
      e = h->entry(t);
    }
    const auto tb0 = std::chrono::steady_clock::now();
    lb_odometry_result& r = e->res;
    const Slot& cur = h->ring[t % R];
    r.status = cur.status;
    if (cur.status != LB_OK) memcpy(r.error, cur.error, sizeof(r.error));
    if (h->method == LB_REG_NDT) {
      if (h->chain && cur.status == LB_OK && cur.n > 0) {
        // stage L still takes this scan's GICP cloud (keyframe transform, ICP covariance, a GICP localization): prepared
        // here, off stage L's critical path, with the odometry GICP params
        int st = lb_gicp_set_source(g, cur.d, cur.n, cur.point_step, (size_t)cur.xyz_off, LB_NO_NORMALS, LB_MEM_DEVICE);
        if (st == LB_OK && h->normals_k) st = lb_gicp_estimate_normals(g, 0, h->normals_k, h->normals_vp);
        if (st == LB_OK) st = lb_gicp_prepare_source(g);
        if (st == LB_OK) st = lb_gicp_share_source(g, &e->loc_cloud);
        if (st != LB_OK) { r.status = st; copy_err(r.error, sizeof(r.error)); }
      }
      const Slot& prv = h->ring[(t + R - 1) % R];
      if (t > 0 && r.status == LB_OK && prv.status == LB_OK && prv.n > 0 && cur.n > 0) {
        lb_ndt* nd = h->ndt[(size_t)w];
        int st = lb_ndt_set_source(nd, cur.d, cur.n, cur.point_step, (size_t)cur.xyz_off, LB_MEM_DEVICE);
        if (st == LB_OK) st = lb_ndt_set_target(nd, prv.d, prv.n, prv.point_step, (size_t)prv.xyz_off, LB_MEM_DEVICE);
        if (st == LB_OK) st = lb_ndt_align(nd, e->job.has_guess ? e->job.guess : nullptr, &r.ndt);
        r.status = st;
        if (st == LB_OK) { r.has_pose = 1; ndt_as_gicp(r.ndt, r.gicp); } else copy_err(r.error, sizeof(r.error));
      }
    } else if (h->share) {
      // this scan's cloud is prepared here, once, and published for the worker of the next registration
      lb_cloud* mine = nullptr;
      int st = cur.status;
      if (st == LB_OK && cur.n > 0) {
        st = lb_gicp_set_source(g, cur.d, cur.n, cur.point_step, (size_t)cur.xyz_off, LB_NO_NORMALS, LB_MEM_DEVICE);
        if (st == LB_OK && h->normals_k) st = lb_gicp_estimate_normals(g, 0, h->normals_k, h->normals_vp);
        if (st == LB_OK) st = lb_gicp_prepare_source(g);
        if (st == LB_OK) st = lb_gicp_share_source(g, &mine);
        // the chain's stage L adopts the same cloud as its localization source: its reference, not the ring slot,
        // keeps the points alive until stage L is done with them
        if (st == LB_OK && h->chain) st = lb_gicp_share_source(g, &e->loc_cloud);
        if (st != LB_OK) { r.status = st; copy_err(r.error, sizeof(r.error)); }
      }
      lb_cloud* prev = nullptr;
      {
        std::unique_lock<std::mutex> lk(h->mu);
        Prepared& p = h->prep[t % R];
        if (p.cloud) lb_cloud_release(p.cloud);       // slot of ticket t-R: both of its users finished long ago
        p.ticket = t; p.cloud = mine; p.ready = true;
        h->cv.notify_all();
        if (t > 0) {
          Prepared& q = h->prep[(t - 1) % R];
          h->cv.wait(lk, [&] { return h->stop || (q.ticket == t - 1 && q.ready); });
          if (!h->stop) prev = q.cloud;
        }
      }
      const bool adopt = t > 0 && mine && prev;
      if (adopt) st = lb_gicp_set_target_cloud(g, prev);       // the handle now holds its own reference
      if (t > 0) {
        // this worker is the only consumer of scan t-1's published reference: give it back now, so that the
        // owner can recycle the object two jobs later instead of R tickets later (no allocation in steady state)
        std::lock_guard<std::mutex> lk(h->mu);
        Prepared& q = h->prep[(t - 1) % R];
        if (q.ticket == t - 1 && q.cloud) { lb_cloud_release(q.cloud); q.cloud = nullptr; }
      }
      if (adopt) {
        if (st == LB_OK) st = lb_gicp_align(g, e->job.has_guess ? e->job.guess : nullptr, &r.gicp);
        r.status = st;
        if (st == LB_OK) r.has_pose = 1; else copy_err(r.error, sizeof(r.error));
      }
    } else if (t > 0 && cur.status == LB_OK) {
      const Slot& prv = h->ring[(t - 1) % R];
      if (prv.status == LB_OK && prv.n > 0 && cur.n > 0) {
        int st = lb_gicp_set_source(g, cur.d, cur.n, cur.point_step, (size_t)cur.xyz_off, LB_NO_NORMALS, LB_MEM_DEVICE);
        if (st == LB_OK && h->normals_k) st = lb_gicp_estimate_normals(g, 0, h->normals_k, h->normals_vp);
        if (st == LB_OK)
          st = lb_gicp_set_target(g, prv.d, prv.n, prv.point_step, (size_t)prv.xyz_off, LB_NO_NORMALS, LB_MEM_DEVICE, nullptr);
        if (st == LB_OK && h->normals_k) st = lb_gicp_estimate_normals(g, 1, h->normals_k, h->normals_vp);
        if (st == LB_OK) st = lb_gicp_align(g, e->job.has_guess ? e->job.guess : nullptr, &r.gicp);
        r.status = st;
        if (st == LB_OK) r.has_pose = 1; else copy_err(r.error, sizeof(r.error));
      }
    }
    {
      std::lock_guard<std::mutex> lk(h->mu);
      if (h->chain) {
        e->aligned = true;
      } else {
        e->done = true;
        advance_done_floor(h);
      }
      h->t_worker_wait += std::chrono::duration<double>(tb0 - tw0).count();
      h->t_worker_busy += std::chrono::duration<double>(std::chrono::steady_clock::now() - tb0).count();
      h->n_registered++;
    }
    h->cv.notify_all();
  }
}

int odometry_create(int device, int depth, size_t max_points, uint32_t max_point_step, bool chain, lb_odometry** out) {
  if (!out || depth < 1 || depth > 16 || max_points == 0 || max_point_step < 12) {
    set_error("lb_odometry_create: need depth in 1..16, max_points > 0, max_point_step >= 12");
    return LB_ERR_INVALID_ARG;
  }
  lb_odometry* h = new lb_odometry;
  h->device = device; h->depth = depth; h->max_points = max_points; h->max_step = max_point_step; h->chain = chain;
  // The VoxelGrid stage is the one serial stage of the pipeline and a chain of ~12 short dependent kernels: on its
  // own high-priority stream its CTAs are placed before the pending CTAs of the workers' k-NN / index kernels.
  int st = LB_OK;
  {
    int lo = 0, hi = 0;
    const char* e = getenv("LB_VOXEL_PRIO");
    if (cudaSetDevice(device) != cudaSuccess || cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&h->voxel_stream, cudaStreamNonBlocking, (e && atoi(e) == 0) ? lo : hi) != cudaSuccess) {
      set_error("lb_odometry_create: stream creation failed: %s", cudaGetErrorString(cudaGetLastError()));
      st = LB_ERR_CUDA;
    }
  }
  if (st == LB_OK) st = lb_voxel_create_on_stream(device, h->voxel_stream, &h->vg);
  // no device allocation in steady state: the VoxelGrid's scratch for raw scans of up to max_points points (a merged
  // scan grows mid-stream when a lidar comes back)
  if (st == LB_OK) st = voxel_reserve(h->vg, max_points, max_point_step);
  for (int i = 0; st == LB_OK && i < depth; i++) {
    lb_gicp* g = nullptr;
    st = lb_gicp_create(device, &g);
    // no device allocation in steady state: clouds of up to max_points points, and enough spare cloud objects for the
    // sharing mode (a prepared cloud stays referenced until the next worker has adopted and used it)
    if (st == LB_OK) h->gicp.push_back(g);
    if (st == LB_OK) st = lb_gicp_reserve(g, max_points, 8);
  }
  if (st == LB_OK) {
    h->ring.resize((size_t)depth + 3);
    h->prep.resize((size_t)depth + 3);
    for (auto& s : h->ring) {
      if (cudaMalloc((void**)&s.d, max_points * (size_t)max_point_step) != cudaSuccess) {
        set_error("lb_odometry_create: ring allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
        st = LB_ERR_CUDA;
        break;
      }
    }
  }
  if (st == LB_OK && cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess) {
    set_error("lb_odometry_create: stream creation failed");
    st = LB_ERR_CUDA;
  }
  if (st != LB_OK) {
    for (auto& s : h->ring) if (s.d) cudaFree(s.d);
    for (auto g : h->gicp) lb_gicp_destroy(g);
    if (h->vg) lb_voxel_destroy(h->vg);
    if (h->voxel_stream) cudaStreamDestroy(h->voxel_stream);
    delete h;
    return st;
  }
  h->vthread = std::thread(voxel_stage, h);
  for (int i = 0; i < depth; i++) h->gthreads.emplace_back(align_stage, h, i);
  *out = h;
  return LB_OK;
}

// The refusals of a registration setting, before anything changes (mu not held): method, NDT params, an idle pipeline,
// a method change after the first scan, and NDT with the normals stage outside lb_locus.
int registration_check(lb_odometry* h, int method, const lb_ndt_params* ndt, const char* who) {
  if (method != LB_REG_GICP && method != LB_REG_NDT) {
    set_error("%s: method must be LB_REG_GICP (0) or LB_REG_NDT (1), got %d", who, method);
    return LB_ERR_INVALID_ARG;
  }
  if (method == LB_REG_NDT) {
    if (!ndt) { set_error("%s: NDT needs its params", who); return LB_ERR_INVALID_ARG; }
    LB_TRY(ndt_check_params(ndt, who));
  }
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->next_return != h->next_ticket) { set_error("%s: pipeline not idle", who); return LB_ERR_INVALID_ARG; }
  if (h->next_ticket != 0 && method != h->method) {
    // the previous scan exists only in the form its method prepared (a GICP worker adopts its shared cloud)
    set_error("%s: change the registration method before the first scan is submitted", who);
    return LB_ERR_UNSUPPORTED;
  }
  if (method == LB_REG_NDT && h->normals_k && !h->chain) {
    set_error("%s: the normals stage has no consumer under NDT registration", who);
    return LB_ERR_UNSUPPORTED;
  }
  return LB_OK;
}

// one lb_ndt per worker, sized like the ring, created the first time NDT is selected
int odometry_ndt_handles(lb_odometry* h) {
  if (!h->ndt.empty()) return LB_OK;
  std::vector<lb_ndt*> v;
  int st = LB_OK;
  for (int i = 0; st == LB_OK && i < h->depth; i++) {
    lb_ndt* n = nullptr;
    st = lb_ndt_create(h->device, &n);
    if (st == LB_OK) v.push_back(n);
    if (st == LB_OK) st = ndt_reserve(n, h->max_points);
  }
  if (st != LB_OK) {
    for (auto n : v) lb_ndt_destroy(n);
    return st;
  }
  h->ndt = v;
  return LB_OK;
}

// after registration_check and odometry_ndt_handles: applies the setting (params already validated)
int odometry_set_registration(lb_odometry* h, int method, const lb_ndt_params* ndt) {
  if (method == LB_REG_NDT)
    for (auto n : h->ndt) LB_TRY(lb_ndt_set_params(n, ndt));
  std::lock_guard<std::mutex> lk(h->mu);
  h->method = method;
  return LB_OK;
}

// the next ticket in submission order once it is done (mu not held); 1 = not done yet and block == 0
int take_next(lb_odometry* h, int block, const char* who, Entry** out) {
  Entry* e = nullptr;
  {
    std::unique_lock<std::mutex> lk(h->mu);
    if (h->next_return == h->next_ticket) { set_error("%s: nothing pending", who); return LB_ERR_NO_ALIGN; }
    e = h->inflight.front();
    if (!e->done) {
      if (!block) return 1;
      h->cv.wait(lk, [&] { return e->done; });
    }
    h->inflight.pop_front();
    h->next_return++;
    advance_done_floor(h);
  }
  h->cv.notify_all();
  *out = e;
  return LB_OK;
}

}  // namespace

extern "C" {

int lb_odometry_create(int device, int depth, size_t max_points, uint32_t max_point_step, lb_odometry** out) {
  return odometry_create(device, depth, max_points, max_point_step, false, out);
}

int lb_odometry_destroy(lb_odometry* h) {
  if (!h) return LB_OK;
  {
    std::lock_guard<std::mutex> lk(h->mu);
    h->stop = true;
  }
  h->cv.notify_all();
  if (h->vthread.joinable()) h->vthread.join();
  for (auto& t : h->gthreads) if (t.joinable()) t.join();
  cudaSetDevice(h->device);
  for (auto& p : h->prep) if (p.cloud) { lb_cloud_release(p.cloud); p.cloud = nullptr; }
  for (auto g : h->gicp) lb_gicp_destroy(g);
  for (auto n : h->ndt) lb_ndt_destroy(n);
  lb_voxel_destroy(h->vg);
  for (auto& s : h->ring) if (s.d) cudaFree(s.d);
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  if (h->voxel_stream) cudaStreamDestroy(h->voxel_stream);
  for (auto e : h->inflight) {
    if (e->loc_cloud) lb_cloud_release(e->loc_cloud);
    delete e;
  }
  delete h;
  return LB_OK;
}

lb_voxel* lb_odometry_voxel(lb_odometry* h) { return h ? h->vg : nullptr; }
lb_gicp* lb_odometry_gicp(lb_odometry* h, int i) { return (h && i >= 0 && i < h->depth) ? h->gicp[(size_t)i] : nullptr; }
int lb_odometry_depth(lb_odometry* h) { return h ? h->depth : 0; }

int lb_odometry_set_gicp_params(lb_odometry* h, const lb_gicp_params* p) {
  if (!h || !p) { set_error("lb_odometry_set_gicp_params: null argument"); return LB_ERR_INVALID_ARG; }
  {
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->next_return != h->next_ticket) { set_error("lb_odometry_set_gicp_params: pipeline not idle"); return LB_ERR_INVALID_ARG; }
  }
  for (auto g : h->gicp) LB_TRY(lb_gicp_set_params(g, p));
  return LB_OK;
}

int lb_odometry_set_cloud_sharing(lb_odometry* h, int on) {
  if (!h) { set_error("lb_odometry_set_cloud_sharing: null handle"); return LB_ERR_INVALID_ARG; }
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->next_return != h->next_ticket) { set_error("lb_odometry_set_cloud_sharing: pipeline not idle"); return LB_ERR_INVALID_ARG; }
  if (h->next_ticket != 0 && (on != 0) != h->share) {
    // the previous scan's cloud exists in one form only (ring slot or prepared cloud): switch before the first scan
    set_error("lb_odometry_set_cloud_sharing: switch before the first scan is submitted");
    return LB_ERR_UNSUPPORTED;
  }
  h->share = on != 0;
  return LB_OK;
}

int lb_odometry_set_normals(lb_odometry* h, int k, const float* viewpoint) {
  if (!h) { set_error("lb_odometry_set_normals: null handle"); return LB_ERR_INVALID_ARG; }
  if (k != 0 && (k < 3 || k > 20)) { set_error("lb_odometry_set_normals: k must be 0 (off) or in [3, 20]"); return LB_ERR_UNSUPPORTED; }
  const float vp[3] = {viewpoint ? viewpoint[0] : 0.f, viewpoint ? viewpoint[1] : 0.f, viewpoint ? viewpoint[2] : 0.f};
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->next_return != h->next_ticket) { set_error("lb_odometry_set_normals: pipeline not idle"); return LB_ERR_INVALID_ARG; }
  if (k != 0 && h->method == LB_REG_NDT && !h->chain) {
    set_error("lb_odometry_set_normals: the normals stage has no consumer under NDT registration");
    return LB_ERR_UNSUPPORTED;
  }
  if (h->next_ticket != 0 && (k != h->normals_k || memcmp(vp, h->normals_vp, sizeof(vp)) != 0)) {
    // the previous scan's prepared cloud was built with the old setting
    set_error("lb_odometry_set_normals: change before the first scan is submitted");
    return LB_ERR_UNSUPPORTED;
  }
  h->normals_k = k;
  memcpy(h->normals_vp, vp, sizeof(vp));
  return LB_OK;
}

int lb_odometry_set_registration(lb_odometry* h, int method, const lb_ndt_params* ndt) {
  if (!h) { set_error("lb_odometry_set_registration: null handle"); return LB_ERR_INVALID_ARG; }
  LB_TRY(registration_check(h, method, ndt, "lb_odometry_set_registration"));
  if (method == LB_REG_NDT) LB_TRY(odometry_ndt_handles(h));
  return odometry_set_registration(h, method, ndt);
}

}  // extern "C"

namespace {

// the checks and the queueing both submit calls share: scan of n_pts points in total; merged: the caller fills
// the Job's inputs into *job_out before it is queued (a callback, so that a refusal allocates nothing)
template <class Fill>
int submit_job(lb_odometry* h, const char* who, size_t n_pts, uint32_t point_step, const lb_field* fields, int n_fields,
               int mem, const float* guess, uint8_t* filtered_out, int mem_filtered, uint64_t* ticket, Fill fill) {
  if (n_pts > h->max_points || point_step > h->max_step) {
    set_error("%s: scan of %zu x %u bytes exceeds the pipeline's ring (%zu x %u)", who, n_pts, point_step,
              h->max_points, h->max_step);
    return LB_ERR_CAPACITY;
  }
  int xo = -1;
  for (int f = 0; f < n_fields; f++)
    if (!strcmp(fields[f].name, "x") && fields[f].datatype == LB_FLOAT32) xo = (int)fields[f].offset;
  if (xo < 0) { set_error("%s: FLOAT32 field 'x' required", who); return LB_ERR_INVALID_ARG; }
  Entry* e = new Entry;
  Job& j = e->job;
  j.n_pts = n_pts; j.point_step = point_step; j.fields.assign(fields, fields + n_fields); j.mem = mem;
  fill(j);
  j.has_guess = guess != nullptr;
  if (guess) memcpy(j.guess, guess, sizeof(j.guess));
  j.filtered_out = filtered_out; j.mem_filtered = mem_filtered; j.xyz_off = xo;
  memset(&e->res, 0, sizeof(e->res));
  {
    std::unique_lock<std::mutex> lk(h->mu);
    const uint64_t limit = 2 * (uint64_t)h->depth + 2;
    h->cv.wait(lk, [&] { return h->next_ticket - h->done_floor < limit; });
    j.ticket = e->res.ticket = h->next_ticket++;
    h->inflight.push_back(e);
    if (ticket) *ticket = j.ticket;
  }
  h->cv.notify_all();
  return LB_OK;
}

}  // namespace

extern "C" {

int lb_odometry_submit(lb_odometry* h, const uint8_t* scan, size_t n_pts, uint32_t point_step, const lb_field* fields,
                       int n_fields, int mem, const float* guess, uint8_t* filtered_out, int mem_filtered,
                       uint64_t* ticket) {
  if (!h || !scan || !fields || n_fields <= 0) { set_error("lb_odometry_submit: null argument"); return LB_ERR_INVALID_ARG; }
  return submit_job(h, "lb_odometry_submit", n_pts, point_step, fields, n_fields, mem, guess, filtered_out, mem_filtered,
                    ticket, [&](Job& j) { j.scan = scan; });
}

int lb_odometry_submit_merged(lb_odometry* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step,
                              const lb_field* fields, int n_fields, int mem, const float* guess, uint8_t* filtered_out,
                              int mem_filtered, uint64_t* ticket) {
  if (!h || !inputs || !fields || n_fields <= 0) { set_error("lb_odometry_submit_merged: null argument"); return LB_ERR_INVALID_ARG; }
  if (n_inputs < 1 || n_inputs > MAX_LIDARS) {
    set_error("lb_odometry_submit_merged: 1 to %d input clouds, got %d", MAX_LIDARS, n_inputs);
    return LB_ERR_INVALID_ARG;
  }
  size_t n_pts = 0;
  for (int i = 0; i < n_inputs; i++) {
    if (inputs[i].n_pts && !inputs[i].data) { set_error("lb_odometry_submit_merged: null input cloud %d", i); return LB_ERR_INVALID_ARG; }
    n_pts += inputs[i].n_pts;
  }
  return submit_job(h, "lb_odometry_submit_merged", n_pts, point_step, fields, n_fields, mem, guess, filtered_out,
                    mem_filtered, ticket, [&](Job& j) {
                      j.n_inputs = n_inputs;
                      for (int i = 0; i < n_inputs; i++) {
                        j.in_data[i] = inputs[i].data; j.in_pts[i] = inputs[i].n_pts;
                        j.has_T[i] = inputs[i].transform != nullptr;     // copied: the caller's array may go now
                        if (j.has_T[i]) memcpy(j.T[i], inputs[i].transform, sizeof(j.T[i]));
                      }
                    });
}

int lb_odometry_next(lb_odometry* h, lb_odometry_result* r, int block) {
  if (!h || !r) { set_error("lb_odometry_next: null argument"); return LB_ERR_INVALID_ARG; }
  Entry* e = nullptr;
  const int st = take_next(h, block, "lb_odometry_next", &e);
  if (st != LB_OK) return st;
  *r = e->res;
  delete e;
  return LB_OK;
}

int lb_odometry_pending(lb_odometry* h, size_t* n) {
  if (!h || !n) return LB_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  *n = (size_t)(h->next_ticket - h->next_return);
  return LB_OK;
}

int lb_odometry_stage_times(lb_odometry* h, double* out6) {
  if (!h || !out6) return LB_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lk(h->mu);
  out6[0] = (double)h->n_filtered; out6[1] = h->t_voxel_busy; out6[2] = h->t_voxel_wait;
  out6[3] = (double)h->n_registered; out6[4] = h->t_worker_busy; out6[5] = h->t_worker_wait;
  return LB_OK;
}

int lb_odometry_launch_count(lb_odometry* h, uint64_t* n) {
  if (!h || !n) return LB_ERR_INVALID_ARG;
  uint64_t tot = 0, v = 0;
  lb_voxel_launch_count(h->vg, &v); tot += v;
  for (auto g : h->gicp) { lb_gicp_launch_count(g, &v); tot += v; }
  for (auto nd : h->ndt) { lb_ndt_launch_count(nd, &v); tot += v; }
  *n = tot;
  return LB_OK;
}

}  // extern "C"

// ================================================================ lb_locus_*: the whole lidar callback
// The core above with stage L behind stage G.  Per ticket, in order, stage L adopts the scan's prepared cloud as the
// source of its own lb_gicp handle, aligns it against the caller's rolling submap and does the pose bookkeeping and map
// updates of Locus.cc:462-543 (lo_pose.h).  With localization_method = NDT the align is that of stage L's lb_ndt handle
// (source = the scan's filtered points in its ring slot, target = the submap's points); the GICP handle then only
// transforms keyframes and, with the ICP covariance on, searches the map.  It is the one stage that depends on the
// previous scan's result, so it is the only serial one; V and G fill and register the following scans meanwhile.
#if !defined(LB_ODOMETRY_STUB) || defined(LB_LOCUS_STUB)

namespace lb {
int submap_device(const lb_submap* m);
}

struct lb_locus {
  lb_odometry* core = nullptr;
  lb_gicp* g = nullptr;            // stage L's handle (own stream); source = the shared cloud, target = the submap
  lb_ndt* ndt = nullptr;           // stage L's NDT handle (own stream), created when localization NDT is first selected
  lb_submap* map = nullptr;        // the caller's
  float* d_xyz = nullptr;          // a keyframe's points in the fixed frame, max_points x 6 floats (xyz, normal)
  lb_locus_params P{};
  // pose state, touched by stage L only (and by set_params while nothing is in flight)
  bool started = false;            // the first scan has been taken
  lo::Pose O, L, KF;               // odometry estimate, localization estimate, last keyframe
  int counter = 0;                 // keyframes since the last Refresh
  double condition_number = NAN;   // the last ICP condition number computed (condition_number_, kept over a NaN fallback)
  double t_busy = 0, t_wait = 0;   // core->mu held when updated
  uint64_t n_localized = 0;
  std::thread lthread;
};

namespace {

int locus_insert(lb_locus* c, size_t n, lb_locus_result& r) {
  float T[16];
  lo::to_mat(c->L, T);
  size_t ins = 0;
  if (c->P.front_end.normals_k) {
    // Locus.cc:530-532: the keyframe enters the map with its normals rotated into the fixed frame
    LB_TRY(lb_gicp_transform_source(c->g, T, c->d_xyz, 24, 0, 12, LB_MEM_DEVICE));
    LB_TRY(lb_submap_insert_with_normals(c->map, c->d_xyz, n, 24, 0, 12, LB_MEM_DEVICE, &ins, nullptr));
  } else {
    LB_TRY(lb_gicp_transform_source(c->g, T, c->d_xyz, 12, 0, LB_NO_NORMALS, LB_MEM_DEVICE));
    LB_TRY(lb_submap_insert(c->map, c->d_xyz, n, 12, 0, LB_MEM_DEVICE, &ins, nullptr));
  }
  r.keyframe = 1;
  r.n_inserted = ins;
  return LB_OK;
}

// MotionUpdate(I) + MeasurementUpdate against the submap + the keyframe branch (PointCloudLocalization.cc:313-382,
// Locus.cc:514-543).  s: the scan's ring slot (its filtered points, the NDT source)
int locus_localize(lb_locus* c, const lo::Pose& I, const Slot& s, lb_locus_result& r) {
  const size_t n = s.n;
  const lo::Pose P = lo::update(c->L, I);
  float guess[16];
  lo::to_mat(P, guess);
  const bool ndt = c->P.localization_method == LB_REG_NDT;
  if (ndt) {
    LB_TRY(lb_ndt_set_source(c->ndt, s.d, s.n, s.point_step, (size_t)s.xyz_off, LB_MEM_DEVICE));
    LB_TRY(lb_ndt_set_target_submap(c->ndt, c->map));      // no device work while the map is unchanged
    LB_TRY(lb_ndt_align(c->ndt, guess, &r.localization_ndt));
    ndt_as_gicp(r.localization_ndt, r.localization);
  } else {
    LB_TRY(lb_gicp_set_target_submap(c->g, c->map));
    LB_TRY(lb_gicp_align(c->g, guess, &r.localization));
  }
  r.has_localization = 1;
  if (c->P.icp_covariance.enabled) {
    // PointCloudLocalization.cc:325-336 searches getSearchMethodTarget(), the target's kd-tree, for NDT too: the GICP
    // handle takes the map as target for the 1-NN (the GICP align has done so already)
    if (ndt) LB_TRY(lb_gicp_set_target_submap(c->g, c->map));
    // PointCloudLocalization.cc:325-336,398-421: the ICP covariance of this align, before the map changes.  The
    // reference's target is the mapper's neighbours in the frame of P (the align's guess); the submap is in the fixed
    // frame, so its normals are rotated by P^-1 (unpinned, DESIGN.md 4i)
    const lo::Pose Pinv = lo::inverse(P);
    float Rf[9];
    for (int i = 0; i < 9; i++) Rf[i] = (float)Pinv.R[i];
    lb_icp_covariance ic;
    LB_TRY(lb_gicp_icp_covariance(c->g, r.localization.final_transformation, nullptr, LB_MEM_HOST, Rf,
                                  c->P.icp_covariance.max_covariance, &ic));
    r.has_icp_covariance = 1;
    memcpy(r.icp_covariance, ic.covariance, sizeof(r.icp_covariance));
    r.icp_covariance_flags = ic.flags;
    if (!(ic.flags & LB_ICPCOV_D_NAN)) c->condition_number = ic.condition_number;
  }
  const lo::Pose U = lo::delta(P, lo::from_mat(r.localization.final_transformation));   // sensor-frame correction
  const lb_locus_thresholds& th = c->P.localization_thresholds;
  r.correction_accepted = lo::passes(U, th.enabled, th.max_translation, th.max_rotation);
  c->L = lo::update(c->L, r.correction_accepted ? lo::update(I, U) : I);
  if (!c->P.add_keyframes || !lo::is_keyframe(lo::delta(c->KF, c->L), c->P.translation_threshold_kf, c->P.rotation_threshold_kf))
    return LB_OK;
  LB_TRY(locus_insert(c, n, r));
  if (++c->counter == c->P.refresh_every) {
    c->counter = 0;
    if (c->P.msw) {
      const float centre[3] = {(float)c->L.t[0], (float)c->L.t[1], (float)c->L.t[2]};
      size_t removed = 0;
      LB_TRY(lb_submap_crop_box(c->map, centre, c->P.window_half_size, &removed));
      r.n_removed = removed;
    }
  }
  c->KF = c->L;
  return LB_OK;
}

void locus_scan(lb_locus* c, Entry* e) {
  const lb_odometry_result& o = e->res;
  lb_locus_result& r = e->loc;
  memset(&r, 0, sizeof(r));
  r.ticket = o.ticket; r.status = o.status; r.n_filtered = o.n_filtered; r.leaf_size = e->leaf;
  memcpy(r.error, o.error, sizeof(r.error));
  r.has_odometry = o.has_pose;
  r.odometry = o.gicp;
  r.odometry_ndt = o.ndt;
  const Slot& slot = c->core->ring[o.ticket % c->core->ring.size()];   // kept until this ticket is done (voxel_stage)
  lb_cloud* cl = e->loc_cloud;
  e->loc_cloud = nullptr;
  lo::Pose I = lo::identity();
  // a failed voxel or odometry stage (or an empty filtered scan) changes no state
  if (o.status == LB_OK && cl) {
    int st = lb_gicp_set_source_cloud(c->g, cl);
    if (st == LB_OK) {
      if (o.has_pose) {
        // PointCloudOdometry.cc:265-316: the increment is stored before the thresholds are tested, and localization
        // receives it either way (Locus.cc:474)
        I = lo::from_mat(o.gicp.final_transformation);
        const lb_locus_thresholds& th = c->P.odometry_thresholds;
        r.odometry_accepted = lo::passes(I, th.enabled, th.max_translation, th.max_rotation);
        if (r.odometry_accepted) c->O = lo::update(c->O, I);
      }
      if (!c->started) {
        // Locus.cc:462-472: the first scan seeds the map at the initial pose -- unless a prior map is loaded, in
        // which case it is localized against it like any other scan (with I = identity)
        c->started = true;
        st = c->P.prior_map ? locus_localize(c, I, slot, r) : locus_insert(c, o.n_filtered, r);
      } else {
        st = locus_localize(c, I, slot, r);
      }
    }
    if (st != LB_OK) { r.status = st; copy_err(r.error, sizeof(r.error)); }
  }
  if (cl) lb_cloud_release(cl);
  lo::to_mat(c->O, r.odometry_pose);
  lo::to_mat(I, r.incremental);
  lo::to_mat(c->L, r.pose);
  lb_submap_size(c->map, &r.map_size);
  if (c->P.icp_covariance.enabled) r.condition_number = c->condition_number;
}

void loc_stage(lb_locus* c) {
  lb_odometry* h = c->core;
  cudaSetDevice(h->device);
  for (uint64_t t = 0;; t++) {
    Entry* e = nullptr;
    const auto tw0 = std::chrono::steady_clock::now();
    {
      std::unique_lock<std::mutex> lk(h->mu);
      h->cv.wait(lk, [&] { return h->stop || (t < h->next_ticket && h->entry(t)->aligned); });
      if (h->stop) return;
      e = h->entry(t);
    }
    const auto tb0 = std::chrono::steady_clock::now();
    locus_scan(c, e);
    {
      std::lock_guard<std::mutex> lk(h->mu);
      e->done = true;
      advance_done_floor(h);
      c->t_wait += std::chrono::duration<double>(tb0 - tw0).count();
      c->t_busy += std::chrono::duration<double>(std::chrono::steady_clock::now() - tb0).count();
      c->n_localized++;
    }
    h->cv.notify_all();
  }
}

int locus_apply_params(lb_locus* c, const lb_locus_params* p) {
  if (p->odometry.k_correspondences != p->localization.k_correspondences || p->odometry.gicp_epsilon != p->localization.gicp_epsilon ||
      p->odometry.index_cell_size != p->localization.index_cell_size) {
    set_error("lb_locus_set_params: odometry and localization must agree on k_correspondences, gicp_epsilon and "
              "index_cell_size (each scan's index and covariances are built once for both)");
    return LB_ERR_INVALID_ARG;
  }
  if (p->odometry.recompute_source_covariance != p->odometry.recompute_target_covariance ||
      p->odometry.recompute_source_covariance != p->localization.recompute_source_covariance) {
    set_error("lb_locus_set_params: the odometry's recompute_source_covariance and recompute_target_covariance and the "
              "localization's recompute_source_covariance must agree (one prepared cloud serves all three)");
    return LB_ERR_INVALID_ARG;
  }
  if (p->refresh_every < 1 || !(p->window_half_size > 0.f)) {
    set_error("lb_locus_set_params: need refresh_every >= 1 and window_half_size > 0");
    return LB_ERR_INVALID_ARG;
  }
  const lb_locus_front_end& fe = p->front_end;
  if ((fe.normals_k != 0 && (fe.normals_k < 3 || fe.normals_k > 20)) || (fe.adaptive_voxelization && fe.points_to_process <= 0)) {
    set_error("lb_locus_set_params: front_end needs normals_k = 0 or in [3, 20], and points_to_process > 0 with "
              "adaptive_voxelization");
    return LB_ERR_INVALID_ARG;
  }
  // checked when the covariance is on, so that parameters filled field by field without it keep working
  if (p->icp_covariance.enabled && (!std::isfinite(p->icp_covariance.max_covariance) || !(p->icp_covariance.max_covariance > 0.0))) {
    set_error("lb_locus_set_params: icp_covariance.max_covariance must be finite and > 0");
    return LB_ERR_INVALID_ARG;
  }
  // registration methods: checked (and their NDT handles made) before anything changes
  LB_TRY(registration_check(c->core, p->odometry_method, &p->odometry_ndt, "lb_locus_set_params"));
  if (p->localization_method != LB_REG_GICP && p->localization_method != LB_REG_NDT) {
    set_error("lb_locus_set_params: localization_method must be LB_REG_GICP (0) or LB_REG_NDT (1)");
    return LB_ERR_INVALID_ARG;
  }
  if (p->localization_method == LB_REG_NDT) LB_TRY(ndt_check_params(&p->localization_ndt, "lb_locus_set_params"));
  bool submitted;
  {
    std::lock_guard<std::mutex> lk(c->core->mu);
    submitted = c->core->next_ticket != 0;
  }
  if (submitted && p->localization_method != c->P.localization_method) {
    set_error("lb_locus_set_params: change the registration method before the first scan is submitted");
    return LB_ERR_UNSUPPORTED;
  }
  if (p->odometry_method == LB_REG_NDT) LB_TRY(odometry_ndt_handles(c->core));
  if (p->localization_method == LB_REG_NDT && !c->ndt) {
    lb_ndt* n = nullptr;
    LB_TRY(lb_ndt_create(c->core->device, &n));
    const int s = ndt_reserve(n, c->core->max_points);       // the scan side; the map side grows with the map
    if (s != LB_OK) { lb_ndt_destroy(n); return s; }
    c->ndt = n;
  }
  LB_TRY(lb_odometry_set_normals(c->core, fe.normals_k, fe.viewpoint));
  int st = lb_gicp_set_params(c->g, &p->localization);
  if (st == LB_OK) {
    st = lb_odometry_set_gicp_params(c->core, &p->odometry);
    if (st != LB_OK) lb_gicp_set_params(c->g, &c->P.localization);   // keep the previous state
  }
  if (st == LB_OK) {
    st = odometry_set_registration(c->core, p->odometry_method, &p->odometry_ndt);
    if (st == LB_OK && p->localization_method == LB_REG_NDT) st = lb_ndt_set_params(c->ndt, &p->localization_ndt);
    if (st != LB_OK) {
      lb_gicp_set_params(c->g, &c->P.localization);
      lb_odometry_set_gicp_params(c->core, &c->P.odometry);
      odometry_set_registration(c->core, c->P.odometry_method, &c->P.odometry_ndt);
    }
  }
  if (st != LB_OK) {
    lb_odometry_set_normals(c->core, c->P.front_end.normals_k, c->P.front_end.viewpoint);
    return st;
  }
  {
    std::lock_guard<std::mutex> lk(c->core->mu);
    c->core->adaptive = fe.adaptive_voxelization != 0;
    c->core->points_to_process = fe.points_to_process;
  }
  c->P = *p;
  if (!c->started) {
    c->O = lo::identity();
    c->L = c->KF = lo::from_mat(p->initial_pose);
  }
  return LB_OK;
}

}  // namespace

extern "C" {

int lb_locus_default_params(lb_locus_params* p) {
  if (!p) { set_error("lb_locus_default_params: null argument"); return LB_ERR_INVALID_ARG; }
  memset(p, 0, sizeof(*p));
  // point_cloud_odometry/config/parameters.yaml icp/*, PointCloudOdometry.cc:147-155
  lb_gicp_default_params(&p->odometry);
  p->odometry.transformation_epsilon = 0.001;
  p->odometry.max_correspondence_distance = 1.0;
  p->odometry.max_iterations = 20;
  p->odometry.ransac_iterations = 0;
  p->odometry.euclidean_fitness_epsilon = 0.005;
  p->odometry.align_points_per_cta = 1024;      // the chain's SM budget (DESIGN.md)
  p->odometry_thresholds = {1, 1.0, 1.0};
  // point_cloud_localization/config/parameters.yaml localization/*
  lb_gicp_default_params(&p->localization);
  p->localization.transformation_epsilon = 0.00001;
  p->localization.max_correspondence_distance = 0.2;
  p->localization.max_iterations = 20;
  p->localization.ransac_iterations = 0;
  p->localization_thresholds = {1, 1.0, 1.0};
  // locus/config/lo_settings.yaml
  p->translation_threshold_kf = 1.0;
  p->rotation_threshold_kf = 0.3;
  p->add_keyframes = 1;
  p->refresh_every = 1;          // map_publishment/meters
  p->msw = 1;                    // b_enable_msw
  p->window_half_size = 20.f;    // box_filter_size
  p->prior_map = 0;              // b_run_with_gt_point_cloud
  for (int i = 0; i < 16; i++) p->initial_pose[i] = (i % 5 == 0) ? 1.0 : 0.0;
  p->icp_covariance.enabled = 0;               // off: the chain computes what it computed without it
  p->icp_covariance.max_covariance = 0.01;     // point_cloud_localization/config/parameters.yaml icp_max_covariance
  // registration_method: gicp in both packages; their NDT settings (PointCloudOdometry.cc:182-195,
  // PointCloudLocalization.cc:267-280) take the same icp_tf_epsilon / icp_iterations (tf_epsilon / iterations) values
  p->odometry_method = LB_REG_GICP;
  p->localization_method = LB_REG_GICP;
  lb_ndt_default_params(&p->odometry_ndt);
  p->odometry_ndt.transformation_epsilon = 0.001;
  p->odometry_ndt.max_iterations = 20;
  lb_ndt_default_params(&p->localization_ndt);
  p->localization_ndt.transformation_epsilon = 0.00001;
  p->localization_ndt.max_iterations = 20;
  return LB_OK;
}

int lb_locus_create(int device, int depth, size_t max_points, uint32_t max_point_step, lb_submap* map, lb_locus** out) {
  if (!out || !map) { set_error("lb_locus_create: null argument"); return LB_ERR_INVALID_ARG; }
  if (lb::submap_device(map) != device) {
    set_error("lb_locus_create: submap on device %d, chain on %d", lb::submap_device(map), device);
    return LB_ERR_INVALID_ARG;
  }
  lb_locus* c = new lb_locus;
  c->map = map;
  lb_locus_params P{};
  lb_locus_default_params(&P);
  int st = odometry_create(device, depth, max_points, max_point_step, true, &c->core);
  if (st == LB_OK) st = lb_gicp_create(device, &c->g);
  if (st == LB_OK) st = lb_gicp_reserve(c->g, max_points, 0);
  if (st == LB_OK && cudaMalloc((void**)&c->d_xyz, max_points * 6 * sizeof(float)) != cudaSuccess) {
    set_error("lb_locus_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    st = LB_ERR_CUDA;
  }
  if (st == LB_OK) st = locus_apply_params(c, &P);
  if (st != LB_OK) {
    if (c->g) lb_gicp_destroy(c->g);
    if (c->ndt) lb_ndt_destroy(c->ndt);
    if (c->core) lb_odometry_destroy(c->core);
    if (c->d_xyz) cudaFree(c->d_xyz);
    delete c;
    return st;
  }
  c->lthread = std::thread(loc_stage, c);
  *out = c;
  return LB_OK;
}

int lb_locus_destroy(lb_locus* c) {
  if (!c) return LB_OK;
  {
    std::lock_guard<std::mutex> lk(c->core->mu);
    c->core->stop = true;
  }
  c->core->cv.notify_all();
  if (c->lthread.joinable()) c->lthread.join();
  cudaSetDevice(c->core->device);
  lb_gicp_destroy(c->g);
  if (c->ndt) lb_ndt_destroy(c->ndt);
  lb_odometry_destroy(c->core);    // joins stages V and G, releases the clouds of the scans still in flight
  cudaFree(c->d_xyz);
  delete c;
  return LB_OK;
}

lb_voxel* lb_locus_voxel(lb_locus* c) { return c ? c->core->vg : nullptr; }

int lb_locus_set_params(lb_locus* c, const lb_locus_params* p) {
  if (!c || !p) { set_error("lb_locus_set_params: null argument"); return LB_ERR_INVALID_ARG; }
  {
    std::lock_guard<std::mutex> lk(c->core->mu);
    if (c->core->next_return != c->core->next_ticket) { set_error("lb_locus_set_params: scans in flight"); return LB_ERR_INVALID_ARG; }
  }
  return locus_apply_params(c, p);
}

int lb_locus_submit(lb_locus* c, const uint8_t* scan, size_t n_pts, uint32_t point_step, const lb_field* fields,
                    int n_fields, int mem, const float* guess, uint8_t* filtered_out, int mem_filtered, uint64_t* ticket) {
  if (!c) { set_error("lb_locus_submit: null handle"); return LB_ERR_INVALID_ARG; }
  return lb_odometry_submit(c->core, scan, n_pts, point_step, fields, n_fields, mem, guess, filtered_out, mem_filtered, ticket);
}

int lb_locus_submit_merged(lb_locus* c, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step, const lb_field* fields,
                           int n_fields, int mem, const float* guess, uint8_t* filtered_out, int mem_filtered, uint64_t* ticket) {
  if (!c) { set_error("lb_locus_submit_merged: null handle"); return LB_ERR_INVALID_ARG; }
  return lb_odometry_submit_merged(c->core, inputs, n_inputs, point_step, fields, n_fields, mem, guess, filtered_out,
                                   mem_filtered, ticket);
}

int lb_locus_next(lb_locus* c, lb_locus_result* r, int block) {
  if (!c || !r) { set_error("lb_locus_next: null argument"); return LB_ERR_INVALID_ARG; }
  Entry* e = nullptr;
  const int st = take_next(c->core, block, "lb_locus_next", &e);
  if (st != LB_OK) return st;
  *r = e->loc;
  delete e;
  return LB_OK;
}

int lb_locus_pending(lb_locus* c, size_t* n) {
  if (!c) return LB_ERR_INVALID_ARG;
  return lb_odometry_pending(c->core, n);
}

int lb_locus_stage_times(lb_locus* c, double* out9) {
  if (!c || !out9) return LB_ERR_INVALID_ARG;
  LB_TRY(lb_odometry_stage_times(c->core, out9));
  std::lock_guard<std::mutex> lk(c->core->mu);
  out9[6] = (double)c->n_localized; out9[7] = c->t_busy; out9[8] = c->t_wait;
  return LB_OK;
}

}  // extern "C"

#endif  // lb_locus
