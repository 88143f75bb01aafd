#!/usr/bin/env python
"""SURVEY 8f row f5 measurement: the outlier filters LOCUS can switch on, as blocking calls on the GPU against the
oracle (oracle/outlier_oracle.c, PCL 1.10's filters restated; serial, like PCL's own) on one host core.

  c2      a VoxelGrid-filtered 64 x 2048 scan (~30 k points, tools/gen_lidar.py): PointCloudFilter's
          StatisticalOutlierRemoval (mean_k 10, std_mul 1.0) and RadiusOutlierRemoval (0.15 m, 3)
  merged  the full-resolution cloud of three 64 x 2048 lidars (~390 k points, gen_lidar.merged_scan): the merger's
          RadiusOutlierRemoval (0.1 m, 3), both of PCL's branches (is_dense true / false)

GPU timings are host wall-clock around blocking calls (each ends in a stream synchronise), averaged over --steps calls
after --warmup calls:
  filter_host_ms     the filter call on the handle's indexed source, host output buffers
  filter_device_ms   the same with device-resident output buffers
  upload_filter_ms   lb_gicp_set_source from a host cloud (upload + voxel-hash index) + the filter call, host buffers:
                     what shim/b200_outlier_pcl.hpp does per scan
cpu_ms is the oracle on the same cloud (kd-tree build included, as PCL's setInputCloud + filter).  The GPU results are
checked against the oracle's (kept indices; mean distances and statistics bit for bit).  One JSON line per case.
    python tools/bench_outliers.py [--steps 50] [--warmup 5] [--cpu-reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import gen_lidar as G  # noqa: E402


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q.splitlines()[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unknown"
    return info


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    return (time.perf_counter() - t0) * 1e3 / steps


def cpu_time(fn, reps):
    best = None
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        dt = (time.perf_counter() - t0) * 1e3
        best = dt if best is None else min(best, dt)
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import locus_b200
    from oracle import oracle as O
    from oracle import outlier_oracle as OO
    assert locus_b200.device_count() > 0, "bench_outliers.py measures the GPU; there is no CPU path to time instead"
    L = locus_b200.lib()
    HOST, DEV = locus_b200.LB_MEM_HOST, locus_b200.LB_MEM_DEVICE
    info = gpu_info()

    scene, poses, blobs = G.stream(2, 1)
    f = O.voxel_filter(blobs[0], G.POINT_STEP, 0.1088, float_fields=G.FLOAT_FIELDS, filter_field_offset=G.Z_OFF,
                       limit_min=-100.0, limit_max=100.0)["out"]
    c2 = np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()
    merged = G.merged_scan(7)

    g = locus_b200.GicpB200(0)
    nmax = max(len(c2), len(merged))
    h_idx = np.zeros(nmax, np.int32); h_md = np.zeros(nmax, np.float32); h_st = np.zeros(3)
    d_idx = torch.zeros(nmax, dtype=torch.int32, device="cuda")
    d_md = torch.zeros(nmax, dtype=torch.float32, device="cuda")
    d_st = torch.zeros(3, dtype=torch.float64, device="cuda")
    m = C.c_size_t(0)

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else t.ctypes.data_as(C.c_void_p)

    def sor_call(mem, mean_k=10, std_mul=1.0):
        b = (d_idx, d_md, d_st) if mem == DEV else (h_idx, h_md, h_st)
        assert L.lb_gicp_statistical_outlier_removal(g._h, 0, mean_k, std_mul, 0, ptr(b[0]), C.byref(m), ptr(b[1]), ptr(b[2]),
                                                     mem) == 0
        return m.value

    def radius_call(mem, radius, k, dense):
        b = d_idx if mem == DEV else h_idx
        assert L.lb_gicp_radius_outlier_removal(g._h, 0, radius, k, int(dense), 0, ptr(b), C.byref(m), mem) == 0
        return m.value

    def run_case(case, filt, pts, call, oracle_fn, check):
        g.setInputSource(pts)
        call(HOST)
        ok = check()
        res = {"case": case, "filter": filt, "points": int(len(pts)), "kept": int(m.value), "matches_oracle": bool(ok)}
        res["filter_host_ms"] = timed(lambda: call(HOST), a.steps, a.warmup)
        res["filter_device_ms"] = timed(lambda: call(DEV), a.steps, a.warmup)
        torch.cuda.synchronize()

        def upload_and_filter():
            g.setInputSource(pts)
            call(HOST)
        res["upload_filter_ms"] = timed(upload_and_filter, a.steps, a.warmup)
        res["cpu_ms"], _ = cpu_time(oracle_fn, a.cpu_reps)
        res["speedup_upload_filter_vs_cpu"] = res["cpu_ms"] / res["upload_filter_ms"]
        res["gpu"] = info
        res["cpu"] = {"cores": 1, "what": "oracle/outlier_oracle.c, serial like PCL's filters"}
        print(json.dumps(res), flush=True)

    # c2: the statistical filter
    def sor_check():
        k, md, st = OO.statistical_outlier_removal(c2, 10, 1.0)
        n = len(c2)
        return (m.value == len(k) and np.array_equal(h_idx[: m.value], k) and
                np.array_equal(h_md[:n].view(np.uint32), md.view(np.uint32)) and np.array_equal(h_st.view(np.uint64), st.view(np.uint64)))
    run_case("c2", "StatisticalOutlierRemoval mean_k=10 std_mul=1.0", c2, lambda mem: sor_call(mem),
             lambda: OO.statistical_outlier_removal(c2, 10, 1.0), sor_check)
    # c2: the radius filter, and the merged cloud's
    for case, pts, r in (("c2", c2, 0.15), ("merged", merged, 0.1)):
        for dense in ((True,) if case == "c2" else (True, False)):
            def rcheck(pts=pts, r=r, dense=dense):
                k = OO.radius_outlier_removal(pts, r, 3, dense)
                return m.value == len(k) and np.array_equal(h_idx[: m.value], k)
            run_case(case, "RadiusOutlierRemoval radius=%g min_neighbors=3 dense=%d" % (r, dense), pts,
                     lambda mem, r=r, dense=dense: radius_call(mem, r, 3, dense),
                     lambda pts=pts, r=r, dense=dense: OO.radius_outlier_removal(pts, r, 3, dense), rcheck)
    g.close()


if __name__ == "__main__":
    main()
