#!/usr/bin/env python
"""Where the VoxelGrid stage of the c2 odometry pipeline spends its time.

bench.py's c2 headline is bounded by the pipeline's one serial stage, the VoxelGrid filter of every scan
(lb_voxel_filter, a stream-ordered chain of small dependent kernels).  This script measures that chain on its own and
inside the pipeline, at bench.py's c2 shape (seeded stream 2, 131072 rays, leaf bisected to ~30k voxels, z limits):

    python tools/bench_voxel.py [--calls 200]                       # CUDA-event time per call, device-resident
    python tools/bench_voxel.py --trace [--out DIR]                 # torch.profiler traces (a separate run)
    python tools/bench_voxel.py --report TRACE [TRACE ...]          # the same report from saved traces, no GPU

The timing run prints one JSON line: ms per call, key_bits (the sort key width, from the grid the leaf gives),
voxels, launches per call, the card name and its power limit.  The trace run writes two Chrome traces under DIR
(default: a new temporary directory) -- (a) standalone calls, (b) a pipelined lb_odometry run at bench.py's c2 settings (depth 8, 1024 points per align CTA)
-- and prints, for every kernel on the VoxelGrid stream, its mean duration and the mean gap before it, plus the
span of one call from its first kernel's start to its last kernel's end.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import gen_lidar as G  # noqa: E402

POINT_STEP = 32
GICP = dict(max_iterations=50, max_inner=20, corr_dist=1.0, tf_eps=1e-3, k=20)     # bench.py's c2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [s.strip() for s in q.stdout.splitlines()[0].split(",")] if q.returncode == 0 and q.stdout else ["?"] * 4
    return {"name": f[0], "power_limit": f[1], "sm_clock_max": f[2], "sm_clock_now": f[3]}


def key_bits(blob, leaf):
    """the sort key width lb_voxel_filter derives on the device: bits of the grid's cell count (PCL's min_b / div_b)"""
    a = blob.view(np.float32).reshape(-1, 8)[:, :3]
    ok = np.isfinite(a).all(1) & (a[:, 2] >= -100.0) & (a[:, 2] <= 100.0)
    p = a[ok]
    inv = np.float32(1.0) / np.float32(leaf)
    mn = np.floor(p.min(0) * inv).astype(np.int64); mx = np.floor(p.max(0) * inv).astype(np.int64)
    cells = int(np.prod(mx - mn + 1))
    return cells.bit_length(), [int(v) for v in (mx - mn + 1)]


def setup(torch, lb, n_scans):
    scene, poses, blobs = G.stream(2, n_scans)
    fields = lb.xyzi_fields()
    vg = lb.VoxelGridB200(0)
    vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    lo, hi = 0.02, 2.0                       # bench.py's bisection (bisect_leaf)
    for _ in range(18):
        mid = 0.5 * (lo + hi)
        vg.setLeafSize(mid)
        if vg.filter(blobs[0], POINT_STEP, fields).shape[0] > 30000:
            lo = mid
        else:
            hi = mid
    leaf = float(np.float32(0.5 * (lo + hi)))
    vg.setLeafSize(leaf)
    d_scans = [torch.from_numpy(b).cuda() for b in blobs]
    return blobs, fields, vg, leaf, d_scans


def standalone(torch, vg, fields, d_scans, d_out, nraw, calls):
    m = 0
    for i in range(calls):
        m = vg.filter_device(d_scans[i % len(d_scans)].data_ptr(), nraw, POINT_STEP, fields, d_out.data_ptr(), nraw)
    return m


def _short(name):
    return name.replace("void ", "").replace("lb::", "").split("(")[0].split("<")[0]


def voxel_stream_kernels(trace_path):
    """kernels and copies of the stream that runs vg_bbox_kernel, in start order: (name, start us, duration us)"""
    with open(trace_path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    streams = {e["args"].get("stream") for e in ev if _short(e["name"]) == "vg_bbox_kernel"}
    ks = sorted((e for e in ev if e["args"].get("stream") in streams), key=lambda e: e["ts"])
    return [(_short(e["name"]), float(e["ts"]), float(e["dur"])) for e in ks]


def chain_report(ks):
    """per kernel name: launches, mean duration, mean gap before it (previous kernel's end on the stream -> its start);
    per call (vg_bbox .. the kernel before the next vg_bbox): mean span, summed kernel time and summed gaps"""
    per = collections.OrderedDict()
    calls, cur = [], []
    prev_end = None
    for name, t, d in ks:
        if name == "vg_bbox_kernel":
            if cur:
                calls.append(cur)
            cur = []
            gap = None                         # the gap before a call's first kernel is the host's, not the chain's
        else:
            gap = t - prev_end if prev_end is not None else None
        cur.append((name, t, d, gap))
        prev_end = t + d
        s = per.setdefault(name, {"n": 0, "dur_us": 0.0, "gap_us": 0.0, "gaps": 0})
        s["n"] += 1; s["dur_us"] += d
        if gap is not None:
            s["gap_us"] += gap; s["gaps"] += 1
    if cur:
        calls.append(cur)
    kern = {k: {"launches": v["n"], "mean_us": v["dur_us"] / v["n"],
                "mean_gap_before_us": (v["gap_us"] / v["gaps"]) if v["gaps"] else None} for k, v in per.items()}
    full = [c for c in calls if len(c) > 1]
    span = [c[-1][1] + c[-1][2] - c[0][1] for c in full]
    busy = [sum(x[2] for x in c) for c in full]
    gaps = [sum(x[3] for x in c[1:] if x[3] is not None) for c in full]
    return {"kernels": kern, "calls": len(full),
            "kernels_per_call": float(np.mean([len(c) for c in full])) if full else 0.0,
            "call_span_us_mean": float(np.mean(span)) if span else 0.0,
            "call_kernel_us_mean": float(np.mean(busy)) if busy else 0.0,
            "call_gap_us_mean": float(np.mean(gaps)) if gaps else 0.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--report", nargs="+", metavar="TRACE", help="only print the voxel-stream report of saved traces")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--trace", action="store_true", help="profiler run: standalone + pipelined traces")
    ap.add_argument("--scans", type=int, default=64, help="pipelined scans traced")
    ap.add_argument("--out", default=None, help="directory for the traces (default: a new temporary directory)")
    args = ap.parse_args()
    if args.report:
        for t in args.report:
            print(json.dumps({"trace": os.path.basename(t), **chain_report(voxel_stream_kernels(t))}))
        return
    import torch
    import locus_b200 as lb
    if lb.device_count() <= 0:
        raise SystemExit("bench_voxel.py: no CUDA device; locus_b200 has no CPU fallback")
    blobs, fields, vg, leaf, d_scans = setup(torch, lb, 8)
    nraw = blobs[0].size // POINT_STEP
    d_out = torch.empty(nraw * POINT_STEP, dtype=torch.uint8, device="cuda")
    kb, div = key_bits(blobs[0], leaf)
    line = {"metric": "voxel_filter_ms_per_call", "card": card(), "library": lb.lib_path(), "points_in": nraw, "leaf_m": leaf,
            "grid": div, "key_bits": kb, "sort_passes": (kb + 7) // 8}
    standalone(torch, vg, fields, d_scans, d_out, nraw, args.warmup)
    torch.cuda.synchronize()
    if not args.trace:
        l0 = vg.launchCount()
        vg.avgCallMs(reset=True)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        m = standalone(torch, vg, fields, d_scans, d_out, nraw, args.calls)
        ev1.record()
        torch.cuda.synchronize()
        line.update({"calls": args.calls, "voxels": int(m), "launches_per_call": (vg.launchCount() - l0) / args.calls,
                     "ms_per_call_wall_events": ev0.elapsed_time(ev1) / args.calls,
                     "ms_per_call_device_events": vg.avgCallMs(reset=True)})
        print(json.dumps(line))
        return
    from torch.profiler import ProfilerActivity, profile
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="bench_voxel_")
    os.makedirs(args.out, exist_ok=True)
    line["trace_dir"] = args.out
    acts = [ProfilerActivity.CPU, ProfilerActivity.CUDA]
    with profile(activities=acts) as prof:
        standalone(torch, vg, fields, d_scans, d_out, nraw, 50)
        torch.cuda.synchronize()
    pa = os.path.join(args.out, "voxel_standalone.pt.trace.json")
    prof.export_chrome_trace(pa)
    line["standalone"] = chain_report(voxel_stream_kernels(pa))
    # (b) the pipeline at bench.py's c2 settings
    odo = lb.OdometryB200(0, depth=8, max_points=nraw, max_point_step=POINT_STEP)
    odo.voxel.setFilterFieldName("z"); odo.voxel.setFilterLimits(-100.0, 100.0); odo.voxel.setLeafSize(leaf)
    odo.setGicpParams(max_iterations=GICP["max_iterations"], max_optimizer_iterations=GICP["max_inner"],
                      max_correspondence_distance=GICP["corr_dist"], transformation_epsilon=GICP["tf_eps"],
                      k_correspondences=GICP["k"], ransac_iterations=0, optimizer=lb.LB_OPT_BFGS,
                      execution=lb.LB_EXEC_STREAM_ORDERED, align_points_per_cta=1024)

    def run(n, k0):
        for i in range(n):
            odo.submit(d_scans[(k0 + i) % len(d_scans)].data_ptr(), nraw, POINT_STEP, fields, mem=lb.LB_MEM_DEVICE)
            r = odo.next(block=False)
            while r is not None:
                r = odo.next(block=False) if odo.pending() else None
        while odo.pending():
            r = odo.next()
            if r.status != 0:
                raise RuntimeError("lb_odometry status %d" % r.status)

    run(32, 0)
    torch.cuda.synchronize()
    st0 = odo.stageTimes()
    with profile(activities=acts) as prof:
        run(args.scans, 32)
        torch.cuda.synchronize()
    st1 = odo.stageTimes()
    pb = os.path.join(args.out, "voxel_pipelined.pt.trace.json")
    prof.export_chrome_trace(pb)
    line["pipelined"] = chain_report(voxel_stream_kernels(pb))
    nf = max(1, st1["filtered"] - st0["filtered"])
    line["pipelined"]["voxel_stage_busy_ms_per_scan_traced"] = 1e3 * (st1["voxel_busy_s"] - st0["voxel_busy_s"]) / nf
    odo.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
