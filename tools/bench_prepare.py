#!/usr/bin/env python
"""Where a registration worker of the c2 odometry pipeline spends its time outside the align: the preparation of one
filtered scan (lb_gicp_set_source + lb_gicp_prepare_source: upload, grid, cell index, k-NN covariances).

At bench.py's c2 shape (seeded stream 2, 131072 rays, leaf bisected to ~30k voxels, z limits):

    python tools/bench_prepare.py [--calls 200]           # CUDA-event time per call, launches / memsets / copies / syncs
    python tools/bench_prepare.py --trace [--out DIR]     # torch.profiler traces (a separate run)

The timing run prints one JSON line: ms per preparation standalone (device-resident filtered scans, one handle),
launches per call from the library's counter, probe rounds per call, the card and its power limit.  The trace run
writes two Chrome traces under DIR (default: a new temporary directory) -- (a) standalone calls, (b) a pipelined
lb_odometry run at bench.py's c2 settings (depth 8, 1024 points per align CTA) -- and prints per preparation its
kernels, memsets and copies, the span from the first kernel's start to the last kernel's end, the summed kernel time
and the gaps; for (b) also, per worker stream, the span of the align that follows each preparation.  Host
synchronisations per call are read from the CPU side of trace (a): cudaStreamSynchronize calls between two gathers.
"""
import argparse
import collections
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import bench_voxel as BV  # noqa: E402

POINT_STEP = BV.POINT_STEP
FIRST, LAST = "gather_cloud_kernel", "knn_cov_tail_kernel"


def stream_events(trace_path):
    """per stream that runs gather_cloud_kernel: its kernels, memsets and copies in start order"""
    with open(trace_path) as f:
        allev = json.load(f)["traceEvents"]
    ev = [e for e in allev if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    streams = sorted({e["args"].get("stream") for e in ev if BV._short(e["name"]) == FIRST})
    out = {}
    for s in streams:
        ks = sorted((e for e in ev if e["args"].get("stream") == s), key=lambda e: e["ts"])
        out[s] = [(BV._short(e["name"]), e["cat"], float(e["ts"]), float(e["dur"])) for e in ks]
    syncs = [e for e in allev if e.get("cat") == "cuda_runtime" and "Synchronize" in e.get("name", "")]
    return out, len(syncs)


def prepare_report(by_stream):
    """a preparation = gather_cloud_kernel .. knn_cov_tail_kernel on one stream; what follows until the next gather is
    the worker's align"""
    preps, aligns = [], []
    per = collections.OrderedDict()
    for ks in by_stream.values():
        cur, after = None, None
        for name, cat, t, d in ks:
            if name == FIRST:
                if after:
                    aligns.append(after[-1][2] + after[-1][3] - after[0][2])
                cur, after = [], None
            if cur is not None:
                cur.append((name, cat, t, d))
                if name == LAST:
                    preps.append(cur)
                    cur, after = None, []
            elif after is not None and cat == "kernel":
                after.append((name, cat, t, d))
    for c in preps:
        prev_end = None
        for name, cat, t, d in c:
            s = per.setdefault(name, {"n": 0, "dur_us": 0.0, "gap_us": 0.0})
            s["n"] += 1; s["dur_us"] += d
            if prev_end is not None:
                s["gap_us"] += t - prev_end
            prev_end = t + d
    n = max(1, len(preps))
    count = lambda cat: sum(1 for c in preps for x in c if x[1] == cat) / n  # noqa: E731
    span = [c[-1][2] + c[-1][3] - c[0][2] for c in preps]
    busy = [sum(x[3] for x in c) for c in preps]
    return {"preparations": len(preps), "kernels_per_call": count("kernel"), "memsets_per_call": count("gpu_memset"),
            "copies_per_call": count("gpu_memcpy"),
            "span_us_mean": float(np.mean(span)) if span else 0.0,
            "kernel_and_copy_us_mean": float(np.mean(busy)) if busy else 0.0,
            "gap_us_mean": float(np.mean(span) - np.mean(busy)) if span else 0.0,
            "align_span_us_mean": float(np.mean(aligns)) if aligns else None,
            "steps": {k: {"per_call": v["n"] / n, "mean_us": v["dur_us"] / v["n"], "mean_gap_before_us": v["gap_us"] / v["n"]}
                      for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--trace", action="store_true", help="profiler run: standalone + pipelined traces")
    ap.add_argument("--scans", type=int, default=64, help="pipelined scans traced")
    ap.add_argument("--out", default=None, help="directory for the traces (default: a new temporary directory)")
    args = ap.parse_args()
    import torch
    import locus_b200 as lb
    if lb.device_count() <= 0:
        raise SystemExit("bench_prepare.py: no CUDA device; locus_b200 has no CPU fallback")
    blobs, fields, vg, leaf, d_scans = BV.setup(torch, lb, 8)
    nraw = blobs[0].size // POINT_STEP
    filt = [np.ascontiguousarray(vg.filter(b, POINT_STEP, fields)) for b in blobs]
    d_filt = [torch.from_numpy(f.view(np.uint8).reshape(-1)).cuda() for f in filt]
    npts = [f.shape[0] for f in filt]
    g = lb.GicpB200(0)
    g.setCorrespondenceRandomness(BV.GICP["k"])
    g.reserve(max(npts))

    def prepare(calls):
        for i in range(calls):
            j = i % len(d_filt)
            g.setInputSource(d_filt[j].data_ptr(), n=npts[j], stride=POINT_STEP)
            g.prepareSource()

    line = {"metric": "gicp_prepare_ms_per_call", "card": BV.card(), "library": lb.lib_path(), "points": npts[0], "leaf_m": leaf}
    prepare(args.warmup)
    torch.cuda.synchronize()
    if not args.trace:
        l0, r0 = g.launchCount(), g.kernelTime("probe_rounds")[0]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        prepare(args.calls)
        ev1.record()
        torch.cuda.synchronize()
        line.update({"calls": args.calls, "launches_per_call": (g.launchCount() - l0) / args.calls,
                     "probe_rounds_per_call": (g.kernelTime("probe_rounds")[0] - r0) / args.calls,
                     "cell_m": g.kernelTime("cell_src")[0],
                     "ms_per_call_wall_events": ev0.elapsed_time(ev1) / args.calls})
        print(json.dumps(line))
        return
    from torch.profiler import ProfilerActivity, profile
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="bench_prepare_")
    os.makedirs(args.out, exist_ok=True)
    line["trace_dir"] = args.out
    acts = [ProfilerActivity.CPU, ProfilerActivity.CUDA]
    with profile(activities=acts) as prof:
        prepare(50)
        torch.cuda.synchronize()
    pa = os.path.join(args.out, "prepare_standalone.pt.trace.json")
    prof.export_chrome_trace(pa)
    by_stream, syncs = stream_events(pa)
    line["standalone"] = prepare_report(by_stream)
    line["standalone"]["host_syncs_per_call"] = (syncs - 1) / 50.0          # minus the torch.cuda.synchronize() that ends the run
    # (b) the pipeline at bench.py's c2 settings
    odo = lb.OdometryB200(0, depth=8, max_points=nraw, max_point_step=POINT_STEP)
    odo.voxel.setFilterFieldName("z"); odo.voxel.setFilterLimits(-100.0, 100.0); odo.voxel.setLeafSize(leaf)
    G_ = BV.GICP
    odo.setGicpParams(max_iterations=G_["max_iterations"], max_optimizer_iterations=G_["max_inner"],
                      max_correspondence_distance=G_["corr_dist"], transformation_epsilon=G_["tf_eps"],
                      k_correspondences=G_["k"], ransac_iterations=0, optimizer=lb.LB_OPT_BFGS,
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
    pb = os.path.join(args.out, "prepare_pipelined.pt.trace.json")
    prof.export_chrome_trace(pb)
    line["pipelined"] = prepare_report(stream_events(pb)[0])
    line["pipelined"]["stage_times_delta"] = {k: st1[k] - st0[k] for k in st1 if isinstance(st1[k], (int, float))}
    odo.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
