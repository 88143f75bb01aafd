#!/usr/bin/env python
"""SURVEY 8f row f6 measurement: the `filtering/extract_features` branch of PointCloudFilter::Filter as a blocking call
on the GPU (lb_voxel_extract_features) against the oracle (oracle/features_oracle.c, the reference's serial algorithm
with its insertion sort) on one host core.

  scan_order   a VLP-16 sweep (16 beams over +-15 deg, 1800 azimuths, tools/gen_lidar.py) in scan order
  voxel_order  the same sweep after the VoxelGrid (lb_voxel_filter, leaf 0.1): voxel-index order, which is what LOCUS's
               lidar callback receives in the shipped launch file

GPU timings are host wall-clock around blocking calls (each ends in a stream synchronise), averaged over --steps calls
after --warmup calls:
  host_ms      host input, host output (upload, three kernels, download)
  device_ms    device input, device output
cpu_ms is the oracle on the same cloud (best of --cpu-reps).  The GPU output is checked against the oracle's bit for bit.
One JSON line per case.
    python tools/bench_features.py [--steps 50] [--warmup 5] [--cpu-reps 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import gen_lidar as G  # noqa: E402
from tools.bench_outliers import cpu_time, gpu_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import locus_b200
    from oracle import features_oracle as FO
    assert locus_b200.device_count() > 0, "bench_features.py measures the GPU; there is no CPU path to time instead"
    info = gpu_info()
    blob = G.scan(G.make_scene(3), np.eye(4), 7, beams=16, az=1800, elev_deg=(-15.0, 15.0))
    vg = locus_b200.VoxelGridB200(0)
    vg.setLeafSize(0.1)
    filtered = vg.filter(blob, G.POINT_STEP, locus_b200.xyzi_fields())
    clouds = {"scan_order": G.blob_xyz(blob), "voxel_order": G.blob_xyz(np.ascontiguousarray(filtered).reshape(-1))}
    for case, xyz in clouds.items():
        ref, rcnt = FO.extract_features(xyz)
        out, cnt = vg.extractFeatures(xyz)
        eq = out.view(np.uint32) == ref.view(np.uint32)
        ok = cnt == rcnt and bool(np.all(eq | (np.isnan(out) & np.isnan(ref))))
        d_in = torch.from_numpy(np.ascontiguousarray(xyz)).cuda()
        d_out = torch.zeros((2 * len(xyz), 4), dtype=torch.float32, device="cuda")
        res = {"case": case, "points": int(len(xyz)), "counts": cnt, "matches_oracle": ok}
        res["host_ms"] = timed(lambda: vg.extractFeatures(xyz), a.steps, a.warmup)
        res["device_ms"] = timed(lambda: vg.extractFeatures(d_in, out=d_out), a.steps, a.warmup)
        res["cpu_ms"], _ = cpu_time(lambda: FO.extract_features(xyz), a.cpu_reps)
        res["speedup_host_vs_cpu"] = res["cpu_ms"] / res["host_ms"]
        res["launches_per_call"] = 3
        res["gpu"] = info
        res["cpu"] = {"cores": 1, "what": "oracle/features_oracle.c, serial like the reference"}
        print(json.dumps(res), flush=True)
    vg.close()


if __name__ == "__main__":
    main()
