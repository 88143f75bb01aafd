"""Time lb_gicp_icp_covariance (the localization's ICP covariance after align) on a C2 scan against a C3-shaped
500 k-point submap with normals and against the previous scan with normals, next to the oracle's serial chain on one
core (oracle/icp_cov_oracle.py: kd-tree 1-NN loop, normalizePCloud, Ap, 6x6 algebra; the kd-tree of the target is built
beforehand, as the reference searches the registration's existing tree).

One process, seeded inputs: 131072-ray scans filtered to ~30 k points (bench.py's leaf), the submap a voxel-merged union
of posed scans of the same scene filtered to ~500 k points (tools/bench_c3.py's recipe), normals k = 20 on the GPU.  Each
GPU call is a host wall-clock span that ends in the call's own synchronisation, median of --reps after --warmup calls;
the oracle chain is timed --cpu-reps times.  Every GPU result is checked against the oracle (the 1-NN index for index, Ap
to 1e-10).  Prints one JSON line with the card's name, power limit and SM clock.

  python tools/bench_icp_covariance.py --reps 50
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import icp_cov_oracle as IC  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tools import gen_lidar as G  # noqa: E402

STEP = 32
SUBMAP_POINTS = 500_000
SCAN_POINTS = 30_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi failed: " + q.stdout.strip()


def _bisect(vg, blob, fields, target, lo, hi, iters):
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        vg.setLeafSize(mid)
        n = vg.filter(blob, STEP, fields).shape[0]
        lo, hi = (mid, hi) if n > target else (lo, mid)
    return float(np.float32(0.5 * (lo + hi)))


def c2_c3_case(seed=2, map_scans=12):
    """(scan0, scan1, submap): two consecutive C2 scans filtered to ~30 k points and a ~500 k-point C3-shaped submap,
    all (n, 3) float32"""
    import locus_b200 as lb
    scene, poses, blobs = G.stream(seed, 2)
    world = G.world_points(scene, G.trajectory(seed + 50, map_scans, t_step=1.5, r_step_deg=20.0), seed + 50)
    fields = lb.xyzi_fields()
    vg = lb.VoxelGridB200()
    vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    wblob = np.zeros((len(world), 8), np.float32)
    wblob[:, :3] = world
    wblob = wblob.view(np.uint8).reshape(-1)
    vg.setLeafSize(_bisect(vg, wblob, fields, SUBMAP_POINTS, 0.005, 0.5, 16))
    submap = np.ascontiguousarray(vg.filter(wblob, STEP, fields)).view(np.float32).reshape(-1, 8)[:, :3].copy()
    vg.setLeafSize(_bisect(vg, blobs[0], fields, SCAN_POINTS, 0.02, 2.0, 18))
    scans = [np.ascontiguousarray(vg.filter(b, STEP, fields)).view(np.float32).reshape(-1, 8)[:, :3].copy() for b in blobs]
    return scans[0], scans[1], submap


def _median_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import locus_b200 as lb
    assert lb.device_count() > 0, "bench_icp_covariance needs a CUDA device; locus_b200 has no CPU fallback"
    scan0, scan1, submap = c2_c3_case()
    g = lb.GicpB200()
    g.setInputSource(submap)
    map_n = g.computeNormals(0, 20)[:, :3].copy()
    g.setInputSource(scan0)
    n0 = g.computeNormals(0, 20)[:, :3].copy()
    line = {"card": card(), "scan_points": len(scan1), "submap_points": len(submap), "arms": {}}
    m = lb.SubmapB200(0, 0.01)
    m.InsertPointsWithNormals(submap, map_n)
    targets = {"vs_submap": (lambda h: h.setTargetSubmap(m), m.points, m.normals, 0.5),
               "vs_previous_scan": (lambda h: h.setInputTarget(np.ascontiguousarray(np.hstack([scan0, n0])), normal_off=12),
                                    lambda: scan0, lambda: n0, 1.0)}
    for name, (set_target, pts, nrm, corr_dist) in targets.items():
        h = lb.GicpB200()
        h.setMaxCorrespondenceDistance(corr_dist); h.setMaximumIterations(20)
        h.setInputSource(scan1); set_target(h)
        h.align()
        T = h.getFinalTransformation()
        r = h.icpCovariance()
        tgt, tgt_n = pts(), nrm()
        tree = O.KdTree(tgt)
        o = IC.icp_covariance(scan1, tgt, tgt_n, T=T, tree=tree)
        idx, _ = h.nearestTarget(h.transformSource())
        ok = bool(np.array_equal(idx, o["correspondences"]) and np.abs(r["Ap"] - o["Ap"]).max() <= 1e-10 * np.abs(o["Ap"]).max())
        gpu_med, gpu_min = _median_ms(h.icpCovariance, a.warmup, a.reps)
        cpu_med, cpu_min = _median_ms(lambda: IC.icp_covariance(scan1, tgt, tgt_n, T=T, tree=tree), 0, a.cpu_reps)
        line["arms"][name] = dict(target_points=len(tgt), gpu_ms_median=gpu_med, gpu_ms_min=gpu_min,
                                  oracle_serial_ms_median=cpu_med, speedup=cpu_med / gpu_med, matches_oracle=ok,
                                  n_used=int(r["n_used"]), flags=int(r["flags"]))
    m.close()
    line["card_after"] = card()
    txt = json.dumps(line)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
