"""Throughput of lb_locus (the whole lidar callback as one pipeline) against the same chain run as blocking calls.

One seeded stream, one process, arms alternated:
  seq_host / seq_device     VoxelGrid -> odometry GICP -> localization GICP against the rolling submap -> keyframe
                            insert / crop, one blocking call after the other (scans on the host / already on the device)
  chain_host / chain_device lb_locus with the same parameters
Every arm starts from the same pre-filled submap and runs the whole stream once untimed, then timed.  The chain's poses
and registration results on the timed scans are checked bit for bit against the sequential arm.  Prints one JSON line
(and writes it to --out) with scans/s, the chain's stage times and the card's name, power limit and SM clock.

  python tools/bench_locus.py --scans 60 --depth 3 --reps 2 --out /tmp/bench_locus.json
"""
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

from oracle import locus_oracle as LO  # noqa: E402
from tools import gen_lidar as G  # noqa: E402

STEP = 32
LEAF = 0.35
MAP_RES = 0.1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi failed: " + q.stdout.strip()


def sequential(lb, blobs, d_blobs, prefill, params, device):
    """the chain as blocking calls; returns (seconds, per-scan records)"""
    import torch
    P = lb.locus_params(**params)
    vg = lb.VoxelGridB200(); vg.setLeafSize(LEAF); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    odo, loc = lb.GicpB200(), lb.GicpB200()
    C.memmove(C.byref(odo._p), C.byref(P.odometry), C.sizeof(P.odometry)); odo._apply()
    C.memmove(C.byref(loc._p), C.byref(P.localization), C.sizeof(P.localization)); loc._apply()
    m = lb.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    n = blobs[0].size // STEP
    d_f = [torch.empty(n * STEP, dtype=torch.uint8, device="cuda") for _ in range(2)]
    d_xyz = torch.empty(n * 3, dtype=torch.float32, device="cuda")
    chain = LO.LocusChain(P)
    fields = lb.xyzi_fields()
    recs = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prev = None
    for k in range(len(blobs)):
        if device:
            cur = d_f[k % 2]
            nf = vg.filter_device(d_blobs[k].data_ptr(), n, STEP, fields, cur.data_ptr(), n)
            src = (cur.data_ptr(), nf, STEP)
        else:
            f = vg.filter(blobs[k], STEP, fields)
            src = (np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy(), None, None)
            nf = src[0].shape[0]
        odoT = None
        if prev is not None:
            odo.setInputSource(*src); odo.setInputTarget(*prev)
            odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(*src)
        out = {}

        def localize(Gs):
            loc.setTargetSubmap(m)
            out["loc"] = loc.align(Gs)
            return loc.getFinalTransformation()

        def insert(T, nf=nf):
            if device:
                t = np.ascontiguousarray(T, np.float32).reshape(16)
                lb.api._check(lb.lib().lb_gicp_transform_source(loc._h, t.ctypes.data_as(C.c_void_p), C.c_void_p(d_xyz.data_ptr()),
                                                                12, 0, -1, lb.LB_MEM_DEVICE))
                return m.insert_device(d_xyz.data_ptr(), nf, 12, 0)
            return m.InsertPoints(loc.transformSource(T))

        rec = chain.scan(True, odoT, localize, insert, lambda c, half: m.Refresh(c, half))
        rec["loc_T"] = np.array(out["loc"].final_transformation, np.float32) if "loc" in out else None
        recs.append(rec)
        prev = src
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    m.close()
    return dt, recs


def pipelined(lb, blobs, d_blobs, prefill, params, device, depth):
    m = lb.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    n = blobs[0].size // STEP
    ch = lb.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **params)
    ch.voxel.setLeafSize(LEAF); ch.voxel.setFilterFieldName("z"); ch.voxel.setFilterLimits(-100.0, 100.0)
    fields = lb.api.VoxelGridB200._fields(lb.xyzi_fields())
    res = []
    t0 = time.perf_counter()
    for k in range(len(blobs)):
        if device:
            ch.submit(d_blobs[k].data_ptr(), n, STEP, fields, mem=lb.LB_MEM_DEVICE)
        else:
            ch.submit(blobs[k], n, STEP, fields)
        r = ch.next(block=False)
        while r is not None:
            res.append(r)
            r = ch.next(block=False)
    while len(res) < len(blobs):
        res.append(ch.next())
    dt = time.perf_counter() - t0
    times = ch.stageTimes()
    ch.close()
    m.close()
    return dt, res, times


def same(res, recs):
    bad = 0
    for r, e in zip(res, recs):
        ok = r.status == 0 and np.array_equal(np.asarray(r.pose, np.float64).view(np.uint64), e["L"].view(np.uint64))
        ok = ok and r.keyframe == e["keyframe"]
        if e["loc_T"] is not None:
            ok = ok and np.array_equal(np.array(r.localization.final_transformation, np.float32).view(np.uint32), e["loc_T"].view(np.uint32))
        bad += not ok
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=60)
    ap.add_argument("--beams", type=int, default=64)
    ap.add_argument("--az", type=int, default=2048)
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import locus_b200 as lb
    assert lb.device_count() > 0, "bench_locus needs a CUDA device"
    scene, poses, blobs = G.stream(a.seed, a.scans, a.beams, a.az)
    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], a.seed, a.beams, a.az)
    vg = lb.VoxelGridB200(); vg.setLeafSize(0.2)
    prefill = np.ascontiguousarray(vg.filter(G.xyz_blob(world), STEP, lb.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
    d_blobs = [torch.from_numpy(b).cuda() for b in blobs]
    params = dict(translation_threshold_kf=0.6, refresh_every=2)
    line = {"scans": a.scans, "raw_points_per_scan": blobs[0].size // STEP, "depth": a.depth, "card": card(),
            "params": dict(params, leaf=LEAF, map_resolution=MAP_RES), "arms": {}}
    ref = None
    for arm in ("seq_host", "chain_host", "seq_device", "chain_device"):     # one untimed pass each: modules, allocations
        dev = arm.endswith("device")
        if arm.startswith("seq"):
            _, recs = sequential(lb, blobs, d_blobs, prefill, params, dev)
            ref = ref or recs
        else:
            pipelined(lb, blobs, d_blobs, prefill, params, dev, a.depth)
    for rep in range(a.reps):
        for arm in ("seq_host", "chain_host", "seq_device", "chain_device"):
            dev = arm.endswith("device")
            if arm.startswith("seq"):
                dt, recs = sequential(lb, blobs, d_blobs, prefill, params, dev)
                extra = {"pose_mismatches_vs_seq_host": sum(not np.array_equal(x["L"].view(np.uint64), y["L"].view(np.uint64))
                                                            for x, y in zip(recs, ref))}
            else:
                dt, res, times = pipelined(lb, blobs, d_blobs, prefill, params, dev, a.depth)
                extra = {"mismatches_vs_seq_host": same(res, ref), "stage_times": times,
                         "keyframes": sum(r.keyframe for r in res), "crops": sum(1 for r in res if r.n_removed),
                         "filtered_points_mean": float(np.mean([r.n_filtered for r in res]))}
            line["arms"].setdefault(arm, []).append(dict(scans_per_s=a.scans / dt, ms_per_scan=1e3 * dt / a.scans, **extra))
    for dev in ("host", "device"):
        s = max(x["scans_per_s"] for x in line["arms"]["seq_" + dev])
        c = max(x["scans_per_s"] for x in line["arms"]["chain_" + dev])
        line["speedup_" + dev] = c / s
    line["card_after"] = card()
    txt = json.dumps(line)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
