"""Throughput of lb_locus (the whole lidar callback as one pipeline) against the same chain run as blocking calls.

One seeded stream, one process, arms alternated:
  seq_host / seq_device     VoxelGrid -> odometry GICP -> localization GICP against the rolling submap -> keyframe
                            insert / crop, one blocking call after the other (scans on the host / already on the device)
  chain_host / chain_device lb_locus with the same parameters
Every arm starts from the same pre-filled submap and runs the whole stream once untimed, then timed.  The chain's poses
and registration results on the timed scans are checked bit for bit against the sequential arm.  Prints one JSON line
(and writes it to --out) with scans/s, the chain's stage times and the card's name, power limit and SM clock.

  python tools/bench_locus.py --scans 60 --depth 3 --reps 2 --out /tmp/bench_locus.json

With --front-end the arms are instead, scans on the host:
  chain_current             lb_locus as above (no normals, k-NN covariances, fixed leaf)
  chain_shipped             lb_locus in LOCUS's shipped front end: normals k = 20, every covariance from normals,
                            adaptive input voxelization at 3000 points from a 0.25 leaf
  seq_shipped               the shipped configuration as blocking calls (computeNormals + an upload with normals,
                            tools/front_end_oracle.FrontEndChain for the leaf)
and the line adds the mean leaf and filtered points and how many timed scans were bit-equal between chain_shipped and
seq_shipped.

  python tools/bench_locus.py --front-end --scans 60 --depth 3 --reps 2

With --icp-covariance the arms are lb_locus in the shipped front end without (shipped_cov_off) and with
(shipped_cov_on) the localization's ICP covariance (icp_covariance.enabled = 1, max_covariance = 0.01), scans on the host,
alternated --reps times (default here 3).  Stage L bounds the chain, so its busy time per scan is the cost a user sees;
the line reports scans/s and stage L busy ms per scan for both arms, and how many timed scans kept bit-equal poses.

  python tools/bench_locus.py --icp-covariance --scans 60 --depth 3 --reps 3

With --lidars 3 every scan is the three lidars of gen_lidar.LIDAR_MOUNTS (tools/gen_lidar.merged_stream, ~390 k raw
points at 64 x 2048), sensor frame, merged in the VoxelGrid stage with their sensor -> base_link transforms, PassThrough
and BodyFilter on.  The arms are those of the default run: seq_* calls lb_voxel_filter_merged and then the blocking
chain, chain_* submits each scan with lb_locus_submit_merged (scans on the host: the pageable host-to-device copy of
the three clouds is part of stage V).  The line adds stage V busy ms per scan of the chain arms.  --leaf sets the
VoxelGrid leaf (default here 0.5, which keeps the filtered scans within the SM budget of DESIGN.md 4i).

  python tools/bench_locus.py --lidars 3 --scans 60 --depth 3 --reps 3

--odometry-method / --localization-method {gicp,ndt} set each package's registration_method in the default run (the
other modes keep GICP): the chain arms register with lb_locus's NDT stages, the seq_* arms with blocking NdtB200 calls
(the odometry against the previous filtered scan, the localization against the submap's points).

  python tools/bench_locus.py --odometry-method ndt --localization-method ndt --scans 60 --depth 3 --reps 3

--ndt-map-rebuild N times what an NDT localization pays after a keyframe: a submap of about N points (posed scans of the
stream, 0.1 m map voxels), one point inserted (a new generation), then lb_ndt_set_target_submap plus the lazy build of the
voxel Gaussians (through lb_ndt_target_voxels, which triggers it), host clock around the blocking calls, --reps x 10
times; and the same call on the unchanged map.

  python tools/bench_locus.py --ndt-map-rebuild 500000
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
from tools import front_end_oracle as FE  # noqa: E402
from tools import gen_lidar as G  # noqa: E402

STEP = 32
LEAF = 0.35
LEAF_SHIPPED = 0.25       # Locus.cc:39, what the shipped launch sets
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
    odo_ndt, loc_ndt = P.odometry_method == lb.api.LB_REG_NDT, P.localization_method == lb.api.LB_REG_NDT
    nodo, nloc = lb.NdtB200(), lb.NdtB200()
    C.memmove(C.byref(nodo._p), C.byref(P.odometry_ndt), C.sizeof(P.odometry_ndt)); nodo._apply()
    C.memmove(C.byref(nloc._p), C.byref(P.localization_ndt), C.sizeof(P.localization_ndt)); nloc._apply()

    def ndt_cloud(h, which, src):
        """an NDT source (which = 0) or target (1) from a host xyz array or a device filtered cloud (ptr, n, stride)"""
        if src[1] is None:
            (h.setInputSource if which == 0 else h.setInputTarget)(src[0])
        else:
            fn = lb.lib().lb_ndt_set_source if which == 0 else lb.lib().lb_ndt_set_target
            lb.api._check(fn(h._h, C.c_void_p(src[0]), src[1], src[2], 0, lb.LB_MEM_DEVICE))

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
        if prev is not None and odo_ndt:
            ndt_cloud(nodo, 0, src); ndt_cloud(nodo, 1, prev)
            nodo.align()
            odoT = nodo.getFinalTransformation()
        elif prev is not None:
            odo.setInputSource(*src); odo.setInputTarget(*prev)
            odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(*src)
        if loc_ndt:
            ndt_cloud(nloc, 0, src)
        out = {}

        def localize(Gs):
            if loc_ndt:
                nloc.setTargetSubmap(m)
                out["loc"] = nloc.align(Gs)
                return nloc.getFinalTransformation()
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


def sequential_front_end(lb, blobs, prefill, prefill_n, params):
    """the shipped front end as blocking calls on the host; returns (seconds, per-scan records)"""
    import torch
    P = lb.locus_params(**params)
    vg = lb.VoxelGridB200(); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    odo, loc, nrm = lb.GicpB200(), lb.GicpB200(), lb.GicpB200()
    C.memmove(C.byref(odo._p), C.byref(P.odometry), C.sizeof(P.odometry)); odo._apply()
    C.memmove(C.byref(loc._p), C.byref(P.localization), C.sizeof(P.localization)); loc._apply()
    m = lb.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    chain = FE.FrontEndChain(P, np.float32(LEAF_SHIPPED))
    fields = lb.xyzi_fields()
    recs = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prev = None
    for b in blobs:
        leaf = chain.next_leaf
        vg.setLeafSize(float(leaf))
        xyz = np.ascontiguousarray(vg.filter(b, STEP, fields)).view(np.float32).reshape(-1, 8)[:, :3].copy()
        chain.filtered(len(xyz))
        nrm.setInputSource(xyz)
        c6 = np.ascontiguousarray(np.hstack([xyz, nrm.computeNormals(0, 20)[:, :3]]))
        odoT = None
        if prev is not None:
            odo.setInputSource(c6, normal_off=12); odo.setInputTarget(prev, normal_off=12)
            odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(c6, normal_off=12)
        out = {}

        def localize(Gs):
            loc.setTargetSubmap(m)
            out["loc"] = loc.align(Gs)
            return loc.getFinalTransformation()

        def insert(T):
            t = loc.transformSource(T, with_normals=True)
            return m.InsertPointsWithNormals(t[:, :3], t[:, 3:])

        rec = chain.scan(True, odoT, localize, insert, lambda c, half: m.Refresh(c, half))
        rec["loc_T"] = np.array(out["loc"].final_transformation, np.float32) if "loc" in out else None
        rec["leaf"] = leaf
        recs.append(rec)
        prev = c6
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    m.close()
    return dt, recs


def pipelined(lb, blobs, d_blobs, prefill, params, device, depth, prefill_n=None, leaf=LEAF):
    m = lb.SubmapB200(0, MAP_RES)
    if prefill_n is None:
        m.InsertPoints(prefill)
    else:
        m.InsertPointsWithNormals(prefill, prefill_n)
    n = blobs[0].size // STEP
    ch = lb.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **params)
    ch.voxel.setLeafSize(leaf); ch.voxel.setFilterFieldName("z"); ch.voxel.setFilterLimits(-100.0, 100.0)
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


def ndt_map_rebuild(lb, a, line):
    """--ndt-map-rebuild: the submap's NDT target rebuilt after a change of the map, and the call on an unchanged map"""
    scene, poses, _ = G.stream(a.seed, 2, a.beams, a.az)
    m = lb.SubmapB200(0, MAP_RES)
    k = 0
    while m.size() < a.ndt_map_rebuild and k < 64:
        # scans from poses around the origin, kept to LOCUS's 20 m window (box_filter_size) around it
        T = G.pose_matrix([4.0 * (k % 7) - 12.0, 3.0 * (k // 7 % 7) - 9.0, 0.0], [0, 0, 0.4 * k])
        w = G.world_points(scene, [T], a.seed + k, a.beams, a.az)
        m.InsertPoints(np.ascontiguousarray(w[(np.abs(w) <= 20.0).all(axis=1)]))
        k += 1
    nd = lb.NdtB200()
    L = lb.lib()
    nv = C.c_size_t(0)

    def target():
        nd.setTargetSubmap(m)
        lb.api._check(L.lb_ndt_target_voxels(nd._h, 0, C.byref(nv), None, None, None, None, None))

    target()                                                  # modules, allocations
    top = m.points().max(axis=0) - np.float32(0.5)            # free space inside the map's box: inserts land there
    rebuild, unchanged = [], []
    j = 0
    for i in range(10 * a.reps):
        while not m.InsertPoints((top - np.float32(0.13) * np.array([j % 50, j // 50, 0], np.float32)).reshape(1, 3)):
            j += 1
        j += 1
        t0 = time.perf_counter(); target(); rebuild.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); target(); unchanged.append(time.perf_counter() - t0)
    line.update(map_points=m.size(), window_half_size=20.0, map_resolution=MAP_RES, searchable_voxels=nv.value, ndt_resolution=nd.getResolution(),
                rebuild_ms_median=1e3 * float(np.median(rebuild)), rebuild_ms_min=1e3 * float(np.min(rebuild)),
                unchanged_ms_median=1e3 * float(np.median(unchanged)))
    m.close()


def merged_inputs(scans, mounts):
    return [[(b, M) for b, M in zip(sc, mounts)] for sc in scans]


def sequential_merged(lb, scans, d_scans, mounts, prefill, params, device, leaf, setup):
    """--lidars: the chain as blocking calls, the lidars merged by lb_voxel_filter_merged (host or device clouds)"""
    import torch
    P = lb.locus_params(**params)
    vg = lb.VoxelGridB200(); setup(vg, leaf)
    odo, loc = lb.GicpB200(), lb.GicpB200()
    C.memmove(C.byref(odo._p), C.byref(P.odometry), C.sizeof(P.odometry)); odo._apply()
    C.memmove(C.byref(loc._p), C.byref(P.localization), C.sizeof(P.localization)); loc._apply()
    m = lb.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    n = max(sum(b.size for b in sc) for sc in scans) // STEP
    d_f = [torch.empty(n * STEP, dtype=torch.uint8, device="cuda") for _ in range(2)]
    chain = LO.LocusChain(P)
    fields = lb.api.VoxelGridB200._fields(lb.xyzi_fields())
    Ts = [np.ascontiguousarray(M, np.float32).reshape(16) for M in mounts]
    recs = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prev = None
    for k in range(len(scans)):
        if device:
            arr = (lb.api.VoxelInput * len(scans[k]))()
            for i, d in enumerate(d_scans[k]):
                arr[i].data = d.data_ptr(); arr[i].n_pts = d.numel() // STEP; arr[i].transform = Ts[i].ctypes.data_as(C.c_void_p).value
            cur = d_f[k % 2]
            nf = C.c_size_t(0)
            lb.api._check(lb.lib().lb_voxel_filter_merged(vg._h, arr, len(scans[k]), STEP, fields, len(fields), C.c_void_p(cur.data_ptr()),
                                                          n, C.byref(nf), None, lb.LB_MEM_DEVICE, lb.LB_MEM_DEVICE))
            src = (cur.data_ptr(), nf.value, STEP)
        else:
            f = vg.filterMerged(scans[k], STEP, lb.xyzi_fields(), mounts)
            src = (np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy(), None, None)
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

        rec = chain.scan(True, odoT, localize, lambda T: m.InsertPoints(loc.transformSource(T)), lambda c, half: m.Refresh(c, half))
        rec["loc_T"] = np.array(out["loc"].final_transformation, np.float32) if "loc" in out else None
        recs.append(rec)
        prev = src
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    m.close()
    return dt, recs


def pipelined_merged(lb, scans, d_scans, mounts, prefill, params, device, depth, leaf, setup):
    m = lb.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    n = max(sum(b.size for b in sc) for sc in scans) // STEP
    ch = lb.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **params)
    setup(ch.voxel, leaf)
    fields = lb.api.VoxelGridB200._fields(lb.xyzi_fields())
    res = []
    t0 = time.perf_counter()
    for k in range(len(scans)):
        if device:
            ch.submit_merged([(d.data_ptr(), d.numel() // STEP) for d in d_scans[k]], STEP, fields, mounts, mem=lb.LB_MEM_DEVICE)
        else:
            ch.submit_merged(scans[k], STEP, fields, mounts)
        r = ch.next(block=False)
        while r is not None:
            res.append(r)
            r = ch.next(block=False)
    while len(res) < len(scans):
        res.append(ch.next())
    dt = time.perf_counter() - t0
    times = ch.stageTimes()
    ch.close()
    m.close()
    return dt, res, times


def lidars(lb, a, line):
    """--lidars 3: three lidars per scan merged in stage V; blocking calls against the pipeline, host and device clouds"""
    import torch
    scene, poses, scans, mounts = G.merged_stream(a.seed, a.scans, a.beams, a.az)
    body = ([-0.6, -0.45, -0.5], [0.6, 0.45, 1.0])

    def setup(v, leaf):
        v.setLeafSize(leaf); v.setFilterFieldName("z"); v.setFilterLimits(-100.0, 100.0)
        v.setInputPassThrough("z", -100.0, 100.0)
        v.setBodyFilter(body[0], body[1], 0.0)

    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], a.seed, a.beams, a.az)
    vg = lb.VoxelGridB200(); vg.setLeafSize(0.2)
    prefill = np.ascontiguousarray(vg.filter(G.xyz_blob(world), STEP, lb.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
    params = dict(translation_threshold_kf=0.6, refresh_every=2)
    leaf = a.leaf if a.leaf else 0.5
    line.update(raw_points_per_scan=int(np.mean([sum(b.size for b in sc) // STEP for sc in scans])), lidars=3,
                params=dict(params, leaf=leaf, map_resolution=MAP_RES, passthrough_z=[-100.0, 100.0], body_filter=body))
    d_scans = [[torch.from_numpy(b).cuda() for b in sc] for sc in scans]
    arms = ("seq_host", "chain_host", "seq_device", "chain_device")

    def run(arm):
        dev = arm.endswith("device")
        if arm.startswith("seq"):
            return sequential_merged(lb, scans, d_scans, mounts, prefill, params, dev, leaf, setup)
        return pipelined_merged(lb, scans, d_scans, mounts, prefill, params, dev, a.depth, leaf, setup)

    ref = None
    for arm in arms:                     # one untimed pass each: modules, allocations
        out = run(arm)
        if arm == "seq_host":
            ref = out[1]
    for rep in range(a.reps):
        for arm in arms:
            out = run(arm)
            dt = out[0]
            entry = dict(scans_per_s=a.scans / dt, ms_per_scan=1e3 * dt / a.scans)
            if arm.startswith("seq"):
                entry["pose_mismatches_vs_seq_host"] = sum(not np.array_equal(x["L"].view(np.uint64), y["L"].view(np.uint64))
                                                           for x, y in zip(out[1], ref))
            else:
                res, times = out[1], out[2]
                entry.update(bit_equal_scans_vs_seq_host=len(res) - same(res, ref), stage_times=times,
                             stage_v_busy_ms_per_scan=1e3 * times["voxel_busy_s"] / max(times["filtered"], 1),
                             filtered_points_mean=float(np.mean([r.n_filtered for r in res])),
                             filtered_points_max=int(max(r.n_filtered for r in res)),
                             keyframes=sum(r.keyframe for r in res), crops=sum(1 for r in res if r.n_removed))
            line["arms"].setdefault(arm, []).append(entry)
    for arm in arms:
        line["best_scans_per_s_" + arm] = max(x["scans_per_s"] for x in line["arms"][arm])
    for dev in ("host", "device"):
        line["median_stage_v_busy_ms_chain_" + dev] = float(np.median([x["stage_v_busy_ms_per_scan"] for x in line["arms"]["chain_" + dev]]))
        line["speedup_" + dev] = line["best_scans_per_s_chain_" + dev] / line["best_scans_per_s_seq_" + dev]


def same(res, recs):
    bad = 0
    for r, e in zip(res, recs):
        ok = r.status == 0 and np.array_equal(np.asarray(r.pose, np.float64).view(np.uint64), e["L"].view(np.uint64))
        ok = ok and r.keyframe == e["keyframe"]
        if e["loc_T"] is not None:
            ok = ok and np.array_equal(np.array(r.localization.final_transformation, np.float32).view(np.uint32), e["loc_T"].view(np.uint32))
        bad += not ok
    return bad


def front_end(lb, a, blobs, prefill, line):
    """--front-end: the current chain, the shipped chain and the shipped chain as blocking calls, alternated"""
    g = lb.GicpB200()
    g.setInputSource(prefill)
    prefill_n = g.computeNormals(0, 20)[:, :3].copy()
    base = dict(translation_threshold_kf=0.6, refresh_every=2)
    shipped = dict(base, **FE.SHIPPED)
    line["params"] = dict(base, leaf=LEAF, shipped_front_end=FE.SHIPPED, shipped_initial_leaf=LEAF_SHIPPED,
                          map_resolution=MAP_RES)
    arms = ("chain_current", "chain_shipped", "seq_shipped")

    def run(arm):
        if arm == "chain_current":
            return pipelined(lb, blobs, None, prefill, base, False, a.depth)
        if arm == "chain_shipped":
            return pipelined(lb, blobs, None, prefill, shipped, False, a.depth, prefill_n=prefill_n, leaf=LEAF_SHIPPED)
        return sequential_front_end(lb, blobs, prefill, prefill_n, shipped)

    for arm in arms:                     # one untimed pass each: modules, allocations
        run(arm)
    for rep in range(a.reps):
        last = {}
        for arm in arms:
            out = run(arm)
            last[arm] = out
            dt = out[0]
            entry = dict(scans_per_s=a.scans / dt, ms_per_scan=1e3 * dt / a.scans)
            if arm.startswith("chain"):
                res, times = out[1], out[2]
                entry.update(stage_times=times, filtered_points_mean=float(np.mean([r.n_filtered for r in res])),
                             leaf_mean=float(np.mean([r.leaf_size for r in res])),
                             keyframes=sum(r.keyframe for r in res), crops=sum(1 for r in res if r.n_removed))
            else:
                entry.update(leaf_mean=float(np.mean([r["leaf"] for r in out[1]])))
            line["arms"].setdefault(arm, []).append(entry)
        res, recs = last["chain_shipped"][1], last["seq_shipped"][1]
        leaves_equal = all(np.float32(r.leaf_size) == e["leaf"] for r, e in zip(res, recs))
        line["arms"]["chain_shipped"][-1]["bit_equal_scans_vs_seq_shipped"] = (len(res) - same(res, recs)) if leaves_equal else 0
    for arm in arms:
        line["best_scans_per_s_" + arm] = max(x["scans_per_s"] for x in line["arms"][arm])


def icp_covariance(lb, a, blobs, prefill, line):
    """--icp-covariance: the shipped chain with the ICP covariance off and on, alternated"""
    g = lb.GicpB200()
    g.setInputSource(prefill)
    prefill_n = g.computeNormals(0, 20)[:, :3].copy()
    base = dict(translation_threshold_kf=0.6, refresh_every=2, **FE.SHIPPED)
    kw = {"shipped_cov_off": dict(base, icp_covariance=dict(enabled=0, max_covariance=0.01)),
          "shipped_cov_on": dict(base, icp_covariance=dict(enabled=1, max_covariance=0.01))}
    line["params"] = dict(base, shipped_initial_leaf=LEAF_SHIPPED, map_resolution=MAP_RES, icp_max_covariance=0.01)

    def run(arm):
        return pipelined(lb, blobs, None, prefill, kw[arm], False, a.depth, prefill_n=prefill_n, leaf=LEAF_SHIPPED)

    for arm in kw:                       # one untimed pass each: modules, allocations
        run(arm)
    for rep in range(a.reps):
        last = {}
        for arm in kw:
            dt, res, times = last[arm] = run(arm)
            line["arms"].setdefault(arm, []).append(dict(
                scans_per_s=a.scans / dt, ms_per_scan=1e3 * dt / a.scans,
                stage_l_busy_ms_per_scan=1e3 * times["localization_busy_s"] / max(times["localized"], 1),
                stage_times=times, covariances=sum(r.has_icp_covariance for r in res)))
        off, on = last["shipped_cov_off"][1], last["shipped_cov_on"][1]
        line["arms"]["shipped_cov_on"][-1]["bit_equal_poses_vs_off"] = sum(
            np.array_equal(np.asarray(x.pose).view(np.uint64), np.asarray(y.pose).view(np.uint64)) for x, y in zip(off, on))
    for arm in kw:
        line["best_scans_per_s_" + arm] = max(x["scans_per_s"] for x in line["arms"][arm])
        line["median_stage_l_busy_ms_" + arm] = float(np.median([x["stage_l_busy_ms_per_scan"] for x in line["arms"][arm]]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=60)
    ap.add_argument("--beams", type=int, default=64)
    ap.add_argument("--az", type=int, default=2048)
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--front-end", action="store_true", help="compare the current chain with LOCUS's shipped front end")
    ap.add_argument("--icp-covariance", action="store_true",
                    help="the shipped chain with and without the localization's ICP covariance (--reps defaults to 3)")
    ap.add_argument("--lidars", type=int, default=1, choices=(1, 3),
                    help="3: every scan is three lidars merged in the VoxelGrid stage (lb_locus_submit_merged)")
    ap.add_argument("--leaf", type=float, default=None, help="VoxelGrid leaf of --lidars 3 (default 0.5)")
    ap.add_argument("--odometry-method", choices=("gicp", "ndt"), default="gicp", help="registration_method of the odometry")
    ap.add_argument("--ndt-map-rebuild", type=int, default=0, metavar="N",
                    help="time the NDT target of an N-point submap after a change of the map")
    ap.add_argument("--localization-method", choices=("gicp", "ndt"), default="gicp",
                    help="registration_method of the localization")
    a = ap.parse_args()
    if a.icp_covariance and "--reps" not in sys.argv:
        a.reps = 3
    import torch
    import locus_b200 as lb
    assert lb.device_count() > 0, "bench_locus needs a CUDA device"
    if a.ndt_map_rebuild:
        line = {"card": card()}
        ndt_map_rebuild(lb, a, line)
        emit(line, a.out)
        return
    if a.lidars == 3:
        line = {"scans": a.scans, "depth": a.depth, "card": card(), "arms": {}}
        lidars(lb, a, line)
        emit(line, a.out)
        return
    scene, poses, blobs = G.stream(a.seed, a.scans, a.beams, a.az)
    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], a.seed, a.beams, a.az)
    vg = lb.VoxelGridB200(); vg.setLeafSize(0.2)
    prefill = np.ascontiguousarray(vg.filter(G.xyz_blob(world), STEP, lb.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
    params = dict(translation_threshold_kf=0.6, refresh_every=2, odometry_method=a.odometry_method,
                  localization_method=a.localization_method)
    line = {"scans": a.scans, "raw_points_per_scan": blobs[0].size // STEP, "depth": a.depth, "card": card(),
            "params": dict(params, leaf=LEAF, map_resolution=MAP_RES), "arms": {}}
    if a.front_end:
        front_end(lb, a, blobs, prefill, line)
        emit(line, a.out)
        return
    if a.icp_covariance:
        icp_covariance(lb, a, blobs, prefill, line)
        emit(line, a.out)
        return
    d_blobs = [torch.from_numpy(b).cuda() for b in blobs]
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
    emit(line, a.out)


def emit(line, out):
    line["card_after"] = card()
    txt = json.dumps(line)
    print(txt)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
