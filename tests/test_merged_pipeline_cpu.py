"""The multi-lidar input of lb_odometry / lb_locus (lb_*_submit_merged) without a GPU.

odometry.cu's host logic is compiled against fake stages (tests/odometry_stub.h, tests/locus_stub.h) with the merged
VoxelGrid call recorded by tests/merged_stub.h.  Checks, at depth 1 and 4:
* every scan's clouds reach stage V in the order given, with their point counts and the transforms given at submit --
  although the test overwrites its transform arrays right after each submit (the pipeline copies them);
* the lidar count changes from scan to scan (3 -> 2 -> 1 -> 3), with an empty input and a lidar that comes back last;
* an all-empty scan filters to nothing and changes no pose, keyframe or map state: the results equal those of the same
  stream submitted one cloud per scan with that scan empty;
* a failed VoxelGrid on a merged scan gives the result a failed single-cloud scan gives;
* each refusal at submit leaves the pending count and the next ticket number as they were;
* the pipeline sizes the VoxelGrid scratch once, at creation, for max_points raw points.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from locus_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP = 16
MAXP = 64
LB_ERR_INVALID_ARG, LB_ERR_CAPACITY = -1, -8


def _build(name, define):
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    so = os.path.join(bdir, name)
    srcs = [os.path.join(ROOT, p) for p in ("tests/merged_harness.cpp", "tests/merged_stub.h", "tests/locus_stub.h",
                                             "tests/odometry_stub.h", "tests/front_end_stub.h", "tests/icp_covariance_stub.h",
                                             "locus_b200/csrc/odometry.cu", "locus_b200/csrc/lo_pose.h", "include/locus_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-O1", "-D" + define,
                               "-x", "c++", srcs[0], "-I", os.path.join(ROOT, "tests"), "-o", so])
    H = C.CDLL(so)
    vp, sz, i32, u64p = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_uint64)
    H.mh_calls.argtypes = [vp, vp, vp, vp, vp, sz]; H.mh_calls.restype = sz
    H.mh_reserves.argtypes = [vp, sz]; H.mh_reserves.restype = sz
    H.mh_last_error.restype = C.c_char_p
    sub = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, u64p]
    merged = [vp, C.POINTER(api.VoxelInput), i32, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, u64p]
    H.lb_odometry_create.argtypes = [i32, i32, sz, C.c_uint32, C.POINTER(vp)]
    H.lb_odometry_destroy.argtypes = [vp]
    H.lb_odometry_submit.argtypes = sub
    H.lb_odometry_submit_merged.argtypes = merged
    H.lb_odometry_next.argtypes = [vp, C.POINTER(api.OdometryResult), i32]
    H.lb_odometry_pending.argtypes = [vp, C.POINTER(sz)]
    if define == "LB_LOCUS_STUB":
        H.mh_submap_create.argtypes = [i32, sz]; H.mh_submap_create.restype = vp
        H.mh_submap_destroy.argtypes = [vp]
        H.mh_events.argtypes = [vp, vp, vp, sz]; H.mh_events.restype = sz
        H.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
        H.lb_locus_destroy.argtypes = [vp]
        H.lb_locus_submit.argtypes = sub
        H.lb_locus_submit_merged.argtypes = merged
        H.lb_locus_next.argtypes = [vp, C.POINTER(api.LocusResult), i32]
        H.lb_locus_pending.argtypes = [vp, C.POINTER(sz)]
    return H


@pytest.fixture(scope="module")
def oh():
    return _build("libmerged_odometry_harness.so", "LB_ODOMETRY_STUB")


@pytest.fixture(scope="module")
def lh():
    return _build("libmerged_locus_harness.so", "LB_LOCUS_STUB")


def _cloud(i, n, flags=0):
    b = np.zeros(max(n, 1) * STEP, dtype=np.uint8)
    b[:8] = np.frombuffer(np.uint64(i).tobytes(), dtype=np.uint8)
    b[8:12] = np.frombuffer(np.uint32(flags).tobytes(), dtype=np.uint8)
    return b


def _fields():
    return api.VoxelGridB200._fields([("x", 0, api.LB_FLOAT32, 1), ("y", 4, api.LB_FLOAT32, 1), ("z", 8, api.LB_FLOAT32, 1)])


def _calls(H):
    cap = 4096
    ni = (C.c_int * cap)(); ids = (C.c_uint64 * (3 * cap))(); n = (C.c_size_t * (3 * cap))(); hT = (C.c_int * (3 * cap))()
    T = (C.c_float * (48 * cap))()
    m = H.mh_calls(ni, ids, n, hT, T, cap)
    Ta = np.ctypeslib.as_array(T).reshape(cap, 3, 16)
    return [dict(n_inputs=ni[c], ids=[ids[3 * c + i] for i in range(ni[c])], n=[n[3 * c + i] for i in range(ni[c])],
                 has_T=[hT[3 * c + i] for i in range(ni[c])], T=Ta[c, :ni[c]].copy()) for c in range(m)]


def _stream(n_scans):
    """per scan: [(id, n_pts, flags, transform or None)] in merge order.  The lidar count runs 3, 2, 1, 3, ..., scan 4
    has an empty middle input, and from scan 5 on lidar 0 has come back LAST (the merger's alive_keys_ after a
    resurrection).  Ids: 1000 * (scan + 1) + 10 * lidar."""
    rng = np.random.default_rng(3)
    out = []
    for k in range(n_scans):
        lidars = [[0, 1, 2], [0, 1], [0], [0, 1, 2], [2, 0, 1]][k % 5] if k < 5 else [1, 2, 0][: 1 + (k % 3)]
        scan = []
        for j, li in enumerate(lidars):
            n = 0 if (k == 4 and j == 1) else 3 + (k + li) % 4
            T = None if (k + li) % 4 == 3 else rng.normal(size=16).astype(np.float32)
            scan.append((1000 * (k + 1) + 10 * li, n, 0, T))
        out.append(scan)
    return out


def _submit_merged(H, fn, h, scan, guess, fa, t):
    """submits one scan; the caller's transform arrays are overwritten right after the call"""
    arr = (api.VoxelInput * len(scan))()
    blobs, Ts = [], []
    for i, (cid, n, fl, T) in enumerate(scan):
        b = _cloud(cid, n, fl)
        blobs.append(b)
        arr[i].data = b.ctypes.data_as(C.c_void_p).value if n else None
        arr[i].n_pts = n
        if T is not None:
            Tc = T.copy()
            Ts.append(Tc)
            arr[i].transform = Tc.ctypes.data_as(C.c_void_p).value
    st = fn(h, arr, len(scan), STEP, fa, 3, 0, guess.ctypes.data_as(C.c_void_p), None, 0, C.byref(t))
    for Tc in Ts:
        Tc[:] = np.nan                        # the pipeline must have copied them
    return st, blobs


def _check_calls(calls, scans):
    assert len(calls) == len(scans)
    for c, scan in zip(calls, scans):
        assert c["n_inputs"] == len(scan)
        assert c["ids"] == [cid if n else 2 ** 64 - 1 for cid, n, _, _ in scan]
        assert c["n"] == [n for _, n, _, _ in scan]
        assert c["has_T"] == [int(T is not None) for _, _, _, T in scan]
        for i, (_, _, _, T) in enumerate(scan):
            want = np.eye(4, dtype=np.float32).reshape(16) if T is None else T
            assert np.array_equal(c["T"][i].view(np.uint32), want.view(np.uint32))


def _first_id(scan):
    return next((cid for cid, n, _, _ in scan if n), None)


@pytest.mark.parametrize("depth", [1, 4])
def test_odometry_inputs_reach_stage_v_in_order(oh, depth):
    oh.mh_reset()
    h = C.c_void_p()
    assert oh.lb_odometry_create(0, depth, MAXP, STEP, C.byref(h)) == 0
    sizes = (C.c_size_t * 8)()
    assert oh.mh_reserves(sizes, 8) == 1 and sizes[0] == MAXP       # the VoxelGrid scratch: once, at creation
    scans = _stream(23)
    fa, t, r = _fields(), C.c_uint64(), api.OdometryResult()
    keep, res = [], []
    for k, scan in enumerate(scans):
        g = np.zeros(16, np.float32); g[3] = k
        st, blobs = _submit_merged(oh, oh.lb_odometry_submit_merged, h, scan, g, fa, t)
        assert st == 0 and t.value == k
        keep.append(blobs)
    for _ in scans:
        assert oh.lb_odometry_next(h, C.byref(r), 1) == 0
        res.append((r.ticket, r.status, r.has_pose, r.n_filtered, list(r.gicp.final_transformation[:5])))
    oh.lb_odometry_destroy(h)
    _check_calls(_calls(oh), scans)
    assert [x[0] for x in res] == list(range(len(scans)))
    assert oh.mh_reserves(sizes, 8) == 1
    for k, (_, st, has_pose, n_f, ft) in enumerate(res):
        assert st == 0
        if k == 0:
            assert not has_pose
            continue
        # the fake VoxelGrid tags the merged scan with its first non-empty input: source = this scan, target = the last
        assert has_pose and ft[0] == _first_id(scans[k]) and ft[1] == _first_id(scans[k - 1]) and ft[4] == k


@pytest.mark.parametrize("depth", [1, 4])
def test_locus_inputs_reach_stage_v_and_the_map_gets_the_merged_scan(lh, depth):
    lh.mh_reset()
    m = lh.mh_submap_create(0, 0)
    h = C.c_void_p()
    assert lh.lb_locus_create(0, depth, MAXP, STEP, m, C.byref(h)) == 0
    scans = _stream(17)
    fa, t, r = _fields(), C.c_uint64(), api.LocusResult()
    keep, res = [], []
    for k, scan in enumerate(scans):
        g = np.eye(4, dtype=np.float32).reshape(16).copy(); g[3] = 1.5       # every scan a keyframe
        st, blobs = _submit_merged(lh, lh.lb_locus_submit_merged, h, scan, g, fa, t)
        assert st == 0 and t.value == k
        keep.append(blobs)
    for _ in scans:
        assert lh.lb_locus_next(h, C.byref(r), 1) == 0
        res.append((r.status, r.n_filtered, r.keyframe, r.n_inserted))
    lh.lb_locus_destroy(h)
    _check_calls(_calls(lh), scans)
    cap = 1024
    kind = (C.c_int * cap)(); ids = (C.c_uint64 * cap)(); n = (C.c_size_t * cap)()
    ne = lh.mh_events(kind, ids, n, cap)
    inserts = [(ids[i], n[i]) for i in range(ne) if kind[i] == 1]
    # the keyframe is the merged scan: all the scan's points, tagged with its first non-empty input
    assert inserts == [(_first_id(s), sum(x[1] for x in s)) for s in scans]
    assert all(st == 0 and kf == 1 and nf == sum(x[1] for x in s) for (st, nf, kf, _), s in zip(res, scans))
    lh.mh_submap_destroy(m)


def _run_locus(H, scans, merged, depth):
    """the results of a stream through lb_locus, one record per scan: merged = lb_locus_submit_merged, else
    lb_locus_submit of the first input's cloud with the scan's total point count (what the fakes make of a merge)"""
    H.mh_reset()
    m = H.mh_submap_create(0, 0)
    h = C.c_void_p()
    assert H.lb_locus_create(0, depth, MAXP, STEP, m, C.byref(h)) == 0
    fa, t, r = _fields(), C.c_uint64(), api.LocusResult()
    keep, out = [], []
    for k, scan in enumerate(scans):
        g = np.eye(4, dtype=np.float32).reshape(16).copy(); g[3] = 0.4 * (k % 3)
        if merged:
            st, blobs = _submit_merged(H, H.lb_locus_submit_merged, h, scan, g, fa, t)
        else:
            cid, _, fl, _ = scan[0]
            blobs = _cloud(cid, max(sum(x[1] for x in scan), 1), fl)
            st = H.lb_locus_submit(h, blobs.ctypes.data_as(C.c_void_p), sum(x[1] for x in scan), STEP, fa, 3, 0,
                                   g.ctypes.data_as(C.c_void_p), None, 0, C.byref(t))
        assert st == 0
        keep.append(blobs)
    for _ in scans:
        assert H.lb_locus_next(h, C.byref(r), 1) == 0
        out.append(dict(status=r.status, error=r.error, n_filtered=r.n_filtered, has_odometry=r.has_odometry,
                        has_localization=r.has_localization, keyframe=r.keyframe, n_inserted=r.n_inserted,
                        map_size=r.map_size, O=list(r.odometry_pose), I=list(r.incremental), L=list(r.pose)))
    H.lb_locus_destroy(h)
    H.mh_submap_destroy(m)
    return out


@pytest.mark.parametrize("depth", [1, 4])
def test_locus_all_empty_scan_changes_no_state(lh, depth):
    # the first input of every scan carries the id in both runs, so the scans have the same ids
    scans = [[(1000 * (k + 1), 0 if k == 6 else 5, 0, None), (1000 * (k + 1) + 10, 0 if k == 6 else 2, 0, None)]
             for k in range(12)]
    merged = _run_locus(lh, scans, True, depth)
    single = _run_locus(lh, scans, False, depth)
    assert merged == single
    e, before = merged[6], merged[5]
    assert e["status"] == 0 and e["n_filtered"] == 0 and not e["keyframe"] and not e["has_localization"]
    assert e["O"] == before["O"] and e["L"] == before["L"] and e["map_size"] == before["map_size"]
    assert not merged[7]["has_odometry"]             # the scan after it has no odometry target, as after an empty scan


@pytest.mark.parametrize("depth", [1, 4])
def test_locus_stage_v_failure_behaves_like_a_single_scan(lh, depth):
    scans = [[(1000 * (k + 1), 6, 1 if k == 5 else 0, None), (1000 * (k + 1) + 10, 3, 0, None)] for k in range(12)]
    merged = _run_locus(lh, scans, True, depth)
    single = _run_locus(lh, scans, False, depth)
    assert merged == single
    assert merged[5]["status"] == LB_ERR_INVALID_ARG and b"stub voxel failure" in merged[5]["error"]
    assert merged[5]["L"] == merged[4]["L"] and merged[5]["map_size"] == merged[4]["map_size"]


def test_odometry_stage_v_failure_and_empty_scan_behave_like_single_scans(oh):
    scans = [[(100 + k, 0 if k == 7 else 4, 1 if k == 3 else 0, None), (900 + k, 0 if k == 7 else 3, 0, None)] for k in range(12)]
    fa, t, r = _fields(), C.c_uint64(), api.OdometryResult()
    runs = []
    for merged in (True, False):
        oh.mh_reset()
        h = C.c_void_p()
        assert oh.lb_odometry_create(0, 4, MAXP, STEP, C.byref(h)) == 0
        keep = []
        for k, scan in enumerate(scans):
            g = np.zeros(16, np.float32)
            if merged:
                st, b = _submit_merged(oh, oh.lb_odometry_submit_merged, h, scan, g, fa, t)
            else:
                b = _cloud(scan[0][0], 8, scan[0][2])
                st = oh.lb_odometry_submit(h, b.ctypes.data_as(C.c_void_p), sum(x[1] for x in scan), STEP, fa, 3, 0,
                                           g.ctypes.data_as(C.c_void_p), None, 0, C.byref(t))
            assert st == 0
            keep.append(b)
        out = []
        for _ in scans:
            assert oh.lb_odometry_next(h, C.byref(r), 1) == 0
            out.append((r.ticket, r.status, r.error, r.has_pose, r.n_filtered, list(r.gicp.final_transformation[:4])))
        oh.lb_odometry_destroy(h)
        runs.append(out)
    assert runs[0] == runs[1]
    assert runs[0][3][1] == LB_ERR_INVALID_ARG and not runs[0][4][3]      # the failed scan, and the one after it
    assert runs[0][7][1] == 0 and runs[0][7][4] == 0 and not runs[0][8][3]


@pytest.mark.parametrize("pipeline", ["odometry", "locus"])
def test_refusals_take_no_ticket(oh, lh, pipeline):
    H = oh if pipeline == "odometry" else lh
    H.mh_reset()
    h = C.c_void_p()
    m = None
    if pipeline == "odometry":
        assert H.lb_odometry_create(0, 2, MAXP, STEP, C.byref(h)) == 0
        submit, nxt, pending, res = H.lb_odometry_submit_merged, H.lb_odometry_next, H.lb_odometry_pending, api.OdometryResult()
    else:
        m = H.mh_submap_create(0, 0)
        assert H.lb_locus_create(0, 2, MAXP, STEP, m, C.byref(h)) == 0
        submit, nxt, pending, res = H.lb_locus_submit_merged, H.lb_locus_next, H.lb_locus_pending, api.LocusResult()
    fa, t = _fields(), C.c_uint64(77)
    a, b = _cloud(1, 8), _cloud(2, 8)
    # one scan in flight, then the refusals
    good = (api.VoxelInput * 2)()
    good[0].data = a.ctypes.data_as(C.c_void_p).value; good[0].n_pts = 8
    good[1].data = b.ctypes.data_as(C.c_void_p).value; good[1].n_pts = 8
    assert submit(h, good, 2, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0 and t.value == 0
    four = (api.VoxelInput * 4)(good[0], good[1], good[0], good[1])
    nul = (api.VoxelInput * 2)(good[0]); nul[1].data = None; nul[1].n_pts = 3
    big = (api.VoxelInput * 2)(good[0]); big[1].data = b.ctypes.data_as(C.c_void_p).value; big[1].n_pts = MAXP - 7
    cases = [(four, 0, STEP, LB_ERR_INVALID_ARG), (four, 4, STEP, LB_ERR_INVALID_ARG), (four, -1, STEP, LB_ERR_INVALID_ARG),
             (None, 2, STEP, LB_ERR_INVALID_ARG), (nul, 2, STEP, LB_ERR_INVALID_ARG), (big, 2, STEP, LB_ERR_CAPACITY),
             (good, 2, STEP + 4, LB_ERR_CAPACITY)]
    n = C.c_size_t()
    for arr, k, step, want in cases:
        t.value = 77
        assert submit(h, arr, k, step, fa, 3, 0, None, None, 0, C.byref(t)) == want, (k, step)
        assert t.value == 77 and H.mh_last_error()
        assert pending(h, C.byref(n)) == 0 and n.value == 1
    ok = (api.VoxelInput * 2)(good[0]); ok[1].data = b.ctypes.data_as(C.c_void_p).value; ok[1].n_pts = MAXP - 8   # exactly max_points
    assert submit(h, ok, 2, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0 and t.value == 1
    assert [nxt(h, C.byref(res), 1) == 0 and res.ticket for _ in range(2)] == [0, 1]
    assert len(_calls(H)) == 2
    if pipeline == "odometry":
        H.lb_odometry_destroy(h)
    else:
        H.lb_locus_destroy(h)
        H.mh_submap_destroy(m)
