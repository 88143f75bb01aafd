"""The front end of lb_locus without a GPU: adaptive input voxelization, the normals stage and keyframes with normals.

* tools/front_end_oracle.adaptive_leaf equals a line-by-line transcription of Locus::ApplyAdaptiveInputVoxelization
  (locus/src/Locus.cc:780-810) on random count sequences that hit both clamps, the forced update every 20 scans, the
  first scan's forced update and changes just above and below 0.01.
* odometry.cu's host logic, compiled against fake stages with the front end's calls logged in order
  (tests/front_end_stub.h): stage V sets exactly the oracle's leaves, each after the scan it follows and before the next
  is filtered, at depth 1 and 4; a failed VoxelGrid changes nothing; leaf_size reports the leaf each scan was filtered
  with; the normals call comes once per scan and before its prepare_source (with cloud sharing), or once per cloud and
  registration (without); keyframes go through the normals insert; lb_locus_set_params refuses a covariance mode the
  shared clouds cannot serve and keeps the previous parameters.
* the submap oracle with normals against a direct numpy restatement.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from locus_b200 import api
from tools import front_end_oracle as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP = 16
MAXP = 4096
LB_ERR_UNSUPPORTED = -9


def _build(name, define):
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    so = os.path.join(bdir, name)
    srcs = [os.path.join(ROOT, p) for p in ("tests/locus_front_end_harness.cpp", "tests/front_end_stub.h", "tests/locus_stub.h",
                                             "tests/odometry_stub.h", "locus_b200/csrc/odometry.cu",
                                             "locus_b200/csrc/lo_pose.h", "include/locus_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-O1", "-D" + define,
                               "-x", "c++", srcs[0], "-I", os.path.join(ROOT, "tests"), "-o", so])
    H = C.CDLL(so)
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    H.fh_set_leaf.argtypes = [vp, C.c_float]
    H.fh_log.argtypes = [vp, vp, vp, vp, vp, sz]; H.fh_log.restype = sz
    H.lb_odometry_create.argtypes = [i32, i32, sz, C.c_uint32, C.POINTER(vp)]
    H.lb_odometry_destroy.argtypes = [vp]
    H.lb_odometry_set_cloud_sharing.argtypes = [vp, i32]
    H.lb_odometry_set_normals.argtypes = [vp, i32, vp]
    H.lb_odometry_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, C.POINTER(C.c_uint64)]
    H.lb_odometry_next.argtypes = [vp, C.POINTER(api.OdometryResult), i32]
    if define == "LB_LOCUS_STUB":
        H.fh_submap_create.argtypes = [i32, sz]; H.fh_submap_create.restype = vp
        H.fh_submap_destroy.argtypes = [vp]
        H.fh_events.argtypes = [vp, vp, sz]; H.fh_events.restype = sz
        H.lb_locus_default_params.argtypes = [C.POINTER(api.LocusParams)]
        H.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
        H.lb_locus_destroy.argtypes = [vp]
        H.lb_locus_voxel.argtypes = [vp]; H.lb_locus_voxel.restype = vp
        H.lb_locus_set_params.argtypes = [vp, C.POINTER(api.LocusParams)]
        H.lb_locus_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, C.POINTER(C.c_uint64)]
        H.lb_locus_next.argtypes = [vp, C.POINTER(api.LocusResult), i32]
    return H


@pytest.fixture(scope="module")
def lh():
    return _build("liblocus_front_end_harness.so", "LB_LOCUS_STUB")


@pytest.fixture(scope="module")
def oh():
    return _build("libodometry_front_end_harness.so", "LB_ODOMETRY_STUB")


def _log(H):
    cap = 1 << 16
    kind = (C.c_char * cap)(); ids = (C.c_uint64 * cap)(); a = (C.c_int * cap)(); b = (C.c_int * cap)()
    v = (C.c_double * cap)()
    n = H.fh_log(kind, ids, a, b, v, cap)
    return [(kind[i].decode(), ids[i], a[i], b[i], v[i]) for i in range(n)]


def _events(H):
    cap = 4096
    kind = (C.c_int * cap)(); ids = (C.c_uint64 * cap)()
    n = H.fh_events(kind, ids, cap)
    return [(kind[i], ids[i]) for i in range(n)]


def _scan(i, n, flags=0):
    b = np.zeros(max(n, 1) * STEP, dtype=np.uint8)
    b[:8] = np.frombuffer(np.uint64(i).tobytes(), dtype=np.uint8)
    b[8:12] = np.frombuffer(np.uint32(flags).tobytes(), dtype=np.uint8)
    return b


def _fields():
    return api.VoxelGridB200._fields([("x", 0, api.LB_FLOAT32, 1), ("y", 4, api.LB_FLOAT32, 1), ("z", 8, api.LB_FLOAT32, 1)])


def _params(H, **kw):
    p = api.LocusParams()
    assert H.lb_locus_default_params(C.byref(p)) == 0
    for k, v in kw.items():
        for kk, vv in v.items():
            setattr(getattr(p, k), kk, vv)
    return p


# ------------------------------------------------------------------------------------------ the leaf rule itself
def _transcription(counts, ptp, leaf0):
    """Locus::ApplyAdaptiveInputVoxelization, statement by statement; returns the published leaves (None = none)"""
    value, counter_voxel_ = leaf0, 0
    out = []
    for size in counts:
        change = False
        dchange_voxel = value * (float(size) / float(ptp))
        if dchange_voxel < 0.01:
            dchange_voxel = 0.01
        if dchange_voxel > 5.0:
            dchange_voxel = 5.0
        if abs(value - dchange_voxel) > 0.01 or counter_voxel_ % 20 == 0:
            value = dchange_voxel
            change = True
            counter_voxel_ = 0
        counter_voxel_ += 1
        out.append(dchange_voxel if change else None)
    return out


def _sequences():
    rng = np.random.default_rng(7)
    seqs = []
    for s in range(40):
        ptp = int(rng.choice([3, 100, 3000]))
        n = int(rng.integers(30, 90))
        kind = s % 4
        if kind == 0:
            c = rng.integers(0, 4 * ptp, n)                      # wide: both clamps
        elif kind == 1:
            c = np.full(n, ptp) + rng.integers(-1, 2, n)         # steady: the forced update every 20 scans
        elif kind == 2:
            c = np.where(rng.random(n) < 0.2, 0, rng.integers(ptp * 30, ptp * 80, n))   # 0.01 and 5.0
        else:
            c = rng.integers(int(ptp * 0.9), int(ptp * 1.1) + 2, n)
        seqs.append((ptp, [int(x) for x in c]))
    # changes of exactly one side of 0.01: 0.25 * 1041/1000 = 0.26025 (> 0.01 away), 0.25 * 1039/1000 = 0.25975 (< 0.01)
    seqs.append((1000, [1000, 1041, 1000, 1039, 1000, 1040, 961, 959, 1000] + [1000] * 25))
    return seqs


def test_adaptive_leaf_equals_transcription():
    hit = set()
    for ptp, counts in _sequences():
        ref = _transcription(counts, ptp, 0.25)
        st = FE.LeafState(0.25)
        for k, (n, r) in enumerate(zip(counts, ref)):
            before, old = st.counter, st.leaf
            changed = FE.adaptive_leaf(st, n, ptp)
            assert changed == (r is not None)
            if changed:
                assert np.float64(st.leaf).view(np.uint64) == np.float64(r).view(np.uint64)
                hit.add("first" if k == 0 else "forced" if before % 20 == 0 and abs(old - r) <= 0.01 else "moved")
            elif abs(old - old * (n / ptp)) > 0.009:
                hit.add("just below")
            hit.add("lo" if st.leaf == 0.01 else "hi" if st.leaf == 5.0 else "mid")
    assert {"first", "forced", "moved", "lo", "hi", "mid", "just below"} <= hit


# ------------------------------------------------------------------------------------------ through the chain
def _run_chain(H, counts, depth, flags=(), leaf0=0.25, ptp=100, normals_k=0, **extra):
    H.fh_reset()
    m = H.fh_submap_create(0, 0)
    h = C.c_void_p()
    assert H.lb_locus_create(0, depth, MAXP, STEP, m, C.byref(h)) == 0
    assert H.fh_set_leaf(H.lb_locus_voxel(h), leaf0) == 0
    P = _params(H, front_end=dict(normals_k=normals_k, adaptive_voxelization=1, points_to_process=ptp), **extra)
    assert H.lb_locus_set_params(h, C.byref(P)) == 0
    H.fh_reset()                       # drop the set-up call from the log
    fa = _fields()
    scans = [_scan(100 + k, n, 1 if k in flags else 0) for k, n in enumerate(counts)]
    t = C.c_uint64(0)
    for k, n in enumerate(counts):
        assert H.lb_locus_submit(h, scans[k].ctypes.data_as(C.c_void_p), n, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0
    res = []
    for _ in counts:
        r = api.LocusResult()
        assert H.lb_locus_next(h, C.byref(r), 1) == 0
        res.append(r)
    H.lb_locus_destroy(h)
    H.fh_submap_destroy(m)
    return res, _log(H), _events(H)


def _oracle_leaves(counts, flags, leaf0, ptp):
    """(leaf each scan was filtered with, [(scan id after which a leaf is set, leaf)])"""
    st = FE.LeafState(np.float32(leaf0))
    cur = np.float32(leaf0)
    used, sets = [], []
    for k, n in enumerate(counts):
        used.append(cur)
        if k in flags:
            continue
        if FE.adaptive_leaf(st, n, ptp):
            cur = np.float32(st.leaf)
            sets.append((100 + k, cur))
    return used, sets


@pytest.mark.parametrize("depth", [1, 4])
def test_stage_v_sets_the_oracle_leaves(lh, depth):
    rng = np.random.default_rng(depth)
    counts = [int(x) for x in rng.integers(0, 400, 60)] + [0, 0, 3000, 3000, 100, 100] + [100] * 24
    flags = {5, 6, 31}
    res, log, _ = _run_chain(lh, counts, depth, flags=flags)
    used, sets = _oracle_leaves(counts, flags, 0.25, 100)
    got = [(i, np.float32(v)) for kind, i, _, _, v in log if kind == "S"]
    assert [i for i, _ in got] == [i for i, _ in sets]
    assert all(a.view(np.uint32) == b.view(np.uint32) for (_, a), (_, b) in zip(got, sets))
    assert [np.float32(r.leaf_size).view(np.uint32) for r in res] == [u.view(np.uint32) for u in used]
    assert any(v == np.float32(0.01) for _, v in sets) and any(v == np.float32(5.0) for _, v in sets)
    for k in flags:
        assert res[k].status != 0


def test_normals_call_before_prepare_with_sharing(lh):
    counts = [8] * 12
    res, log, events = _run_chain(lh, counts, 3, normals_k=20)
    calls = [(kind, i, a, b) for kind, i, a, b, _ in log if kind in "NP"]
    for k in range(len(counts)):
        mine = [c for c in calls if c[1] == 100 + k]
        assert mine == [("N", 100 + k, 0, 20), ("P", 100 + k, 0, 0)], mine
    # every keyframe (the first scan at least) went through the normals insert, at stride 24 with the normal at 12
    ins = [(kind, i, a, b) for kind, i, a, b, _ in log if kind == "I"]
    assert ins and all(a == 24 and b == 12 for _, _, a, b in ins)
    assert {k for k, _ in events if k in (1, 3)} == {3}
    # normals off: no normals call, plain inserts
    res, log, events = _run_chain(lh, counts, 3, normals_k=0)
    assert not [c for c in log if c[0] in "NI"]
    assert {k for k, _ in events if k in (1, 3)} == {1}


def test_normals_for_source_and_target_without_sharing(oh):
    oh.fh_reset()
    h = C.c_void_p()
    assert oh.lb_odometry_create(0, 2, MAXP, STEP, C.byref(h)) == 0
    assert oh.lb_odometry_set_cloud_sharing(h, 0) == 0
    assert oh.lb_odometry_set_normals(h, 2, None) == LB_ERR_UNSUPPORTED
    assert oh.lb_odometry_set_normals(h, 12, None) == 0
    fa = _fields()
    scans = [_scan(200 + k, 8) for k in range(10)]
    t = C.c_uint64(0)
    for s in scans:
        assert oh.lb_odometry_submit(h, s.ctypes.data_as(C.c_void_p), 8, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0
    for _ in scans:
        r = api.OdometryResult()
        assert oh.lb_odometry_next(h, C.byref(r), 1) == 0 and r.status == 0
    assert oh.lb_odometry_set_normals(h, 20, None) != 0              # after the first scan: refused
    assert oh.lb_odometry_set_normals(h, 12, None) == 0              # the same setting is fine
    oh.lb_odometry_destroy(h)
    log = [(kind, i, a, b) for kind, i, a, b, _ in _log(oh)]
    assert not [c for c in log if c[0] == "P"]
    # registration k (k >= 1): the source k, then the target k - 1, each once; scan 0 registers nothing
    for k in range(1, 10):
        assert sorted(c for c in log if c[0] == "N" and (c[1], c[2]) in ((200 + k, 0), (200 + k - 1, 1))) == \
            sorted([("N", 200 + k, 0, 12), ("N", 200 + k - 1, 1, 12)])
    assert len([c for c in log if c[0] == "N"]) == 2 * 9


def test_set_params_refuses_a_mode_the_shared_clouds_cannot_serve(lh):
    lh.fh_reset()
    m = lh.fh_submap_create(0, 0)
    h = C.c_void_p()
    assert lh.lb_locus_create(0, 1, MAXP, STEP, m, C.byref(h)) == 0
    nr = dict(recompute_source_covariance=0, recompute_target_covariance=0)
    good = _params(lh, odometry=nr, localization=nr)
    assert lh.lb_locus_set_params(h, C.byref(good)) == 0
    # the odometry's two flags, or the odometry and the localization source, disagree; bad front-end values
    def flags(os_, ot, ls, lt=0, **fe):
        return _params(lh, odometry=dict(recompute_source_covariance=os_, recompute_target_covariance=ot),
                       localization=dict(recompute_source_covariance=ls, recompute_target_covariance=lt), front_end=fe)
    bad = [flags(0, 1, 0, normals_k=20), flags(1, 0, 0, normals_k=20), flags(0, 0, 1, normals_k=20), flags(1, 1, 0),
           flags(0, 0, 0, normals_k=2), flags(0, 0, 0, normals_k=21), flags(0, 0, 0, adaptive_voxelization=1, points_to_process=0)]
    for p in bad:
        assert lh.lb_locus_set_params(h, C.byref(p)) == -1
    # the localization's target flag is free
    assert lh.lb_locus_set_params(h, C.byref(flags(0, 0, 0, lt=1))) == 0
    assert lh.lb_locus_set_params(h, C.byref(flags(1, 1, 1, lt=0))) == 0
    # the previous parameters stayed in place: no normals, no leaf changes
    fa = _fields()
    scans = [_scan(300 + k, 8) for k in range(6)]
    t = C.c_uint64(0)
    for s in scans:
        assert lh.lb_locus_submit(h, s.ctypes.data_as(C.c_void_p), 8, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0
    for _ in scans:
        r = api.LocusResult()
        assert lh.lb_locus_next(h, C.byref(r), 1) == 0 and r.status == 0
    assert not [c for c in _log(lh) if c[0] in "NIS"]
    # normals_k cannot change once scans have been through the pipeline
    assert lh.lb_locus_set_params(h, C.byref(_params(lh, odometry=nr, localization=nr, front_end=dict(normals_k=20)))) != 0
    lh.lb_locus_destroy(h)
    lh.fh_submap_destroy(m)


# ------------------------------------------------------------------------------------------ the submap oracle
def test_submap_oracle_with_normals_against_numpy():
    rng = np.random.default_rng(3)
    res = np.float32(0.5)
    o = FE.SubmapNormalsOracle(res)
    pts = np.zeros((0, 3), np.float32); nrm = np.zeros((0, 3), np.float32)
    for step in range(6):
        p = (rng.normal(size=(400, 3)) * 4).astype(np.float32)
        p[rng.integers(0, 400, 5)] = np.nan
        q = (rng.normal(size=(400, 3))).astype(np.float32) if step % 3 else None
        added = o.insert(p, q)
        # numpy: the first finite point of every voxel not occupied yet, in input order
        occ = {tuple(v) for v in np.floor(pts / res).astype(np.int64)}
        keep = []
        for i in range(len(p)):
            if not np.isfinite(p[i]).all():
                continue
            v = tuple(np.floor(p[i] / res).astype(np.int64))
            if v not in occ:
                occ.add(v); keep.append(i)
        assert np.array_equal(added, p[keep])
        pts = np.concatenate([pts, p[keep]])
        nrm = np.concatenate([nrm, q[keep] if q is not None else np.full((len(keep), 3), np.nan, np.float32)])
        if step % 2:
            c = rng.normal(size=3).astype(np.float32); h = np.float32(6.0)
            inside = np.all((pts >= c - h) & (pts <= c + h), axis=1)
            assert o.crop(c, h) == int((~inside).sum())
            pts, nrm = pts[inside], nrm[inside]
        assert np.array_equal(o.pts.view(np.uint32), pts.view(np.uint32))
        assert np.array_equal(o.nrm.view(np.uint32), nrm.view(np.uint32))
    eps = 1e-3
    n = nrm.astype(np.float64)
    direct = np.eye(3)[None] - (1.0 - eps) * np.einsum("ni,nj->nij", n, n)
    got = o.normal_covariances(eps)
    fin = np.isfinite(n).all(axis=1)
    assert np.allclose(got[fin], direct[fin], rtol=1e-14, atol=1e-14) and np.isnan(got[~fin]).all()
