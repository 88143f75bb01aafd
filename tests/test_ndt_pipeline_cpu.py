"""NDT registration inside lb_odometry and lb_locus, without a GPU.

The pipelines' host logic (locus_b200/csrc/odometry.cu) is built against fake stages (tests/locus_stub.h and
tests/ndt_stub.h, which log every NDT call and every GICP align) and checked for:
* routing: NDT odometry registers filtered k against filtered k-1 on the worker's NDT handle with the prior as guess and
  makes no GICP align -- and under lb_locus still prepares and shares every scan's GICP cloud; NDT localization sets the
  submap as target and aligns with the guess P of the GICP path, and builds no GICP map target unless the ICP covariance
  asks for one; O / I / L, keyframes, inserts and crops equal oracle.locus_oracle.LocusChain driven with the fakes'
  outputs, for (ndt, gicp), (gicp, ndt) and (ndt, ndt) at depth 1 and 4;
* errors: a failed NDT stage changes no state; a method change after the first scan, invalid NDT params and NDT with the
  normals stage in plain lb_odometry are refused, and the previous settings stay;
* layout: sizeof / offsetof of every changed struct, printed by a compiled probe, equal the ctypes mirrors.
The GPU twin is test_ndt_pipeline_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from locus_b200 import api
from oracle import locus_oracle as LO
from test_locus_cpu import NPTS, STEP, _corrections, _d, _dp, _fake_align, _fields, _increments, _pose, _rot, _same, _scan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GICP, NDT = api.LB_REG_GICP, api.LB_REG_NDT
ID0 = 100


def _build(name, src, deps, cmd):
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    out = os.path.join(bdir, name)
    srcs = [os.path.join(ROOT, p) for p in [src] + deps]
    if not os.path.exists(out) or any(os.path.getmtime(f) > os.path.getmtime(out) for f in srcs):
        subprocess.check_call(cmd + [srcs[0], "-o", out])
    return out


@pytest.fixture(scope="module")
def nh():
    so = _build("libndt_pipeline_harness.so", "tests/ndt_pipeline_harness.cpp",
                ["tests/ndt_stub.h", "tests/locus_stub.h", "locus_b200/csrc/odometry.cu", "locus_b200/csrc/lo_pose.h",
                 "include/locus_b200.h"],
                ["g++", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-O1", "-I",
                 os.path.join(ROOT, "tests"), "-x", "c++"])
    H = C.CDLL(so)
    vp, sz, i32, u64p = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_uint64)
    H.nh_submap_create.argtypes = [i32, sz]; H.nh_submap_create.restype = vp
    H.nh_submap_destroy.argtypes = [vp]
    H.nh_set_correction.argtypes = [C.c_uint64, C.POINTER(C.c_double)]
    H.nh_events.argtypes = [vp, vp, vp, vp, sz]; H.nh_events.restype = sz
    H.nh_ndt_log.argtypes = [vp, vp, vp, vp, vp, sz]; H.nh_ndt_log.restype = sz
    H.nh_prepared.argtypes = [vp, sz]; H.nh_prepared.restype = sz
    H.nh_fe_count.argtypes = [C.c_char]; H.nh_fe_count.restype = sz
    H.nh_icp_calls.argtypes = [vp, vp, vp, sz]; H.nh_icp_calls.restype = sz
    H.lb_odometry_create.argtypes = [i32, i32, sz, C.c_uint32, C.POINTER(vp)]
    H.lb_odometry_destroy.argtypes = [vp]
    H.lb_odometry_set_registration.argtypes = [vp, i32, C.POINTER(api.NdtParams)]
    H.lb_odometry_set_normals.argtypes = [vp, i32, vp]
    H.lb_odometry_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, u64p]
    H.lb_odometry_next.argtypes = [vp, C.POINTER(api.OdometryResult), i32]
    H.nh_ndt_default_params.argtypes = [C.POINTER(api.NdtParams)]; H.nh_ndt_default_params.restype = None
    H.lb_locus_default_params.argtypes = [C.POINTER(api.LocusParams)]
    H.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
    H.lb_locus_destroy.argtypes = [vp]
    H.lb_locus_set_params.argtypes = [vp, C.POINTER(api.LocusParams)]
    H.lb_locus_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, u64p]
    H.lb_locus_next.argtypes = [vp, C.POINTER(api.LocusResult), i32]
    return H


def _log(nh):
    cap = 4096
    kind = (C.c_char * cap)(); src = np.zeros(cap, np.uint64); tgt = np.zeros(cap, np.uint64)
    is_map = np.zeros(cap, np.int32); g = np.zeros((cap, 16), np.float32)
    n = nh.nh_ndt_log(kind, src.ctypes.data, tgt.ctypes.data, is_map.ctypes.data, g.ctypes.data, cap)
    assert n <= cap
    return [(kind[i].decode(), int(src[i]), int(tgt[i]), int(is_map[i]), g[i].reshape(4, 4).copy()) for i in range(n)]


def _prepared(nh):
    ids = np.zeros(4096, np.uint64)
    n = nh.nh_prepared(ids.ctypes.data, 4096)
    return [int(x) for x in ids[:n]]


def _ndt_params(nh, **kw):
    p = api.NdtParams()
    nh.nh_ndt_default_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


# ------------------------------------------------------------------------------------------------- lb_odometry
def _odometry(nh, depth, method=NDT, ndt=None):
    h = C.c_void_p()
    assert nh.lb_odometry_create(0, depth, NPTS, STEP, C.byref(h)) == 0
    if method is not None:
        assert nh.lb_odometry_set_registration(h, method, C.byref(ndt or _ndt_params(nh, max_iterations=17))) == 0
    return h


def _odo_run(nh, h, ids, incs, flags=None):
    fa = _fields()
    scans = [_scan(i, (flags or {}).get(i, 0)) for i in ids]
    t = C.c_uint64(0)
    for k, s in enumerate(scans):
        g = np.ascontiguousarray(incs[k], np.float32).reshape(16)
        assert nh.lb_odometry_submit(h, s.ctypes.data_as(C.c_void_p), NPTS, STEP, fa, 3, 0, g.ctypes.data_as(C.c_void_p),
                                     None, 0, C.byref(t)) == 0
    out = []
    for _ in scans:
        r = api.OdometryResult()
        assert nh.lb_odometry_next(h, C.byref(r), 1) == 0
        out.append(r)
    return out


@pytest.mark.parametrize("depth", [1, 4])
def test_odometry_ndt_registers_k_against_k_minus_1(nh, depth):
    nh.nh_reset()
    n = 24
    incs = _increments(n, 11)
    h = _odometry(nh, depth)
    res = _odo_run(nh, h, [ID0 + k for k in range(n)], incs)
    assert nh.lb_odometry_destroy(h) == 0
    log = _log(nh)
    assert not [e for e in log if e[0] == "G"]                         # no GICP align
    assert _prepared(nh) == []                                           # nothing to share outside lb_locus
    aligns = sorted((e for e in log if e[0] == "A"), key=lambda e: e[1])
    assert [(e[1], e[2], e[3]) for e in aligns] == [(ID0 + k, ID0 + k - 1, 0) for k in range(1, n)]
    for k, r in enumerate(res):
        assert r.ticket == k and r.status == 0
        if k == 0:
            assert r.has_pose == 0 and bytes(r.ndt) == bytes(api.NdtResult())
            continue
        assert r.has_pose == 1
        np.testing.assert_array_equal(aligns[k - 1][4], incs[k])        # the prior is the guess
        F = np.array(r.ndt.final_transformation, np.float32).reshape(4, 4)
        assert np.array_equal(F, incs[k])
        assert (r.ndt.nr_iterations, r.ndt.converged, r.ndt.n_evaluations) == (17, 1, 3 + (ID0 + k) % 7)
        assert r.ndt.n_target_voxels == ID0 + k - 1 and r.ndt.trans_probability == ID0 + k + 0.25
        # gicp carries the pose, converged, iterations and status only
        want = api.GicpResult()
        want.final_transformation[:] = list(r.ndt.final_transformation)
        want.converged, want.iterations, want.status = 1, 17, 0
        assert bytes(r.gicp) == bytes(want)


def test_odometry_ndt_failure_changes_nothing(nh):
    nh.nh_reset()
    n = 12
    incs = _increments(n, 12)
    h = _odometry(nh, 3)
    res = _odo_run(nh, h, [ID0 + k for k in range(n)], incs, flags={ID0 + 4: 2, ID0 + 7: 1})
    assert nh.lb_odometry_destroy(h) == 0
    assert res[4].status != 0 and res[4].has_pose == 0 and b"NDT align failure" in res[4].error
    assert bytes(res[4].ndt) == bytes(api.NdtResult())
    assert res[5].status == 0 and res[5].has_pose == 1                  # scan 4's filtered cloud is still a target
    assert res[7].status != 0 and res[8].status == 0 and res[8].has_pose == 0     # no target after a failed VoxelGrid
    assert res[9].has_pose == 1


def test_odometry_registration_refusals(nh):
    nh.nh_reset()
    h = _odometry(nh, 2, method=None)
    good = _ndt_params(nh)
    # NDT + normals, in either order
    assert nh.lb_odometry_set_normals(h, 20, None) == 0
    assert nh.lb_odometry_set_registration(h, NDT, C.byref(good)) == -9
    assert nh.lb_odometry_set_normals(h, 0, None) == 0
    assert nh.lb_odometry_set_registration(h, NDT, C.byref(good)) == 0
    assert nh.lb_odometry_set_normals(h, 20, None) == -9
    # invalid params, an unknown method, NDT without params
    for bad in (dict(resolution=0.0), dict(min_points_per_voxel=2), dict(outlier_ratio=1.0), dict(transformation_epsilon=0.0)):
        assert nh.lb_odometry_set_registration(h, NDT, C.byref(_ndt_params(nh, **bad))) == -1, bad
    assert nh.lb_odometry_set_registration(h, NDT, C.byref(_ndt_params(nh, search_method=4))) == -9
    assert nh.lb_odometry_set_registration(h, 2, C.byref(good)) == -1
    assert nh.lb_odometry_set_registration(h, NDT, None) == -1
    # the previous settings stay: NDT with max_iterations 35, normals off
    res = _odo_run(nh, h, [ID0, ID0 + 1, ID0 + 2], _increments(3, 1))
    assert [r.ndt.nr_iterations for r in res] == [0, 35, 35] and nh.nh_fe_count(b"N") == 0
    assert not [e for e in _log(nh) if e[0] == "G"]
    # the method is fixed once a scan was submitted; the params may still change while idle
    assert nh.lb_odometry_set_registration(h, GICP, None) == -9
    assert nh.lb_odometry_set_registration(h, NDT, C.byref(_ndt_params(nh, max_iterations=9))) == 0
    res = _odo_run(nh, h, [ID0 + 3], _increments(1, 2))
    assert res[0].ndt.nr_iterations == 9
    assert nh.lb_odometry_destroy(h) == 0
    assert nh.nh_ndt_alive() == 0


# ------------------------------------------------------------------------------------------------- lb_locus
def _locus_params(nh, odo, loc, **kw):
    p = api.LocusParams()
    assert nh.lb_locus_default_params(C.byref(p)) == 0
    p.odometry_method, p.localization_method = odo, loc
    for k, v in kw.items():
        if isinstance(v, dict):
            for kk, vv in v.items():
                setattr(getattr(p, k), kk, vv)
        elif k == "initial_pose":
            p.initial_pose[:] = [float(x) for x in np.asarray(v).reshape(16)]
        else:
            setattr(p, k, v)
    return p


def _locus_run(nh, n, odo, loc, depth=2, flags=None, incs=None, corr=None, map_n=0, **params):
    flags = flags or {}
    incs = incs if incs is not None else _increments(n, 3)
    corr = corr or {}
    nh.nh_reset()
    for k, Cm in corr.items():
        nh.nh_set_correction(ID0 + k, _dp(_d(Cm)))
    m = nh.nh_submap_create(0, map_n)
    h = C.c_void_p()
    assert nh.lb_locus_create(0, depth, NPTS, STEP, m, C.byref(h)) == 0
    P = _locus_params(nh, odo, loc, **params)
    assert nh.lb_locus_set_params(h, C.byref(P)) == 0
    fa = _fields()
    scans = [_scan(ID0 + k, flags.get(k, 0)) for k in range(n)]
    t = C.c_uint64(0)
    for k in range(n):
        g = np.ascontiguousarray(incs[k], dtype=np.float32).reshape(16)
        assert nh.lb_locus_submit(h, scans[k].ctypes.data_as(C.c_void_p), NPTS, STEP, fa, 3, 0, g.ctypes.data_as(C.c_void_p),
                                  None, 0, C.byref(t)) == 0
    res = []
    for _ in range(n):
        r = api.LocusResult()
        assert nh.lb_locus_next(h, C.byref(r), 1) == 0
        res.append(r)
    assert nh.lb_locus_destroy(h) == 0
    nh.nh_submap_destroy(m)
    assert nh.nh_clouds_alive() == 0 and nh.nh_ndt_alive() == 0
    cap = 4 * n + 8
    kind = np.zeros(cap, np.int32); ids = np.zeros(cap, np.uint64); v = np.zeros((cap, 16)); cnt = np.zeros(cap, np.uint64)
    ne = nh.nh_events(kind.ctypes.data, ids.ctypes.data, v.ctypes.data, cnt.ctypes.data, cap)
    events = [(int(kind[i]), int(ids[i]), v[i].copy(), int(cnt[i])) for i in range(ne)]
    return res, events, P, incs


def _replay(res, P, corr, map_n=0, fail_loc=()):
    """LocusChain with the fakes' outputs; returns its records, the map calls and the localization guesses per scan"""
    chain = LO.LocusChain(P)
    calls, guesses, recs = [], {}, []
    size = [map_n]
    for k, r in enumerate(res):
        def localize(G, k=k):
            guesses[k] = G
            if k in fail_loc:
                return None
            return _fake_align(G, corr.get(k, np.eye(4)))

        def insert(T, k=k):
            calls.append((1, ID0 + k, T.reshape(16).astype(np.float64), NPTS))
            size[0] += NPTS
            return NPTS

        def crop(c, half):
            rm = size[0] // 2
            calls.append((2, 0, np.array([c[0], c[1], c[2], np.float32(half)] + [0.0] * 12), rm))
            size[0] -= rm
            return rm

        ok = r.status == 0 or k in fail_loc
        odo = np.array(r.odometry.final_transformation, np.float32).reshape(4, 4) if r.has_odometry else None
        recs.append(chain.scan(ok, odo, localize, insert, crop))
        recs[-1]["map_size"] = size[0]
    return recs, calls, guesses


def _check(res, recs, events, calls):
    for k, (r, e) in enumerate(zip(res, recs)):
        assert r.ticket == k
        for f in ("odometry_accepted", "has_localization", "correction_accepted", "keyframe", "n_inserted", "n_removed", "map_size"):
            assert getattr(r, f) == e[f], (k, f, getattr(r, f), e[f])
        assert _same(r.odometry_pose, e["O"]) and _same(r.incremental, e["I"]) and _same(r.pose, e["L"]), k
    assert len(events) == len(calls)
    for a, b in zip(events, calls):
        assert a[0] == b[0] and a[1] == b[1] and a[3] == b[3] and _same(a[2], b[2])


@pytest.mark.parametrize("depth", [1, 4])
@pytest.mark.parametrize("odo,loc", [(NDT, GICP), (GICP, NDT), (NDT, NDT)])
def test_locus_ndt_equals_oracle(nh, odo, loc, depth):
    n = 40
    incs = _increments(n, 5, big=(10,))
    corr = _corrections(n, 6, big=(15,))
    init = _pose(_rot([0, 0, 1], 0.3), [1.0, -2.0, 0.5])
    res, events, P, _ = _locus_run(nh, n, odo, loc, depth=depth, incs=incs, corr=corr, refresh_every=2, window_half_size=7.5,
                                   initial_pose=init)
    assert all(r.status == 0 for r in res)
    recs, calls, guesses = _replay(res, P, corr)
    _check(res, recs, events, calls)
    assert sum(r.keyframe for r in res) >= 6 and any(r.n_removed for r in res)
    log = _log(nh)
    scan_aligns = sorted(((e[1], e[2], e[4]) for e in log if e[0] in "AG" and not e[3] and (e[0] == "A") == (odo == NDT)))
    assert [(s, t) for s, t, _ in scan_aligns] == [(ID0 + k, ID0 + k - 1) for k in range(1, n)]
    for s, _, g in scan_aligns:
        assert np.array_equal(g, incs[s - ID0])                           # the prior is the odometry guess
    # the other method makes no scan-to-scan align; every scan's GICP cloud is still prepared for stage L
    assert not [e for e in log if not e[3] and e[0] in "AG" and (e[0] == "A") != (odo == NDT)]
    assert sorted(_prepared(nh)) == [ID0 + k for k in range(n)]
    # localization: only the chosen method aligns against the map, with the guess P of LocusChain
    map_aligns = [e for e in log if e[3] and e[0] in "AG"]
    assert {e[0] for e in map_aligns} == {"A" if loc == NDT else "G"}
    assert [e[1] - ID0 for e in map_aligns] == sorted(guesses)
    for e in map_aligns:
        assert np.array_equal(e[4], guesses[e[1] - ID0])
    if loc == NDT:
        kinds = [e[0] for e in log if e[3] and e[0] in "MA"]
        assert kinds == ["M", "A"] * len(map_aligns)                     # the submap target before every align
        assert not [e for e in log if e[0] == "g"]                       # no GICP index of the map without the covariance
    zero = bytes(api.NdtResult())
    for r in res:
        for method, has, g, nd in ((odo, r.has_odometry, r.odometry, r.odometry_ndt),
                                   (loc, r.has_localization, r.localization, r.localization_ndt)):
            if method == GICP or not has:
                assert bytes(nd) == zero
                continue
            assert nd.nr_iterations == 20 and nd.converged == 1
            assert list(g.final_transformation) == list(nd.final_transformation) and g.iterations == 20
            assert g.n_correspondences == 0 and g.delta == 0.0 and g.n_objective_evals == 0


def test_locus_ndt_localization_icp_covariance(nh):
    n = 16
    corr = _corrections(n, 7)
    res, events, P, _ = _locus_run(nh, n, GICP, NDT, corr=corr, icp_covariance={"enabled": 1, "max_covariance": 0.01})
    recs, calls, _ = _replay(res, P, corr)
    _check(res, recs, [e for e in events if e[0] != 4], calls)          # kind 4: the covariance calls, checked below
    ids = np.zeros(64, np.uint64); T = np.zeros((64, 16), np.float32); is_map = np.zeros(64, np.int32)
    m = nh.nh_icp_calls(ids.ctypes.data, T.ctypes.data, is_map.ctypes.data, 64)
    loc = [k for k in range(n) if res[k].has_localization]
    assert [int(i) - ID0 for i in ids[:m]] == loc and all(is_map[:m] == 1)
    for j, k in enumerate(loc):
        assert np.array_equal(T[j], np.array(res[k].localization_ndt.final_transformation, np.float32))   # the NDT pose
        assert res[k].has_icp_covariance == 1
    kinds = [e[0] for e in _log(nh) if e[3] and e[0] in "MAg"]
    assert kinds == ["M", "A", "g"] * len(loc)                           # the map as GICP target for the 1-NN, after the align


def test_locus_ndt_failures_change_no_state(nh):
    n = 28
    flags = {5: 1, 12: 2, 20: 4}
    corr = _corrections(n, 8)
    res, events, P, _ = _locus_run(nh, n, NDT, NDT, depth=3, flags=flags, corr=corr)
    recs, calls, _ = _replay(res, P, corr, fail_loc=(20,))
    _check(res, recs, events, calls)
    for k in (5, 12, 20):
        assert res[k].status != 0 and res[k].error and res[k].has_localization == 0 and res[k].keyframe == 0
        assert _same(res[k].pose, res[k - 1].pose)
    assert res[6].has_odometry == 0 and res[13].has_odometry == 1 and res[21].has_localization == 1
    assert not _same(res[20].odometry_pose, res[19].odometry_pose)       # odometry itself succeeded


def test_locus_registration_refusals(nh):
    nh.nh_reset()
    m = nh.nh_submap_create(0, 0)
    h = C.c_void_p()
    assert nh.lb_locus_create(0, 2, NPTS, STEP, m, C.byref(h)) == 0
    # invalid NDT params are refused only where the method is NDT
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, GICP, GICP, localization_ndt={"resolution": 0.0}))) == 0
    for bad in (dict(localization_ndt={"resolution": 0.0}), dict(odometry_ndt={"min_points_per_voxel": 1}),
                dict(localization_ndt={"step_size": -1.0})):
        assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, NDT, NDT, **bad))) == -1, bad
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, 2, GICP))) == -1
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, GICP, 2))) == -1
    # normals stay allowed under lb_locus: the shared GICP cloud carries them
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, NDT, GICP, front_end={"normals_k": 20}))) == 0
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, NDT, GICP))) == 0
    fa = _fields()
    t = C.c_uint64(0)
    s = [_scan(ID0 + k) for k in range(3)]
    r = api.LocusResult()
    assert nh.lb_locus_submit(h, s[0].ctypes.data_as(C.c_void_p), NPTS, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0
    assert nh.lb_locus_next(h, C.byref(r), 1) == 0 and r.status == 0
    # after the first scan: a method change is refused and the previous methods stay
    for odo, loc in ((GICP, GICP), (NDT, NDT), (GICP, NDT)):
        assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, odo, loc))) == -9
    assert nh.lb_locus_set_params(h, C.byref(_locus_params(nh, NDT, GICP, odometry_ndt={"max_iterations": 7}))) == 0
    for k in (1, 2):
        assert nh.lb_locus_submit(h, s[k].ctypes.data_as(C.c_void_p), NPTS, STEP, fa, 3, 0, None, None, 0, C.byref(t)) == 0
        assert nh.lb_locus_next(h, C.byref(r), 1) == 0 and r.status == 0
        assert r.odometry_ndt.nr_iterations == 7 and r.has_localization == 1 and r.localization_ndt.nr_iterations == 0
    log = _log(nh)
    assert [e[0] for e in log if e[0] in "AG"] == ["A", "G", "A", "G"]
    assert nh.lb_locus_destroy(h) == 0
    nh.nh_submap_destroy(m)


def test_default_registration_is_gicp():
    import locus_b200
    p = locus_b200.locus_params()
    assert (p.odometry_method, p.localization_method) == (GICP, GICP)
    o, lo_ = p.odometry_ndt, p.localization_ndt
    assert (o.transformation_epsilon, o.max_iterations) == (0.001, 20)
    assert (lo_.transformation_epsilon, lo_.max_iterations) == (0.00001, 20)
    for q in (o, lo_):
        assert (q.resolution, q.step_size, q.outlier_ratio, q.min_points_per_voxel, q.search_method) == (1.0, 0.1, 0.55, 6, 0)
    p = locus_b200.locus_params(odometry_method="ndt", localization_method="ndt", localization_ndt={"resolution": 2.0})
    assert (p.odometry_method, p.localization_method, p.localization_ndt.resolution) == (NDT, NDT, 2.0)


# ------------------------------------------------------------------------------------------------- layout
def test_struct_layout_matches_ctypes():
    exe = _build("ndt_layout_probe", "tests/ndt_layout_probe.c", ["include/locus_b200.h"],
                 ["gcc", "-std=c99", "-O0", "-I", os.path.join(ROOT, "include")])
    out = subprocess.run([exe], stdout=subprocess.PIPE, text=True, check=True).stdout.split("\n")
    got = dict(line.split() for line in out if line)
    mirrors = {"lb_ndt_params": api.NdtParams, "lb_ndt_result": api.NdtResult, "lb_odometry_result": api.OdometryResult,
               "lb_locus_params": api.LocusParams, "lb_locus_result": api.LocusResult}
    seen = 0
    for key, v in got.items():
        name, _, field = key.partition(".")
        M = mirrors[name]
        want = getattr(M, field).offset if field else C.sizeof(M)
        assert int(v) == want, (key, v, want)
        seen += 1
    # every field of the three changed structs is probed
    assert seen == 2 + sum(1 + len(mirrors[s]._fields_) for s in ("lb_odometry_result", "lb_locus_params", "lb_locus_result"))
