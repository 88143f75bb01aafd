"""lb_locus_* without a GPU.

* lo_pose.h (the chain's pose bookkeeping), built into a g++ harness with the library's host flags, is bit-equal to
  oracle/locus_oracle.py's pure-Python restatement: random poses, both quaternion branches, values exactly at every
  threshold.
* The chain's host logic (locus_b200/csrc/odometry.cu: the pipeline core plus the localization stage), built against
  fake stages (tests/locus_stub.h), reports exactly what oracle.locus_oracle.LocusChain computes from the same stage
  outputs: order, first-scan insert, prior map, keyframe and crop cadence, discarded odometry increments, rejected
  corrections, failed stages, add_keyframes = 0, destroy with scans in flight and the parameter refusals.
The GPU twin is test_locus_gpu.py."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from locus_b200 import api
from oracle import locus_oracle as LO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP = 16
NPTS = 8
D16 = C.c_double * 16


def _build(name, src, deps, flags):
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    so = os.path.join(bdir, name)
    srcs = [os.path.join(ROOT, p) for p in [src] + deps]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off"] + flags +
                              ["-x", "c++", srcs[0], "-I", os.path.join(ROOT, "tests"), "-o", so])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def lp():
    H = _build("liblo_pose_harness.so", "tests/lo_pose_harness.cpp", ["locus_b200/csrc/lo_pose.h"], ["-O2"])
    dp, fp, d = C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_double
    for f in ("lp_update", "lp_delta"):
        getattr(H, f).argtypes = [dp, dp, dp]
    H.lp_from_float.argtypes = [fp, dp]
    H.lp_to_float.argtypes = [dp, fp]
    H.lp_euler.argtypes = [dp, dp]
    for f in ("lp_euler_norm", "lp_translation_norm", "lp_quat_w", "lp_keyframe_angle"):
        getattr(H, f).argtypes = [dp]
        getattr(H, f).restype = d
    H.lp_passes.argtypes = [dp, C.c_int, d, d]
    H.lp_is_keyframe.argtypes = [dp, d, d]
    return H


@pytest.fixture(scope="module")
def lh():
    return _load_harness()


def _load_harness():
    H = _build("liblocus_harness.so", "tests/locus_harness.cpp",
               ["tests/locus_stub.h", "locus_b200/csrc/odometry.cu", "locus_b200/csrc/lo_pose.h", "include/locus_b200.h"], ["-O1"])
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    H.lh_submap_create.argtypes = [i32, sz]; H.lh_submap_create.restype = vp
    H.lh_submap_destroy.argtypes = [vp]
    H.lh_set_correction.argtypes = [C.c_uint64, C.POINTER(C.c_double)]
    H.lh_events.argtypes = [vp, vp, vp, vp, sz]; H.lh_events.restype = sz
    H.lb_locus_default_params.argtypes = [C.POINTER(api.LocusParams)]
    H.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
    H.lb_locus_destroy.argtypes = [vp]
    H.lb_locus_set_params.argtypes = [vp, C.POINTER(api.LocusParams)]
    H.lb_locus_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, C.POINTER(C.c_uint64)]
    H.lb_locus_next.argtypes = [vp, C.POINTER(api.LocusResult), i32]
    H.lb_locus_pending.argtypes = [vp, C.POINTER(sz)]
    H.lb_locus_stage_times.argtypes = [vp, C.POINTER(C.c_double)]
    return H


# ------------------------------------------------------------------------------------------------- lo_pose.h
def _rot(axis, angle):
    a = np.asarray(axis, float)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K)


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def _random_poses(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        ang = rng.uniform(0, math.pi) if i % 3 else rng.uniform(0, 0.3)
        out.append(_pose(_rot(rng.normal(size=3), ang), rng.normal(size=3) * (0.2 if i % 2 else 3.0)))
    # large angles and exact special cases: both branches of Eigen's quaternion, each choice of its index i
    for axis in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0.2, -1, 0.7]):
        for ang in (math.pi, 2.5, 2 * math.pi / 3, 2.0, 1e-9, 0.0):
            out.append(_pose(_rot(axis, ang), [0.5, -0.25, 1.0]))
    out.append(_pose(np.diag([1.0, -1.0, -1.0]), [0, 0, 0]))
    out.append(_pose(np.diag([-1.0, 1.0, -1.0]), [0, 0, 0]))
    out.append(_pose(np.diag([-1.0, -1.0, 1.0]), [0, 0, 0]))
    out.append(_pose(np.diag([1.0000001, 1.0, 1.0]), [0, 0, 0]))     # acos / asin argument outside [-1, 1]: NaN
    out.append(_pose(_rot([0, 1, 0], math.pi / 2) * 1.0000001, [0, 0, 0]))
    return out


def _d(a):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(16))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _same(a, b):
    a = np.asarray(a, np.float64).reshape(-1); b = np.asarray(b, np.float64).reshape(-1)
    return a.view(np.uint64).tolist() == b.view(np.uint64).tolist()


def _same_scalar(a, b):
    return np.float64(a).view(np.uint64) == np.float64(b).view(np.uint64)


def test_pose_math_bit_equal_to_oracle(lp):
    poses = _random_poses(120, 1)
    branches = set()
    for a, b in zip(poses, poses[1:] + poses[:1]):
        A, B = _d(a), _d(b)
        pa, pb = LO.from_mat(A), LO.from_mat(B)
        out = np.zeros(16)
        lp.lp_update(_dp(A), _dp(B), _dp(out))
        assert _same(out, LO.to_mat(LO.update(pa, pb)))
        lp.lp_delta(_dp(A), _dp(B), _dp(out))
        assert _same(out, LO.to_mat(LO.delta(pa, pb)))
        rpy = np.zeros(3)
        lp.lp_euler(_dp(A), _dp(rpy))
        assert _same(rpy, LO.euler_zyx(pa))
        assert _same_scalar(lp.lp_euler_norm(_dp(A)), LO.euler_norm(pa))
        assert _same_scalar(lp.lp_translation_norm(_dp(A)), LO.translation_norm(pa))
        assert _same_scalar(lp.lp_quat_w(_dp(A)), LO.quat_w(pa))
        assert _same_scalar(lp.lp_keyframe_angle(_dp(A)), LO.keyframe_angle(pa))
        branches.add(LO.sum3(pa.R[0], pa.R[4], pa.R[8]) > 0.0)
        # float(P) and double(float) conversions
        f = np.zeros(16, np.float32)
        lp.lp_to_float(_dp(A), f.ctypes.data_as(C.POINTER(C.c_float)))
        assert np.array_equal(f.view(np.uint32), LO.to_mat(pa, np.float32).view(np.uint32))
        lp.lp_from_float(f.ctypes.data_as(C.POINTER(C.c_float)), _dp(out))
        assert _same(out, LO.to_mat(LO.from_mat(f)))
    assert branches == {True, False}
    # in the trace <= 0 branch Eigen makes the largest-diagonal component positive, so w < 0 when that axis component
    # is negative: 2 acos(w) > pi
    A = _d(_pose(_rot([-1, 0.2, 0.1], 2.5), [0, 0, 0]))
    assert LO.quat_w(LO.from_mat(A)) < 0 and _same_scalar(lp.lp_quat_w(_dp(A)), LO.quat_w(LO.from_mat(A)))


def test_thresholds_exactly_at_the_limit(lp):
    for T in _random_poses(30, 7)[:30]:
        A = _d(T)
        p = LO.from_mat(A)
        tn, rn, ang = LO.translation_norm(p), LO.euler_norm(p), LO.keyframe_angle(p)
        below = lambda x: math.nextafter(x, -math.inf)   # noqa: E731
        for enabled in (0, 1):
            for mt, mr in ((tn, rn), (below(tn), rn), (tn, below(rn)), (below(tn), below(rn))):
                want = LO.passes(p, enabled, mt, mr)
                assert bool(lp.lp_passes(_dp(A), enabled, mt, mr)) == want
                if enabled:
                    assert want == (mt == tn and mr == rn)        # <= at the limit passes, one ulp below fails
        for tk, rk in ((tn, ang), (below(tn), ang), (tn, below(ang)), (math.inf, math.inf)):
            want = LO.is_keyframe(p, tk, rk)
            assert bool(lp.lp_is_keyframe(_dp(A), tk, rk)) == want
            assert want == (tk < tn or rk < ang)                   # > : exactly at the limit is no keyframe


# ------------------------------------------------------------------------------------------------- the chain
def _scan(i, flags=0):
    b = np.zeros(NPTS * STEP, dtype=np.uint8)
    b[:8] = np.frombuffer(np.uint64(i).tobytes(), dtype=np.uint8)
    b[8:12] = np.frombuffer(np.uint32(flags).tobytes(), dtype=np.uint8)
    return b


def _fields():
    return api.VoxelGridB200._fields([("x", 0, api.LB_FLOAT32, 1), ("y", 4, api.LB_FLOAT32, 1), ("z", 8, api.LB_FLOAT32, 1)])


def _params(lh, **kw):
    p = api.LocusParams()
    assert lh.lb_locus_default_params(C.byref(p)) == 0
    for k, v in kw.items():
        if isinstance(v, dict):
            for kk, vv in v.items():
                setattr(getattr(p, k), kk, vv)
        elif k == "initial_pose":
            p.initial_pose[:] = [float(x) for x in np.asarray(v).reshape(16)]
        else:
            setattr(p, k, v)
    return p


def _increments(n, seed, big=()):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        t = rng.uniform(-0.35, 0.35, 3) if k not in big else np.array([3.0, 0.0, 0.0])
        out.append(_pose(_rot(rng.normal(size=3), rng.uniform(0, 0.08)), t).astype(np.float32))
    return out


def _corrections(n, seed, big=()):
    rng = np.random.default_rng(seed)
    out = {}
    for k in range(n):
        if k in big:
            out[k] = _pose(np.eye(3), [2.0, 0.0, 0.0])
        elif k % 3:
            out[k] = _pose(_rot(rng.normal(size=3), rng.uniform(0, 0.01)), rng.uniform(-0.02, 0.02, 3))
    return out


def _fake_align(G, Cm):
    """what the stub's localization align computes: float(guess * C), double sums in k order"""
    F = np.zeros(16, np.float32)
    g = [float(x) for x in np.asarray(G, np.float32).reshape(16)]
    c = [float(x) for x in np.asarray(Cm, np.float64).reshape(16)]
    for r in range(4):
        for col in range(4):
            s = 0.0
            for k in range(4):
                s += g[4 * r + k] * c[4 * k + col]
            F[4 * r + col] = s
    return F.reshape(4, 4)


def _run(lh, n, depth=2, flags=None, incs=None, corr=None, map_n=0, map_device=0, id0=100, destroy_early=False, **params):
    flags = flags or {}
    incs = incs if incs is not None else _increments(n, 3)
    corr = corr or {}
    lh.lh_reset()
    for k, Cm in corr.items():
        lh.lh_set_correction(id0 + k, _dp(_d(Cm)))
    m = lh.lh_submap_create(map_device, map_n)
    h = C.c_void_p()
    st = lh.lb_locus_create(0, depth, NPTS, STEP, m, C.byref(h))
    if st != 0:
        lh.lh_submap_destroy(m)
        return st, None, None, None
    P = _params(lh, **params)
    assert lh.lb_locus_set_params(h, C.byref(P)) == 0
    fa = _fields()
    scans = [_scan(id0 + k, flags.get(k, 0)) for k in range(n)]
    res = []
    t = C.c_uint64(0)
    for k in range(n):
        g = np.ascontiguousarray(incs[k], dtype=np.float32).reshape(16)
        assert lh.lb_locus_submit(h, scans[k].ctypes.data_as(C.c_void_p), NPTS, STEP, fa, 3, 0, g.ctypes.data_as(C.c_void_p),
                                  None, 0, C.byref(t)) == 0
        assert t.value == k
        while not destroy_early:
            r = api.LocusResult()
            s = lh.lb_locus_next(h, C.byref(r), 0)
            if s != 0:
                assert s in (1, -10)
                break
            res.append(r)
    if destroy_early:
        assert lh.lb_locus_destroy(h) == 0
        lh.lh_submap_destroy(m)
        return 0, res, None, P
    while len(res) < n:
        r = api.LocusResult()
        assert lh.lb_locus_next(h, C.byref(r), 1) == 0
        res.append(r)
    pend = C.c_size_t(9)
    assert lh.lb_locus_pending(h, C.byref(pend)) == 0 and pend.value == 0
    times = (C.c_double * 9)()
    assert lh.lb_locus_stage_times(h, times) == 0 and times[6] == n
    assert lh.lb_locus_destroy(h) == 0
    lh.lh_submap_destroy(m)
    cap = 4 * n + 8
    kind = np.zeros(cap, np.int32); ids = np.zeros(cap, np.uint64); v = np.zeros((cap, 16)); cnt = np.zeros(cap, np.uint64)
    ne = lh.lh_events(kind.ctypes.data, ids.ctypes.data, v.ctypes.data, cnt.ctypes.data, cap)
    events = [(int(kind[i]), int(ids[i]), v[i].copy(), int(cnt[i])) for i in range(ne)]
    return 0, res, events, P


def _replay(res, P, corr, map_n, id0=100, fail_loc=()):
    """oracle.LocusChain fed with the same stage outputs; returns its records and the map calls it makes"""
    chain = LO.LocusChain(P)
    calls = []
    size = [map_n]
    recs = []
    for k, r in enumerate(res):
        def localize(G, k=k):
            if k in fail_loc:
                return None
            F = _fake_align(G, corr.get(k, np.eye(4)))
            assert np.array_equal(np.array(r.localization.final_transformation, np.float32).reshape(4, 4), F)
            return F

        def insert(T, k=k):
            calls.append((1, id0 + k, T.reshape(16).astype(np.float64), NPTS))
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
    return recs, calls


def _check(res, recs, events, calls):
    for k, (r, e) in enumerate(zip(res, recs)):
        assert r.ticket == k
        for f in ("odometry_accepted", "has_localization", "correction_accepted", "keyframe", "n_inserted", "n_removed", "map_size"):
            assert getattr(r, f) == e[f], (k, f, getattr(r, f), e[f])
        assert _same(r.odometry_pose, e["O"]), k
        assert _same(r.incremental, e["I"]), k
        assert _same(r.pose, e["L"]), k
    assert len(events) == len(calls)
    for a, b in zip(events, calls):
        assert a[0] == b[0] and a[1] == b[1] and a[3] == b[3] and _same(a[2], b[2])


@pytest.mark.parametrize("depth", [1, 2, 4])
def test_chain_equals_oracle(lh, depth):
    n = 48
    incs = _increments(n, 5, big=(10,))
    corr = _corrections(n, 6, big=(15,))
    init = _pose(_rot([0, 0, 1], 0.3), [1.0, -2.0, 0.5])
    st, res, events, P = _run(lh, n, depth=depth, incs=incs, corr=corr, refresh_every=2, window_half_size=7.5,
                              initial_pose=init)
    assert st == 0
    recs, calls = _replay(res, P, corr, 0)
    _check(res, recs, events, calls)
    assert all(r.status == 0 for r in res)
    # the first scan seeds the map at the initial pose, without localization
    assert res[0].keyframe == 1 and res[0].has_localization == 0 and res[0].has_odometry == 0
    assert events[0][0] == 1 and events[0][1] == 100 and _same(events[0][2], init.astype(np.float32).reshape(16).astype(np.float64))
    # keyframes and the crop cadence: every second keyframe after the first scan crops around L
    kf = [k for k in range(1, n) if res[k].keyframe]
    crops = [k for k in range(n) if res[k].n_removed]
    assert len(kf) >= 6 and crops == kf[1::2]
    for k in crops:
        ev = [e for e in events if e[0] == 2]
        assert any(_same(e[2][:3], np.array(res[k].pose, np.float64).reshape(4, 4)[:3, 3].astype(np.float32).astype(np.float64)) for e in ev)
    # a discarded odometry increment: O stays, but the prediction (and so L) still moves by it
    assert res[10].has_odometry and not res[10].odometry_accepted
    O9, O10 = (np.array(res[k].odometry_pose).reshape(4, 4) for k in (9, 10))
    L9, L10 = (np.array(res[k].pose).reshape(4, 4) for k in (9, 10))
    assert np.array_equal(O9, O10)
    assert np.linalg.norm(L10[:3, 3] - L9[:3, 3]) > 2.5
    # a rejected localization correction: L = L_prev * I exactly
    assert res[15].has_localization and not res[15].correction_accepted
    L14 = LO.from_mat(np.array(res[14].pose))
    assert _same(res[15].pose, LO.to_mat(LO.update(L14, LO.from_mat(np.array(res[15].incremental)))))
    assert sum(r.correction_accepted for r in res) >= n - 3


def test_failed_stages_leave_the_state_unchanged(lh):
    n = 30
    flags = {5: 1, 12: 2, 20: 4, 0: 0}
    corr = _corrections(n, 8)
    st, res, events, P = _run(lh, n, depth=3, flags=flags, corr=corr)
    assert st == 0
    recs, calls = _replay(res, P, corr, 0, fail_loc=(20,))
    _check(res, recs, events, calls)
    for k in (5, 12):
        assert res[k].status != 0 and res[k].error
        assert res[k].has_localization == 0 and res[k].keyframe == 0
        for f in ("odometry_pose", "pose"):
            assert _same(getattr(res[k], f), getattr(res[k - 1], f))
        # after a failed VoxelGrid the next scan has no odometry target; a failed align still leaves its prepared cloud
        assert res[k + 1].status == 0 and res[k + 1].has_odometry == (k == 12)
        assert res[k + 1].has_localization == 1
    assert res[20].status != 0 and res[20].has_localization == 0 and _same(res[20].pose, res[19].pose)
    assert not _same(res[20].odometry_pose, res[19].odometry_pose)              # odometry itself succeeded


def test_first_scan_failure_moves_the_map_seed(lh):
    st, res, events, P = _run(lh, 6, flags={0: 1})
    assert res[0].status != 0 and res[0].keyframe == 0
    assert res[1].keyframe == 1 and res[1].has_localization == 0 and events[0][1] == 101


def test_prior_map(lh):
    n = 12
    corr = _corrections(n, 9)
    st, res, events, P = _run(lh, n, corr=corr, map_n=500, prior_map=1)
    assert st == 0
    recs, calls = _replay(res, P, corr, 500)
    _check(res, recs, events, calls)
    assert res[0].has_localization == 1 and res[0].has_odometry == 0 and _same(res[0].incremental, np.eye(4))
    assert all(e[1] != 100 for e in events if e[0] == 1) or res[0].keyframe == 1


def test_prior_map_empty_is_reported(lh):
    st, res, events, P = _run(lh, 3, map_n=0, prior_map=1)
    assert res[0].status == -5 and res[0].has_localization == 0


def test_no_keyframes(lh):
    n = 30
    st, res, events, P = _run(lh, n, add_keyframes=0)
    recs, calls = _replay(res, P, {}, 0)
    _check(res, recs, events, calls)
    assert [e[1] for e in events] == [100] and sum(r.keyframe for r in res) == 1 and all(r.has_localization for r in res[1:])


def test_destroy_with_scans_in_flight(lh):
    for depth in (1, 3):
        st, res, _, _ = _run(lh, 20, depth=depth, destroy_early=True)
        assert st == 0
        assert lh.lh_clouds_alive() == 0


def test_parameter_refusals(lh):
    m = lh.lh_submap_create(1, 10)
    h = C.c_void_p()
    assert lh.lb_locus_create(0, 2, NPTS, STEP, m, C.byref(h)) == -1                 # submap on another device
    lh.lh_submap_destroy(m)
    m = lh.lh_submap_create(0, 10)
    assert lh.lb_locus_create(0, 2, NPTS, STEP, None, C.byref(h)) == -1
    assert lh.lb_locus_create(0, 2, NPTS, STEP, m, C.byref(h)) == 0
    for bad in (dict(odometry={"k_correspondences": 15}), dict(localization={"gicp_epsilon": 1e-4}),
                dict(localization={"index_cell_size": 0.5}), dict(refresh_every=0), dict(window_half_size=0.0)):
        P = _params(lh, **bad)
        assert lh.lb_locus_set_params(h, C.byref(P)) == -1, bad
    same = _params(lh, odometry={"k_correspondences": 15}, localization={"k_correspondences": 15})
    assert lh.lb_locus_set_params(h, C.byref(same)) == 0
    # refused while a scan is in flight, accepted again once it has been returned
    s = _scan(7)
    t = C.c_uint64(0)
    assert lh.lb_locus_submit(h, s.ctypes.data_as(C.c_void_p), NPTS, STEP, _fields(), 3, 0, None, None, 0, C.byref(t)) == 0
    assert lh.lb_locus_set_params(h, C.byref(same)) == -1
    r = api.LocusResult()
    assert lh.lb_locus_next(h, C.byref(r), 1) == 0 and r.status == 0
    assert lh.lb_locus_next(h, C.byref(r), 1) == -10
    assert lh.lb_locus_set_params(h, C.byref(same)) == 0
    assert lh.lb_locus_destroy(h) == 0
    lh.lh_submap_destroy(m)


def test_default_params_are_the_shipped_values():
    import locus_b200
    p = locus_b200.locus_params()
    o, lo_ = p.odometry, p.localization
    assert (o.transformation_epsilon, o.max_correspondence_distance, o.max_iterations) == (0.001, 1.0, 20)
    assert (lo_.transformation_epsilon, lo_.max_correspondence_distance, lo_.max_iterations) == (0.00001, 0.2, 20)
    assert o.align_points_per_cta == 1024 and lo_.align_points_per_cta == 0
    assert o.k_correspondences == lo_.k_correspondences and o.gicp_epsilon == lo_.gicp_epsilon
    for th in (p.odometry_thresholds, p.localization_thresholds):
        assert (th.enabled, th.max_translation, th.max_rotation) == (1, 1.0, 1.0)
    assert (p.translation_threshold_kf, p.rotation_threshold_kf, p.add_keyframes, p.refresh_every, p.msw) == (1.0, 0.3, 1, 1, 1)
    assert p.window_half_size == 20.0 and p.prior_map == 0 and list(p.initial_pose) == list(np.eye(4).reshape(16))


def test_new_symbols_exported():
    import locus_b200
    L = locus_b200.lib()
    new = ["lb_gicp_set_source_cloud", "lb_locus_default_params", "lb_locus_create", "lb_locus_destroy", "lb_locus_voxel",
           "lb_locus_set_params", "lb_locus_submit", "lb_locus_next", "lb_locus_pending", "lb_locus_stage_times"]
    for s in new:
        assert hasattr(L, s) and s in api.SYMBOLS
