"""The localization's ICP covariance without a GPU.

* oracle/icp_cov_oracle.py reproduces the reference's two known answers (test_point_cloud_localization.cpp:398-477):
  one plane -> exactly 0.01 I through the D-NaN fallback; three orthogonal planes rotated 30 deg and offset 1 mm -> 1e-6 I.
* locus_b200/csrc/icp_cov.h, built with g++ and the library's host flags, equals the oracle bit for bit, flags
  included, on a well-conditioned Ap, a D > max clamp, a non-positive LDLT pivot, a singular Ap and an Ap with inf;
  against numpy: the unclamped covariance is 0.0025 inv(Ap), the condition number the ratio of numpy's singular values,
  and a clamp rebuild with the unclamped D gives the pivot-permuted covariance (the reference's step 7 as written).
* stage L of lb_locus (odometry.cu against fake stages, tests/icp_covariance_stub.h): the call comes after every
  localization and before its insert, with F and the float rotation of P^-1; none on an unlocalized first scan, one
  with prior_map; none when disabled; the condition number carries over a fallback scan; set_params refuses a bad
  max_covariance; the defaults leave the feature off.
* tests/icp_covariance_cpp_harness.cpp (the C++ mirror and the PCL shim's member template, instantiated with a 6x6
  type) compiles and links.
The GPU twin is test_icp_covariance_gpu.py."""
import ctypes as C
import itertools
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from locus_b200 import api
from oracle import icp_cov_oracle as IC
from oracle import locus_oracle as LO
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fixtures as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP = 16
NPTS = 8


def _so(name, src, deps, flags):
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    so = os.path.join(bdir, name)
    srcs = [os.path.join(ROOT, p) for p in [src] + deps]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off"] + flags +
                              ["-x", "c++", srcs[0], "-I", os.path.join(ROOT, "tests"), "-o", so])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def ic():
    L = _so("libicp_cov_harness.so", "tests/icp_cov_harness.cpp", ["locus_b200/csrc/icp_cov.h"], ["-O2"])
    L.ic_compute.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]
    return L


def _header(L, Ap, max_cov=0.01):
    Ap = np.ascontiguousarray(Ap, dtype=np.float64).reshape(36)
    cov = np.zeros(36)
    cond = C.c_double(0); flags = C.c_int(-1)
    L.ic_compute(Ap.ctypes.data, max_cov, cov.ctypes.data, C.byref(cond), C.byref(flags))
    return cov.reshape(6, 6), cond.value, flags.value


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


# ------------------------------------------------------------------------------------------ known answers
def _plane_with_normals():
    xyz, _ = F.plane()
    nrm = O.normals_knn(xyz, k=10)[:, :3]           # addNormal(*dummy_cloud, dummy_cloud, 10)
    return O.normalize_pcloud(xyz), nrm             # normalizePCloud keeps the normals (transformPointCloud)


def test_single_plane_is_max_identity():
    xyz, nrm = _plane_with_normals()
    r = IC.icp_covariance(xyz, xyz, nrm, correspondences=np.arange(len(xyz)), max_cov=0.01)
    assert r["flags"] == IC.D_NAN and math.isnan(r["condition_number"])
    assert np.array_equal(r["covariance"], 0.01 * np.eye(6))


def test_three_planes_give_1e6():
    xyz, nrm = _plane_with_normals()
    T1 = np.array([[1, 0, 0, 0], [0, 0, -1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], np.float32)
    T2 = np.array([[0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0], [0, 0, 0, 1]], np.float32)
    pts = np.concatenate([xyz, IC.transform(xyz, T1), IC.transform(xyz, T2)])
    nr = np.concatenate([nrm, IC.rotate_normals(nrm, T1[:3, :3]), IC.rotate_normals(nrm, T2[:3, :3])])
    tf = np.zeros((4, 4), np.float32)
    tf[0, 0] = 0.866; tf[0, 1] = -0.5; tf[1, 0] = 0.5; tf[1, 1] = 0.866; tf[0, 3] = 0.001; tf[3, 3] = 1
    offset = IC.transform(pts, tf)
    r = IC.icp_covariance(offset, pts, nr, correspondences=np.arange(len(pts)), max_cov=0.01)
    assert np.abs(r["covariance"] - 1e-6 * np.eye(6)).max() < 1e-4
    assert r["n_used"] == len(pts)


# ------------------------------------------------------------------------------------------ icp_cov.h vs oracle
def _spd(seed, lo=10.0):
    rng = np.random.default_rng(seed)
    B = rng.normal(size=(6, 6))
    return B @ B.T + lo * np.eye(6)


def _cases():
    rng = np.random.default_rng(7)
    well = _spd(1)
    big_d = _spd(2, lo=0.0) * 1e-3 + np.diag([5e3, 4e3, 0.05, 3e3, 1e3, 2e3])   # small eigenvalues: D > max
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    indefinite = Q @ np.diag([50.0, 40.0, -30.0, 20.0, 10.0, 5.0]) @ Q.T            # a negative pivot in the LDLT
    singular = np.diag([1.0, 2.0, 3.0, 4.0, 5.0, 0.0]); singular[0, 1] = singular[1, 0] = 0.5
    xyz, nrm = _plane_with_normals()
    plane = O.compute_ap(O.normalize_pcloud(xyz), nrm, np.arange(len(xyz)))
    with_inf = _spd(3); with_inf[2, 4] = with_inf[4, 2] = np.inf
    return {"well": well, "big_d": big_d, "indefinite": indefinite, "singular": singular, "plane": plane,
            "with_inf": with_inf}


@pytest.mark.parametrize("name", ["well", "big_d", "indefinite", "singular", "plane", "with_inf"])
def test_header_equals_oracle_bitwise(ic, name):
    Ap = _cases()[name]
    cov_h, cond_h, fl_h = _header(ic, Ap)
    cov_o, cond_o, fl_o = IC.covariance(Ap, 0.01)
    assert fl_h == fl_o
    assert np.array_equal(_bits(cov_h), _bits(cov_o))
    assert _bits(cond_h) == _bits(cond_o) or (math.isnan(cond_h) and math.isnan(cond_o))
    expect = {"well": 0, "big_d": IC.CLAMPED, "indefinite": IC.CLAMPED}
    if name in expect:
        assert fl_h == expect[name]
    elif name == "with_inf":                        # inf rows and columns of the inverse are 0: the clamp rebuilds
        assert fl_h & IC.CLAMPED and np.isfinite(cov_h).all()
    else:                                           # singular: the LU divides by zero -> the D-NaN fallback
        assert fl_h & IC.D_NAN and np.array_equal(cov_h, 0.01 * np.eye(6))


@pytest.mark.parametrize("seed", range(8))
def test_random_spd_bitwise(ic, seed):
    Ap = _spd(100 + seed, lo=float(seed) * 0.1)
    cov_h, cond_h, fl_h = _header(ic, Ap)
    cov_o, cond_o, fl_o = IC.covariance(Ap, 0.01)
    assert fl_h == fl_o and np.array_equal(_bits(cov_h), _bits(cov_o)) and _bits(cond_h) == _bits(cond_o)


def test_unclamped_against_numpy(ic):
    Ap = _cases()["well"]
    cov, cond, fl = _header(ic, Ap)
    assert fl == 0
    ref = 0.0025 * np.linalg.inv(Ap)
    assert np.abs(cov - ref).max() <= 1e-12 * np.abs(ref).max()
    s = np.linalg.svd(cov, compute_uv=False)
    assert abs(cond - s[0] / s[-1]) <= 1e-10 * (s[0] / s[-1])


def test_clamped_condition_number_against_numpy(ic):
    cov, cond, fl = _header(ic, _cases()["big_d"])
    assert fl == IC.CLAMPED
    s = np.linalg.svd(cov, compute_uv=False)
    assert abs(cond - s[0] / s[-1]) <= 1e-10 * (s[0] / s[-1])


def test_clamp_rebuild_is_pivot_permuted():
    """step 7 as written: L diag(D) L^T with the UNclamped D is P cov P^T for Eigen's pivot permutation P, not cov"""
    Ap = _cases()["big_d"]
    cov0 = 0.05 * 0.05 * np.array(IC.lu_inverse(Ap.tolist()))
    m, D = IC.ldlt(cov0.tolist())
    L = np.tril(np.array(m), -1) + np.eye(6)
    rebuilt = L @ np.diag(D) @ L.T
    tol = 1e-9 * np.abs(cov0).max()
    assert np.abs(rebuilt - cov0).max() > tol
    perms = [p for p in itertools.permutations(range(6))
             if np.abs(rebuilt - cov0[np.ix_(p, p)]).max() <= tol]
    assert perms and all(list(p) != list(range(6)) for p in perms)


# ------------------------------------------------------------------------------------------ stage L (fake stages)
@pytest.fixture(scope="module")
def ih():
    L = _so("libicp_covariance_harness.so", "tests/icp_covariance_harness.cpp",
            ["tests/icp_covariance_stub.h", "tests/locus_stub.h", "tests/front_end_stub.h", "locus_b200/csrc/odometry.cu",
             "locus_b200/csrc/lo_pose.h", "include/locus_b200.h"], ["-O1", "-DLB_LOCUS_STUB"])
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    L.ih_set_fallback.argtypes = [C.c_uint64]
    L.ih_set_correction.argtypes = [C.c_uint64, vp]
    L.ih_calls.argtypes = [vp, vp, vp, vp, vp, sz]; L.ih_calls.restype = sz
    L.ih_events.argtypes = [vp, vp, sz]; L.ih_events.restype = sz
    L.ih_submap_create.argtypes = [i32, sz]; L.ih_submap_create.restype = vp
    L.ih_submap_destroy.argtypes = [vp]
    L.lb_locus_default_params.argtypes = [C.POINTER(api.LocusParams)]
    L.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
    L.lb_locus_destroy.argtypes = [vp]
    L.lb_locus_set_params.argtypes = [vp, C.POINTER(api.LocusParams)]
    L.lb_locus_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(api.Field), i32, i32, vp, vp, i32, C.POINTER(C.c_uint64)]
    L.lb_locus_next.argtypes = [vp, C.POINTER(api.LocusResult), i32]
    return L


def _scan(i, flags=0):
    b = np.zeros(NPTS * STEP, dtype=np.uint8)
    b[:8] = np.frombuffer(np.uint64(i).tobytes(), dtype=np.uint8)
    b[8:12] = np.frombuffer(np.uint32(flags).tobytes(), dtype=np.uint8)
    return b


def _fields():
    return api.VoxelGridB200._fields([("x", 0, api.LB_FLOAT32, 1), ("y", 4, api.LB_FLOAT32, 1), ("z", 8, api.LB_FLOAT32, 1)])


def _pose(theta, t):
    c, s = math.cos(theta), math.sin(theta)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    return T


def _run(ih, n, depth=2, map_n=0, fallback=(), corrections=None, id0=100, **params):
    ih.ih_reset()
    for k in fallback:
        ih.ih_set_fallback(id0 + k)
    for k, Cm in (corrections or {}).items():
        c16 = np.ascontiguousarray(Cm, np.float64).reshape(16)
        ih.ih_set_correction(id0 + k, c16.ctypes.data)
    m = ih.ih_submap_create(0, map_n)
    h = C.c_void_p()
    assert ih.lb_locus_create(0, depth, NPTS, STEP, m, C.byref(h)) == 0
    P = api.LocusParams()
    assert ih.lb_locus_default_params(C.byref(P)) == 0
    for k, v in params.items():
        if isinstance(v, dict):
            for kk, vv in v.items():
                setattr(getattr(P, k), kk, vv)
        else:
            setattr(P, k, v)
    assert ih.lb_locus_set_params(h, C.byref(P)) == 0
    fa = _fields()
    scans = [_scan(id0 + k) for k in range(n)]
    incs = [_pose(0.05 * (k % 3), [0.3 * k % 0.7, 0.1, 0.0]).astype(np.float32) for k in range(n)]
    t = C.c_uint64(0)
    res = []
    for k in range(n):
        g = np.ascontiguousarray(incs[k]).reshape(16)
        assert ih.lb_locus_submit(h, scans[k].ctypes.data, NPTS, STEP, fa, 3, 0, g.ctypes.data, None, 0, C.byref(t)) == 0
    for k in range(n):
        r = api.LocusResult()
        assert ih.lb_locus_next(h, C.byref(r), 1) == 0
        res.append(r)
    assert ih.lb_locus_destroy(h) == 0
    ih.ih_submap_destroy(m)
    cap = 8 * n + 8
    ids = np.zeros(cap, np.uint64); T = np.zeros((cap, 16), np.float32); R = np.zeros((cap, 9), np.float32)
    mx = np.zeros(cap); is_map = np.zeros(cap, np.int32)
    nc = ih.ih_calls(ids.ctypes.data, T.ctypes.data, R.ctypes.data, mx.ctypes.data, is_map.ctypes.data, cap)
    calls = [(int(ids[i]), T[i].reshape(4, 4).copy(), R[i].reshape(3, 3).copy(), mx[i], int(is_map[i])) for i in range(nc)]
    kind = np.zeros(cap, np.int32); eid = np.zeros(cap, np.uint64)
    ne = ih.ih_events(kind.ctypes.data, eid.ctypes.data, cap)
    events = [(int(kind[i]), int(eid[i])) for i in range(ne)]
    return res, calls, events, P


def _expected_rotation(prev_pose, inc):
    """the float rotation of P^-1, P = update(L_{k-1}, I_k), as lo_pose.h computes it"""
    P = LO.update(LO.from_mat(np.asarray(prev_pose).reshape(4, 4)), LO.from_mat(np.asarray(inc).reshape(4, 4)))
    return np.array(LO.inverse(P).R, dtype=np.float64).reshape(3, 3).astype(np.float32)


@pytest.mark.parametrize("depth", [1, 3])
def test_call_after_every_localization_before_insert(ih, depth):
    n = 8
    corr = {k: _pose(0.002 * k, [0.01 * k, 0.0, 0.0]) for k in range(n)}
    res, calls, events, P = _run(ih, n, depth=depth, corrections=corr, icp_covariance={"enabled": 1, "max_covariance": 0.02})
    assert res[0].has_localization == 0 and res[0].has_icp_covariance == 0 and res[0].keyframe == 1
    assert not any(res[0].icp_covariance) and res[0].icp_covariance_flags == 0
    assert [c[0] for c in calls] == [100 + k for k in range(1, n)]
    init = np.asarray(P.initial_pose).reshape(4, 4)
    for k in range(1, n):
        r = res[k]
        idk, T, R, mx, is_map = calls[k - 1]
        assert r.status == 0 and r.has_localization and r.has_icp_covariance and is_map == 1 and mx == 0.02
        assert np.array_equal(T, np.array(r.localization.final_transformation, np.float32).reshape(4, 4))
        prev = np.asarray(res[k - 1].pose) if k > 0 else init
        assert np.array_equal(R, _expected_rotation(prev, np.asarray(r.incremental)))
        assert list(r.icp_covariance) == [idk + i / 64.0 for i in range(36)]
        assert r.condition_number == 100.0 + idk
    # before the insert and crop of the same scan
    for idk in [c[0] for c in calls]:
        pos = [i for i, e in enumerate(events) if e[1] == idk]
        kinds = [events[i][0] for i in pos]
        assert kinds[0] == 4 and kinds.count(4) == 1
    assert any(e[0] in (1, 3) and e[1] > 100 for e in events)       # some keyframe was inserted after its call


def test_prior_map_first_scan_has_a_call(ih):
    res, calls, events, P = _run(ih, 3, map_n=500, prior_map=1, icp_covariance={"enabled": 1})
    assert [c[0] for c in calls] == [100, 101, 102]
    assert res[0].has_icp_covariance == 1 and calls[0][3] == 0.01
    init = np.asarray(P.initial_pose).reshape(4, 4)
    assert np.array_equal(calls[0][2], _expected_rotation(init, np.asarray(res[0].incremental)))


def test_disabled_makes_no_call(ih):
    res, calls, events, P = _run(ih, 5)
    assert P.icp_covariance.enabled == 0 and P.icp_covariance.max_covariance == 0.01
    assert calls == [] and all(e[0] != 4 for e in events)
    for r in res:
        assert r.has_icp_covariance == 0 and not any(r.icp_covariance) and r.condition_number == 0.0 and r.icp_covariance_flags == 0


def test_condition_number_carries_over_a_fallback(ih):
    res, calls, events, P = _run(ih, 6, fallback=(3, 4), icp_covariance={"enabled": 1})
    assert math.isnan(res[0].condition_number)                       # nothing computed yet
    assert [r.condition_number for r in res[1:3]] == [201.0, 202.0]     # 100 + scan id
    for k in (3, 4):
        assert res[k].icp_covariance_flags == api.LB_ICPCOV_D_NAN and res[k].has_icp_covariance == 1
        assert res[k].condition_number == 202.0
        assert np.array_equal(np.asarray(res[k].icp_covariance).reshape(6, 6), 0.01 * np.eye(6))
    assert res[5].condition_number == 205.0


@pytest.mark.parametrize("bad", [0.0, -0.01, float("nan"), float("inf")])
def test_set_params_refuses_bad_max_covariance(ih, bad):
    m = ih.ih_submap_create(0, 0)
    h = C.c_void_p()
    assert ih.lb_locus_create(0, 1, NPTS, STEP, m, C.byref(h)) == 0
    P = api.LocusParams()
    assert ih.lb_locus_default_params(C.byref(P)) == 0
    P.icp_covariance.enabled = 1
    P.icp_covariance.max_covariance = bad
    assert ih.lb_locus_set_params(h, C.byref(P)) == -1
    P.icp_covariance.max_covariance = 0.01
    assert ih.lb_locus_set_params(h, C.byref(P)) == 0
    assert ih.lb_locus_destroy(h) == 0
    ih.ih_submap_destroy(m)


def test_defaults_leave_the_feature_off(ih):
    P = api.LocusParams()
    assert ih.lb_locus_default_params(C.byref(P)) == 0
    assert P.icp_covariance.enabled == 0 and P.icp_covariance.max_covariance == 0.01


# ------------------------------------------------------------------------------------------ C++ mirror and PCL shim
def build_cpp_harness():
    """tests/icp_covariance_cpp_harness.cpp: B200Gicp::icpCovariance and the shim's computePoint2PlaneICPCovariance
    (instantiated with a 6x6 type) against the C ABI; the GPU test runs it"""
    out = os.path.join(ROOT, "tests", "_build", "icp_covariance_cpp_harness")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "pcl_stub"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "shim"),
                           "-I", os.path.join(ROOT, "locus_b200", "host"),
                           os.path.join(ROOT, "tests", "icp_covariance_cpp_harness.cpp"), "-L", os.path.join(ROOT, "locus_b200"),
                           "-llocus_b200", "-Wl,-rpath," + os.path.join(ROOT, "locus_b200"), "-pthread", "-o", out])
    return out


def test_cpp_mirror_and_shim_compile_and_link():
    import locus_b200
    exe = build_cpp_harness()
    if locus_b200.device_count() <= 0:
        r = subprocess.run([exe], stdout=subprocess.PIPE, text=True, timeout=120)
        assert r.returncode == 3 and "no_device=1" in r.stdout
