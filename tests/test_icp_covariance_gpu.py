"""lb_gicp_icp_covariance and lb_locus's icp_covariance on the GPU.

* The reference's known answers through the C ABI with explicit correspondences, host and device buffers.
* A filtered scan against the previous scan with normals and against a submap with normals (rotated normals): the
  1-NN equals lb_gicp_nn_target on lb_gicp_transform_source's output and the oracle's kd-tree index for index; Ap is
  within 1e-10 of oracle/icp_cov_oracle.py; covariance, condition number and flags equal the oracle's 6x6 algebra on the
  returned Ap bit for bit (the oracle equals icp_cov.h bit for bit, test_icp_covariance_cpu.py), and are within 1e-9 of
  the oracle end to end; repeated calls give identical bits.
* A target without normals takes the fallback; a map with mixed normals skips exactly the oracle's rows.
* Errors leave the handle as it was.
* lb_locus in the shipped front end at depth 1 and 3: every scan's covariance, condition number and flags equal
  lb_gicp_icp_covariance called in blocking calls driven by tools/front_end_oracle.FrontEndChain (after the align, with
  F, the map before the insert and the chain oracle's rotation of P^-1; the condition number carried over fallbacks);
  with the covariance off every pose, keyframe flag, localization result and leaf are the same bits.
* The C++ mirror (B200Gicp::icpCovariance) and the PCL shim (computePoint2PlaneICPCovariance) give the C call's bits,
  the shim leaves the condition number alone on the D-NaN fallback and refuses a target uploaded without normals.
* A C2 scan (~30 k points) against a C3-shaped ~500 k-point submap with normals and against the previous scan.
"""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import icp_cov_oracle as IC
from oracle import oracle as O
from tools import front_end_oracle as FE
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

STEP = 32
SEED = 11
N_SCANS = 12
MAP_RES = 0.1
PARAMS = dict(translation_threshold_kf=0.6, rotation_threshold_kf=0.3, refresh_every=2, window_half_size=9.0)


def _bits(a):
    return np.asarray(a, np.float64).reshape(-1).view(np.uint64)


def _same(a, b):
    a = np.asarray(a, np.float64).reshape(-1); b = np.asarray(b, np.float64).reshape(-1)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(_bits(np.where(np.isnan(a), 0, a)), _bits(np.where(np.isnan(b), 0, b)))


def _check_6x6(r):
    """covariance, condition number and flags are the 6x6 algebra of the returned Ap, bit for bit"""
    cov, cond, fl = IC.covariance(r["Ap"], 0.01)
    assert fl == r["flags"]
    assert _same(cov, r["covariance"]) and _same(cond, r["condition_number"])


def _filtered(vg, blob):
    import locus_b200
    f = vg.filter(blob, STEP, locus_b200.xyzi_fields())
    return np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()


@pytest.fixture(scope="module")
def data():
    import locus_b200
    scene, poses, blobs = G.stream(SEED, N_SCANS, beams=32, az=1024)
    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], SEED, beams=32, az=1024)
    vg = locus_b200.VoxelGridB200()
    vg.setLeafSize(0.2)
    prefill = _filtered(vg, G.xyz_blob(world))
    g = locus_b200.GicpB200()
    g.setInputSource(prefill)
    prefill_n = g.computeNormals(0, 20)[:, :3].copy()
    vg.setLeafSize(0.35); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    scans = [_filtered(vg, b) for b in blobs[:3]]
    g.setInputSource(scans[0])
    n0 = g.computeNormals(0, 20)[:, :3].copy()
    return poses, blobs, prefill, prefill_n, scans, n0


# ------------------------------------------------------------------------------------------ known answers
def _planes():
    xyz = np.array([(np.float32(i) * np.float32(0.1), np.float32(j) * np.float32(0.1), np.float32(0)) for i in range(10)
                    for j in range(10)], np.float32)          # tests/fixtures.py plane()
    nrm = O.normals_knn(xyz, k=10)[:, :3]
    return O.normalize_pcloud(xyz), nrm


@pytest.mark.parametrize("device", [False, True])
def test_known_answers_through_the_c_abi(device):
    import locus_b200
    import torch
    xyz, nrm = _planes()
    T1 = np.array([[1, 0, 0, 0], [0, 0, -1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], np.float32)
    T2 = np.array([[0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0], [0, 0, 0, 1]], np.float32)
    g = locus_b200.GicpB200()
    # one plane: Ap singular -> 0.01 I with the D-NaN flag
    g.setInputSource(xyz)
    g.setInputTarget(np.ascontiguousarray(np.hstack([xyz, nrm])), normal_off=12)
    co = np.arange(len(xyz), dtype=np.int32)
    arg = torch.from_numpy(co).cuda() if device else co
    r = g.icpCovariance(correspondences=arg, device=device)
    assert r["flags"] == locus_b200.api.LB_ICPCOV_D_NAN and np.array_equal(r["covariance"], 0.01 * np.eye(6))
    assert math.isnan(r["condition_number"]) and r["n_used"] == len(xyz)
    _check_6x6(r)
    # three planes, rotated 30 deg and offset 1 mm: ~1e-6 I
    pts = np.concatenate([xyz, IC.transform(xyz, T1), IC.transform(xyz, T2)])
    nr = np.concatenate([nrm, IC.rotate_normals(nrm, T1[:3, :3]), IC.rotate_normals(nrm, T2[:3, :3])])
    tf = np.zeros((4, 4), np.float32)
    tf[0, 0] = 0.866; tf[0, 1] = -0.5; tf[1, 0] = 0.5; tf[1, 1] = 0.866; tf[0, 3] = 0.001; tf[3, 3] = 1
    off = IC.transform(pts, tf)
    g.setInputSource(off)
    g.setInputTarget(np.ascontiguousarray(np.hstack([pts, nr])), normal_off=12)
    co = np.arange(len(pts), dtype=np.int32)
    arg = torch.from_numpy(co).cuda() if device else co
    r = g.icpCovariance(correspondences=arg, device=device)
    assert np.abs(r["covariance"] - 1e-6 * np.eye(6)).max() < 1e-4
    o = IC.icp_covariance(off, pts, nr, correspondences=co)
    assert np.abs(r["Ap"] - o["Ap"]).max() <= 1e-10 * np.abs(o["Ap"]).max()
    _check_6x6(r)


# ------------------------------------------------------------------------------------------ scan-sized inputs
def _against_oracle(g, src, tgt, tgt_n, T, R=None):
    r = g.icpCovariance(normal_rotation=R)
    o = IC.icp_covariance(src, tgt, tgt_n, T=T, normal_rotation=R)
    idx, _ = g.nearestTarget(g.transformSource())
    assert np.array_equal(idx, o["correspondences"])
    assert r["n_query"] == len(src) and r["n_used"] == o["n_used"]
    assert np.abs(r["Ap"] - o["Ap"]).max() <= 1e-10 * np.abs(o["Ap"]).max()
    _check_6x6(r)
    assert r["flags"] == o["flags"]
    assert np.abs(r["covariance"] - o["covariance"]).max() <= 1e-9 * np.abs(o["covariance"]).max()
    if not math.isnan(o["condition_number"]):
        assert abs(r["condition_number"] - o["condition_number"]) <= 1e-9 * o["condition_number"]
    again = g.icpCovariance(normal_rotation=R)
    for k in ("Ap", "covariance", "condition_number"):
        assert _same(again[k], r[k])
    return r


def test_scan_against_previous_scan(data):
    import locus_b200
    _, _, _, _, scans, n0 = data
    g = locus_b200.GicpB200()
    g.setMaxCorrespondenceDistance(1.0); g.setMaximumIterations(20)
    g.setInputTarget(np.ascontiguousarray(np.hstack([scans[0], n0])), normal_off=12)
    g.setInputSource(scans[1])
    g.align()
    r = _against_oracle(g, scans[1], scans[0], n0, g.getFinalTransformation())
    assert r["n_used"] > 0.9 * len(scans[1])


def test_scan_against_submap_with_rotated_normals(data):
    import locus_b200
    _, _, prefill, prefill_n, scans, _ = data
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    g = locus_b200.GicpB200()
    g.setMaxCorrespondenceDistance(0.5); g.setMaximumIterations(20)
    g.setInputSource(scans[1]); g.setTargetSubmap(m)
    g.align()
    R = np.array([[0.9950042, -0.0998334, 0.0], [0.0998334, 0.9950042, 0.0], [0.0, 0.0, 1.0]], np.float32)
    _against_oracle(g, scans[1], m.points(), m.normals(), g.getFinalTransformation(), R)
    # a map change after set_target_submap is refused until the target is set again
    m.InsertPoints(scans[1] + np.float32(50.0))
    with pytest.raises(locus_b200.LocusB200Error) as e:
        g.icpCovariance()
    assert e.value.status == -1
    g.setTargetSubmap(m)
    g.icpCovariance()
    m.close()


def test_target_without_normals_takes_the_fallback(data):
    import locus_b200
    _, _, _, _, scans, _ = data
    g = locus_b200.GicpB200()
    g.setInputTarget(scans[0]); g.setInputSource(scans[1])
    g.align()
    r = g.icpCovariance()
    assert r["n_used"] == 0 and not r["Ap"].any()
    assert r["flags"] == locus_b200.api.LB_ICPCOV_D_NAN and np.array_equal(r["covariance"], 0.01 * np.eye(6))


def test_mixed_normals_skip_the_oracles_rows(data):
    import locus_b200
    _, _, prefill, prefill_n, scans, _ = data
    m = locus_b200.SubmapB200(0, MAP_RES)
    half = len(prefill) // 2
    m.InsertPoints(prefill[:half])
    m.InsertPointsWithNormals(prefill[half:], prefill_n[half:])
    g = locus_b200.GicpB200()
    g.setMaxCorrespondenceDistance(0.5); g.setMaximumIterations(20)
    g.setInputSource(scans[1]); g.setTargetSubmap(m)
    g.align()
    nrm = m.normals()
    assert np.isnan(nrm).any() and (~np.isnan(nrm).any(1)).any()
    r = _against_oracle(g, scans[1], m.points(), nrm, g.getFinalTransformation())
    assert 0 < r["n_used"] < len(scans[1])
    m.close()


def test_errors_leave_the_handle_as_it_was(data):
    import locus_b200
    _, _, _, _, scans, n0 = data
    g = locus_b200.GicpB200()
    with pytest.raises(locus_b200.LocusB200Error) as e:
        g.icpCovariance()
    assert e.value.status == -4                                         # no source
    g.setInputSource(scans[1])
    with pytest.raises(locus_b200.LocusB200Error) as e:
        g.icpCovariance()
    assert e.value.status == -5                                         # no target
    g.setInputTarget(np.ascontiguousarray(np.hstack([scans[0], n0])), normal_off=12)
    with pytest.raises(locus_b200.LocusB200Error) as e:
        g.icpCovariance()
    assert e.value.status == -10                                        # no align yet
    r0 = g.align()
    T0 = g.getFinalTransformation().copy()
    good = g.icpCovariance()
    bad = np.zeros(len(scans[1]), np.int32); bad[7] = len(scans[0])
    for kw in (dict(correspondences=bad), dict(max_covariance=0.0), dict(max_covariance=float("nan"))):
        with pytest.raises(locus_b200.LocusB200Error) as e:
            g.icpCovariance(**kw)
        assert e.value.status == -1
    assert np.array_equal(g.getFinalTransformation(), T0)
    again = g.icpCovariance()
    assert _same(again["Ap"], good["Ap"]) and _same(again["covariance"], good["covariance"])
    r1 = g.align()
    assert np.array_equal(g.getFinalTransformation(), T0) and r1.iterations == r0.iterations


# ------------------------------------------------------------------------------------------ the chain
LEAF0 = 0.25


def _kw(on):
    return {**PARAMS, **FE.SHIPPED, "icp_covariance": {"enabled": int(on), "max_covariance": 0.01}}


def _voxel(v, leaf):
    v.setLeafSize(leaf); v.setFilterFieldName("z"); v.setFilterLimits(-100.0, 100.0)


def _gicp(params):
    import locus_b200
    g = locus_b200.GicpB200()
    C.memmove(C.byref(g._p), C.byref(params), C.sizeof(params))
    g._apply()
    return g


def _cloud6(g, xyz):
    g.setInputSource(xyz)
    n = g.computeNormals(0, 20)
    return np.ascontiguousarray(np.hstack([xyz, n[:, :3]]))


def _sequential(blobs, prefill, prefill_n):
    """the chain as blocking calls driven by tools/front_end_oracle.FrontEndChain; after every localization align,
    lb_gicp_icp_covariance with the align's F, the map before the insert and the chain oracle's rotation of P^-1"""
    import locus_b200
    P = locus_b200.locus_params(**_kw(True))
    vg = locus_b200.VoxelGridB200()
    odo, loc = _gicp(P.odometry), _gicp(P.localization)
    nrm = locus_b200.GicpB200()
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    chain = FE.FrontEndChain(P, np.float32(LEAF0))
    out, prev = [], None
    for b in blobs:
        _voxel(vg, float(chain.next_leaf))
        xyz = _filtered(vg, b)
        chain.filtered(len(xyz))
        c6 = _cloud6(nrm, xyz)
        rec = {"icp": None}
        odoT = None
        if prev is not None:
            odo.setInputSource(c6, normal_off=12); odo.setInputTarget(prev, normal_off=12)
            odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(c6, normal_off=12)

        def localize(Gs):
            loc.setTargetSubmap(m)
            loc.align(Gs)
            rec["icp"] = loc.icpCovariance(normal_rotation=chain.normal_rotation, max_covariance=0.01)
            return loc.getFinalTransformation()

        def insert(T):
            t = loc.transformSource(T, with_normals=True)
            return m.InsertPointsWithNormals(t[:, :3], t[:, 3:])

        rec.update(chain.scan(True, odoT, localize, insert, lambda c, half: m.Refresh(c, half)))
        rec["condition_number"] = chain.published_condition_number(rec["icp"])
        out.append(rec)
        prev = c6
    m.close()
    return out


def _chain(blobs, prefill, prefill_n, depth, on):
    import locus_b200
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    n = blobs[0].size // STEP
    ch = locus_b200.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **_kw(on))
    _voxel(ch.voxel, LEAF0)
    for b in blobs:
        ch.submit(b, n, STEP, locus_b200.xyzi_fields())
    res = [ch.next() for _ in blobs]
    ch.close()
    pts = m.points()
    m.close()
    return res, pts


@pytest.fixture(scope="module")
def blocking(data):
    _, blobs, prefill, prefill_n, _, _ = data
    return _sequential(blobs, prefill, prefill_n)


@pytest.mark.parametrize("depth", [1, 3])
def test_chain_covariance_equals_blocking_calls(data, blocking, depth):
    """every scan's covariance, condition number and flags are those of lb_gicp_icp_covariance called after the
    blocking align with F, the pre-insert map and the rotation of P^-1; the chain is otherwise bit-equal to itself
    with the covariance off"""
    _, blobs, prefill, prefill_n, _, _ = data
    off, map_off = _chain(blobs, prefill, prefill_n, depth, False)
    on, map_on = _chain(blobs, prefill, prefill_n, depth, True)
    assert np.array_equal(map_off, map_on)
    n_loc = n_fallback = 0
    for a, b, ref in zip(off, on, blocking):
        assert a.status == 0 and b.status == 0
        for f in ("pose", "odometry_pose", "incremental"):
            assert np.array_equal(np.array(getattr(a, f)), np.array(getattr(b, f)))
            assert np.array_equal(np.array(getattr(b, f)), np.asarray(ref[{"pose": "L", "odometry_pose": "O", "incremental": "I"}[f]]).reshape(16))
        assert a.keyframe == b.keyframe == ref["keyframe"] and a.leaf_size == b.leaf_size
        assert a.has_localization == b.has_localization == ref["has_localization"]
        assert np.array_equal(np.array(a.localization.final_transformation), np.array(b.localization.final_transformation))
        assert a.has_icp_covariance == 0 and a.condition_number == 0.0
        assert b.has_icp_covariance == b.has_localization
        if ref["icp"] is None:
            assert not any(b.icp_covariance) and b.icp_covariance_flags == 0
        else:
            n_loc += 1
            n_fallback += bool(ref["icp"]["flags"] & 2)
            assert _same(np.array(b.icp_covariance), ref["icp"]["covariance"])
            assert b.icp_covariance_flags == ref["icp"]["flags"]
        assert _same(b.condition_number, ref["condition_number"])
    assert n_loc >= len(blobs) - 1


# ------------------------------------------------------------------------------------------ C++ mirror and PCL shim
def test_cpp_mirror_and_shim_equal_the_c_call():
    import subprocess
    from test_icp_covariance_cpu import build_cpp_harness
    r = subprocess.run([build_cpp_harness()], stdout=subprocess.PIPE, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    kv = dict(line.split("=", 1) for line in r.stdout.split())
    assert kv["planes3_c_status"] == "0" and kv["planes3_c_flags"] != "2"
    assert kv["plane1_c_status"] == "0" and kv["plane1_c_flags"] == "2"          # one plane: the D-NaN fallback
    for tag in ("planes3", "plane1"):
        assert kv[tag + "_mirror_equal"] == "1" and kv[tag + "_shim_equal"] == "1", r.stdout
        assert kv[tag + "_shim_refuses_without_normals"] == "1"
    assert kv["plane1_shim_condition_kept"] == "1" and kv["planes3_shim_condition_kept"] == "0"


# ------------------------------------------------------------------------------------------ C2 scan, C3-shaped submap
def test_c2_scan_against_c3_submap_and_previous_scan():
    """bench sizes: a ~30 k-point C2 scan against a ~500 k-point submap with normals (where the 1-NN kernel is chosen
    by the map's density) and against the previous scan"""
    import locus_b200
    from tools.bench_icp_covariance import c2_c3_case
    scan0, scan1, submap = c2_c3_case()
    assert len(submap) > 400_000 and len(scan1) > 20_000
    g = locus_b200.GicpB200()
    g.setInputSource(submap)
    map_n = g.computeNormals(0, 20)[:, :3].copy()
    g.setInputSource(scan0)
    n0 = g.computeNormals(0, 20)[:, :3].copy()
    m = locus_b200.SubmapB200(0, 0.01)
    m.InsertPointsWithNormals(submap, map_n)
    h = locus_b200.GicpB200()
    h.setMaxCorrespondenceDistance(0.5); h.setMaximumIterations(20)
    h.setInputSource(scan1); h.setTargetSubmap(m)
    h.align()
    R = np.array([[0.9950042, -0.0998334, 0.0], [0.0998334, 0.9950042, 0.0], [0.0, 0.0, 1.0]], np.float32)
    _against_oracle(h, scan1, m.points(), m.normals(), h.getFinalTransformation(), R)
    m.close()
    h2 = locus_b200.GicpB200()
    h2.setMaxCorrespondenceDistance(1.0); h2.setMaximumIterations(20)
    h2.setInputSource(scan1); h2.setInputTarget(np.ascontiguousarray(np.hstack([scan0, n0])), normal_off=12)
    h2.align()
    _against_oracle(h2, scan1, scan0, n0, h2.getFinalTransformation())
