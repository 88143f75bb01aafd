"""The front end LOCUS ships, on the GPU: normals in the prepared clouds, a map whose points keep their normals, and the
whole chain with normals, covariances from normals and adaptive input voxelization.

* lb_gicp_estimate_normals gives the normals, covariances and pose of lb_gicp_compute_normals followed by a re-upload
  of the cloud with those normals, bit for bit, for the source and the target; the normals agree with
  oracle/normals_oracle.c at the bar of tests/test_normals_gpu.py; a prepared, shared cloud aligns as the uploaded one.
* lb_submap_insert_with_normals / crops / lb_submap_normals equal tools/front_end_oracle.SubmapNormalsOracle; with
  recompute_target_covariance = 0 the map's covariances are cov_from_normal of the stored normals, and a map holding one
  point without a normal takes the k-NN cache exactly as before.
* lb_locus in the shipped configuration (normals k = 20, every covariance from normals, adaptive leaf at 3000 points)
  equals, at depth 1 and 4, a blocking sequential restatement on the pre-existing public calls driven by
  tools/front_end_oracle.FrontEndChain; L stays near the generator's ground truth.  lb_odometry with normals gives the
  chain's odometry.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tools import front_end_oracle as FE
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

STEP = 32
LEAF0 = 0.25                  # Locus.cc:39, what the shipped launch sets
MAP_RES = 0.1
N_SCANS = 24
SEED = 11
PARAMS = dict(translation_threshold_kf=0.6, rotation_threshold_kf=0.3, refresh_every=2, window_half_size=9.0)
RESULT_FIELDS = ("final_transformation", "transformation", "converged", "iterations", "n_correspondences", "delta",
                 "n_objective_evals", "n_inner_iterations", "status")


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_nan(a, b):
    """bit-equal, with every NaN counted equal to every NaN"""
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_u32(np.where(na, 0, a)), _u32(np.where(nb, 0, b)))


def _same_result(a, b):
    for f in RESULT_FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        if f in ("final_transformation", "transformation"):
            if not np.array_equal(_u32(np.array(x, np.float32)), _u32(np.array(y, np.float32))):
                return False
        elif x != y:
            return False
    return True


def _bits(a):
    return np.asarray(a, np.float64).reshape(-1).view(np.uint64)


def _gicp(params=None, **kw):
    import locus_b200
    g = locus_b200.GicpB200()
    if params is not None:
        C.memmove(C.byref(g._p), C.byref(params), C.sizeof(params))
    for k, v in kw.items():
        setattr(g._p, k, v)
    g._apply()
    return g


def _filtered(vg, blob):
    import locus_b200
    f = vg.filter(blob, STEP, locus_b200.xyzi_fields())
    return np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()


def _voxel(v, leaf):
    v.setLeafSize(leaf); v.setFilterFieldName("z"); v.setFilterLimits(-100.0, 100.0)


@pytest.fixture(scope="module")
def data():
    import locus_b200
    scene, poses, blobs = G.stream(SEED, N_SCANS, beams=32, az=1024)
    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], SEED, beams=32, az=1024)
    vg = locus_b200.VoxelGridB200()
    vg.setLeafSize(0.2)
    prefill = np.ascontiguousarray(vg.filter(G.xyz_blob(world), STEP, locus_b200.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
    g = locus_b200.GicpB200()
    g.setInputSource(prefill)
    prefill_n = g.computeNormals(0, 20)[:, :3].copy()
    _voxel(vg, 0.35)
    scans = [_filtered(vg, b) for b in blobs[:2]]
    return poses, blobs, prefill, prefill_n, scans


# ------------------------------------------------------------------------------------------ normals in a cloud
@pytest.mark.parametrize("which", [0, 1])
def test_estimate_normals_equals_compute_and_reupload(data, which):
    _, _, _, _, (tgt, src) = data
    nr = dict(recompute_source_covariance=0, recompute_target_covariance=0)
    a, b = _gicp(**nr), _gicp(**nr)
    for g in (a, b):
        g.setInputSource(src); g.setInputTarget(tgt)
    a.estimateNormals(which, 20)
    nb = b.computeNormals(which, 20)
    cloud6 = np.ascontiguousarray(np.hstack([(src, tgt)[which], nb[:, :3]]))
    (b.setInputSource if which == 0 else b.setInputTarget)(cloud6, normal_off=12)
    # the normals: a's as the identity transform returns them (source), and the oracle's
    if which == 0:
        assert np.array_equal(_u32(a.transformSource(np.eye(4), with_normals=True)[:, 3:]), _u32(nb[:, :3]))
    # oracle/normals_oracle.c, at the bar of tests/test_normals_gpu.py (PCL's float eigen solver is not reproduced to
    # the last bit)
    ref = O.normals_knn((src, tgt)[which], 20)
    assert (np.abs(nb[:, :3] - ref[:, :3]).max(axis=1) < 1e-5).mean() >= 0.995
    ra, rb = a.align(), b.align()
    assert _same_result(ra, rb)
    for w in (0, 1):
        assert np.array_equal(a.covariances(w).view(np.uint64), b.covariances(w).view(np.uint64))
    # with normals the covariances really come from them (the k-NN ones differ)
    assert not np.array_equal(a.covariances(which), _knn_covariances((src, tgt)[which], (tgt, src)[which], which))


def _knn_covariances(cloud, other, which):
    g = _gicp()
    if which == 0:
        g.setInputSource(cloud); g.setInputTarget(other)
    else:
        g.setInputSource(other); g.setInputTarget(cloud)
    g.align()
    return g.covariances(which)


def test_shared_cloud_with_normals_aligns_as_the_upload(data):
    _, _, _, _, (tgt, src) = data
    nr = dict(recompute_source_covariance=0, recompute_target_covariance=0)
    a, b, c = _gicp(**nr), _gicp(**nr), _gicp(**nr)
    a.setInputSource(src); a.estimateNormals(0, 20); a.prepareSource()
    cl = a.shareSource()
    b.setSourceCloud(cl)
    type(a).releaseCloud(cl)
    with pytest.raises(Exception):
        b.estimateNormals(0, 20)                   # an adopted cloud is immutable
    c.setInputSource(src)
    n_src = c.computeNormals(0, 20)
    c.setInputSource(np.ascontiguousarray(np.hstack([src, n_src[:, :3]])), normal_off=12)
    g = _gicp(**nr)
    g.setInputSource(tgt)
    n_tgt = g.computeNormals(0, 20)
    t6 = np.ascontiguousarray(np.hstack([tgt, n_tgt[:, :3]]))
    for h in (b, c):
        h.setInputTarget(t6, normal_off=12)
    rb, rc = b.align(), c.align()
    assert _same_result(rb, rc)
    assert np.array_equal(_u32(b.transformSource(with_normals=True)), _u32(c.transformSource(with_normals=True)))


# ------------------------------------------------------------------------------------------ the map with normals
def test_map_with_normals_equals_oracle(data):
    import locus_b200
    _, _, prefill, prefill_n, (s0, s1) = data
    m = locus_b200.SubmapB200(0, MAP_RES)
    o = FE.SubmapNormalsOracle(MAP_RES)
    rng = np.random.default_rng(5)

    def check():
        assert np.array_equal(_u32(m.points()), _u32(o.pts))
        assert _same_nan(m.normals(), o.nrm)

    m.InsertPoints(s0[:200]); o.insert(s0[:200])                 # no normals yet: NaN rows
    check()
    n1 = rng.normal(size=(len(prefill), 3)).astype(np.float32)
    n1[3] = np.nan                                             # a NaN normal is still a normal
    assert m.InsertPointsWithNormals(prefill, n1) == len(o.insert(prefill, n1))
    check()
    for c, half in (([0.0, 0.0, 0.0], 8.0), ([1.0, 0.5, 0.0], 5.0)):
        assert m.Refresh(c, half) == o.crop(c, half)
        check()
    s1n = rng.normal(size=(len(s1), 3)).astype(np.float32)
    m.InsertPointsWithNormals(s1 + 0.03, s1n); o.insert(s1 + 0.03, s1n)
    m.InsertPoints(s0 + 0.05); o.insert(s0 + 0.05)
    check()
    m.Refresh([0.0, 0.0, 0.0], 30.0); o.crop([0.0, 0.0, 0.0], 30.0)
    check()
    m.close()


def test_map_covariances_from_normals(data):
    import locus_b200
    _, _, prefill, prefill_n, (s0, s1) = data
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    m.Refresh([0.0, 0.0, 0.0], 12.0)
    g = _gicp(recompute_target_covariance=0)
    eps = g._p.gicp_epsilon
    g.setInputSource(s1)
    g.setTargetSubmap(m)
    want = FE.cov_from_normals(m.normals(), eps)
    assert np.array_equal(g.covariances(1).view(np.uint64), want.view(np.uint64))
    r_normals = g.align()
    # one point without a normal: the k-NN cache, exactly as a map of the same points without normals gets it today
    m.InsertPoints(np.array([[40.0, 40.0, 40.0]], np.float32))
    plain = locus_b200.SubmapB200(0, MAP_RES)
    assert plain.InsertPoints(m.points()) == m.size()
    knn = _gicp()
    g.setInputSource(s1); g.setTargetSubmap(m)
    knn.setInputSource(s1); knn.setTargetSubmap(plain)
    assert np.array_equal(g.covariances(1).view(np.uint64), knn.covariances(1).view(np.uint64))
    assert _same_result(g.align(), knn.align())
    assert r_normals.converged
    m.close(); plain.close()


def test_map_without_normals_is_unchanged(data):
    """a map that never had a normal: recompute_target_covariance = 0 takes the k-NN cache of today's chain"""
    import locus_b200
    _, _, prefill, _, (s0, s1) = data
    ms = [locus_b200.SubmapB200(0, MAP_RES) for _ in range(2)]
    hs = [_gicp(recompute_target_covariance=0), _gicp()]
    for m, h in zip(ms, hs):
        m.InsertPoints(prefill)
        h.setInputSource(s1)
        h.setTargetSubmap(m)
    assert np.array_equal(hs[0].covariances(1).view(np.uint64), hs[1].covariances(1).view(np.uint64))
    assert _same_result(hs[0].align(), hs[1].align())
    assert np.isnan(ms[0].normals()).all()
    for m in ms:
        m.close()


# ------------------------------------------------------------------------------------------ the shipped chain
def _shipped(**kw):
    """keywords of locus_params: the test's keyframe settings in the shipped front-end configuration"""
    return {**PARAMS, **FE.SHIPPED, **kw}


def _cloud6(g, xyz):
    """computeNormals, then an upload with normal_off: the pre-existing public path to a cloud with normals"""
    g.setInputSource(xyz)
    n = g.computeNormals(0, 20)
    return np.ascontiguousarray(np.hstack([xyz, n[:, :3]]))


def _sequential(blobs, prefill, prefill_n, kw):
    import locus_b200
    P = locus_b200.locus_params(**kw)
    vg = locus_b200.VoxelGridB200()
    odo, loc, nrm = _gicp(P.odometry), _gicp(P.localization), _gicp()
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    chain = FE.FrontEndChain(P, np.float32(LEAF0))
    out, prev = [], None
    for b in blobs:
        leaf = chain.next_leaf
        _voxel(vg, float(leaf))
        xyz = _filtered(vg, b)
        used = chain.filtered(len(xyz))
        assert used == leaf
        c6 = _cloud6(nrm, xyz)
        rec = {"odometry": None, "localization": None, "leaf": leaf}
        odoT = None
        if prev is not None:
            odo.setInputSource(c6, normal_off=12); odo.setInputTarget(prev, normal_off=12)
            rec["odometry"] = odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(c6, normal_off=12)

        def localize(Gs):
            loc.setTargetSubmap(m)
            rec["localization"] = loc.align(Gs)
            return loc.getFinalTransformation()

        def insert(T):
            t = loc.transformSource(T, with_normals=True)
            return m.InsertPointsWithNormals(t[:, :3], t[:, 3:])

        rec.update(chain.scan(True, odoT, localize, insert, lambda c, half: m.Refresh(c, half)))
        rec["map_size"] = m.size()
        out.append(rec)
        prev = c6
    res = out, m.points(), m.normals()
    m.close()
    return res


def _chain(blobs, prefill, prefill_n, kw, depth, device_input=False):
    import locus_b200
    import torch
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPointsWithNormals(prefill, prefill_n)
    n = blobs[0].size // STEP
    ch = locus_b200.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **kw)
    _voxel(ch.voxel, LEAF0)
    keep = [torch.from_numpy(b).cuda() for b in blobs] if device_input else blobs
    for b in keep:
        if device_input:
            ch.submit(b.data_ptr(), n, STEP, locus_b200.xyzi_fields(), mem=locus_b200.LB_MEM_DEVICE)
        else:
            ch.submit(b, n, STEP, locus_b200.xyzi_fields())
    res = [ch.next() for _ in blobs]
    ch.close()
    out = res, m.points(), m.normals()
    m.close()
    return out


@pytest.fixture(scope="module")
def reference(data):
    poses, blobs, prefill, prefill_n, _ = data
    return _sequential(blobs, prefill, prefill_n, _shipped())


@pytest.mark.parametrize("depth", [1, 4])
def test_shipped_chain_equals_sequential_calls(data, reference, depth):
    poses, blobs, prefill, prefill_n, _ = data
    ref, ref_pts, ref_nrm = reference
    res, pts, nrm = _chain(blobs, prefill, prefill_n, _shipped(), depth, device_input=(depth == 4))
    assert [r.ticket for r in res] == list(range(len(blobs)))
    for k, (r, e) in enumerate(zip(res, ref)):
        assert r.status == 0, (k, r.error)
        assert np.float32(r.leaf_size) == e["leaf"], k
        assert r.has_odometry == (e["odometry"] is not None)
        if r.has_odometry:
            assert _same_result(r.odometry, e["odometry"]), k
        assert r.has_localization == e["has_localization"]
        if r.has_localization:
            assert _same_result(r.localization, e["localization"]), k
        for f in ("odometry_accepted", "correction_accepted", "keyframe", "n_inserted", "n_removed", "map_size"):
            assert getattr(r, f) == e[f], (k, f)
        assert np.array_equal(_bits(r.odometry_pose), _bits(e["O"])), k
        assert np.array_equal(_bits(r.incremental), _bits(e["I"])), k
        assert np.array_equal(_bits(r.pose), _bits(e["L"])), k
    assert np.array_equal(_u32(pts), _u32(ref_pts))
    assert _same_nan(nrm, ref_nrm)
    # the leaf moved towards ~3000 filtered points
    assert len({r.leaf_size for r in res}) > 1
    kf = [k for k, r in enumerate(res) if r.keyframe]
    assert len(kf) >= 4 and sum(1 for r in res if r.n_removed) >= 1, (kf, [r.n_removed for r in res])
    err_t = max(float(np.linalg.norm(np.array(r.pose).reshape(4, 4)[:3, 3] - T[:3, 3])) for r, T in zip(res, poses))
    err_r = max(float(np.arccos(np.clip((np.trace(np.array(r.pose).reshape(4, 4)[:3, :3].T @ T[:3, :3]) - 1) / 2, -1, 1)))
                for r, T in zip(res, poses))
    assert err_t < 0.2 and err_r < 0.03, (err_t, err_r)


def test_odometry_with_normals_equals_chain_odometry(data):
    """lb_odometry's normals stage = the chain's (fixed leaf: lb_odometry has no adaptive voxelization)"""
    import locus_b200
    poses, blobs, prefill, prefill_n, _ = data
    kw = _shipped(front_end=dict(normals_k=20, adaptive_voxelization=0, points_to_process=0))
    res, _, _ = _chain(blobs, prefill, prefill_n, kw, 2)
    P = locus_b200.locus_params(**kw)
    n = blobs[0].size // STEP
    odo = locus_b200.OdometryB200(0, depth=3, max_points=n, max_point_step=STEP)
    _voxel(odo.voxel, LEAF0)
    odo.setGicpParams(**{k: getattr(P.odometry, k) for k, _ in locus_b200.GicpParams._fields_})
    odo.setNormals(20)
    for b in blobs:
        odo.submit(b, n, STEP, locus_b200.xyzi_fields())
    rs = [odo.next() for _ in blobs]
    odo.close()
    assert sum(r.has_pose for r in rs) == len(blobs) - 1
    for r, e in zip(rs, res):
        assert r.status == 0 and bool(r.has_pose) == bool(e.has_odometry)
        if r.has_pose:
            assert _same_result(r.gicp, e.odometry)
