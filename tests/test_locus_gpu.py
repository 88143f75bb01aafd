"""lb_locus_* on the GPU: the whole lidar callback as one pipeline must compute what the blocking calls compute.

On a generated stream with several keyframes and crops, starting from a pre-filled submap, every odometry and
localization lb_gicp_result, O/I/L, the keyframe flags and the final map are bit-identical to a sequential restatement:
blocking VoxelGridB200 / GicpB200 / SubmapB200 calls driven by oracle/locus_oracle.py.  Depth 1 and depth 4 agree, the
chain's odometry equals lb_odometry's, and L stays near the generator's ground truth."""
import numpy as np
import pytest

from oracle import locus_oracle as LO
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

STEP = 32
LEAF = 0.35
MAP_RES = 0.1
N_SCANS = 24
SEED = 11
PARAMS = dict(translation_threshold_kf=0.6, rotation_threshold_kf=0.3, refresh_every=2, window_half_size=9.0)
RESULT_FIELDS = ("final_transformation", "transformation", "converged", "iterations", "n_correspondences", "delta",
                 "n_objective_evals", "n_inner_iterations", "status")


@pytest.fixture(scope="module")
def data():
    import locus_b200
    scene, poses, blobs = G.stream(SEED, N_SCANS, beams=32, az=1024)
    world = G.world_points(scene, [poses[0], G.pose_matrix([1.0, 0.5, 0.0], [0, 0, 0.3])], SEED, beams=32, az=1024)
    vg = locus_b200.VoxelGridB200()
    vg.setLeafSize(0.2)
    prefill = vg.filter(G.xyz_blob(world), STEP, locus_b200.xyzi_fields())
    prefill = np.ascontiguousarray(prefill).view(np.float32).reshape(-1, 8)[:, :3].copy()
    return poses, blobs, prefill


def _voxel(v):
    v.setLeafSize(LEAF); v.setFilterFieldName("z"); v.setFilterLimits(-100.0, 100.0)


def _gicp(params):
    import locus_b200
    import ctypes as C
    g = locus_b200.GicpB200()
    C.memmove(C.byref(g._p), C.byref(params), C.sizeof(params))
    g._apply()
    return g


def _sequential(blobs, prefill):
    import locus_b200
    P = locus_b200.locus_params(**PARAMS)
    vg = locus_b200.VoxelGridB200(); _voxel(vg)
    odo, loc = _gicp(P.odometry), _gicp(P.localization)
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    chain = LO.LocusChain(P)
    out, prev = [], None
    for b in blobs:
        f = vg.filter(b, STEP, locus_b200.xyzi_fields())
        xyz = np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()
        rec = {"odometry": None, "localization": None}
        odoT = None
        if prev is not None:
            odo.setInputSource(xyz); odo.setInputTarget(prev)
            rec["odometry"] = odo.align()
            odoT = odo.getFinalTransformation()
        loc.setInputSource(xyz)

        def localize(Gs):
            loc.setTargetSubmap(m)
            rec["localization"] = loc.align(Gs)
            return loc.getFinalTransformation()

        rec.update(chain.scan(True, odoT, localize, lambda T: m.InsertPoints(loc.transformSource(T)),
                              lambda c, half: m.Refresh(c, half)))
        rec["map_size"] = m.size()
        out.append(rec)
        prev = xyz
    return out, m.points()


def _chain(blobs, prefill, depth, device_input=False):
    import locus_b200
    import torch
    m = locus_b200.SubmapB200(0, MAP_RES)
    m.InsertPoints(prefill)
    n = blobs[0].size // STEP
    ch = locus_b200.LocusB200(m, 0, depth=depth, max_points=n, max_point_step=STEP, **PARAMS)
    _voxel(ch.voxel)
    keep = [torch.from_numpy(b).cuda() for b in blobs] if device_input else blobs
    for b in keep:
        if device_input:
            ch.submit(b.data_ptr(), n, STEP, locus_b200.xyzi_fields(), mem=locus_b200.LB_MEM_DEVICE)
        else:
            ch.submit(b, n, STEP, locus_b200.xyzi_fields())
    res = [ch.next() for _ in blobs]
    times = ch.stageTimes()
    ch.close()
    pts = m.points()
    m.close()
    return res, pts, times


def _same_result(a, b):
    for f in RESULT_FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        if f in ("final_transformation", "transformation"):
            if not np.array_equal(np.array(x, np.float32).view(np.uint32), np.array(y, np.float32).view(np.uint32)):
                return False
        elif x != y:
            return False
    return True


def _bits(a):
    return np.asarray(a, np.float64).reshape(-1).view(np.uint64)


@pytest.fixture(scope="module")
def reference(data):
    poses, blobs, prefill = data
    return _sequential(blobs, prefill)


@pytest.mark.parametrize("depth", [1, 4])
def test_chain_equals_sequential_calls(data, reference, depth):
    poses, blobs, prefill = data
    ref, ref_map = reference
    res, pts, times = _chain(blobs, prefill, depth, device_input=(depth == 4))
    assert [r.ticket for r in res] == list(range(len(blobs)))
    for k, (r, e) in enumerate(zip(res, ref)):
        assert r.status == 0, (k, r.error)
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
    assert np.array_equal(pts.view(np.uint32), ref_map.view(np.uint32))
    kf = [k for k, r in enumerate(res) if r.keyframe]
    assert len(kf) >= 4 and sum(1 for r in res if r.n_removed) >= 1, (kf, [r.n_removed for r in res])
    assert times["localized"] == len(blobs)
    # L stays near the generator's ground truth (the stream starts at the identity, as L_0 does)
    err_t = max(float(np.linalg.norm(np.array(r.pose).reshape(4, 4)[:3, 3] - T[:3, 3])) for r, T in zip(res, poses))
    err_r = max(float(np.arccos(np.clip((np.trace(np.array(r.pose).reshape(4, 4)[:3, :3].T @ T[:3, :3]) - 1) / 2, -1, 1)))
                for r, T in zip(res, poses))
    assert err_t < 0.2 and err_r < 0.03, (err_t, err_r)


def test_chain_odometry_equals_lb_odometry(data, reference):
    import locus_b200
    poses, blobs, prefill = data
    ref, _ = reference
    P = locus_b200.locus_params()
    n = blobs[0].size // STEP
    odo = locus_b200.OdometryB200(0, depth=3, max_points=n, max_point_step=STEP)
    _voxel(odo.voxel)
    odo.setGicpParams(**{k: getattr(P.odometry, k) for k, _ in locus_b200.GicpParams._fields_})
    for b in blobs:
        odo.submit(b, n, STEP, locus_b200.xyzi_fields())
    rs = [odo.next() for _ in blobs]
    odo.close()
    for r, e in zip(rs, ref):
        assert r.status == 0 and bool(r.has_pose) == (e["odometry"] is not None)
        if r.has_pose:
            assert _same_result(r.gicp, e["odometry"])


def test_set_source_cloud_equals_upload(data):
    import locus_b200
    poses, blobs, prefill = data
    vg = locus_b200.VoxelGridB200(); _voxel(vg)
    xyz = [np.ascontiguousarray(vg.filter(b, STEP, locus_b200.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
           for b in blobs[:2]]
    a, b, c = locus_b200.GicpB200(), locus_b200.GicpB200(), locus_b200.GicpB200()
    a.setInputSource(xyz[1]); a.prepareSource()
    cl = a.shareSource()
    b.setSourceCloud(cl)
    locus_b200.GicpB200.releaseCloud(cl)               # b holds its own reference
    a.setInputSource(xyz[0])                            # a switches to another object: the shared one stays intact
    for g in (b, c):
        g.setInputTarget(xyz[0])
    c.setInputSource(xyz[1])
    rb, rc = b.align(), c.align()
    assert _same_result(rb, rc)
    assert np.array_equal(b.transformSource(), c.transformSource())
    assert b.getFitnessScore(1.0) == c.getFitnessScore(1.0)
