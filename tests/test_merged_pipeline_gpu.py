"""Three lidars per scan through lb_locus / lb_odometry (lb_*_submit_merged), on the GPU.

Streams of 16-beam scans from tools/gen_lidar.merged_stream: per scan the three sensor-frame clouds of the lidars
of gen_lidar.LIDAR_MOUNTS and their sensor -> base_link transforms, with PassThrough and BodyFilter set on the
pipeline's voxel handle.
* lb_locus_submit_merged at depth 1 (host input) and depth 4 (device input) equals blocking calls --
  VoxelGridB200.filterMerged, GicpB200 and SubmapB200 driven by oracle/locus_oracle.py (tools/front_end_oracle.py for
  the front end) -- bit for bit: every odometry and localization result, O / I / L, the keyframe flags, the filtered
  clouds and the final map.  Once in the default configuration and once in the shipped front end (normals k = 20,
  adaptive voxelization, ICP covariance).
* The lidar count changes mid-stream (3 -> 2 -> 1 -> 3, a lidar that comes back passed last, an empty input, and in
  the default configuration an all-empty scan): still bit-equal to the blocking calls fed the same clouds in the same
  order.
* One cloud without a transform through submit_merged is bit-equal to submit, for both pipelines.
* lb_odometry_submit_merged's poses equal lb_locus's odometry results.
* From the second scan to the end of a stream whose lidar count grows, the process makes no device allocation.
* A two-input scan in a layout other than x, y, z, intensity reports LB_ERR_UNSUPPORTED and changes no state.
"""
import ctypes as C

import numpy as np
import pytest

from tools import front_end_oracle as FE
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

STEP = 32
LEAF0 = 0.25
MAP_RES = 0.1
SEED = 5
N_SCANS = 14
BEAMS, AZ = 16, 1024
BODY = ([-0.6, -0.45, -0.5], [0.6, 0.45, 1.0])
PARAMS = dict(translation_threshold_kf=0.6, rotation_threshold_kf=0.3, refresh_every=2, window_half_size=9.0)
SHIPPED = {**PARAMS, **FE.SHIPPED, "icp_covariance": {"enabled": 1, "max_covariance": 0.01}}
RESULT_FIELDS = ("final_transformation", "transformation", "converged", "iterations", "n_correspondences", "delta",
                 "n_objective_evals", "n_inner_iterations", "status")
LB_ERR_UNSUPPORTED = -9

# lidar lists per scan (indices into the three mounts, in merge order; None = an empty input)
THREE = [[0, 1, 2]] * N_SCANS
VARYING = [[0, 1, 2], [0, 1, 2], [0, 1], [0], [0, 1, 2], [0, 2], [0, 2, 1], [0, None, 2], [], [0, 1, 2], [1, 2],
           [1, 2, 0], [1, 2, 0], [0, 1, 2]]
VARYING_SHIPPED = [x if x else [0, 1, 2] for x in VARYING]       # an all-empty scan would clamp the adaptive leaf


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _bits(a):
    return np.asarray(a, np.float64).reshape(-1).view(np.uint64)


def _same_result(a, b):
    for f in RESULT_FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        if f in ("final_transformation", "transformation"):
            if not np.array_equal(_u32(np.array(x, np.float32)), _u32(np.array(y, np.float32))):
                return False
        elif x != y:
            return False
    return True


def _same_nan(a, b):
    a = np.asarray(a, np.float64).reshape(-1); b = np.asarray(b, np.float64).reshape(-1)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
        np.array_equal(_bits(np.where(np.isnan(a), 0, a)), _bits(np.where(np.isnan(b), 0, b)))


@pytest.fixture(scope="module")
def data():
    _, poses, scans, mounts = G.merged_stream(SEED, N_SCANS, beams=BEAMS, az=AZ)
    return poses, scans, mounts


def _inputs(data, lists):
    """per scan: [(blob, transform)] in merge order; an empty input is a zero-length blob"""
    _, scans, mounts = data
    empty = np.zeros(0, np.uint8)
    out = []
    for k, li in enumerate(lists):
        if not li:
            out.append([(empty, mounts[0]), (empty, mounts[1]), (empty, mounts[2])])
        else:
            out.append([(empty, mounts[0]) if i is None else (scans[k][i], mounts[i]) for i in li])
    return out


def _setup(v, leaf=LEAF0):
    v.setLeafSize(leaf); v.setFilterFieldName("z"); v.setFilterLimits(-100.0, 100.0)
    v.setInputPassThrough("z", -100.0, 100.0)
    v.setBodyFilter(BODY[0], BODY[1], 0.0)


def _gicp(params):
    import locus_b200
    g = locus_b200.GicpB200()
    C.memmove(C.byref(g._p), C.byref(params), C.sizeof(params))
    g._apply()
    return g


def _max_points(inputs):
    return max(sum(b.size // STEP for b, _ in s) for s in inputs)


def _sequential(inputs, kw):
    """the chain as blocking calls: filterMerged, then GicpB200 / SubmapB200 driven by FrontEndChain"""
    import locus_b200
    P = locus_b200.locus_params(**kw)
    shipped = P.front_end.normals_k != 0
    icp = bool(P.icp_covariance.enabled)
    vg = locus_b200.VoxelGridB200()
    _setup(vg)
    odo, loc = _gicp(P.odometry), _gicp(P.localization)
    nrm = locus_b200.GicpB200()
    m = locus_b200.SubmapB200(0, MAP_RES)
    chain = FE.FrontEndChain(P, np.float32(LEAF0))
    no = dict(normal_off=12) if shipped else {}
    out, prev = [], None
    for scan in inputs:
        leaf = chain.next_leaf
        vg.setLeafSize(float(leaf))
        f = vg.filterMerged([b for b, _ in scan], STEP, locus_b200.xyzi_fields(), [T for _, T in scan])
        xyz = np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()
        chain.filtered(len(xyz))
        rec = {"odometry": None, "localization": None, "icp": None, "leaf": leaf, "filtered": np.ascontiguousarray(f).copy()}
        if len(xyz) == 0:               # an empty scan: no cloud, no state change, no odometry target for the next
            rec.update(chain.scan(False, None, None, None, None))
            prev = None
        else:
            if shipped:
                nrm.setInputSource(xyz)
                cloud = np.ascontiguousarray(np.hstack([xyz, nrm.computeNormals(0, P.front_end.normals_k)[:, :3]]))
            else:
                cloud = xyz
            odoT = None
            if prev is not None:
                odo.setInputSource(cloud, **no); odo.setInputTarget(prev, **no)
                rec["odometry"] = odo.align()
                odoT = odo.getFinalTransformation()
            loc.setInputSource(cloud, **no)

            def localize(Gs):
                loc.setTargetSubmap(m)
                rec["localization"] = loc.align(Gs)
                if icp:
                    rec["icp"] = loc.icpCovariance(normal_rotation=chain.normal_rotation, max_covariance=0.01)
                return loc.getFinalTransformation()

            def insert(T):
                if shipped:
                    t = loc.transformSource(T, with_normals=True)
                    return m.InsertPointsWithNormals(t[:, :3], t[:, 3:])
                return m.InsertPoints(loc.transformSource(T))

            rec.update(chain.scan(True, odoT, localize, insert, lambda c, half: m.Refresh(c, half)))
            prev = cloud
        rec["map_size"] = m.size()
        if icp:
            rec["condition_number"] = chain.published_condition_number(rec["icp"])
        out.append(rec)
    pts = m.points()
    m.close()
    return out, pts


def _chain(inputs, kw, depth, device_input=False):
    import locus_b200
    import torch
    m = locus_b200.SubmapB200(0, MAP_RES)
    mp = _max_points(inputs)
    ch = locus_b200.LocusB200(m, 0, depth=depth, max_points=mp, max_point_step=STEP, **kw)
    _setup(ch.voxel)
    keep, outs = [], []
    for scan in inputs:
        n = sum(b.size // STEP for b, _ in scan)
        if device_input:
            d = [torch.from_numpy(b).cuda() if b.size else None for b, _ in scan]
            fo = torch.zeros(max(n, 1) * STEP, dtype=torch.uint8, device="cuda")
            ch.submit_merged([(0, 0) if x is None else (x.data_ptr(), x.numel() // STEP) for x in d], STEP,
                             locus_b200.xyzi_fields(), [T for _, T in scan], mem=locus_b200.LB_MEM_DEVICE,
                             filtered_out=fo.data_ptr(), mem_filtered=locus_b200.LB_MEM_DEVICE)
            keep.append(d)
        else:
            fo = np.zeros(max(n, 1) * STEP, np.uint8)
            ch.submit_merged([b for b, _ in scan], STEP, locus_b200.xyzi_fields(), [T for _, T in scan], filtered_out=fo)
        outs.append(fo)
    res = [ch.next() for _ in inputs]
    ch.close()
    filtered = [(o.cpu().numpy() if hasattr(o, "cpu") else o)[: r.n_filtered * STEP] for o, r in zip(outs, res)]
    pts = m.points()
    m.close()
    return res, filtered, pts


def _compare(res, filtered, pts, ref, ref_pts, icp):
    assert [r.ticket for r in res] == list(range(len(ref)))
    for k, (r, e) in enumerate(zip(res, ref)):
        assert r.status == 0, (k, r.error)
        assert np.float32(r.leaf_size) == e["leaf"], k
        assert np.array_equal(filtered[k], e["filtered"].reshape(-1)), k
        assert r.has_odometry == (e["odometry"] is not None), k
        if r.has_odometry:
            assert _same_result(r.odometry, e["odometry"]), k
        assert r.has_localization == e["has_localization"], k
        if r.has_localization:
            assert _same_result(r.localization, e["localization"]), k
        for f in ("odometry_accepted", "correction_accepted", "keyframe", "n_inserted", "n_removed", "map_size"):
            assert getattr(r, f) == e[f], (k, f)
        assert np.array_equal(_bits(r.odometry_pose), _bits(e["O"])), k
        assert np.array_equal(_bits(r.incremental), _bits(e["I"])), k
        assert np.array_equal(_bits(r.pose), _bits(e["L"])), k
        if icp:
            assert r.has_icp_covariance == (e["icp"] is not None), k
            if e["icp"] is not None:
                assert _same_nan(np.array(r.icp_covariance), e["icp"]["covariance"]), k
                assert r.icp_covariance_flags == e["icp"]["flags"], k
            assert _same_nan(r.condition_number, e["condition_number"]), k
    assert np.array_equal(_u32(pts), _u32(ref_pts))


CONFIGS = {"default": PARAMS, "shipped": SHIPPED}


@pytest.fixture(scope="module")
def blocking(data):
    memo = {}

    def get(name, lists):
        key = (name, str(lists))
        if key not in memo:
            memo[key] = _sequential(_inputs(data, lists), CONFIGS[name])
        return memo[key]
    return get


@pytest.mark.parametrize("config", ["default", "shipped"])
@pytest.mark.parametrize("depth", [1, 4])
def test_three_lidars_equal_blocking_calls(data, blocking, config, depth):
    inputs = _inputs(data, THREE)
    ref, ref_pts = blocking(config, THREE)
    res, filtered, pts = _chain(inputs, CONFIGS[config], depth, device_input=(depth == 4))
    _compare(res, filtered, pts, ref, ref_pts, config == "shipped")
    assert sum(r.keyframe for r in res) >= 2 and all(r.has_localization for r in res[1:])
    poses = data[0]
    err_t = max(float(np.linalg.norm(np.array(r.pose).reshape(4, 4)[:3, 3] - T[:3, 3])) for r, T in zip(res, poses))
    assert err_t < 0.2, err_t


@pytest.mark.parametrize("config", ["default", "shipped"])
@pytest.mark.parametrize("depth", [1, 4])
def test_varying_lidar_count_equals_blocking_calls(data, blocking, config, depth):
    lists = VARYING if config == "default" else VARYING_SHIPPED
    inputs = _inputs(data, lists)
    ref, ref_pts = blocking(config, lists)
    res, filtered, pts = _chain(inputs, CONFIGS[config], depth, device_input=(depth == 4))
    _compare(res, filtered, pts, ref, ref_pts, config == "shipped")
    if config == "default":
        e = VARYING.index([])
        assert res[e].n_filtered == 0 and not res[e].keyframe and not res[e].has_localization
        assert np.array_equal(_bits(res[e].pose), _bits(res[e - 1].pose)) and res[e].map_size == res[e - 1].map_size
        assert not res[e + 1].has_odometry


def test_one_cloud_without_transform_equals_submit(data):
    import locus_b200
    _, scans, _ = data
    blobs = [s[0] for s in scans]
    n = blobs[0].size // STEP
    out = {}
    for how in ("submit", "merged"):
        m = locus_b200.SubmapB200(0, MAP_RES)
        ch = locus_b200.LocusB200(m, 0, depth=2, max_points=n, max_point_step=STEP, **PARAMS)
        odo = locus_b200.OdometryB200(0, depth=2, max_points=n, max_point_step=STEP)
        for v in (ch.voxel, odo.voxel):
            _setup(v)
        for b in blobs:
            for p in (ch, odo):
                if how == "submit":
                    p.submit(b, n, STEP, locus_b200.xyzi_fields())
                else:
                    p.submit_merged([b], STEP, locus_b200.xyzi_fields())
        out[how] = ([ch.next() for _ in blobs], [odo.next() for _ in blobs], m.points())
        ch.close(); odo.close(); m.close()
    (la, oa, pa), (lb, ob, pb) = out["submit"], out["merged"]
    assert np.array_equal(_u32(pa), _u32(pb))
    for a, b in zip(la, lb):
        assert a.status == b.status == 0 and a.n_filtered == b.n_filtered and a.keyframe == b.keyframe
        assert a.has_odometry == b.has_odometry and (not a.has_odometry or _same_result(a.odometry, b.odometry))
        assert a.has_localization == b.has_localization and (not a.has_localization or _same_result(a.localization, b.localization))
        assert np.array_equal(_bits(a.pose), _bits(b.pose)) and np.array_equal(_bits(a.odometry_pose), _bits(b.odometry_pose))
    for a, b in zip(oa, ob):
        assert a.status == b.status == 0 and a.has_pose == b.has_pose and a.n_filtered == b.n_filtered
        assert not a.has_pose or _same_result(a.gicp, b.gicp)


def test_odometry_merged_equals_locus_odometry(data):
    import locus_b200
    inputs = _inputs(data, VARYING)
    mp = _max_points(inputs)
    res, _, _ = _chain(inputs, PARAMS, 2)
    P = locus_b200.locus_params(**PARAMS)
    odo = locus_b200.OdometryB200(0, depth=3, max_points=mp, max_point_step=STEP)
    _setup(odo.voxel)
    odo.setGicpParams(**{k: getattr(P.odometry, k) for k, _ in locus_b200.GicpParams._fields_})
    for scan in inputs:
        odo.submit_merged([b for b, _ in scan], STEP, locus_b200.xyzi_fields(), [T for _, T in scan])
    rs = [odo.next() for _ in inputs]
    odo.close()
    assert sum(r.has_pose for r in rs) >= len(inputs) - 4
    for r, e in zip(rs, res):
        assert r.status == 0 and bool(r.has_pose) == bool(e.has_odometry) and r.n_filtered == e.n_filtered
        if r.has_pose:
            assert _same_result(r.gicp, e.odometry)


def test_no_device_allocation_when_the_lidar_count_changes(data):
    import locus_b200
    lists = [[0, 1], [0, 1], [0, 1, 2], [0], [], [1, 2, 0], [0, 1, 2], [2]]
    inputs = _inputs(data, lists)
    mp = _max_points(inputs)
    probe = locus_b200.GicpB200()
    # one registration worker, so that the first two scans have used every handle once (a worker's first index build
    # sizes its sort's look-back state: a first use, not a change of the lidar count)
    odo = locus_b200.OdometryB200(0, depth=1, max_points=mp, max_point_step=STEP)
    _setup(odo.voxel)
    for scan in inputs[:2]:
        odo.submit_merged([b for b, _ in scan], STEP, locus_b200.xyzi_fields(), [T for _, T in scan])
    rs = [odo.next() for _ in range(2)]
    a0 = probe.kernelTime("dbuf_allocs")[0]
    for scan in inputs[2:]:
        odo.submit_merged([b for b, _ in scan], STEP, locus_b200.xyzi_fields(), [T for _, T in scan])
    rs += [odo.next() for _ in inputs[2:]]
    a1 = probe.kernelTime("dbuf_allocs")[0]
    odo.close()
    assert all(r.status == 0 for r in rs)
    assert rs[2].n_filtered > rs[1].n_filtered            # the third lidar arrived: a larger raw and filtered scan
    assert a1 == a0, (a0, a1)


def test_non_xyzi_layout_is_refused_in_the_result(data):
    import locus_b200
    inputs = _inputs(data, [[0, 1, 2], [0, 1], [0, 1, 2], [0, 1, 2]])
    m = locus_b200.SubmapB200(0, MAP_RES)
    ch = locus_b200.LocusB200(m, 0, depth=2, max_points=_max_points(inputs), max_point_step=STEP, **PARAMS)
    _setup(ch.voxel)
    f32 = locus_b200.api.LB_FLOAT32
    xyz_only = [("x", 0, f32, 1), ("y", 4, f32, 1), ("z", 8, f32, 1)]
    for k, scan in enumerate(inputs):
        f = xyz_only if k == 1 else locus_b200.xyzi_fields()
        ch.submit_merged([b for b, _ in scan], STEP, f, [T for _, T in scan])
    res = [ch.next() for _ in inputs]
    ch.close(); m.close()
    bad, before = res[1], res[0]
    assert res[0].status == 0 and res[2].status == 0 and res[3].status == 0
    assert bad.status == LB_ERR_UNSUPPORTED and b"x, y, z, intensity" in bad.error
    assert bad.n_filtered == 0 and not bad.keyframe and not bad.has_localization and not bad.has_odometry
    assert np.array_equal(_bits(bad.pose), _bits(before.pose)) and np.array_equal(_bits(bad.odometry_pose), _bits(before.odometry_pose))
    assert bad.map_size == before.map_size
    assert not res[2].has_odometry and res[3].has_odometry            # as after any failed VoxelGrid
