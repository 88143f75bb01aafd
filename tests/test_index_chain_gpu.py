"""The GICP index build as one stream-ordered chain (gather + grid on the device -> keys + occupancy + sort histograms
-> one scatter per sort pass -> reorder + cell offsets -> the two k-NN kernels): what is built on the index -- covariances
and exact nearest neighbours with ties -- against the oracle at every key width and on every path of the cell-size
choice, the pipeline against the blocking calls, and the number of kernels, memsets and copies one prepared cloud costs."""
import json
import os

import numpy as np
import pytest

import fixtures as F
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

# cells per axis at cell size 1.0 whose cell count needs exactly this many key bits
GRIDS = {8: (8, 8, 4), 9: (8, 8, 6), 16: (64, 32, 32), 17: (64, 64, 24), 25: (256, 256, 384)}


def _clustered(dims, seed, n_cells=3000):
    """1..7 points per occupied cell, both corner cells occupied (the grid is exactly `dims` at cell size 1), some exact
    duplicates (distance ties are broken by the original index), input order shuffled"""
    rng = np.random.default_rng(seed)
    dims = np.asarray(dims)
    cells = rng.integers(0, dims, size=(n_cells, 3))
    cells[0] = 0; cells[1] = dims - 1
    c = np.repeat(cells, rng.integers(1, 8, size=n_cells), axis=0)
    p = (c + rng.uniform(0.05, 0.95, size=c.shape)).astype(np.float32)
    p[0] = 0; p[1] = dims                                # the box is [0, dims]: floor(dims / 1.0) + 1 cells would be one too
    p[1] -= np.float32(0.5)                              # many, so the far corner sits inside the last cell
    p = np.concatenate([p, p[rng.integers(0, len(p), 300)]])
    return np.ascontiguousarray(p[rng.permutation(len(p))])


def _c2_scans(count):
    """filtered scans of bench.py's c2 stream (131072 rays, ~30 k voxels): lidar-like clouds, whose first probe round
    is accepted"""
    import locus_b200
    scene, poses, blobs = G.stream(2, count)
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(0.1088); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    return [np.ascontiguousarray(vg.filter(b, 32, locus_b200.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
            for b in blobs]


def _check_index(g, oracle, pts, k=20, seed=5):
    """covariances of the source (k-NN through the index, sums in neighbour order) and 1-NN on the target"""
    g.setCorrespondenceRandomness(k)
    g.setInputSource(pts); g.prepareSource()
    gc, oc = g.covariances(0), oracle.covariances(pts, k, 1e-3, 4)
    assert np.allclose(gc, oc, rtol=0, atol=1e-12)
    assert (gc == oc).mean() > 0.99
    rng = np.random.default_rng(seed)
    q = np.concatenate([pts[rng.integers(0, len(pts), 600)] + rng.normal(0, 0.3, (600, 3)).astype(np.float32),
                        pts[rng.integers(0, len(pts), 200)]]).astype(np.float32)
    g.setInputTarget(pts)
    idx, d2 = g.nearestTarget(q)
    oi, od = oracle.KdTree(pts).nn_batch(q)
    assert np.array_equal(d2, od) and np.array_equal(idx, oi)


@pytest.mark.parametrize("bits", sorted(GRIDS))
def test_key_widths_fixed_cell(oracle, bits):
    import locus_b200
    dims = GRIDS[bits]
    cells = int(np.prod(dims))
    assert max(1, (cells - 1).bit_length()) == bits
    pts = _clustered(dims, 300 + bits)
    g = locus_b200.GicpB200(); g.setIndexCellSize(1.0)
    _check_index(g, oracle, pts)
    assert g.kernelTime("cell_src")[0] == 1.0 and g.kernelTime("probe_rounds")[0] == 0
    _check_index(g, oracle, pts[::-1].copy())            # again on the handle's warm buffers


def test_automatic_cell_one_round(oracle):
    """a lidar scan: the device's first round is accepted once the handle has room for its marks, and the grid is the
    one a handle that ran the round from the host chose"""
    import locus_b200
    pts = _c2_scans(1)[0]
    cold = locus_b200.GicpB200()
    _check_index(cold, oracle, pts)
    g = locus_b200.GicpB200(); g.reserve(len(pts))
    r0 = g.kernelTime("probe_rounds")[0]
    _check_index(g, oracle, pts)
    assert g.kernelTime("probe_rounds")[0] - r0 == 2     # source and target, one round each
    assert g.kernelTime("cell_src")[0] == cold.kernelTime("cell_src")[0]
    assert np.array_equal(g.covariances(0), cold.covariances(0))


def test_rejected_first_round(oracle):
    """two dense blobs far apart: the bounding-box guess puts each in one cell, so more rounds follow (from the host)"""
    import locus_b200
    rng = np.random.default_rng(31)
    a = rng.uniform(0, 1, (3000, 3)); b = rng.uniform(0, 1, (3000, 3)) + 20.0
    pts = np.concatenate([a, b]).astype(np.float32)[rng.permutation(6000)]
    g = locus_b200.GicpB200(); g.reserve(len(pts))
    g.setInputSource(pts)
    assert g.kernelTime("probe_rounds")[0] > 1
    cell = g.kernelTime("cell_src")[0]
    _check_index(g, oracle, pts)
    assert g.kernelTime("cell_src")[0] == cell
    _check_index(g, oracle, F.random_scene(6000, 32))    # an accepted round after the rejected ones, same scratch


def test_tiny_and_single_cell_clouds(oracle):
    import locus_b200
    g = locus_b200.GicpB200(); g.reserve(1024)
    pts = np.random.default_rng(41).uniform(-1, 1, (7, 3)).astype(np.float32)
    _check_index(g, oracle, pts, k=5)                     # N <= 8: the first round stands whatever it counted
    g.setIndexCellSize(100.0)
    _check_index(g, oracle, F.random_scene(3000, 42), k=20)   # every point in one cell
    g.setIndexCellSize(0.0)
    line = np.zeros((500, 3), np.float32); line[:, 0] = np.linspace(0, 10, 500)
    _check_index(g, oracle, line, k=10)                   # a degenerate box: zero area


def test_non_finite_cloud_is_refused_and_the_cloud_kept(oracle):
    import locus_b200
    pts = F.random_scene(4000, 51)
    g = locus_b200.GicpB200(); g.reserve(len(pts))
    _check_index(g, oracle, pts)
    cov = g.covariances(0)
    bad = F.random_scene(5000, 52); bad[1234, 1] = np.nan
    with pytest.raises(locus_b200.LocusB200Error):
        g.setInputSource(bad)
    with pytest.raises(locus_b200.LocusB200Error):
        g.setInputTarget(bad)
    assert g.cloudSize(0) == len(pts) and np.array_equal(g.covariances(0), cov)
    _check_index(g, oracle, F.random_scene(5000, 53))     # and the scratch is clean for the next cloud


def test_target_equal_to_previous_source_is_adopted():
    import locus_b200
    scans = [F.random_scene(8000, 60 + i) for i in range(3)]

    def run(g):
        out = []
        g.setInputSource(scans[0]); g.setInputTarget(scans[1]); g.align()
        for i in (1, 2):
            g.setInputSource(scans[i]); g.setInputTarget(scans[i - 1])
            g.align()
            out.append(g.getFinalTransformation())
        return out

    g = locus_b200.GicpB200(); g.setMaximumIterations(5); g.reserve(8000)
    got = run(g)
    assert g.kernelTime("adopted_targets")[0] == 2
    ref = []
    for i in (1, 2):
        f = locus_b200.GicpB200(); f.setMaximumIterations(5)
        f.setInputSource(scans[i]); f.setInputTarget(scans[i - 1]); f.align()
        ref.append(f.getFinalTransformation())
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))


@pytest.mark.parametrize("sharing", [True, False])
def test_pipeline_equals_blocking_calls(sharing):
    import locus_b200
    scene = G.make_scene(3)
    poses = G.trajectory(3, 5)
    scans = [G.scan(scene, poses[i], 70 + i, beams=16, az=512) for i in range(5)]
    n = scans[0].size // 32
    cfg = dict(transformation_epsilon=1e-3, max_correspondence_distance=1.0, max_iterations=20)
    odo = locus_b200.OdometryB200(0, depth=3, max_points=n, max_point_step=32)
    odo.voxel.setLeafSize(0.3)
    odo.setGicpParams(**cfg); odo.setCloudSharing(sharing)
    for b in scans:
        odo.submit(b, n, 32, locus_b200.xyzi_fields())
    rs = [odo.next() for _ in scans]
    odo.close()
    assert all(r.status == 0 for r in rs)
    vg = locus_b200.VoxelGridB200(0); vg.setLeafSize(0.3)
    f = [np.ascontiguousarray(vg.filter(b, 32, locus_b200.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy() for b in scans]
    g = locus_b200.GicpB200(0)
    g.setTransformationEpsilon(1e-3); g.setMaxCorrespondenceDistance(1.0); g.setMaximumIterations(20)
    for i in range(1, 5):
        g.setInputSource(f[i]); g.setInputTarget(f[i - 1]); g.align()
        Tp = np.array(rs[i].gicp.final_transformation, dtype=np.float32).reshape(4, 4)
        assert np.array_equal(Tp, g.getFinalTransformation()), i


def test_launch_shape_of_a_prepared_cloud(tmp_path):
    """set_source + prepare_source of a ~30 k-point lidar scan on a reserved handle: gather, keys, one scatter per sort pass,
    reorder, two k-NN kernels; no memset, one device-to-host copy (the state block) and the host-to-device upload"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import locus_b200
    clouds = _c2_scans(4)
    g = locus_b200.GicpB200(); g.reserve(max(len(c) for c in clouds))
    for c in clouds[:2]:
        g.setInputSource(c); g.prepareSource()
    torch.cuda.synchronize()
    l0, r0 = g.launchCount(), g.kernelTime("probe_rounds")[0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in clouds:
            g.setInputSource(c); g.prepareSource()
        torch.cuda.synchronize()
    launches = (g.launchCount() - l0) / len(clouds)
    assert g.kernelTime("probe_rounds")[0] - r0 == len(clouds)
    path = os.path.join(str(tmp_path), "prepare.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        ev = json.load(fh)["traceEvents"]
    ours = [e for e in ev if e.get("cat") == "kernel" and "lb::" in e["name"]]
    names = [e["name"].split("lb::")[1].split("(")[0].split("<")[0] for e in ours]
    per = {n: names.count(n) / len(clouds) for n in set(names)}
    sort_passes = per.pop("rs_onesweep_kernel")
    assert 2.0 <= sort_passes <= 3.0, per                  # 16..24 key bits, scan by scan
    assert per == {"gather_cloud_kernel": 1.0, "grid_index_keys_kernel": 1.0, "grid_reorder_kernel": 1.0,
                   "knn_cov_quadreg_kernel": 1.0, "knn_cov_tail_kernel": 1.0}, per
    assert launches == 5 + sort_passes
    assert sum(1 for e in ev if e.get("cat") == "gpu_memset") == 0
    copies = [e["name"] for e in ev if e.get("cat") == "gpu_memcpy"]
    assert sum("DtoH" in c for c in copies) == len(clouds), copies        # the state block, once per cloud
    assert len(copies) <= 2 * len(clouds), copies                         # the rest is the upload of the host array
