"""Row f5 on the GPU: lb_gicp_statistical_outlier_removal / lb_gicp_radius_outlier_removal against the oracle's
restatement of PCL 1.10 (oracle/outlier_oracle.c), bit-exact: the same kept indices, the same per-point mean distances
and the same {mean, stddev, threshold}.  The neighbour sets are exact on both sides, the mean distance is a serial
double sum of correctly rounded sqrtf values in neighbour order, and the statistics are serial double sums in input
order on both sides."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fixtures as F
from test_outliers_cpu import _build_outlier_shim_harness, scene_with_outliers
from tools import gen_lidar as G

pytestmark = pytest.mark.gpu


def _handle(pts, which):
    import locus_b200
    g = locus_b200.GicpB200()
    if which == 0:
        g.setInputSource(pts)
    else:
        g.setInputTarget(pts)
    return g


def _check_sor(g, pts, which, mean_k, std_mul, negative):
    from oracle import outlier_oracle as O
    kept, md, st = g.statisticalOutlierRemoval(which, mean_k, std_mul, negative)
    rk, rmd, rst = O.statistical_outlier_removal(pts, mean_k, std_mul, negative)
    assert np.array_equal(md.view(np.uint32), rmd.view(np.uint32))
    assert np.array_equal(st.view(np.uint64), rst.view(np.uint64)), (st, rst)
    assert np.array_equal(kept, rk)
    return kept, md, st


def _check_radius(g, pts, which, radius, min_neighbors, dense, negative):
    from oracle import outlier_oracle as O
    kept = g.radiusOutlierRemoval(which, radius, min_neighbors, dense, negative)
    assert np.array_equal(kept, O.radius_outlier_removal(pts, radius, min_neighbors, dense, negative))
    return kept


def _c2_filtered_scan():
    """the filter's real input in LOCUS: a VoxelGrid-filtered 64 x 2048 scan (~30 k points)"""
    import locus_b200
    scene, poses, blobs = G.stream(2, 1)
    vg = locus_b200.VoxelGridB200()
    vg.setLeafSize(0.1088); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    f = vg.filter(blobs[0], 32, locus_b200.xyzi_fields())
    return np.ascontiguousarray(f).view(np.float32).reshape(-1, 8)[:, :3].copy()


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("negative", [False, True])
def test_sor_scene_with_outliers(which, negative):
    pts = scene_with_outliers(20000, 11, n_out=300)
    g = _handle(pts, which)
    kept, _, _ = _check_sor(g, pts, which, 10, 1.0, negative)
    assert 0 < len(kept) < len(pts)
    _check_sor(g, pts, which, 19, 2.5, negative)
    _check_sor(g, pts, which, 1, 0.0, negative)


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("dense", [True, False])
@pytest.mark.parametrize("negative", [False, True])
def test_radius_scene_with_outliers(which, dense, negative):
    pts = scene_with_outliers(20000, 12, n_out=300)
    g = _handle(pts, which)
    kept = _check_radius(g, pts, which, 0.15, 3, dense, negative)
    assert 0 < len(kept) < len(pts)
    _check_radius(g, pts, which, 0.4, 12, dense, negative)
    assert np.array_equal(_check_radius(g, pts, which, 0.15, 0, dense, False), np.arange(len(pts)))


def test_radius_boundary_and_duplicates():
    """points exactly r apart (d2 == r^2): counted by the dense branch only; duplicated points count once each"""
    centres = np.array([[10.0 * i, 0.0, 0.0] for i in range(6)], np.float32)
    pts = np.concatenate([centres, centres + np.float32([0.5, 0, 0])]).astype(np.float32)
    g = _handle(pts, 0)
    assert np.array_equal(_check_radius(g, pts, 0, 0.5, 1, True, False), np.arange(12))
    assert len(_check_radius(g, pts, 0, 0.5, 1, False, False)) == 0
    rng = np.random.default_rng(4)
    base = rng.uniform(-2, 2, (3000, 3)).astype(np.float32)
    dup = np.concatenate([base, base[:1000], base[:400]])[rng.permutation(4400)].copy()
    g = _handle(dup, 1)
    for dense in (True, False):
        _check_radius(g, dup, 1, 0.2, 2, dense, False)
    _check_sor(g, dup, 1, 10, 1.0, False)
    small = base[:11].copy()                                 # n = mean_k + 1
    _check_sor(_handle(small, 0), small, 0, 10, 1.0, False)


def test_c2_filtered_scan_host_and_device_memory():
    """SOR 10 / 1.0 and radius 0.15 / 3 (PointCloudFilter's settings) on a filtered scan; device-resident buffers give
    the bits of the host path, and two runs give identical bits"""
    import torch
    import locus_b200
    pts = _c2_filtered_scan()
    g = _handle(pts, 0)
    kept, md, st = _check_sor(g, pts, 0, 10, 1.0, False)
    kept2, md2, st2 = g.statisticalOutlierRemoval(0, 10, 1.0, False)
    assert np.array_equal(kept, kept2) and np.array_equal(md.view(np.uint32), md2.view(np.uint32)) and np.array_equal(st, st2)
    rk = {d: _check_radius(g, pts, 0, 0.15, 3, d, False) for d in (True, False)}
    assert np.array_equal(rk[True], g.radiusOutlierRemoval(0, 0.15, 3, True, False))
    L = locus_b200.lib()
    n = len(pts)
    d_idx = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_md = torch.zeros(n, dtype=torch.float32, device="cuda")
    d_st = torch.zeros(3, dtype=torch.float64, device="cuda")
    m = C.c_size_t(0)
    assert L.lb_gicp_statistical_outlier_removal(g._h, 0, 10, 1.0, 0, C.c_void_p(d_idx.data_ptr()), C.byref(m),
                                                 C.c_void_p(d_md.data_ptr()), C.c_void_p(d_st.data_ptr()),
                                                 locus_b200.LB_MEM_DEVICE) == 0
    assert m.value == len(kept) and np.array_equal(d_idx.cpu().numpy()[: m.value], kept)
    assert np.array_equal(d_md.cpu().numpy().view(np.uint32), md.view(np.uint32)) and np.array_equal(d_st.cpu().numpy(), st)
    # nullable outputs on the device path
    assert L.lb_gicp_statistical_outlier_removal(g._h, 0, 10, 1.0, 1, C.c_void_p(d_idx.data_ptr()), C.byref(m), None, None,
                                                 locus_b200.LB_MEM_DEVICE) == 0
    assert m.value == n - len(kept)
    for dense in (True, False):
        assert L.lb_gicp_radius_outlier_removal(g._h, 0, 0.15, 3, int(dense), 0, C.c_void_p(d_idx.data_ptr()), C.byref(m),
                                                locus_b200.LB_MEM_DEVICE) == 0
        assert np.array_equal(d_idx.cpu().numpy()[: m.value], rk[dense])


def test_merged_cloud_radius():
    """the merger's case: radius 0.1 / 3 on the ~390 k-point full-resolution cloud of three lidars, both branches, as
    source and as target, host and device memory"""
    import torch
    import locus_b200
    pts = G.merged_scan(7)
    assert len(pts) > 380_000
    g = locus_b200.GicpB200()
    g.setInputSource(pts); g.setInputTarget(pts)
    for dense in (True, False):
        k0 = _check_radius(g, pts, 0, 0.1, 3, dense, False)
        assert 0 < len(k0) < len(pts)
        assert np.array_equal(g.radiusOutlierRemoval(1, 0.1, 3, dense, False), k0)
        d_idx = torch.full((len(pts),), -1, dtype=torch.int32, device="cuda")
        m = C.c_size_t(0)
        assert locus_b200.lib().lb_gicp_radius_outlier_removal(g._h, 1, 0.1, 3, int(dense), 1, C.c_void_p(d_idx.data_ptr()),
                                                               C.byref(m), locus_b200.LB_MEM_DEVICE) == 0
        neg = d_idx.cpu().numpy()[: m.value]
        assert len(neg) + len(k0) == len(pts) and not np.isin(neg, k0).any()


def _align(g, src, tgt):
    g.setTransformationEpsilon(1e-3); g.setMaxCorrespondenceDistance(1.0); g.setMaximumIterations(20)
    g.setInputSource(src); g.setInputTarget(tgt)


def test_align_after_filters_is_unchanged():
    """the filter calls leave the clouds, their index and covariances as they were: the pose bits do not move"""
    import locus_b200
    box = F.hollow_cube(); moved = box.copy(); moved[:, 0] += np.float32(0.05); moved[:, 1] += np.float32(0.05)
    g1 = locus_b200.GicpB200(); _align(g1, moved, box)
    T1 = g1.align(); T1 = g1.getFinalTransformation()
    g2 = locus_b200.GicpB200(); _align(g2, moved, box)
    for which in (0, 1):
        g2.statisticalOutlierRemoval(which, 10, 1.0)
        g2.radiusOutlierRemoval(which, 0.15, 3, True)
        g2.radiusOutlierRemoval(which, 0.15, 3, False)
    g2.align()
    assert np.array_equal(g2.getFinalTransformation(), T1)
    for which in (0, 1):                                   # after an align (covariances cached) and before the next
        g2.statisticalOutlierRemoval(which, 5, 0.5, True)
        g2.radiusOutlierRemoval(which, 0.3, 8, False, True)
    g2.align()
    assert np.array_equal(g2.getFinalTransformation(), T1)


def test_errors_leave_state_unchanged():
    import locus_b200
    from locus_b200 import api
    g = locus_b200.GicpB200()
    for call, status in ((lambda: g.statisticalOutlierRemoval(0), -4), (lambda: g.statisticalOutlierRemoval(1), -5),
                         (lambda: g.radiusOutlierRemoval(0), -4), (lambda: g.radiusOutlierRemoval(1), -5)):
        with pytest.raises(api.LocusB200Error) as e:
            call()
        assert e.value.status == status
    pts = scene_with_outliers(2000, 13)
    g.setInputSource(pts)
    ref = _check_sor(g, pts, 0, 10, 1.0, False)
    for call, status in ((lambda: g.statisticalOutlierRemoval(0, 0), -1), (lambda: g.statisticalOutlierRemoval(0, 20), -9),
                         (lambda: g.radiusOutlierRemoval(0, 0.0), -1), (lambda: g.radiusOutlierRemoval(0, -1.0), -1),
                         (lambda: g.radiusOutlierRemoval(0, 0.1, -1), -1)):
        with pytest.raises(api.LocusB200Error) as e:
            call()
        assert e.value.status == status
    L = locus_b200.lib()
    m = C.c_size_t(7)
    assert L.lb_gicp_radius_outlier_removal(g._h, 2, 0.1, 3, 1, 0, C.c_void_p(1), C.byref(m), 0) == -1
    assert L.lb_gicp_statistical_outlier_removal(g._h, 0, 10, 1.0, 0, None, C.byref(m), None, None, 0) == -1
    g.setInputTarget(pts[:10])
    with pytest.raises(api.LocusB200Error) as e:
        g.statisticalOutlierRemoval(1, 10)                 # n < mean_k + 1
    assert e.value.status == -6
    assert g.cloudSize(0) == len(pts) and g.cloudSize(1) == 10
    again = _check_sor(g, pts, 0, 10, 1.0, False)
    assert all(np.array_equal(a, b) for a, b in zip(ref, again))


def test_outlier_shim_runs(tmp_path):
    """shim/b200_outlier_pcl.hpp as LOCUS calls it (in place, chained, negative, a cloud with is_dense = false) gives the
    oracle's points"""
    from oracle import outlier_oracle as O
    exe = _build_outlier_shim_harness()
    pts = _c2_filtered_scan()
    src = tmp_path / "in.bin"
    pts.tofile(src)
    pre = str(tmp_path) + os.sep
    r = subprocess.run([exe, str(src), pre], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert r.returncode == 0 and "ok=1" in r.stdout, (r.stdout, r.stderr)

    def load(name):
        return np.fromfile(pre + name, dtype=np.float32).reshape(-1, 3)
    sor = pts[O.statistical_outlier_removal(pts, 10, 1.0)[0]]
    assert np.array_equal(load("sor.bin"), sor)
    assert np.array_equal(load("sor_rad.bin"), sor[O.radius_outlier_removal(sor, 0.15, 3, dense=True)])
    assert np.array_equal(load("sor_neg.bin"), pts[O.statistical_outlier_removal(pts, 10, 1.0, negative=True)[0]])
    assert np.array_equal(load("rad_sparse.bin"), pts[O.radius_outlier_removal(pts, 0.1, 3, dense=False)])
