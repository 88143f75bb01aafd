"""Row f5 without a GPU: the oracle's restatement of pcl::StatisticalOutlierRemoval / pcl::RadiusOutlierRemoval
(oracle/outlier_oracle.c) against an independent numpy + scipy.cKDTree restatement of the same PCL 1.10 semantics.
Kept indices are identical; per-point mean distances and the statistics are bit-identical.  The numpy side takes the
radius filter's dense branch in its count form (at least min_neighbors + 1 points with (double)d2 <= r^2), the oracle in
PCL's literal k-NN form, so the tests also show that the two forms agree -- the GPU kernel uses the count form."""
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import conftest
import fixtures as F

ROOT = conftest.ROOT


@pytest.fixture(scope="module")
def outliers():
    from oracle import outlier_oracle
    outlier_oracle.build()
    return outlier_oracle


def _d2(q, pts):
    """float32 squared distances ((dx*dx)+(dy*dy))+(dz*dz), no FMA (FLANN L2_Simple<float>)"""
    d = (pts - q).astype(np.float32)
    s = d[:, 0] * d[:, 0]
    s = s + d[:, 1] * d[:, 1]
    return s + d[:, 2] * d[:, 2]


def _candidates(tree, pts, radii):
    """every point within radii[i] (double) of pts[i], with a margin that covers float32 rounding of d2"""
    return tree.query_ball_point(pts.astype(np.float64), radii * (1.0 + 1e-5) + 1e-30)


def np_mean_dist(pts, mean_k):
    tree = cKDTree(pts.astype(np.float64))
    dk, _ = tree.query(pts.astype(np.float64), k=mean_k + 1)
    cand = _candidates(tree, pts, dk[:, -1])
    out = np.zeros(len(pts), np.float32)
    for i, c in enumerate(cand):
        c = np.asarray(c, np.int64)
        d2 = _d2(pts[i], pts[c])
        order = np.lexsort((c, d2))[: mean_k + 1]                      # ascending (d2, index)
        s = np.cumsum(np.sqrt(d2[order][1:]).astype(np.float64))[-1]   # sqrtf, then a serial double sum
        out[i] = np.float32(s / mean_k)
    return out


def np_sor_threshold(dist, std_mul, negative):
    n = len(dist)
    s = np.cumsum(dist.astype(np.float64))[-1]
    sq = np.cumsum((dist * dist).astype(np.float64))[-1]              # float product, double sum
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = s / n
        var = (sq - s * s / n) / (n - 1.0)
        std = np.sqrt(np.float64(var))
    thr = mean + std_mul * std
    d = dist.astype(np.float64)
    with np.errstate(invalid="ignore"):
        removed = (d <= thr) if negative else (d > thr)
    return np.nonzero(~removed)[0].astype(np.int32), np.array([mean, std, thr])


def np_radius(pts, radius, min_neighbors, dense, negative):
    tree = cKDTree(pts.astype(np.float64))
    cand = _candidates(tree, pts, np.full(len(pts), radius))
    r2 = radius * radius
    keep = []
    for i, c in enumerate(cand):
        d2 = _d2(pts[i], pts[np.asarray(c, np.int64)])
        cnt = int((d2.astype(np.float64) <= r2).sum()) if dense else int((d2 < np.float32(r2)).sum())
        if (cnt >= min_neighbors + 1) != bool(negative):
            keep.append(i)
    return np.array(keep, np.int32)


def scene_with_outliers(n, seed, n_out=60):
    rng = np.random.default_rng(seed)
    p = F.random_scene(n, seed, extent=(4.0, 3.0, 1.5))
    out = rng.uniform(-6, 6, (n_out, 3)).astype(np.float32)
    p = np.concatenate([p, out])
    return p[rng.permutation(len(p))].copy()


@pytest.mark.parametrize("mean_k,std_mul,negative", [(10, 1.0, False), (10, 1.0, True), (5, 0.5, False), (19, 2.0, False)])
def test_sor_oracle_vs_numpy(outliers, mean_k, std_mul, negative):
    pts = scene_with_outliers(3000, 1)
    kept, md, st = outliers.statistical_outlier_removal(pts, mean_k, std_mul, negative)
    ref_md = np_mean_dist(pts, mean_k)
    assert np.array_equal(md.view(np.uint32), ref_md.view(np.uint32))
    ref_kept, ref_st = np_sor_threshold(ref_md, std_mul, negative)
    assert np.array_equal(st.view(np.uint64), ref_st.view(np.uint64))
    assert np.array_equal(kept, ref_kept) and 0 < len(kept) < len(pts)


def test_sor_duplicates_and_smallest_cloud(outliers):
    rng = np.random.default_rng(2)
    base = rng.uniform(-1, 1, (400, 3)).astype(np.float32)
    pts = np.concatenate([base, base[:150], base[:40]])[rng.permutation(590)].copy()     # twins and triplets
    kept, md, st = outliers.statistical_outlier_removal(pts, 10, 1.0)
    ref_md = np_mean_dist(pts, 10)
    assert np.array_equal(md.view(np.uint32), ref_md.view(np.uint32))
    rk, rst = np_sor_threshold(ref_md, 1.0, False)
    assert np.array_equal(kept, rk) and np.array_equal(st.view(np.uint64), rst.view(np.uint64))
    # n = mean_k + 1: every neighbourhood is the whole cloud
    small = base[:11].copy()
    kept, md, st = outliers.statistical_outlier_removal(small, 10, 1.0)
    ref_md = np_mean_dist(small, 10)
    rk, rst = np_sor_threshold(ref_md, 1.0, False)
    assert np.array_equal(md.view(np.uint32), ref_md.view(np.uint32)) and np.array_equal(kept, rk)
    assert np.array_equal(st.view(np.uint64), rst.view(np.uint64))


def test_sor_single_point_threshold_is_nan(outliers):
    """PCL's n == 1 case (variance = 0 / 0): the threshold is NaN, no comparison holds, every point is kept"""
    for negative in (False, True):
        kept, st = outliers.sor_threshold(np.array([0.25], np.float32), 1.0, negative)
        assert list(kept) == [0] and np.isnan(st[1]) and np.isnan(st[2]) and st[0] == 0.25
        rk, rst = np_sor_threshold(np.array([0.25], np.float32), 1.0, negative)
        assert np.array_equal(kept, rk)


@pytest.mark.parametrize("radius,min_neighbors", [(0.15, 3), (0.1, 3), (0.3, 8)])
@pytest.mark.parametrize("dense", [True, False])
@pytest.mark.parametrize("negative", [False, True])
def test_radius_oracle_vs_count_form(outliers, radius, min_neighbors, dense, negative):
    pts = scene_with_outliers(4000, 3)
    kept = outliers.radius_outlier_removal(pts, radius, min_neighbors, dense, negative)
    assert np.array_equal(kept, np_radius(pts, radius, min_neighbors, dense, negative))
    assert 0 < len(kept) < len(pts)


def test_radius_boundary_at_exactly_r(outliers):
    """pairs of points exactly r = 0.5 apart (d2 = 0.25 in float32, == r^2 in double): the dense branch counts the
    partner (!(0.25 < 0.25)), the radius-search branch does not (0.25 < float(0.25) is false)"""
    centres = np.array([[10.0 * i, 0.0, 0.0] for i in range(6)], np.float32)
    pts = np.concatenate([centres, centres + np.float32([0.5, 0, 0])]).astype(np.float32)
    assert (_d2(pts[0], pts[6:7]) == np.float32(0.25)).all()
    assert np.array_equal(outliers.radius_outlier_removal(pts, 0.5, 1, dense=True), np.arange(12))
    assert len(outliers.radius_outlier_removal(pts, 0.5, 1, dense=False)) == 0
    assert len(outliers.radius_outlier_removal(pts, 0.5, 1, dense=True, negative=True)) == 0
    assert np.array_equal(outliers.radius_outlier_removal(pts, 0.5, 1, dense=False, negative=True), np.arange(12))
    for dense in (True, False):
        assert np.array_equal(outliers.radius_outlier_removal(pts, 0.5, 1, dense), np_radius(pts, 0.5, 1, dense, False))


def test_radius_duplicates_and_min_neighbors_zero(outliers):
    rng = np.random.default_rng(4)
    base = rng.uniform(-2, 2, (500, 3)).astype(np.float32)
    pts = np.concatenate([base, base[:200], base[:200]])[rng.permutation(900)].copy()
    for dense in (True, False):
        assert np.array_equal(outliers.radius_outlier_removal(pts, 0.2, 2, dense), np_radius(pts, 0.2, 2, dense, False))
        assert np.array_equal(outliers.radius_outlier_removal(pts, 0.2, 0, dense), np.arange(len(pts)))     # keeps all
    assert len(outliers.radius_outlier_removal(pts, 0.2, len(pts), True)) == 0          # more than n neighbours: none


def test_error_cases(outliers):
    pts = scene_with_outliers(100, 5, n_out=0)
    with pytest.raises(ValueError):
        outliers.statistical_outlier_removal(pts, 0)
    with pytest.raises(ValueError):
        outliers.statistical_outlier_removal(pts[:10], 10)            # n < mean_k + 1
    for r in (0.0, -0.1):
        with pytest.raises(ValueError):
            outliers.radius_outlier_removal(pts, r, 3)
    with pytest.raises(ValueError):
        outliers.radius_outlier_removal(pts, 0.1, -1)


def _build_outlier_shim_harness():
    out = os.path.join(ROOT, "tests", "_build", "outlier_shim_harness")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "pcl_stub"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "shim"),
                           os.path.join(ROOT, "tests", "outlier_shim_harness.cpp"), "-L", os.path.join(ROOT, "locus_b200"),
                           "-llocus_b200", "-Wl,-rpath," + os.path.join(ROOT, "locus_b200"), "-pthread", "-o", out])
    return out


def test_outlier_shim_compiles_and_links():
    """shim/b200_outlier_pcl.hpp parses and links against the PCL mock and the C ABI; without a GPU the filters'
    constructor throws -- no CPU path behind the seam"""
    import locus_b200
    exe = _build_outlier_shim_harness()
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
    if locus_b200.device_count() <= 0:
        assert r.returncode == 3 and "no_device=" in r.stdout
    else:
        assert r.returncode == 0 and "constructed=1" in r.stdout
