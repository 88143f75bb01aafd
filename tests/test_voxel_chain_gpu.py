"""VoxelGrid chain (bbox -> keys + sort histograms -> one scatter per sort pass -> segment/centroid): the sort's key
width across pass boundaries, the sort-width retry of a handle whose previous call needed fewer passes, and the number
of kernels one call enqueues.  Every result bit-exact against the oracle."""
import numpy as np
import pytest

from tools import gen_lidar as G

pytestmark = pytest.mark.gpu

# grids (cells per axis at leaf 1.0) whose cell count needs exactly this many key bits
GRIDS = {8: (8, 8, 3), 9: (8, 8, 6), 16: (64, 32, 24), 17: (64, 64, 24), 24: (256, 256, 192), 25: (256, 256, 384)}


def _key_bits(dims):
    cells = int(np.prod(dims))
    return max(1, cells.bit_length())


def _cloud(dims, seed, n_vox=6000):
    """points clustered 1..7 to a voxel, the two corner cells occupied so that the grid is exactly `dims` at leaf 1"""
    rng = np.random.default_rng(seed)
    dims = np.asarray(dims)
    cells = rng.integers(0, dims, size=(n_vox, 3))
    cells[0] = 0; cells[1] = dims - 1
    reps = rng.integers(1, 8, size=n_vox)
    c = np.repeat(cells, reps, axis=0)
    p = np.zeros((len(c), 8), np.float32)
    p[:, :3] = (c + rng.uniform(0.05, 0.95, size=(len(c), 3))).astype(np.float32)
    p[:, 4] = rng.uniform(0.0, 100.0, len(c)).astype(np.float32)
    p = p[rng.permutation(len(p))]                # voxels' points scattered through the input order
    return np.ascontiguousarray(p).view(np.uint8).reshape(-1)


def _filter(vg, blob, min_pts=0):
    import locus_b200
    from oracle import oracle as O
    vg.setMinimumPointsNumberPerVoxel(min_pts)
    out, vidx = vg.filter(blob, 32, locus_b200.xyzi_fields(), want_voxel_idx=True)
    r = O.voxel_filter(blob, 32, 1.0, float_fields=G.FLOAT_FIELDS, min_points_per_voxel=min_pts)
    assert r["rc"] == 0
    assert np.array_equal(vidx, r["voxel_idx"])
    assert np.array_equal(out, r["out"])
    assert [int(v) for v in r["div_b"]] == [int(v) for v in _dims_of(blob)]
    return out


def _dims_of(blob):
    a = blob.view(np.float32).reshape(-1, 8)[:, :3]
    return np.floor(a.max(0)).astype(np.int64) - np.floor(a.min(0)).astype(np.int64) + 1


@pytest.mark.parametrize("bits", sorted(GRIDS))
@pytest.mark.parametrize("min_pts", [0, 3])
def test_key_width_across_pass_boundaries(bits, min_pts):
    import locus_b200
    dims = GRIDS[bits]
    assert _key_bits(dims) == bits
    blob = _cloud(dims, 100 + bits)
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(1.0)
    out = _filter(vg, blob, min_pts)
    assert out.shape[0] > 100
    _filter(vg, blob, min_pts)                    # again on a handle that enqueues exactly the passes the key needs


def test_sort_width_retry():
    """the handle enqueues the passes its previous call needed; a wider key re-runs the chain with all four"""
    import locus_b200
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(1.0)
    small, wide = _cloud(GRIDS[8], 7), _cloud(GRIDS[17], 8)
    _filter(vg, small)
    _filter(vg, small)
    l0 = vg.launchCount()
    _filter(vg, wide)
    assert vg.launchCount() - l0 == (3 + 1) + (3 + 4)       # one pass enqueued, three needed: the chain runs again
    l0 = vg.launchCount()
    _filter(vg, wide)
    assert vg.launchCount() - l0 == 3 + 3
    _filter(vg, small)                            # fewer passes than enqueued: the extra ones return at once
    _filter(vg, _cloud(GRIDS[25], 9), min_pts=2)


@pytest.mark.parametrize("bits", [8, 16, 17, 25])
def test_launches_per_call(bits):
    """bbox, keys (+ sort histograms), one scatter per pass, segment/centroid: 3 + passes kernels and no copy; the first
    call of a handle enqueues four passes.  min_points_per_voxel adds none."""
    import locus_b200
    blob = _cloud(GRIDS[bits], 200 + bits)
    passes = (bits + 7) // 8
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(1.0)
    l0 = vg.launchCount()
    _filter(vg, blob)
    assert vg.launchCount() - l0 == 3 + 4
    for min_pts in (0, 4):
        l0 = vg.launchCount()
        _filter(vg, blob, min_pts)
        assert vg.launchCount() - l0 == 3 + passes


def test_c2_scan_launches():
    """bench.py's c2 shape: a 131072-ray scan at ~0.108 m needs 22 key bits, so a repeated call is six kernels"""
    import locus_b200
    from oracle import oracle as O
    scene, poses, blobs = G.stream(2, 2)
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(0.1088); vg.setFilterFieldName("z"); vg.setFilterLimits(-100.0, 100.0)
    vg.filter(blobs[0], 32, locus_b200.xyzi_fields())
    l0 = vg.launchCount()
    out, vidx = vg.filter(blobs[1], 32, locus_b200.xyzi_fields(), want_voxel_idx=True)
    assert vg.launchCount() - l0 == 6
    r = O.voxel_filter(blobs[1], 32, 0.1088, float_fields=G.FLOAT_FIELDS, filter_field_offset=8, limit_min=-100.0, limit_max=100.0)
    assert np.array_equal(vidx, r["voxel_idx"]) and np.array_equal(out, r["out"])
    assert 17 <= int(np.prod(r["div_b"])).bit_length() <= 24
