"""Row f6 on the GPU: lb_voxel_extract_features against the oracle (oracle/features_oracle.c), bit-exact in the counts
and in every output word (NaN-aware), on the fixtures of tests/test_features_cpu.py, a 64-beam scan whose rings take the
global-memory path, a stream of scans, host and device buffers, repeated calls, the error paths and the two host
layers (the C++ mirror and the PCL shim)."""
import os
import subprocess

import numpy as np
import pytest

import conftest
from test_features_cpu import CASE_NAMES, case, same_bits

pytestmark = pytest.mark.gpu
ROOT = conftest.ROOT


@pytest.fixture(scope="module")
def fo():
    from oracle import features_oracle
    features_oracle.build()
    return features_oracle


@pytest.fixture(scope="module")
def vg():
    import locus_b200
    return locus_b200.VoxelGridB200(0)


def _check(vg, fo, xyz, **prm):
    out, cnt = vg.extractFeatures(xyz, **prm)
    ref, rcnt = fo.extract_features(xyz, **prm)
    assert cnt == rcnt, (cnt, rcnt)
    assert same_bits(out, ref)
    return out, cnt


@pytest.mark.parametrize("name", CASE_NAMES)
def test_gpu_matches_oracle(vg, fo, name):
    xyz, prm = case(name)
    _check(vg, fo, xyz, **prm)


def test_large_rings_global_path(vg, fo):
    """64 beams x 2048 azimuths through the default +-15 deg window: about 10 k points per ring, above the shared-memory
    stage of a ring CTA"""
    from test_features_cpu import _scene_scan
    xyz = _scene_scan(64, 2048, (-24.8, 2.0), seed=3)
    _, cnt = _check(vg, fo, xyz)
    from oracle import features_oracle as FO
    from test_features_cpu import np_arrange
    _, ring, _ = np_arrange(xyz, FO.params())
    assert np.bincount(ring[ring >= 0]).max() > 2048 and cnt["n_out"] > 0


def test_stream_of_scans(vg, fo):
    from tools import gen_lidar as G
    scene = G.make_scene(3)
    poses = G.trajectory(4, 5)
    for i, T in enumerate(poses):
        xyz = G.blob_xyz(G.scan(scene, T, 100 + i, beams=16, az=1800, elev_deg=(-15.0, 15.0)))
        _check(vg, fo, xyz)


def test_host_and_device_buffers(vg, fo):
    import torch
    xyz, _ = case("vlp16_scan_order")
    ref, rcnt = fo.extract_features(xyz)
    padded = np.zeros((len(xyz), 8), np.float32); padded[:, 2:5] = xyz
    blob = padded.view(np.uint8).reshape(-1)
    out_h, c1 = vg.extractFeatures(blob, stride=32, xyz_off=8)                        # host in, host out
    assert c1 == rcnt and same_bits(out_h, ref)
    d_in = torch.from_numpy(np.ascontiguousarray(xyz)).cuda()
    out_dh, c2 = vg.extractFeatures(d_in)                                               # device in, host out
    d_out = torch.zeros((rcnt["n_out"] + 5, 4), dtype=torch.float32, device="cuda")
    out_dd, c3 = vg.extractFeatures(d_in, out=d_out)                                   # device in, device out
    d_out2 = torch.zeros((rcnt["n_out"], 4), dtype=torch.float32, device="cuda")
    out_hd, c4 = vg.extractFeatures(xyz, out=d_out2)                                   # host in, device out
    assert c2 == c3 == c4 == rcnt
    assert same_bits(out_dh, ref) and same_bits(out_dd.cpu().numpy(), ref) and same_bits(out_hd.cpu().numpy(), ref)
    assert (d_out[rcnt["n_out"]:] == 0).all()


def test_repeated_calls_identical(vg):
    xyz, _ = case("vlp16_voxel_order")
    a, ca = vg.extractFeatures(xyz)
    n0 = vg.launchCount()
    for _ in range(3):
        b, cb = vg.extractFeatures(xyz)
        assert ca == cb and np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert vg.launchCount() - n0 == 9                  # three kernels per call


def _voxel_bits(v, blob):
    import locus_b200
    v.setLeafSize(0.25)
    v.setFilterFieldName("z"); v.setFilterLimits(-2.0, 3.0)
    return v.filter(blob, 32, locus_b200.xyzi_fields())


def test_errors_leave_the_handle(fo):
    import locus_b200
    import torch
    from tools import gen_lidar as G
    blob = G.scan(G.make_scene(3), np.eye(4), 9, beams=16, az=512)
    xyz, _ = case("vlp16_scan_order")
    _, rcnt = fo.extract_features(xyz)
    h = locus_b200.VoxelGridB200(0)
    first = _voxel_bits(h, blob)
    # capacity: reports the size needed and writes nothing
    small = torch.full((rcnt["n_out"] - 1, 4), 7.0, dtype=torch.float32, device="cuda")
    with pytest.raises(locus_b200.LocusB200Error) as e:
        h.extractFeatures(xyz, out=small)
    assert e.value.status == -8 and (small == 7.0).all()
    import ctypes as C
    from locus_b200 import api
    r = api.FeaturesResult()
    p = h.featureParams()
    a = np.ascontiguousarray(xyz)
    s = api.lib().lb_voxel_extract_features(h._h, a.ctypes.data_as(C.c_void_p), len(a), 12, 0, 0, C.byref(p),
                                            small.data_ptr(), small.shape[0], C.byref(r), 1)
    assert s == -8 and r.n_out == rcnt["n_out"] and (small == 7.0).all()
    # invalid parameters and empty input
    for bad in (dict(n_rings=0), dict(n_rings=129), dict(lower_deg=15.0, upper_deg=15.0), dict(curvature_region=0),
                dict(curvature_region=33), dict(n_feature_regions=0), dict(less_flat_leaf=0.0), dict(max_corner_sharp=-1),
                dict(max_corner_less_sharp=-1), dict(max_surface_flat=-1)):
        with pytest.raises(locus_b200.LocusB200Error) as e:
            h.extractFeatures(xyz, **bad)
        assert e.value.status == -1, bad
    with pytest.raises(locus_b200.LocusB200Error) as e:
        h.extractFeatures(np.zeros((0, 3), np.float32))
    assert e.value.status == -4
    after = h.filter(blob, 32, locus_b200.xyzi_fields())
    fresh = _voxel_bits(locus_b200.VoxelGridB200(0), blob)
    assert np.array_equal(first, fresh) and np.array_equal(after, fresh)
    assert np.array_equal(h.getLeafSize(), np.float32([0.25, 0.25, 0.25]))


def _run_harness(exe, xyz, tmp_path):
    src = tmp_path / "in.bin"; dst = tmp_path / "out.bin"
    np.ascontiguousarray(xyz, np.float32).tofile(src)
    r = subprocess.run([exe, str(src), str(dst)], stdout=subprocess.PIPE, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return np.fromfile(dst, np.float32).reshape(-1, 4)


def test_cpp_mirror_matches_oracle(fo, tmp_path):
    exe = os.path.join(ROOT, "tests", "_build", "features_mirror_harness")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    host = os.path.join(ROOT, "locus_b200", "host")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", host,
                           os.path.join(ROOT, "tests", "features_mirror_harness.cpp"), "-L", os.path.join(ROOT, "locus_b200"),
                           "-llocus_b200", "-Wl,-rpath," + os.path.join(ROOT, "locus_b200"), "-pthread", "-o", exe])
    for name in ("vlp16_scan_order", "vlp16_voxel_order"):
        xyz, _ = case(name)
        ref, _ = fo.extract_features(xyz)
        assert same_bits(_run_harness(exe, xyz, tmp_path), ref), name


def test_shim_matches_oracle(fo, tmp_path):
    exe = os.path.join(ROOT, "tests", "_build", "features_shim_harness")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "pcl_stub"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "shim"),
                           os.path.join(ROOT, "tests", "features_shim_harness.cpp"), "-L", os.path.join(ROOT, "locus_b200"),
                           "-llocus_b200", "-Wl,-rpath," + os.path.join(ROOT, "locus_b200"), "-pthread", "-o", exe])
    for name in ("vlp16_scan_order", "nan_point0"):
        xyz, _ = case(name)
        ref, _ = fo.extract_features(xyz)
        assert same_bits(_run_harness(exe, xyz, tmp_path), ref), name
