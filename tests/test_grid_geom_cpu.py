"""The grid geometry rule of the GICP index (locus_b200/csrc/grid.h: grid_auto_geom, grid_make_geom, grid_probe_accept),
built for the host by g++, against a numpy restatement of the rule as the host driver used to spell it out: automatic
cell size from the bounding box and the point count, the 1.5x growth under the dimension and cell-count caps, the
occupancy band and the sqrt(target / occupancy) rescale.  GridGeom is compared bit for bit: the device evaluates the same
function, and the cell size decides the order of the align's sums."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64
MAXDIM, MAXCELLS, TARGET = 16384, 64.0 * 1024 * 1024, 6.0


@pytest.fixture(scope="module")
def gg():
    bdir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(bdir, exist_ok=True)
    so = os.path.join(bdir, "libgrid_geom_harness.so")
    src = os.path.join(ROOT, "tests", "grid_geom_harness.cpp")
    hdrs = [os.path.join(ROOT, "locus_b200", "csrc", h) for h in ("hd.h", "grid.h")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in [src] + hdrs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    H = C.CDLL(so)
    vp = C.c_void_p
    H.gg_auto_geom.argtypes = [vp, vp, C.c_uint32, vp, vp]
    H.gg_make_geom.argtypes = [vp, vp, C.c_float, vp]
    H.gg_probe_accept.argtypes = [C.c_uint32, C.c_uint32, C.c_float, vp]
    H.gg_probe_accept.restype = C.c_int
    return H


# ---- the rule, restated
def ref_make_geom(mn, ext, cell):
    cell = f32(cell)
    with np.errstate(all="ignore"):
        while True:
            inv_h = f32(1.0) / cell
            fx, fy, fz = (np.floor(f64(f32(ext[d] * inv_h))) + 1 for d in range(3))
            if fx <= MAXDIM and fy <= MAXDIM and fz <= MAXDIM and fx * fy * fz <= MAXCELLS:
                return (f32(mn[0]), f32(mn[1]), f32(mn[2]), inv_h, cell, int(fx), int(fy), int(fz))
            cell = f32(cell * f32(1.5))


def ref_auto_cell(ext, n):
    e = [f64(v) for v in ext]
    area = f64(2.0) * ((e[0] * e[1] + e[1] * e[2]) + e[0] * e[2])
    diag = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
    if not area > 0:
        area = diag * diag
    spacing = np.sqrt(area / f64(n if n else 1))
    cell = f32(f64(1.3) * spacing)
    if not cell > 0:
        cell = f32(1.0)
    return cell


def ref_accept(n, n_occ, h):
    occ = f64(n) / f64(n_occ if n_occ else 1)
    if TARGET / 2 <= occ <= TARGET * 2:
        return True, None
    if n <= 8 or n_occ <= 1:
        return True, None
    scale = np.sqrt(f64(TARGET) / occ)
    scale = min(max(scale, f64(0.25)), f64(4.0))
    return False, f32(f32(h) * f32(scale))


def bits(g):
    return [int(np.array(v, f32).view(np.int32)) for v in g[:5]] + list(g[5:])


def lib_auto(gg, mn, mx, n):
    mn, mx = np.asarray(mn, f32), np.asarray(mx, f32)
    out = np.zeros(8, np.int32); kb = C.c_int(0)
    gg.gg_auto_geom(mn.ctypes.data, mx.ctypes.data, n, out.ctypes.data, C.byref(kb))
    return [int(v) for v in out], kb.value


def boxes(seed, count):
    """bounding boxes and point counts: lidar-sized rooms, lines, planes, single points, tiny and huge extents"""
    rng = np.random.default_rng(seed)
    for i in range(count):
        kind = i % 8
        mn = rng.uniform(-200, 200, 3).astype(f32)
        ext = (10.0 ** rng.uniform(-3, 2.5, 3)).astype(f32)
        if kind == 1:
            ext[rng.integers(3)] = 0                              # a plane
        elif kind == 2:
            ext[[(a := rng.integers(3)), (a + 1) % 3]] = 0         # a line
        elif kind == 3:
            ext[:] = 0                                            # a single point
        elif kind == 4:
            ext = (10.0 ** rng.uniform(2, 5, 3)).astype(f32)      # far beyond a scan
        elif kind == 5:
            ext = (10.0 ** rng.uniform(-6, -3, 3)).astype(f32)
        n = int(10 ** rng.uniform(0, 6.3)) if kind != 6 else int(rng.integers(1, 12))
        yield mn, (mn + ext).astype(f32), n


def test_auto_geometry_bit_for_bit(gg):
    checked = 0
    for mn, mx, n in boxes(1, 4000):
        ext = (mx - mn).astype(f32)
        want = ref_make_geom(mn, ext, ref_auto_cell(ext, n))
        got, kb = lib_auto(gg, mn, mx, n)
        assert got == bits(want), (mn, mx, n)
        cells = want[5] * want[6] * want[7]
        assert kb == max(1, int(cells - 1).bit_length()) and (1 << kb) >= cells
        checked += 1
    assert checked == 4000


def test_growth_under_the_caps(gg):
    """cells far smaller than the extent: the 1.5x loop runs until both the 16384-per-axis and the 64 Mi-cell cap hold"""
    rng = np.random.default_rng(2)
    grown = 0
    for _ in range(1500):
        mn = rng.uniform(-50, 50, 3).astype(f32)
        ext = (10.0 ** rng.uniform(0, 3, 3)).astype(f32)
        if rng.integers(2):
            ext[rng.integers(3)] = f32(0)
        mx = (mn + ext).astype(f32)
        cell = f32(10.0 ** rng.uniform(-4, -1))
        e = (mx - mn).astype(f32)
        want = ref_make_geom(mn, e, cell)
        out = np.zeros(8, np.int32)
        gg.gg_make_geom(mn.ctypes.data, mx.ctypes.data, cell, out.ctypes.data)
        assert [int(v) for v in out] == bits(want)
        assert max(want[5:]) <= MAXDIM and want[5] * want[6] * want[7] <= MAXCELLS
        grown += int(want[4] != cell)
    assert grown > 500
    # a million points filling a cube: the first guess already meets the caps; a huge flat sheet does not
    got, _ = lib_auto(gg, [0, 0, 0], [1e5, 1e5, 0], 4_000_000_000)
    assert got[5] <= MAXDIM and got[6] <= MAXDIM and got[7] == 1


def test_extent_that_overflows_ends_in_one_cell(gg):
    got, kb = lib_auto(gg, [-3e38, 0, 0], [3e38, 1, 1], 1000)
    assert got[5:] == [1, 1, 1] and kb == 1


def test_occupancy_band_and_rescale(gg):
    rng = np.random.default_rng(3)
    cases = []
    for n in (1, 8, 9, 600, 30000, 500000):
        for occ in (1, 2, n // 13, n // 12, n // 12 + 1, n // 6, n // 3 - 1, n // 3, n // 3 + 1, n // 2, n):
            cases.append((n, max(0, occ)))
        cases.append((n, 0))
    for _ in range(3000):
        n = int(10 ** rng.uniform(0, 6))
        cases.append((n, int(rng.integers(0, n + 1))))
    rejected = 0
    for n, n_occ in cases:
        h = f32(10.0 ** rng.uniform(-2, 1))
        nxt = C.c_float(-1.0)
        ok = gg.gg_probe_accept(n, n_occ, h, C.byref(nxt))
        want_ok, want_next = ref_accept(n, n_occ, h)
        assert bool(ok) == want_ok, (n, n_occ)
        if not want_ok:
            rejected += 1
            assert f32(nxt.value).view(np.int32) == want_next.view(np.int32), (n, n_occ, h)
            assert f32(0.25) * h <= nxt.value <= f32(4.0) * h
    assert rejected > 300
    # both edges of the band are inside it
    for n, n_occ in ((1200, 400), (1200, 100)):
        assert gg.gg_probe_accept(n, n_occ, f32(1.0), C.byref(C.c_float()))
    for n, n_occ in ((1200, 401), (1200, 99)):
        assert not gg.gg_probe_accept(n, n_occ, f32(1.0), C.byref(C.c_float()))
