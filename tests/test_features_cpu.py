"""Row f6 without a GPU: the oracle's restatement of LOCUS's LOAM feature extraction (oracle/features_oracle.c) against
an independent numpy restatement (step-by-step float32 arithmetic, Python loops for the pick walk, stable argsort, a
voxel grid of its own), and the serial build of locus_b200/csrc/features.h (tests/features_harness.cpp) against the
oracle.  Counts are equal and every output word is bit-identical (NaN-aware).  The fixtures below are shared with
tests/test_features_gpu.py."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import conftest

ROOT = conftest.ROOT
f32 = np.float32
PI = math.pi


# ------------------------------------------------------------------ fixtures
def _scene_scan(beams, az, elev, seed=7):
    from tools import gen_lidar as G
    blob = G.scan(G.make_scene(3), np.eye(4), seed, beams=beams, az=az, elev_deg=elev)
    return G.blob_xyz(blob)


def vlp16_sweep():
    """a VLP-16 sweep (16 beams over +-15 deg, 1800 azimuths) in scan order, sensor frame, with drop-outs"""
    return _scene_scan(16, 1800, (-15.0, 15.0))


def vlp16_voxel_filtered(leaf=0.1):
    """the same sweep after the VoxelGrid (voxel-index order, what LOCUS's lidar callback receives)"""
    from oracle import oracle as O
    from tools import gen_lidar as G
    blob = G.scan(G.make_scene(3), np.eye(4), 7, beams=16, az=1800, elev_deg=(-15.0, 15.0))
    out = O.voxel_filter(blob, 32, leaf, float_fields=G.FLOAT_FIELDS)["out"]
    return G.blob_xyz(np.ascontiguousarray(out).reshape(-1))


def nan_first():
    p = vlp16_sweep().copy()
    p[0] = np.nan
    return p


def invalid_points():
    """zero points, non-finite coordinates and points outside the vertical window mixed into the sweep"""
    p = vlp16_sweep().copy()
    rng = np.random.default_rng(5)
    idx = rng.choice(len(p), 300, replace=False)
    p[idx[:60]] = 0.0
    p[idx[60:70], 0] = np.inf
    p[idx[70:80], 1] = -np.inf
    p[idx[80:100], 2] = np.nan
    p[idx[100:110]] = f32(0.003)                       # |p|^2 < 1e-4
    r = np.linalg.norm(p[idx[110:300]], axis=1, keepdims=True)
    el = np.deg2rad(rng.choice([40.0, -40.0, 15.9, -15.9, -16.5], (190, 1)))
    az = rng.uniform(0, 2 * np.pi, (190, 1))
    p[idx[110:300]] = np.concatenate([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1) * np.nan_to_num(r, nan=5.0)
    return p.astype(np.float32)


def _ring_points(ring, n, radius=5.0, n_rings=16, lo=-15.0, hi=15.0, a0=0.0, da=0.004):
    el = np.deg2rad(lo + ring * (hi - lo) / (n_rings - 1))
    a = a0 + da * np.arange(n)
    r = radius + 0.3 * np.sin(7 * a)
    return np.stack([r * np.cos(el) * np.cos(a), r * np.cos(el) * np.sin(a), r * np.sin(el) * np.ones_like(a)], 1)


def short_rings():
    """empty rings, rings of <= 2*cr + 1 points (skipped), the smallest unskipped ring and rings whose regions are
    too short (ep <= sp for some regions)"""
    parts = [_ring_points(1, 3), _ring_points(3, 11), _ring_points(4, 12), _ring_points(6, 15), _ring_points(7, 16),
             _ring_points(9, 40), _ring_points(12, 2)]
    return np.concatenate(parts).astype(np.float32)


def curvature_ties():
    """exact curvature ties between DISTINCT points (distinct positions, orientations and intensities), with dyadic
    coordinates so that every curvature is exact:
      ring 8 (elevation 0): 160 equally spaced collinear points, curvature exactly 0 -- the flat walk sees ties only;
      ring 12 (z = 2): a zig-zag of period 2, curvature exactly 0.5625 at every point -- the corner walk sees ties only.
    The steps stay below 0.0002 * range^2 so that no unreliable mark hides them.  A walk that took tied candidates in
    the other order picks different points (test_ties_pin_the_order)."""
    k = np.arange(160, dtype=np.float64)
    line = np.stack([np.full_like(k, 12.0), -10.0 + 0.125 * k, np.zeros_like(k)], 1)
    zig = np.stack([12.0 + 0.125 * (k % 2), -5.0 + 0.0625 * k, np.full_like(k, 2.0)], 1)
    return np.concatenate([line, zig]).astype(np.float32)


def huge_coordinates():
    """finite coordinates whose arithmetic leaves the float range.  Ring 8: a line of 60 points with three consecutive
    (3e38, 0, 0) points in its middle -- NaN curvatures (-inf + inf) and an infinite less-flat extent.  Ring 4: 40
    points 5e8 m away -- a finite extent, but min * inverse leaf beyond int32.  Both less-flat sets pass through the
    VoxelGrid (features.h, "Less-flat set")."""
    k = np.arange(60, dtype=np.float64)
    line = np.stack([np.full_like(k, 12.0), -4.0 + 0.125 * k, np.zeros_like(k)], 1)
    line = np.concatenate([line[:30], [[3e38, 0.0, 0.0]] * 3, line[30:]])
    k = np.arange(40, dtype=np.float64)
    distant = np.stack([np.full_like(k, 5e8), 32.0 * k - 640.0, np.full_like(k, -6.14e7)], 1)
    return np.concatenate([line, distant]).astype(np.float32)


def voxel_overflow_params():
    return dict(less_flat_leaf=1e-5)


def custom_scan():
    return _scene_scan(32, 1024, (-25.0, 5.0), seed=11)


CUSTOM_PARAMS = dict(n_rings=32, lower_deg=-25.0, upper_deg=5.0, scan_period=0.05, curvature_region=3,
                     n_feature_regions=8, max_corner_sharp=3, max_corner_less_sharp=15, max_surface_flat=6,
                     curvature_threshold=0.05, less_flat_leaf=0.3)


def cases():
    """(name, xyz, params) of every fixture"""
    return [
        ("vlp16_scan_order", vlp16_sweep(), {}),
        ("vlp16_voxel_order", vlp16_voxel_filtered(), {}),
        ("nan_point0", nan_first(), {}),
        ("invalid_points", invalid_points(), {}),
        ("short_rings", short_rings(), {}),
        ("curvature_ties", curvature_ties(), {}),
        ("huge_coordinates", huge_coordinates(), {}),
        ("voxel_overflow", vlp16_sweep(), voxel_overflow_params()),
        ("custom_params", custom_scan(), CUSTOM_PARAMS),
    ]


CASE_NAMES = [
    "vlp16_scan_order", "vlp16_voxel_order", "nan_point0", "invalid_points", "short_rings", "curvature_ties",
    "huge_coordinates", "voxel_overflow", "custom_params"]


def case(name):
    for n, x, p in cases():
        if n == name:
            return x, p
    raise KeyError(name)


def same_bits(a, b):
    """bit-identical float32 arrays, any NaN equal to any NaN"""
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape:
        return False
    eq = a.view(np.uint32) == b.view(np.uint32)
    return bool(np.all(eq | (np.isnan(a) & np.isnan(b))))


# ------------------------------------------------------------------ independent numpy restatement
_libm = C.CDLL("libm.so.6")
_libm.atanf.restype = C.c_float; _libm.atanf.argtypes = [C.c_float]
_libm.atan2f.restype = C.c_float; _libm.atan2f.argtypes = [C.c_float, C.c_float]


def _atan(v, libm_float):
    if libm_float:
        return np.array([_libm.atanf(float(t)) for t in v], np.float32)
    return np.array([math.atan(float(t)) for t in v], np.float64).astype(np.float32)


def _atan2(y, x, libm_float):
    if libm_float:
        return np.array([_libm.atan2f(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    return np.array([math.atan2(float(a), float(b)) for a, b in zip(y, x)], np.float64).astype(np.float32)


def np_arrange(xyz, P, libm_float=False):
    """arrangePCLInScanLines: (ring-major list of (m, 4) float32 rings, per-input ring (-1 dropped), intensity)"""
    xyz = np.asarray(xyz, np.float32)
    n = len(xyz)
    factor = f32(f32(P["n_rings"] - 1) / f32(f32(P["upper_deg"]) - f32(P["lower_deg"])))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        so = -_atan2(xyz[:1, 1], xyz[:1, 0], libm_float)[0]
        eo = f32(-_atan2(xyz[-1:, 1], xyz[-1:, 0], libm_float)[0] + f32(2) * f32(PI))
        d = float(f32(eo - so))
        if d > 3 * PI:
            eo = f32(float(eo) - 2 * PI)
        elif d < PI:
            eo = f32(float(eo) + 2 * PI)
        x, y, z = xyz[:, 1].copy(), xyz[:, 2].copy(), xyz[:, 0].copy()
        keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
        s2 = (x * x + y * y) + z * z
        keep &= ~(s2.astype(np.float64) < 0.0001)
        ring = np.full(n, -1, np.int64)
        ki = np.nonzero(keep)[0]
        ang = _atan(y[ki] / np.sqrt(x[ki] * x[ki] + z[ki] * z[ki]), libm_float)
        v = ((ang * f32(180)).astype(np.float64) / PI - float(f32(P["lower_deg"]))) * float(factor) + 0.5
        rk = np.trunc(v).astype(np.int64)
        ok = (rk >= 0) & (rk < P["n_rings"])
        ki, rk = ki[ok], rk[ok]
        ring[ki] = rk
        ori0 = -_atan2(x[ki], z[ki], libm_float)
        inten = np.full(n, np.nan, np.float32)
        half = False
        sp_ = f32(P["scan_period"])
        for t, i in enumerate(ki):
            ori = ori0[t]
            if not half:
                if float(ori) < float(so) - PI / 2:
                    ori = f32(float(ori) + 2 * PI)
                elif float(ori) > float(so) + PI * 3 / 2:
                    ori = f32(float(ori) - 2 * PI)
                if float(f32(ori - so)) > PI:
                    half = True
            else:
                ori = f32(float(ori) + 2 * PI)
                if float(ori) < float(eo) - PI * 3 / 2:
                    ori = f32(float(ori) + 2 * PI)
                elif float(ori) > float(eo) + PI / 2:
                    ori = f32(float(ori) - 2 * PI)
            rel = f32(f32(sp_ * f32(ori - so)) / f32(eo - so))
            inten[i] = f32(f32(rk[t]) + rel)
    rings = []
    for r in range(P["n_rings"]):
        idx = np.nonzero(ring == r)[0]
        rings.append(np.stack([x[idx], y[idx], z[idx], inten[idx]], 1).astype(np.float32).reshape(-1, 4))
    return rings, ring, inten


def _sqd(a, b):
    d = (a[..., :3] - b[..., :3]).astype(np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _sqdw(a, b, w):
    d0 = a[..., 0] - b[..., 0] * w; d1 = a[..., 1] - b[..., 1] * w; d2 = a[..., 2] - b[..., 2] * w
    return (d0 * d0 + d1 * d1) + d2 * d2


def _sqn(a):
    return (a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2]


def np_voxel(pts, leaf):
    """pcl::VoxelGrid<PointF> on one ring's less-flat points (m, 4), ascending position inside a voxel"""
    if len(pts) == 0:
        return pts
    inv = f32(f32(1) / f32(leaf))
    mn = pts[:, :3].min(0); mx = pts[:, :3].max(0)
    with np.errstate(over="ignore", invalid="ignore"):
        ext = [f32((mx[d] - mn[d]) * inv) for d in range(3)]
        lo = [np.floor(f32(mn[d] * inv)) for d in range(3)]
        hi = [np.floor(f32(mx[d] * inv)) for d in range(3)]
    # PCL's guard; where PCL's arithmetic is undefined (extent * inv not below 2^31, min / max * inv outside int32)
    # the set passes through as well
    if not all(e < 2.0**31 and -2.0**31 <= a < 2.0**31 and -2.0**31 <= b < 2.0**31 for e, a, b in zip(ext, lo, hi)):
        return pts.copy()
    dxyz = [int(e) + 1 for e in ext]
    if dxyz[0] * dxyz[1] * dxyz[2] > 2**31 - 1:
        return pts.copy()
    min_b = [int(v) for v in lo]
    div_b = [int(hi[d]) - min_b[d] + 1 for d in range(3)]
    ijk = [(np.floor(pts[:, d] * inv) - f32(min_b[d])).astype(np.int64) for d in range(3)]
    key = ijk[0] + ijk[1] * div_b[0] + ijk[2] * (div_b[0] * div_b[1])
    order = np.argsort(key, kind="stable")
    out = []
    s = 0
    while s < len(order):
        e = s + 1
        while e < len(order) and key[order[e]] == key[order[s]]:
            e += 1
        acc = pts[order[s]].copy()
        for t in range(s + 1, e):
            acc = (acc + pts[order[t]]).astype(np.float32)
        out.append(acc / f32(e - s))
        s = e
    return np.array(out, np.float32).reshape(-1, 4)


def np_rotation():
    def aa(axis):
        th = f32(PI / 2)
        a = np.zeros(3, np.float32); a[axis] = 1
        s_, c_ = f32(math.sin(float(th))), f32(math.cos(float(th)))
        sa = s_ * a; ca = (f32(1) - c_) * a
        R = np.zeros((3, 3), np.float32)
        R[0, 1] = ca[0] * a[1] - sa[2]; R[1, 0] = ca[0] * a[1] + sa[2]
        R[0, 2] = ca[0] * a[2] + sa[1]; R[2, 0] = ca[0] * a[2] - sa[1]
        R[1, 2] = ca[1] * a[2] - sa[0]; R[2, 1] = ca[1] * a[2] + sa[0]
        for d in range(3):
            R[d, d] = ca[d] * a[d] + c_
        return R

    def mm(A, B):
        Cm = np.zeros((3, 3), np.float32)
        for i in range(3):
            for j in range(3):
                Cm[i, j] = (A[i, 0] * B[0, j] + A[i, 1] * B[1, j]) + A[i, 2] * B[2, j]
        return Cm
    return mm(mm(np.eye(3, dtype=np.float32), aa(1)), aa(2))


def insertion_order(c, reverse_ties=False):
    """the order the reference's insertion sort (no early exit, `<`) leaves: NaNs stay in place and nothing passes
    them; between them a stable ascending sort.  reverse_ties: equal curvatures the other way round (a mutation the
    fixtures must detect)"""
    order = np.arange(len(c))
    nan = np.isnan(c)
    s = 0
    while s < len(c):
        if nan[s]:
            s += 1
            continue
        e = s
        while e < len(c) and not nan[e]:
            e += 1
        seg = np.arange(s, e)
        if reverse_ties:
            seg = seg[::-1]
        order[s:e] = seg[np.argsort(c[seg], kind="stable")]
        s = e
    return order


def np_extract(xyz, stats=None, reverse_ties=False, **kw):
    from oracle import features_oracle as FO
    P = FO.params(**kw)
    rings, _, _ = np_arrange(xyz, P)
    cr, R = P["curvature_region"], P["n_feature_regions"]
    thr = f32(P["curvature_threshold"])
    sharp, less, flat, lflat = [], [], [], []
    blocked_across = 0
    for X in rings:
        m = len(X)
        if m <= 2 * cr + 1:
            continue
        picked = np.zeros(m, bool)
        pick_marked = np.zeros(m, bool)              # marks of markAsPicked only
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            i = np.arange(cr, m - 1 - cr)
            pt, nx, pv = X[i], X[i + 1], X[i - 1]
            dn = _sqd(nx, pt)
            d1 = np.sqrt(_sqn(pt)); d2 = np.sqrt(_sqn(nx))
            big = dn.astype(np.float64) > 0.1
            w1 = np.sqrt(_sqdw(nx, pt, d2 / d1)) / d2
            w2 = np.sqrt(_sqdw(pt, nx, d1 / d2)) / d1
            fa = big & (d1 > d2) & (w1.astype(np.float64) < 0.1)
            fb = big & ~(d1 > d2) & (w2.astype(np.float64) < 0.1)
            dis = _sqn(pt).astype(np.float64)
            fc = ~fa & (dn.astype(np.float64) > 0.0002 * dis) & (_sqd(pt, pv).astype(np.float64) > 0.0002 * dis)
        for t in np.nonzero(fa)[0]:
            picked[i[t] - cr: i[t] + 1] = True
        for t in np.nonzero(fb)[0]:
            picked[i[t] + 1: i[t] + cr + 2] = True
        picked[i[fc]] = True
        curv = np.zeros(m, np.float32)
        c = np.arange(cr, m - cr)
        with np.errstate(invalid="ignore", over="ignore"):
            dxyz = f32(-2 * cr) * X[c, :3]
            for j in range(1, cr + 1):
                dxyz = dxyz + (X[c + j, :3] + X[c - j, :3])
            curv[c] = (dxyz[:, 0] * dxyz[:, 0] + dxyz[:, 1] * dxyz[:, 1]) + dxyz[:, 2] * dxyz[:, 2]

        def mark(k):
            picked[k] = pick_marked[k] = True
            with np.errstate(invalid="ignore", over="ignore"):
                for a in range(1, cr + 1):
                    if float(_sqd(X[k + a], X[k + a - 1])) > 0.05:
                        break
                    picked[k + a] = pick_marked[k + a] = True
                for a in range(1, cr + 1):
                    if float(_sqd(X[k - a], X[k - a + 1])) > 0.05:
                        break
                    picked[k - a] = pick_marked[k - a] = True

        lf = []
        D = m - 1 - 2 * cr
        prev_ep = None
        for j in range(R):
            sp = cr + (j * D) // R
            ep = cr + ((j + 1) * D) // R - 1
            if ep <= sp:
                continue
            if prev_ep is not None and prev_ep + 1 == sp:
                blocked_across += int(pick_marked[sp: sp + cr].any())      # the previous region's picks reach into this one
            order = sp + insertion_order(curv[sp: ep + 1], reverse_ties)
            label = np.zeros(ep - sp + 1, np.int64)
            taken = 0
            for k in order[::-1]:
                if taken >= P["max_corner_less_sharp"]:
                    break
                if not picked[k] and curv[k] > thr:
                    taken += 1
                    if taken <= P["max_corner_sharp"]:
                        label[k - sp] = 2; sharp.append(X[k])
                    else:
                        label[k - sp] = 1
                    less.append(X[k])
                    mark(k)
            taken = 0
            for k in order:
                if taken >= P["max_surface_flat"]:
                    break
                if not picked[k] and curv[k] < thr:
                    taken += 1
                    label[k - sp] = -1; flat.append(X[k])
                    mark(k)
            lf.extend(X[sp + np.nonzero(label <= 0)[0]])
            prev_ep = ep
        lflat.append(np_voxel(np.array(lf, np.float32).reshape(-1, 4), P["less_flat_leaf"]))
    parts = [np.array(a, np.float32).reshape(-1, 4) for a in (sharp, less, flat)] + [np.concatenate(lflat) if lflat else np.zeros((0, 4), np.float32)]
    allp = np.concatenate(parts).astype(np.float32)
    M = np_rotation()
    out = np.empty_like(allp)
    for d in range(3):
        out[:, d] = M[d, 0] * allp[:, 0] + (M[d, 1] * allp[:, 1] + (M[d, 2] * allp[:, 2] + f32(0)))
    out[:, 3] = allp[:, 3]
    counts = dict(n_arranged=sum(len(r) for r in rings), n_sharp=len(parts[0]), n_less_sharp=len(parts[1]),
                  n_flat=len(parts[2]), n_less_flat=len(parts[3]), n_out=len(out))
    if stats is not None:
        stats["blocked_across_regions"] = blocked_across
    return out, counts


# ------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def fo():
    from oracle import features_oracle
    features_oracle.build()
    return features_oracle


@pytest.fixture(scope="module")
def all_cases():
    return cases()


@pytest.mark.parametrize("name", CASE_NAMES)
def test_oracle_matches_numpy(fo, all_cases, name):
    xyz, prm = [(x, p) for n, x, p in all_cases if n == name][0]
    out, cnt = fo.extract_features(xyz, **prm)
    ref, rcnt = np_extract(xyz, **prm)
    assert cnt == rcnt, (cnt, rcnt)
    assert same_bits(out, ref)
    if name in ("vlp16_scan_order", "custom_params"):
        assert cnt["n_sharp"] > 0 and cnt["n_flat"] > 0 and cnt["n_less_flat"] > 0 and cnt["n_less_sharp"] > cnt["n_sharp"]
    if name == "nan_point0":
        assert np.isnan(out[:, 3]).all() and cnt["n_out"] > 0
    if name == "voxel_overflow":
        base, _ = fo.extract_features(xyz)
        assert cnt["n_less_flat"] > 0 and cnt["n_out"] > len(base)


def test_fixtures_cover_the_corner_cases(fo, all_cases):
    """the cases really contain what they are named for"""
    from oracle import features_oracle as FO
    P = FO.params()
    _, ring, _ = np_arrange(case("short_rings")[0], P)
    counts = np.bincount(ring[ring >= 0], minlength=16)
    cr = P["curvature_region"]
    assert (counts == 0).any() and ((counts > 0) & (counts <= 2 * cr + 1)).any() and (counts == 2 * cr + 2).any()
    D = counts[counts > 2 * cr + 1] - 1 - 2 * cr
    assert any(any(((j + 1) * d) // 6 - (j * d) // 6 <= 1 for j in range(6)) for d in D)     # a region with ep <= sp
    xyz = case("invalid_points")[0]
    _, ring, _ = np_arrange(xyz, P)
    # +-40 deg points leave the window; -16.5 deg gives -0.25, which int() truncates to ring 0
    assert (ring[np.isfinite(xyz).all(1) & (np.abs(xyz).sum(1) > 0)] < 0).sum() >= 60
    stats = {}
    np_extract(vlp16_sweep(), stats=stats)
    assert stats["blocked_across_regions"] > 0, "no pick near a region's end reached into the next region"


def test_ties_pin_the_order(fo):
    """curvature_ties holds exact ties between distinct points in both walks: the oracle's output differs from what
    a walk that took equal curvatures in the other order would give"""
    from oracle import features_oracle as FO
    xyz = case("curvature_ties")[0]
    rings, _, _ = np_arrange(xyz, FO.params())
    assert len(rings[8]) == 160 and len(rings[12]) == 160
    assert len(np.unique(rings[8][:, 3])) == 160 and len(np.unique(rings[12][:, 3])) == 160      # distinct intensities
    ref, cnt = fo.extract_features(xyz)
    assert cnt["n_sharp"] > 0 and cnt["n_flat"] > 0
    rev, rcnt = np_extract(xyz, reverse_ties=True)
    assert rcnt != cnt or not same_bits(rev, ref)


def test_huge_coordinates_reach_nan_curvature_and_passthrough(fo):
    from oracle import features_oracle as FO
    xyz = case("huge_coordinates")[0]
    P = FO.params()
    rings, _, _ = np_arrange(xyz, P)
    X = rings[8]
    cr = P["curvature_region"]
    c = np.arange(cr, len(X) - cr)
    with np.errstate(invalid="ignore", over="ignore"):
        d = f32(-2 * cr) * X[c, 2]
        for j in range(1, cr + 1):
            d = d + (X[c + j, 2] + X[c - j, 2])
    assert np.isnan(d).any() and np.isinf(d).any() and len(rings[4]) == 40
    _, cnt = fo.extract_features(xyz)
    assert cnt["n_less_flat"] > 0


def test_region_bounds_forms_agree():
    """the reference's size_t form on global ring-major positions equals the ring-local form of features.h"""
    for start in (0, 7, 1000, 123457):
        for cr in (1, 3, 5, 32):
            for R in (1, 2, 6, 7, 64):
                for cnt in range(2 * cr + 2, 2 * cr + 90):
                    S, E = start, start + cnt - 1
                    D = cnt - 1 - 2 * cr
                    for j in range(R):
                        sp = ((S + cr) * (R - j) + (E - cr) * j) // R
                        ep = ((S + cr) * (R - 1 - j) + (E - cr) * (j + 1)) // R - 1
                        assert sp - S == cr + (j * D) // R and ep - S == cr + ((j + 1) * D) // R - 1


def test_stable_sort_is_the_insertion_sort():
    """the reference's insertion sort without early exit == insertion_order (== features.h's feat_region_rank): a
    stable ascending sort between NaNs, which keep their places (ties and NaNs included)"""
    rng = np.random.default_rng(1)
    for t in range(200):
        c = rng.integers(0, 5, rng.integers(1, 40)).astype(np.float32)
        if t % 2:
            c[rng.random(len(c)) < 0.2] = np.nan
        idx = list(range(len(c)))
        for i in range(1, len(c)):
            for j in range(i, 0, -1):
                if c[idx[j]] < c[idx[j - 1]]:
                    idx[j], idx[j - 1] = idx[j - 1], idx[j]
        assert idx == list(insertion_order(c))


def test_generator_default_unchanged():
    """tools/gen_lidar.py: the elev_deg keyword leaves the default scan byte-identical"""
    from tools import gen_lidar as G
    sc = G.make_scene(3)
    a = G.scan(sc, np.eye(4), 5, beams=16, az=256)
    b = G.scan(sc, np.eye(4), 5, beams=16, az=256, elev_deg=(-24.8, 2.0))
    d = G._ray_dirs(16, 256)
    el = np.deg2rad(np.linspace(-24.8, 2.0, 16))
    assert np.array_equal(a, b) and np.array_equal(d[::256, 2], np.sin(el))


def _build(name, src, extra):
    out = os.path.join(ROOT, "tests", "_build", name)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-Wno-unknown-pragmas", "-ffp-contract=off"] + extra + [src, "-o", out])
    return out


@pytest.fixture(scope="module")
def harness():
    return _build("features_harness", os.path.join(ROOT, "tests", "features_harness.cpp"),
                  ["-iquote", os.path.join(ROOT, "locus_b200", "csrc")])   # -iquote: glibc has a <features.h> of its own


def run_harness(exe, xyz, tmp_path, **kw):
    from oracle import features_oracle as FO
    P = FO.params(**kw)
    src = tmp_path / "in.bin"; dst = tmp_path / "out.bin"
    np.ascontiguousarray(xyz, np.float32)[:, :3].tofile(src)
    args = [str(P[k]) for k in ("n_rings", "lower_deg", "upper_deg", "scan_period", "curvature_region", "n_feature_regions",
                                "max_corner_sharp", "max_corner_less_sharp", "max_surface_flat", "curvature_threshold",
                                "less_flat_leaf")]
    r = subprocess.run([exe, str(src), str(dst)] + args, stdout=subprocess.PIPE, text=True, timeout=300, check=True)
    vals = [int(v) for v in r.stdout.split()]
    counts = dict(zip(FO.COUNT_NAMES, vals))
    return np.fromfile(dst, np.float32).reshape(-1, 4), counts


@pytest.mark.parametrize("name", CASE_NAMES)
def test_harness_matches_oracle(fo, all_cases, harness, tmp_path, name):
    xyz, prm = [(x, p) for n, x, p in all_cases if n == name][0]
    out, cnt = run_harness(harness, xyz, tmp_path, **prm)
    ref, rcnt = fo.extract_features(xyz, **prm)
    assert cnt == rcnt and same_bits(out, ref)


def test_libm_float_census(fo, all_cases):
    """how many points change ring or intensity when glibc's atanf / atan2f replace the pinned (float)atan((double)x)
    reading; recorded in DESIGN.md section 2"""
    from oracle import features_oracle as FO
    total = changed_ring = changed_int = 0
    for name, xyz, prm in all_cases:
        P = FO.params(**prm)
        _, r0, i0 = np_arrange(xyz, P)
        _, r1, i1 = np_arrange(xyz, P, libm_float=True)
        kept = (r0 >= 0) | (r1 >= 0)
        total += int(kept.sum())
        changed_ring += int((r0 != r1).sum())
        changed_int += int((~((i0.view(np.uint32) == i1.view(np.uint32)) | (np.isnan(i0) & np.isnan(i1))) & kept & (r0 == r1)).sum())
    print("\nlibm atanf/atan2f census: %d arranged points, %d change ring, %d change intensity" % (total, changed_ring, changed_int))
    assert total > 0


def test_shim_compiles_and_links():
    """shim/b200_feature_extraction_pcl.hpp against the PCL mock (tests/pcl_stub) and the C ABI; without a GPU the
    harness reports that there is no device"""
    import locus_b200
    exe = os.path.join(ROOT, "tests", "_build", "features_shim_harness")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "pcl_stub"),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "shim"),
                           os.path.join(ROOT, "tests", "features_shim_harness.cpp"), "-L", os.path.join(ROOT, "locus_b200"),
                           "-llocus_b200", "-Wl,-rpath," + os.path.join(ROOT, "locus_b200"), "-pthread", "-o", exe])
    r = subprocess.run([exe], stdout=subprocess.PIPE, text=True, timeout=120)
    if locus_b200.device_count() <= 0:
        assert r.returncode == 3 and "no_device=" in r.stdout
