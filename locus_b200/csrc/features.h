// features.h -- scalar logic of LOCUS's LOAM-style feature extraction (SURVEY 8f row f6), shared by the sm_90a kernels
// of features.cu and the serial CPU harness tests/features_harness.cpp.
//
// Restates point_cloud_filter/src/PointCloudFilter.cc:144-173 (the `filtering/extract_features` branch of Filter())
// and :179-515 (arrangePCLInScanLines, extractFeatures, setRegionBuffersFor, setScanBuffersFor, markAsPicked,
// getRingForAngle), with the constants of PointCloudFilter.h:79-96.  The reference holds no test of this code, so
// parity is unpinned; the pinned readings are listed in DESIGN.md section 2.
//
// Semantics, in the order the reference applies them:
//   Arrangement.  Axes swap x <- y, y <- z, z <- x.  A point is dropped when a coordinate is not finite, when
//     (x*x + y*y) + z*z < 1e-4 (float sum, double compare), or when its ring is outside [0, n_rings).  ring =
//     int(((angle*180)/pi - lower) * factor + 0.5): angle*180 in float, the rest in double, int() truncates toward
//     zero; factor = float(n_rings - 1) / (upper - lower).  startOri / endOri come from input points 0 and n-1 (raw
//     y, x), NaN included; a NaN there makes every intensity NaN.  halfPassed switches on AFTER the first kept point
//     whose branch-A orientation has ori - startOri > pi, so a point uses branch A iff its input index is <= that
//     point's index (one min-reduction).  Every `ori +/-= 2*M_PI` is computed in double and stored in float.
//     intensity = float(ring) + scan_period * (ori - startOri) / (endOri - startOri).  Output order: ring-major,
//     input order within a ring.
//   Regions.  A ring of cnt points is skipped when cnt <= 2*cr + 1.  Region j of R covers the ring-local positions
//     [cr + floor(j*D/R), cr + floor((j+1)*D/R) - 1], D = cnt - 1 - 2*cr (the reference's size_t form on global
//     positions reduces to this); it is skipped when it has fewer than 2 points.  Positions outside every region
//     never reach the output.
//   Unreliable marks (setScanBuffersFor) of the positions [cr, cnt-1-cr): they only ever set flags, so they are
//     evaluated in parallel and OR-ed.  Curvature: diff = -2cr*x, then diff += (x[i+j] + x[i-j]) for j = 1..cr,
//     curvature = (dx*dx + dy*dy) + dz*dz.
//   Sort.  The reference's insertion sort has no early exit and compares with `<`.  A NaN curvature (finite
//     coordinates near FLT_MAX give -inf + inf) never moves and nothing moves past it, so the order is: every NaN at
//     its own position, and between them a stable ascending sort by curvature (feat_region_rank).  The corner walk
//     takes candidates from the top of that order (among equal curvatures the higher position first), the flat walk
//     from the bottom; a NaN curvature is neither a corner nor a flat candidate.
//   Picks.  The `picked` flags belong to the ring, so a pick near the end of region j can block region j+1: the
//     regions of a ring are walked in order.  Corner: picked == 0 and curvature > threshold, at most max_less_sharp,
//     the first max_sharp of them sharp; flat: picked == 0 and curvature < threshold, at most max_flat.  Each pick
//     runs markAsPicked (neighbours within cr while the squared step is <= 0.05).
//   Less-flat set.  Every point of an unskipped region that is not a corner (flat points included), in position
//     order, through PCL 1.10 VoxelGrid<PointF> with leaf less_flat_leaf per ring: bounding box, the dx*dy*dz >
//     INT_MAX guard (tripped: the ring's set passes through unchanged), min_b = floor(min*inv), keys as in voxel.cu,
//     points of a voxel summed in ascending position (x, y, z, intensity, float), divided by the float count, voxels
//     in ascending index.  Where PCL's arithmetic is undefined -- an extent * inverse leaf that is not a float below
//     2^31, a dx*dy*dz product beyond int64, min or max * inverse leaf outside int32 -- the ring's set passes through,
//     as when the guard trips.
//   Output.  sharp (all rings) + less-sharp (which includes the sharp points again) + flat + less-flat, rotated by
//     Affine3f::Identity().rotate(AngleAxisf(pi/2, Y)).rotate(AngleAxisf(pi/2, Z)) with pcl::transformPointCloud's
//     association; intensity is carried, normals and curvature are zero.
//   Transcendentals.  atanf / atan2f / sinf / cosf are read as the double function rounded to float (hd.h).
#pragma once

#include "hd.h"

namespace lb {

constexpr double kFeatPi = 3.14159265358979323846;   // M_PI
constexpr int FEAT_MAX_RINGS = 128;
constexpr int FEAT_MAX_CURVATURE_REGION = 32;
constexpr int FEAT_MAX_REGIONS = 1024;
constexpr signed char FEAT_NO_REGION = 3;            // label of a position outside every unskipped region
constexpr signed char FEAT_CORNER_SHARP = 2, FEAT_CORNER_LESS_SHARP = 1, FEAT_SURFACE_LESS_FLAT = 0, FEAT_SURFACE_FLAT = -1;

struct FeatParams {
  int n_rings;
  float lower, upper, scan_period;
  int cr, n_regions, max_sharp, max_less_sharp, max_flat;
  float curv_thr, leaf;
  float factor;                                      // float(n_rings - 1) / (upper - lower)
};

LB_HD float feat_atan(float x) { return (float)atan((double)x); }
LB_HD float feat_atan2(float y, float x) { return (float)atan2((double)y, (double)x); }

// startOri / endOri from the raw x, y of input points 0 and n-1
LB_HD void feat_scan_bounds(float x0, float y0, float xl, float yl, float& start, float& end) {
  start = -feat_atan2(y0, x0);
  end = -feat_atan2(yl, xl) + 2.0f * (float)kFeatPi;
  if (end - start > 3 * kFeatPi) end = (float)(end - 2 * kFeatPi);
  else if (end - start < kFeatPi) end = (float)(end + 2 * kFeatPi);
}

// ring of one input point (raw ix, iy, iz), -1 when it is dropped; (x, y, z) receive the swapped coordinates
LB_HD int feat_ring(float ix, float iy, float iz, const FeatParams& p, float& x, float& y, float& z) {
  x = iy; y = iz; z = ix;
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return -1;
  if ((double)(x * x + y * y + z * z) < 0.0001) return -1;
  const float angle = feat_atan(y / sqrtf(x * x + z * z));
  const int ring = (int)(((double)(angle * 180.0f) / kFeatPi - (double)p.lower) * (double)p.factor + 0.5);
  return (ring >= p.n_rings || ring < 0) ? -1 : ring;
}

// orientation before halfPassed (branch A) and whether this point switches halfPassed on
LB_HD float feat_ori_a(float x, float z, float start) {
  float ori = -feat_atan2(x, z);
  if (ori < start - kFeatPi / 2) ori = (float)(ori + 2 * kFeatPi);
  else if (ori > start + kFeatPi * 3 / 2) ori = (float)(ori - 2 * kFeatPi);
  return ori;
}
LB_HD bool feat_half_passes(float ori_a, float start) { return ori_a - start > kFeatPi; }
// orientation after halfPassed (branch B)
LB_HD float feat_ori_b(float x, float z, float end) {
  float ori = -feat_atan2(x, z);
  ori = (float)(ori + 2 * kFeatPi);
  if (ori < end - kFeatPi * 3 / 2) ori = (float)(ori + 2 * kFeatPi);
  else if (ori > end + kFeatPi / 2) ori = (float)(ori - 2 * kFeatPi);
  return ori;
}
LB_HD float feat_intensity(int ring, float ori, float start, float end, float scan_period) {
  const float rel = scan_period * (ori - start) / (end - start);
  return (float)ring + rel;
}

// ------------------------------------------------------------------ per ring (P: the ring's points, ring-local index)
LB_HD float feat_sqdiff(const f4& a, const f4& b) {
  const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
  return dx * dx + dy * dy + dz * dz;
}
LB_HD float feat_sqdiff_w(const f4& a, const f4& b, float wb) {
  const float dx = a.x - b.x * wb, dy = a.y - b.y * wb, dz = a.z - b.z * wb;
  return dx * dx + dy * dy + dz * dz;
}
LB_HD float feat_sqnorm(const f4& p) { return p.x * p.x + p.y * p.y + p.z * p.z; }

LB_HD bool feat_ring_skipped(long long cnt, int cr) { return cnt <= 2ll * cr + 1; }

// region j of a ring of cnt points: [sp, ep], ring-local; skipped when ep <= sp
LB_HD void feat_region(long long cnt, int cr, int n_regions, int j, long long& sp, long long& ep) {
  const long long d = cnt - 1 - 2ll * cr;
  sp = cr + ((long long)j * d) / n_regions;
  ep = cr + ((long long)(j + 1) * d) / n_regions - 1;
}

// setScanBuffersFor at position i in [cr, cnt-1-cr): sets flags only
LB_HD void feat_unreliable_marks(const f4* P, long long i, int cr, unsigned char* picked) {
  const f4 prev = P[i - 1], pt = P[i], next = P[i + 1];
  const float diff_next = feat_sqdiff(next, pt);
  if (diff_next > 0.1) {
    const float d1 = sqrtf(feat_sqnorm(pt)), d2 = sqrtf(feat_sqnorm(next));
    if (d1 > d2) {
      const float w = sqrtf(feat_sqdiff_w(next, pt, d2 / d1)) / d2;
      if (w < 0.1) {
        for (int k = 0; k <= cr; k++) picked[i - cr + k] = 1;
        return;
      }
    } else {
      const float w = sqrtf(feat_sqdiff_w(pt, next, d1 / d2)) / d1;
      if (w < 0.1)
        for (int k = 0; k <= cr; k++) picked[i + 1 + k] = 1;
    }
  }
  const float diff_prev = feat_sqdiff(pt, prev);
  const float dis = feat_sqnorm(pt);
  if (diff_next > 0.0002 * dis && diff_prev > 0.0002 * dis) picked[i] = 1;
}

LB_HD float feat_curvature(const f4* P, long long i, int cr) {
  const float w = (float)(-2 * cr);
  float dx = w * P[i].x, dy = w * P[i].y, dz = w * P[i].z;
  for (int j = 1; j <= cr; j++) {
    dx += P[i + j].x + P[i - j].x;
    dy += P[i + j].y + P[i - j].y;
    dz += P[i + j].z + P[i - j].z;
  }
  return dx * dx + dy * dy + dz * dz;
}

LB_HD bool feat_corner_candidate(unsigned char picked, float curv, float thr) { return picked == 0 && curv > thr; }
LB_HD bool feat_flat_candidate(unsigned char picked, float curv, float thr) { return picked == 0 && curv < thr; }

// Position of region point a (sp <= a <= ep) in the order the reference's insertion sort leaves: a NaN keeps its
// place; any other point ranks after the points of its NaN-free segment with a smaller curvature, or an equal one at a
// lower position.  A permutation of [0, ep - sp] for every input.
// no_nan: the caller knows that [sp, ep] holds no NaN (skips the search for the segment)
LB_HD long long feat_region_rank(const float* curv, long long sp, long long ep, long long a, bool no_nan = false) {
  const float c = curv[a];
  if (isnan(c)) return a - sp;
  long long lo = a, hi = a;
  if (no_nan) {
    lo = sp; hi = ep;
  } else {
    while (lo > sp && !isnan(curv[lo - 1])) lo--;
    while (hi < ep && !isnan(curv[hi + 1])) hi++;
  }
  long long rank = lo - sp;
  for (long long b = lo; b <= hi; b++) {
    const float cb = curv[b];
    rank += (cb < c || (cb == c && b < a)) ? 1 : 0;
  }
  return rank;
}

LB_HD void feat_mark_as_picked(const f4* P, long long i, int cr, unsigned char* picked) {
  picked[i] = 1;
  for (int k = 1; k <= cr; k++) {
    if (feat_sqdiff(P[i + k], P[i + k - 1]) > 0.05) break;
    picked[i + k] = 1;
  }
  for (int k = 1; k <= cr; k++) {
    if (feat_sqdiff(P[i - k], P[i - k + 1]) > 0.05) break;
    picked[i - k] = 1;
  }
}

// ------------------------------------------------------------------ per-ring VoxelGrid<PointF> (PCL 1.10)
struct FeatGrid {
  float inv;
  int min_b[3], div_b[3];
  bool overflow;                                     // the cloud passes through unchanged
};
LB_HD bool feat_below_2p31(float v) { return v >= -2147483648.0f && v < 2147483648.0f; }   // false for NaN / inf
// PCL's dx*dy*dz > INT_MAX guard; the cases where PCL's own arithmetic is undefined also pass through (see the top)
LB_HD FeatGrid feat_grid(const float mn[3], const float mx[3], float leaf) {
  FeatGrid g;
  g.inv = 1.0f / leaf;
  g.overflow = false;
  long long d[3];
  for (int k = 0; k < 3; k++) {
    const float e = (mx[k] - mn[k]) * g.inv;
    const float lo = floorf(mn[k] * g.inv), hi = floorf(mx[k] * g.inv);
    if (!feat_below_2p31(e) || !feat_below_2p31(lo) || !feat_below_2p31(hi)) { g.overflow = true; d[k] = 1; continue; }
    d[k] = (long long)e + 1;
    g.min_b[k] = (int)lo;
    g.div_b[k] = (int)hi - g.min_b[k] + 1;
  }
  if (!g.overflow) g.overflow = d[0] * d[1] > 2147483647ll || d[0] * d[1] * d[2] > 2147483647ll;
  return g;
}
LB_HD int feat_voxel_key(const FeatGrid& g, float x, float y, float z) {
  const int i0 = (int)(floorf(x * g.inv) - (float)g.min_b[0]);
  const int i1 = (int)(floorf(y * g.inv) - (float)g.min_b[1]);
  const int i2 = (int)(floorf(z * g.inv) - (float)g.min_b[2]);
  return i0 + i1 * g.div_b[0] + i2 * (g.div_b[0] * g.div_b[1]);
}

// ------------------------------------------------------------------ output rotation
// Eigen's AngleAxisf::toRotationMatrix (float), row-major 3x3
LB_HD void feat_angle_axis(float theta, int axis, float* R) {
  float a[3] = {0.f, 0.f, 0.f};
  a[axis] = 1.f;
  const float s = (float)sin((double)theta), c = (float)cos((double)theta);
  const float sa[3] = {s * a[0], s * a[1], s * a[2]};
  const float ca[3] = {(1.f - c) * a[0], (1.f - c) * a[1], (1.f - c) * a[2]};
  float t;
  t = ca[0] * a[1]; R[1] = t - sa[2]; R[3] = t + sa[2];
  t = ca[0] * a[2]; R[2] = t + sa[1]; R[6] = t - sa[1];
  t = ca[1] * a[2]; R[5] = t - sa[0]; R[7] = t + sa[0];
  R[0] = ca[0] * a[0] + c; R[4] = ca[1] * a[1] + c; R[8] = ca[2] * a[2] + c;
}
// C = A * B, Eigen's coefficient order ((a0*b0 + a1*b1) + a2*b2)
LB_HD void feat_matmul3(const float* A, const float* B, float* C) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
}
// Affine3f::Identity().rotate(AngleAxisf(pi/2, UnitY)).rotate(AngleAxisf(pi/2, UnitZ)) as row-major 3x4 [M | 0]
LB_HD void feat_rotation(float* T) {
  const float theta = (float)(kFeatPi / 2);
  float I[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f}, Ry[9], Rz[9], A[9], M[9];
  feat_angle_axis(theta, 1, Ry);
  feat_angle_axis(theta, 2, Rz);
  feat_matmul3(I, Ry, A);
  feat_matmul3(A, Rz, M);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = M[3 * r + c];
    T[4 * r + 3] = 0.f;
  }
}

}  // namespace lb
