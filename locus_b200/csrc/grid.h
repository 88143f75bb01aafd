// grid.h -- dense voxel-hash index over a point cloud and exact ring searches.
//
// Replaces the FLANN KD-tree the reference reaches through
// pcl::search::KdTree (gicp.hpp:108 k-NN for covariances, gicp.h:385-391 1-NN
// correspondences, PointCloudLocalization.cc:327-336 post-align 1-NN).
//
// Layout in HBM (built once per cloud by gicp.cu):
//   pts[n]        float4, sorted by cell (x fastest, then y, then z); .w holds the
//                 ORIGINAL index of the point (int bits).
//   cell_start[ncells+1]  uint32 CSR offsets into pts.
// Because x is the fastest-varying cell coordinate, the cells (cx-r..cx+r, y, z)
// of one row are ONE contiguous run of float4 in memory: a 3x3x3 probe is nine
// contiguous runs, which is what makes the loads coalesce / hit L2 sectors.
//
// Exactness: a candidate is better iff (d2, original index) is lexicographically
// smaller; d2 = ((dx*dx)+(dy*dy))+(dz*dz) in float32 without FMA (FLANN
// L2_Simple<float>).  A search stops after ring r only when the current worst
// kept d2 is strictly below the squared distance from the query to the border
// of the scanned block, shrunk by a safety margin that covers float rounding of
// the cell assignment -- so results equal an exhaustive scan (tests/test_hd_grid).
#pragma once

#include "hd.h"

namespace lb {

struct GridView {
  const f4* pts;               // sorted by cell; w = original index bits
  const uint32_t* cell_start;  // ncells + 1
  float ox, oy, oz;            // origin (min corner)
  float inv_h, h;              // cell size
  int nx, ny, nz;
  int n;                       // number of points
};

// ---- the grid a cloud gets (origin, cell size, dimensions) --------------------------------------------------------
// One set of functions for the host driver and for the kernels of the index build, so that the geometry the device
// chooses for a cloud and the one the host fills into GridView are the same bits.  float and double arithmetic only
// (+, *, /, sqrt, floor: correctly rounded on both sides; the library is built without FMA contraction).  The cell size
// decides the order of the points in memory, hence the summation order of the align and the bits of the pose.
struct GridGeom {
  float ox, oy, oz, inv_h, h;
  int nx, ny, nz;
};

constexpr int GRID_MAXDIM = 16384;
constexpr double GRID_MAXCELLS = 64.0 * 1024 * 1024;
constexpr double GRID_TARGET_OCC = 6.0;      // points per occupied cell the automatic cell size aims at
constexpr int GRID_PROBE_ROUNDS = 4;

// Grid of cell size `cell` over the box [mn, mn + ext]; the cell grows by 1.5x until the grid fits the caps.  The loop is
// bounded: an extent that is not finite (coordinates near FLT_MAX) can never fit and ends in a single cell.
LB_HD GridGeom grid_make_geom(const float* mn, const float* ext, float cell) {
  GridGeom g;
  g.ox = mn[0]; g.oy = mn[1]; g.oz = mn[2];
  for (int grow = 0; grow < 512; grow++) {
    g.h = cell; g.inv_h = 1.0f / cell;
    double fx = floor((double)(ext[0] * g.inv_h)) + 1, fy = floor((double)(ext[1] * g.inv_h)) + 1, fz = floor((double)(ext[2] * g.inv_h)) + 1;
    if (fx <= GRID_MAXDIM && fy <= GRID_MAXDIM && fz <= GRID_MAXDIM && fx * fy * fz <= GRID_MAXCELLS) {
      g.nx = (int)fx; g.ny = (int)fy; g.nz = (int)fz;
      return g;
    }
    cell *= 1.5f;
  }
  g.nx = g.ny = g.nz = 1;
  return g;
}

// First guess of the automatic cell size: aim at ~6 points per occupied cell (h ~ 2.5 x point spacing on a surface, so
// the 20-NN radius is about one cell and a 1-NN probe rarely leaves the 3x3x3 block).  Lidar scans concentrate their
// points, so the bbox-surface spacing overestimates: 1.3x lands inside the accepted occupancy band in one round.
LB_HD float grid_auto_cell(const float* ext, uint32_t n) {
  double area = 2.0 * ((double)ext[0] * ext[1] + (double)ext[1] * ext[2] + (double)ext[0] * ext[2]);
  double diag = sqrt((double)ext[0] * ext[0] + (double)ext[1] * ext[1] + (double)ext[2] * ext[2]);
  if (!(area > 0)) area = diag * diag;
  double spacing = sqrt(area / (double)(n ? n : 1));
  float cell = (float)(1.3 * spacing);
  if (!(cell > 0.f)) cell = 1.0f;
  return cell;
}

// The grid of the first probe round for the finite bounding box [mn, mx] of n points.
LB_HD GridGeom grid_auto_geom(const float* mn, const float* mx, uint32_t n) {
  const float ext[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
  return grid_make_geom(mn, ext, grid_auto_cell(ext, n));
}

// A probe round counted n_occ occupied cells at cell size h: true when the grid is kept (occupancy inside
// [target / 2, 2 target], or nothing to gain from another round); otherwise *next_cell is the next round's cell size.
LB_HD bool grid_probe_accept(uint32_t n, uint32_t n_occ, float h, float* next_cell) {
  double occ = (double)n / (double)(n_occ ? n_occ : 1);
  if (occ >= GRID_TARGET_OCC / 2 && occ <= GRID_TARGET_OCC * 2) return true;
  if (n <= 8 || n_occ <= 1) return true;
  double scale = sqrt(GRID_TARGET_OCC / occ);
  if (scale > 4) scale = 4;
  if (scale < 0.25) scale = 0.25;
  *next_cell = h * (float)scale;
  return false;
}

// width of a cell key of a grid of ncells cells
LB_HD int grid_key_bits(uint64_t ncells) {
  int key_bits = 1;
  while (key_bits < 32 && (1ull << key_bits) < ncells) key_bits++;
  return key_bits;
}

LB_HD float dist2(float ax, float ay, float az, float bx, float by, float bz) {
  float dx = ax - bx, dy = ay - by, dz = az - bz;
  float d = dx * dx;
  d = d + dy * dy;
  d = d + dz * dz;
  return d;
}

LB_HD bool better(float d2a, int ia, float d2b, int ib) { return (d2a < d2b) || (d2a == d2b && ia < ib); }

LB_HD int iabs_(int a) { return a < 0 ? -a : a; }
LB_HD int imax_(int a, int b) { return a > b ? a : b; }
LB_HD int imin_(int a, int b) { return a < b ? a : b; }

// cell coordinate of a query (may lie outside the grid); frac = distance (in cells)
// from the query to the nearest face of its cell.
LB_HD void query_cell(const GridView& g, float qx, float qy, float qz, int& cx, int& cy, int& cz, float& minfrac) {
  float ux = (qx - g.ox) * g.inv_h, uy = (qy - g.oy) * g.inv_h, uz = (qz - g.oz) * g.inv_h;
  // clamp to a sane range so the float->int conversion is defined for far-away queries
  const float LIM = 1.0e9f;
  ux = fminf(fmaxf(ux, -LIM), LIM); uy = fminf(fmaxf(uy, -LIM), LIM); uz = fminf(fmaxf(uz, -LIM), LIM);
  float fx = floorf(ux), fy = floorf(uy), fz = floorf(uz);
  cx = (int)fx; cy = (int)fy; cz = (int)fz;
  float ax = ux - fx, ay = uy - fy, az = uz - fz;
  float m = fminf(fminf(fminf(ax, 1.0f - ax), fminf(ay, 1.0f - ay)), fminf(az, 1.0f - az));
  minfrac = m;
}

// squared lower bound on the distance from the query to any point outside the
// scanned block of Chebyshev radius r (conservative: 0.01 cell safety margin).
LB_HD float ring_bound2(const GridView& g, int r, float minfrac) {
  float b = ((float)r + minfrac - 0.01f) * g.h;
  if (b <= 0.0f) return 0.0f;
  b = b * 0.9999f;
  return b * b;
}

// Visit every point in the shell of Chebyshev radius r around (cx,cy,cz).
// F(float x, float y, float z, int orig_index, int sorted_index)
template <class F>
LB_HD void visit_shell(const GridView& g, int cx, int cy, int cz, int r, F&& f) {
  int z0 = imax_(cz - r, 0), z1 = imin_(cz + r, g.nz - 1);
  int y0 = imax_(cy - r, 0), y1 = imin_(cy + r, g.ny - 1);
  for (int z = z0; z <= z1; z++) {
    bool zface = (iabs_(z - cz) == r);
    for (int y = y0; y <= y1; y++) {
      bool face = zface || (iabs_(y - cy) == r);
      int base = (z * g.ny + y) * g.nx;
      if (face) {
        int xa = imax_(cx - r, 0), xb = imin_(cx + r, g.nx - 1);
        if (xa > xb) continue;
        uint32_t s = g.cell_start[base + xa], e = g.cell_start[base + xb + 1];
        for (uint32_t i = s; i < e; i++) {
          f4 p = g.pts[i];
          f(p.x, p.y, p.z, float_to_bits(p.w), (int)i);
        }
      } else {
        // interior row of the shell: only the two end cells x = cx-r and x = cx+r
        int xs[2] = {cx - r, cx + r};
        for (int k = 0; k < 2; k++) {
          int x = xs[k];
          if (x < 0 || x >= g.nx) continue;
          uint32_t s = g.cell_start[base + x], e = g.cell_start[base + x + 1];
          for (uint32_t i = s; i < e; i++) {
            f4 p = g.pts[i];
            f(p.x, p.y, p.z, float_to_bits(p.w), (int)i);
          }
        }
      }
    }
  }
}

// rings between cell c and the cell range [0, n) along one axis (0 inside).  Written as branches: ptxas for sm_90a
// (CUDA 12.9, -O1 and above) folds the equivalent max(max(-c, c - (n - 1)), 0) into a wrong value for c inside the range.
LB_HD int cell_ring_dist(int c, int n) {
  if (c < 0) return -c;
  if (c > n - 1) return c - (n - 1);
  return 0;
}

// first ring that can contain grid cells, and the ring after which the whole grid is covered
LB_HD void ring_range(const GridView& g, int cx, int cy, int cz, int& r_first, int& r_last) {
  const int fx = cell_ring_dist(cx, g.nx), fy = cell_ring_dist(cy, g.ny), fz = cell_ring_dist(cz, g.nz);
  r_first = imax_(fx, imax_(fy, fz));
  int lx = imax_(iabs_(cx), iabs_(g.nx - 1 - cx));
  int ly = imax_(iabs_(cy), iabs_(g.ny - 1 - cy));
  int lz = imax_(iabs_(cz), iabs_(g.nz - 1 - cz));
  r_last = imax_(lx, imax_(ly, lz));
}

// Exact nearest neighbour with a strict gate d2 < max_d2 (gicp.hpp:483).
// Returns the SORTED index of the neighbour (or -1); orig index and d2 by reference.
LB_HD int nn1(const GridView& g, float qx, float qy, float qz, float max_d2, int& best_orig, float& best_d2) {
  int cx, cy, cz; float minfrac;
  query_cell(g, qx, qy, qz, cx, cy, cz, minfrac);
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  float bd2 = max_d2; int bi = -1; int bs = -1;
  bool found = false;
  for (int r = r0; r <= r1; r++) {
    if (r > r0 || r0 > 0) {
      // everything not yet scanned is at least this far away
      float lb2 = ring_bound2(g, r - 1, minfrac);
      if (lb2 >= max_d2) break;
      if (found && bd2 < lb2) break;
    }
    visit_shell(g, cx, cy, cz, r, [&](float x, float y, float z, int oi, int si) {
      float d = dist2(qx, qy, qz, x, y, z);
      if (!found) {
        if (d < max_d2) { found = true; bd2 = d; bi = oi; bs = si; }
      } else if (better(d, oi, bd2, bi)) {
        bd2 = d; bi = oi; bs = si;
      }
    });
  }
  best_orig = bi; best_d2 = bd2;
  return bs;
}

// Same result as nn1(), with far fewer candidates: what the correspondence step of align() calls.
// nn1() scans every cell of a Chebyshev shell.  Here a cell (or a whole x-row of a shell) is only opened when the box it
// covers can still hold a point closer than the best one found so far: per axis the gap between the query and the cell,
// in cells, is (|i| - 1 + distance to the facing cell wall), so a lower bound of the distance to anything in the cell is
// h * sqrt(gx^2 + gy^2 + gz^2), shrunk by the same safety margin as ring_bound2 (it covers the float rounding of the
// cell assignment).  The centre cell goes first, so when the clouds are nearly aligned -- every outer iteration after
// the first -- the search ends after a handful of cells instead of 27.  Exactness: a cell is skipped only if its lower
// bound is strictly greater than the best d2 (or not below the gate), so neither a closer point nor an equidistant one
// with a lower index can be missed; ties are still broken by (d2, original index).
LB_HD float nn1_gap(int i, float f) {      // gap in cells along one axis between the query and cell offset i (f = fractional position in its own cell)
  if (i == 0) return 0.0f;
  float g = (i > 0) ? ((float)(i - 1) + (1.0f - f)) : ((float)(-i - 1) + f);
  g = g - 0.01f;
  return g > 0.0f ? g : 0.0f;
}
LB_HD int nn1_pruned(const GridView& g, float qx, float qy, float qz, float max_d2, int& best_orig, float& best_d2) {
  float ux = (qx - g.ox) * g.inv_h, uy = (qy - g.oy) * g.inv_h, uz = (qz - g.oz) * g.inv_h;
  const float LIM = 1.0e9f;
  ux = fminf(fmaxf(ux, -LIM), LIM); uy = fminf(fmaxf(uy, -LIM), LIM); uz = fminf(fmaxf(uz, -LIM), LIM);
  const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
  const int cx = (int)flx, cy = (int)fly, cz = (int)flz;
  const float fx = ux - flx, fy = uy - fly, fz = uz - flz;
  const float minfrac = fminf(fminf(fminf(fx, 1.0f - fx), fminf(fy, 1.0f - fy)), fminf(fz, 1.0f - fz));
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  const float hs = g.h * 0.9999f;
  const float hh = hs * hs;
  float bd2 = max_d2; int bi = -1; int bs = -1;
  bool found = false;
  // candidates [s, e) of the cell-sorted cloud: four loads in flight per trip (every lane of a warp reads its own
  // addresses, and with one CTA per SM nothing else hides the L2 latency of a load -> use -> branch loop)
  auto scan = [&](uint32_t s, uint32_t e) {
    for (uint32_t i = s; i < e; i += 4) {
      f4 pv[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
      for (uint32_t u = 0; u < 4; u++) pv[u] = g.pts[(i + u < e) ? (i + u) : (e - 1)];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
      for (uint32_t u = 0; u < 4; u++) {
        if (i + u >= e) break;
        const float d = dist2(qx, qy, qz, pv[u].x, pv[u].y, pv[u].z);
        const int oi = float_to_bits(pv[u].w);
        if (!found) {
          if (d < max_d2) { found = true; bd2 = d; bi = oi; bs = (int)(i + u); }
        } else if (better(d, oi, bd2, bi)) {
          bd2 = d; bi = oi; bs = (int)(i + u);
        }
      }
    }
  };
  // ---- step 1: the 3x3x3 block, cell by cell, centre first, each cell only while it can still hold a closer point
  if (r0 <= 1) {
    const int ORD[3] = {0, -1, 1};
    for (int a = 0; a < 3; a++) {
      const int z = cz + ORD[a];
      if (z < 0 || z >= g.nz) continue;
      const float gz = nn1_gap(ORD[a], fz);
      for (int b = 0; b < 3; b++) {
        const int y = cy + ORD[b];
        if (y < 0 || y >= g.ny) continue;
        const float gy = nn1_gap(ORD[b], fy);
        const float row2 = (gy * gy + gz * gz) * hh;
        if (row2 > bd2 || row2 >= max_d2) continue;
        const int base = (z * g.ny + y) * g.nx;
        // the row's four CSR offsets (cells cx-1, cx, cx+1) are fetched together, then centre, left, right
        uint32_t cs4[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int c = 0; c < 4; c++) {
          const int x = cx - 1 + c;
          cs4[c] = (x >= 0 && x <= g.nx) ? g.cell_start[base + x] : 0u;
        }
        for (int c = 0; c < 3; c++) {
          const int x = cx + ORD[c];
          if (x < 0 || x >= g.nx) continue;
          const float gx = nn1_gap(ORD[c], fx);
          const float c2 = row2 + (gx * gx) * hh;
          if (c2 > bd2 || c2 >= max_d2) continue;
          scan(cs4[ORD[c] + 1], cs4[ORD[c] + 2]);
        }
      }
    }
    const float lb2 = ring_bound2(g, 1, minfrac);
    if (r1 <= 1 || lb2 >= max_d2 || (found && bd2 < lb2)) { best_orig = bi; best_d2 = bd2; return bs; }
    // ---- step 2: the block could not decide (the nearest point is farther than a cell away, or there is none in
    // the block).  Everything that can still matter lies in the cube of cells whose lower bound is within the current
    // bound (best so far, else the gate).  Its x-rows are visited ring by ring; a row costs TWO look-ups (the CSR
    // offsets of the ends of its x-window, which shrinks with the remaining distance budget) and most rows of a
    // surface-like cloud are empty -- the look-ups of 8 rows are issued together so their latencies overlap.
    const float bound2 = found ? bd2 : max_d2;
    const float G = sqrtf(bound2) / hs;
    if (G < 12.0f) {
      const int Rc = (int)(G + 1.01f) + 1;
      for (int ring = 0; ring <= Rc; ring++) {
        if (ring > 1) {
          // every row of this ring is at least (ring - 1 + frac - 0.01) cells away in y or z: stop when that exceeds the bound
          const float gmin = nn1_gap(ring, fmaxf(fmaxf(fy, 1.0f - fy), fmaxf(fz, 1.0f - fz)));   // (ring - 1) + the smallest distance to a y / z cell wall
          if (gmin * gmin * hh > bd2 || gmin * gmin * hh >= max_d2) break;
        }
        const int side = 2 * ring + 1;
        const int nrows = ring == 0 ? 1 : 8 * ring;             // rows on the perimeter of the (2 ring + 1)^2 square
        for (int jb = 0; jb < nrows; jb += 8) {
          uint32_t rs[8], re[8];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
          for (int u = 0; u < 8; u++) {
            rs[u] = 0; re[u] = 0;
            const int j = jb + u;
            if (j >= nrows) continue;
            // perimeter walk: top edge, bottom edge, then the two sides without their corners
            int dy, dz;
            if (ring == 0) { dy = 0; dz = 0; }
            else if (j < side) { dz = -ring; dy = j - ring; }
            else if (j < 2 * side) { dz = ring; dy = j - side - ring; }
            else if (j < 2 * side + (side - 2)) { dy = -ring; dz = j - 2 * side - ring + 1; }
            else { dy = ring; dz = j - 2 * side - (side - 2) - ring + 1; }
            const int z = cz + dz, y = cy + dy;
            if (z < 0 || z >= g.nz || y < 0 || y >= g.ny) continue;
            const float gy = nn1_gap(dy, fy), gz = nn1_gap(dz, fz);
            const float row2 = (gy * gy + gz * gz) * hh;
            if (row2 > bd2 || row2 >= max_d2) continue;
            // x-window: cells whose gap fits into what is left of the bound
            const float rem = fminf(bd2, max_d2) - row2;
            const int wx = (int)(sqrtf(rem > 0.f ? rem : 0.f) / hs + 1.01f) + 1;
            const int xlo = imax_(cx - wx, 0), xhi = imin_(cx + wx, g.nx - 1);
            if (xlo > xhi) continue;
            const int base = (z * g.ny + y) * g.nx;
            rs[u] = g.cell_start[base + xlo];
            re[u] = g.cell_start[base + xhi + 1];
          }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
          for (int u = 0; u < 8; u++) scan(rs[u], re[u]);
        }
      }
      best_orig = bi; best_d2 = bd2;
      return bs;
    }
  }
  // ---- far queries (outside the grid, or an unbounded search that found nothing nearby): shell by shell like nn1
  for (int r = (r0 <= 1 ? 2 : r0); r <= r1; r++) {
    if (r > r0 || r0 > 0) {
      const float lb2 = ring_bound2(g, r - 1, minfrac);      // everything not yet scanned is at least this far away
      if (lb2 >= max_d2) break;
      if (found && bd2 < lb2) break;
    }
    visit_shell(g, cx, cy, cz, r, [&](float x, float y, float z, int oi, int si) {
      float d = dist2(qx, qy, qz, x, y, z);
      if (!found) {
        if (d < max_d2) { found = true; bd2 = d; bi = oi; bs = si; }
      } else if (better(d, oi, bd2, bi)) {
        bd2 = d; bi = oi; bs = si;
      }
    });
  }
  best_orig = bi; best_d2 = bd2;
  return bs;
}

// ---- the cells a ball around a query touches (what the staged search of nn_staged.cuh enumerates) -------------------
// Rows (dy, dz) and, per row, the x-window of the cells whose conservative lower-bound distance (nn1_gap: 0.01 cell
// safety margin, cell size shrunk by 0.9999) does not exceed the radius.  The windows may be too wide, never too narrow:
// sqrt is allowed to be an approximation that errs upwards (the device uses rsqrt).  Shared by the device code and by
// nn1_ball_serial(), the serial restatement the CPU tests run against the kd-tree.
struct BallGeom {
  int cx, cy, cz;          // cell of the query (may lie outside the grid)
  float fx, fy, fz;        // position inside that cell, [0, 1)
  float hs, hh, inv_hs;    // shrunk cell size, its square, its reciprocal rounded up
};
LB_HD float ball_sqrt_up(float x) {
#if defined(__CUDA_ARCH__)
  return x > 0.f ? x * rsqrtf(x) * 1.00001f : 0.f;
#else
  return x > 0.f ? sqrtf(x) * 1.00001f : 0.f;
#endif
}
LB_HD void ball_geom(const GridView& g, float qx, float qy, float qz, BallGeom& b) {
  float ux = (qx - g.ox) * g.inv_h, uy = (qy - g.oy) * g.inv_h, uz = (qz - g.oz) * g.inv_h;
  const float LIM = 1.0e9f;
  ux = fminf(fmaxf(ux, -LIM), LIM); uy = fminf(fmaxf(uy, -LIM), LIM); uz = fminf(fmaxf(uz, -LIM), LIM);
  const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
  b.cx = (int)flx; b.cy = (int)fly; b.cz = (int)flz;
  b.fx = ux - flx; b.fy = uy - fly; b.fz = uz - flz;
  b.hs = g.h * 0.9999f;
  b.hh = b.hs * b.hs;
  b.inv_hs = 1.0002f / b.hs;
}
// radius of the ball in cells (+ margin); rows dy in [ylo, yhi], dz in [zlo, zhi] (not clamped to the grid)
LB_HD float ball_rows(const BallGeom& b, float b2, int& ylo, int& yhi, int& zlo, int& zhi) {
  const float S = sqrtf(b2) / b.hs + 1.0e-4f;
  if (S < 1.0e6f) {
    ylo = -(int)(S + 1.01f - b.fy); yhi = (int)(S + b.fy + 0.01f);
    zlo = -(int)(S + 1.01f - b.fz); zhi = (int)(S + b.fz + 0.01f);
  } else { ylo = yhi = zlo = zhi = 0; }
  return S;
}
// x-window of row (dy, dz) for squared radius e2; false when the row lies outside the ball or the grid
LB_HD bool ball_window(const GridView& g, const BallGeom& b, int dy, int dz, float e2, int& xlo, int& xhi) {
  const int z = b.cz + dz, y = b.cy + dy;
  if (z < 0 || z >= g.nz || y < 0 || y >= g.ny) return false;
  const float gy = nn1_gap(dy, b.fy), gz = nn1_gap(dz, b.fz);
  const float row2 = (gy * gy + gz * gz) * b.hh;
  if (!(row2 <= e2)) return false;
  const float Sx = ball_sqrt_up(e2 - row2) * b.inv_hs + 1.0e-3f;
  xlo = imax_(b.cx - (int)(Sx + 1.01f - b.fx), 0);
  xhi = imin_(b.cx + (int)(Sx + b.fx + 0.01f), g.nx - 1);
  return xlo <= xhi;
}

// Serial restatement of the staged search (nn_staged.cuh): first look = the ball that guarantees completeness (the
// known bound ub2 when have_ub, else the gate) cut to r0cut cells; final when the ball was complete or its best lies
// inside it; otherwise the remaining ball (best so far / bound / gate), shrinking row by row; huge balls fall back to
// nn1_pruned.  Same answers as nn1() / nn1_pruned() -- tests/test_hd_cpu.py checks that against the kd-tree.
LB_HD int nn1_ball_serial(const GridView& g, float qx, float qy, float qz, float max_d2, bool have_ub, float ub2, float r0cut,
                          int& best_orig, float& best_d2) {
  BallGeom b;
  ball_geom(g, qx, qy, qz, b);
  int r0, r1;
  ring_range(g, b.cx, b.cy, b.cz, r0, r1);
  if (r0 > 1 || !(max_d2 > 0.f)) return nn1_pruned(g, qx, qy, qz, max_d2, best_orig, best_d2);
  float bd2 = max_d2; int bi = -1, bs = -1;
  bool found = false;
  auto scan_ball = [&](float b2, bool shrink) {
    int ylo, yhi, zlo, zhi;
    ball_rows(b, b2, ylo, yhi, zlo, zhi);
    for (int dz = zlo; dz <= zhi; dz++)
      for (int dy = ylo; dy <= yhi; dy++) {
        const float e2 = (shrink && found) ? fminf(b2, bd2) : b2;
        int xlo, xhi;
        if (!ball_window(g, b, dy, dz, e2, xlo, xhi)) continue;
        const int base = ((b.cz + dz) * g.ny + (b.cy + dy)) * g.nx;
        for (uint32_t i = g.cell_start[base + xlo]; i < g.cell_start[base + xhi + 1]; i++) {
          const f4 p = g.pts[i];
          const float d = dist2(qx, qy, qz, p.x, p.y, p.z);
          const int oi = float_to_bits(p.w);
          if (!found) { if (d < max_d2) { found = true; bd2 = d; bi = oi; bs = (int)i; } }
          else if (better(d, oi, bd2, bi)) { bd2 = d; bi = oi; bs = (int)i; }
        }
      }
  };
  const bool hub = have_ub && ub2 < max_d2;
  const float need2 = hub ? ub2 : max_d2;
  const float cap2 = r0cut > 0.f ? (r0cut * r0cut) * b.hh : need2;
  const float b2 = fminf(need2, cap2);
  bool decided = false;
  if (sqrtf(b2) / b.hs + 1.0e-4f < 4.0f) {
    scan_ball(b2, true);
    decided = (need2 <= cap2) || (found && bd2 <= b2);
  }
  if (!decided) {
    const float ball2 = fminf(found ? bd2 : max_d2, need2);
    if (sqrtf(ball2) / b.hs + 1.0e-4f < 24.0f) scan_ball(ball2, true);
    else return nn1_pruned(g, qx, qy, qz, max_d2, best_orig, best_d2);
  }
  best_orig = bi; best_d2 = bd2;
  return bs;
}

// Exact k nearest neighbours (unbounded radius, like FLANN nearestKSearch).
// Kept ascending by (d2, orig index) in d2s/idx/sidx (arrays of length >= K).
// Returns the number found (min(K, n)).
template <int KMAX>
struct KnnList {
  float d2[KMAX];
  int oi[KMAX];   // original index
  int si[KMAX];   // sorted index
  int k, cnt;
  LB_HD void init(int k_) {
    k = k_; cnt = 0;
#pragma unroll
    for (int i = 0; i < KMAX; i++) { d2[i] = 3.0e38f; oi[i] = 0x7fffffff; si[i] = -1; }
  }
  LB_HD float worst() const { return d2[k - 1]; }
  LB_HD void push(float d, int o, int s) {
    // list is padded with (+huge, INT_MAX): a plain "better than last" test works while filling
    if (!better(d, o, d2[k - 1], oi[k - 1])) return;
    if (cnt < k) cnt++;
    // insert by bubbling up from the last slot (static indices when unrolled)
    d2[k - 1] = d; oi[k - 1] = o; si[k - 1] = s;
#pragma unroll
    for (int j = KMAX - 1; j > 0; j--) {
      if (j <= k - 1 && better(d2[j], oi[j], d2[j - 1], oi[j - 1])) {
        float td = d2[j]; d2[j] = d2[j - 1]; d2[j - 1] = td;
        int to = oi[j]; oi[j] = oi[j - 1]; oi[j - 1] = to;
        int ts = si[j]; si[j] = si[j - 1]; si[j - 1] = ts;
      }
    }
  }
};

// Sorted candidate list with STATIC indexing only, so that a fully unrolled build keeps it in registers (a list
// indexed by a loop-carried position lives in local memory and every insertion becomes a chain of dependent
// loads and stores).  Order = better(): ascending (d2, original index), packed into one 64-bit key -- d2 >= 0, so
// its float bits are monotone as an unsigned integer.  Unfilled entries hold the all-ones sentinel.  Only the key
// is kept: the point itself is fetched again through its original index when it is needed.
// `gate`: an extra rejection threshold the caller may tighten (see knn_cov_quadreg_kernel); candidates with
// key >= gate are known not to belong to the result.
template <int K>
struct RegList {
  unsigned long long key[K];
  unsigned long long gate;
  int cnt;
  LB_HD static unsigned long long make_key(float d2, int orig) {
    return ((unsigned long long)(uint32_t)float_to_bits(d2) << 32) | (uint32_t)orig;
  }
  LB_HD void init() {
    cnt = 0; gate = ~0ull;
#pragma unroll
    for (int i = 0; i < K; i++) key[i] = ~0ull;
  }
  LB_HD void push(float d2, int orig, int /*sorted position: not kept*/ = 0) {
    const unsigned long long k = make_key(d2, orig);
    if (k >= key[K - 1] || k >= gate) return;
    cnt += (cnt < K) ? 1 : 0;
    bool here = true;                       // k < (old) key[j]
#pragma unroll
    for (int j = K - 1; j > 0; j--) {
      const bool up = k < key[j - 1];       // the new entry belongs below j: slot j takes its lower neighbour
      key[j] = up ? key[j - 1] : (here ? k : key[j]);
      here = up;
    }
    if (here) key[0] = k;
  }
};

template <int KMAX>
LB_HD int knn(const GridView& g, float qx, float qy, float qz, int k, KnnList<KMAX>& L) {
  L.init(k);
  int cx, cy, cz; float minfrac;
  query_cell(g, qx, qy, qz, cx, cy, cz, minfrac);
  int r0, r1;
  ring_range(g, cx, cy, cz, r0, r1);
  for (int r = r0; r <= r1; r++) {
    if (L.cnt == k && r > 0) {
      float lb2 = ring_bound2(g, r - 1, minfrac);
      if (L.worst() < lb2) break;
    }
    visit_shell(g, cx, cy, cz, r, [&](float x, float y, float z, int oi, int si) {
      L.push(dist2(qx, qy, qz, x, y, z), oi, si);
    });
  }
  return L.cnt;
}

}  // namespace lb
