/*
 * features_oracle.c -- CPU restatement of the `filtering/extract_features` branch of PointCloudFilter::Filter
 * (point_cloud_filter/src/PointCloudFilter.cc:144-173, arrangePCLInScanLines / extractFeatures / setRegionBuffersFor /
 * setScanBuffersFor / markAsPicked / getRingForAngle :179-515, constants PointCloudFilter.h:79-96), followed by
 * pcl::VoxelGrid<PointF> (PCL 1.10) on each ring's less-flat points and pcl::transformPointCloud with the fixed
 * rotation of Filter().
 * TEST INFRASTRUCTURE ONLY.  Written in the reference's own shape: global ring-major indices, size_t region bounds, the
 * O(n^2) insertion sort without early exit, one serial pass per ring.
 * The reference holds no test of this code -> PARITY UNPINNED; pinned readings (DESIGN.md section 2):
 *   - atanf / atan2f / sinf / cosf are the double function rounded to float;
 *   - inside a voxel the points are summed in ascending position (PCL sorts with std::sort, which is unstable);
 *   - the rotation is built as Eigen does for 3x3 float: coefficient ((a0*b0 + a1*b1) + a2*b2).
 * Compile with -ffp-contract=off.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct of_params {
  int n_rings;
  float lower_deg, upper_deg, scan_period;
  int curvature_region, n_feature_regions, max_corner_sharp, max_corner_less_sharp, max_surface_flat;
  float curvature_threshold, less_flat_leaf;
} of_params;

typedef struct { float x, y, z, intensity; } of_pt;

enum { CORNER_SHARP = 2, CORNER_LESS_SHARP = 1, SURFACE_LESS_FLAT = 0, SURFACE_FLAT = -1 };

#define OF_PI 3.14159265358979323846

static float of_atan(float x) { return (float)atan((double)x); }
static float of_atan2(float y, float x) { return (float)atan2((double)y, (double)x); }

static float sq_diff(const of_pt* a, const of_pt* b) {
  float dx = a->x - b->x, dy = a->y - b->y, dz = a->z - b->z;
  return dx * dx + dy * dy + dz * dz;
}
static float sq_diff_w(const of_pt* a, const of_pt* b, float wb) {
  float dx = a->x - b->x * wb, dy = a->y - b->y * wb, dz = a->z - b->z * wb;
  return dx * dx + dy * dy + dz * dz;
}
static float pt_dist(const of_pt* p) { return sqrtf(p->x * p->x + p->y * p->y + p->z * p->z); }
static float pt_sqdist(const of_pt* p) { return p->x * p->x + p->y * p->y + p->z * p->z; }

/* a growable point list */
typedef struct { of_pt* p; size_t n, cap; } of_cloud;
static void push(of_cloud* c, of_pt v) {
  if (c->n == c->cap) { c->cap = c->cap ? 2 * c->cap : 64; c->p = (of_pt*)realloc(c->p, c->cap * sizeof(of_pt)); }
  c->p[c->n++] = v;
}
static void append(of_cloud* c, const of_cloud* b) { for (size_t i = 0; i < b->n; i++) push(c, b->p[i]); }

typedef struct { int idx; size_t pos; } vox_ix;
static int cmp_vox(const void* a, const void* b) {
  const vox_ix* x = (const vox_ix*)a; const vox_ix* y = (const vox_ix*)b;
  if (x->idx != y->idx) return x->idx < y->idx ? -1 : 1;
  return (x->pos > y->pos) - (x->pos < y->pos);
}

/* pcl::VoxelGrid<PointF> (PCL 1.10 voxel_grid.hpp applyFilter), dense cloud, no filter field, all data averaged */
static void voxel_grid(const of_cloud* in, float leaf, of_cloud* out) {
  if (in->n == 0) return;
  float inv = 1.0f / leaf;
  float mn[3] = {in->p[0].x, in->p[0].y, in->p[0].z}, mx[3] = {in->p[0].x, in->p[0].y, in->p[0].z};
  for (size_t i = 1; i < in->n; i++) {
    float v[3] = {in->p[i].x, in->p[i].y, in->p[i].z};
    for (int d = 0; d < 3; d++) { if (v[d] < mn[d]) mn[d] = v[d]; if (v[d] > mx[d]) mx[d] = v[d]; }
  }
  /* PCL: dx*dy*dz > INT_MAX -> output = *input_.  Where PCL's own arithmetic is undefined (an extent * inv that is not a
   * float below 2^31, min / max * inv outside int32) the set passes through as well (pinned, DESIGN.md section 2). */
  int64_t dd[3];
  int min_b[3], div_b[3];
  for (int d = 0; d < 3; d++) {
    float e = (mx[d] - mn[d]) * inv, lo = floorf(mn[d] * inv), hi = floorf(mx[d] * inv);
    if (!(e < 2147483648.0f) || !(lo >= -2147483648.0f && lo < 2147483648.0f) || !(hi >= -2147483648.0f && hi < 2147483648.0f)) {
      append(out, in);
      return;
    }
    dd[d] = (int64_t)e + 1;
    min_b[d] = (int)lo;
    div_b[d] = (int)hi - min_b[d] + 1;
  }
  if (dd[0] * dd[1] > (int64_t)INT32_MAX || dd[0] * dd[1] * dd[2] > (int64_t)INT32_MAX) { append(out, in); return; }
  vox_ix* iv = (vox_ix*)malloc(in->n * sizeof(vox_ix));
  for (size_t i = 0; i < in->n; i++) {
    int i0 = (int)(floorf(in->p[i].x * inv) - (float)min_b[0]);
    int i1 = (int)(floorf(in->p[i].y * inv) - (float)min_b[1]);
    int i2 = (int)(floorf(in->p[i].z * inv) - (float)min_b[2]);
    iv[i].idx = i0 + i1 * div_b[0] + i2 * (div_b[0] * div_b[1]);
    iv[i].pos = i;
  }
  qsort(iv, in->n, sizeof(vox_ix), cmp_vox);
  for (size_t a = 0; a < in->n;) {
    size_t e = a + 1;
    while (e < in->n && iv[e].idx == iv[a].idx) e++;
    of_pt c = in->p[iv[a].pos];
    for (size_t j = a + 1; j < e; j++) {
      const of_pt* q = &in->p[iv[j].pos];
      c.x = c.x + q->x; c.y = c.y + q->y; c.z = c.z + q->z; c.intensity = c.intensity + q->intensity;
    }
    float cnt = (float)(e - a);
    c.x = c.x / cnt; c.y = c.y / cnt; c.z = c.z / cnt; c.intensity = c.intensity / cnt;
    push(out, c);
    a = e;
  }
  free(iv);
}

static void angle_axis(float theta, int axis, float R[9]) {
  float a[3] = {0.f, 0.f, 0.f};
  a[axis] = 1.f;
  float s = (float)sin((double)theta), c = (float)cos((double)theta);
  float sa[3] = {s * a[0], s * a[1], s * a[2]};
  float ca[3] = {(1.f - c) * a[0], (1.f - c) * a[1], (1.f - c) * a[2]};
  float t;
  t = ca[0] * a[1]; R[1] = t - sa[2]; R[3] = t + sa[2];
  t = ca[0] * a[2]; R[2] = t + sa[1]; R[6] = t - sa[1];
  t = ca[1] * a[2]; R[5] = t - sa[0]; R[7] = t + sa[0];
  R[0] = ca[0] * a[0] + c; R[4] = ca[1] * a[1] + c; R[8] = ca[2] * a[2] + c;
}
static void matmul3(const float* A, const float* B, float* C) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
}

/* xyz: n points, `stride_floats` floats apart.  counts[6] = arranged, sharp, less-sharp, flat, less-flat, out.
 * Returns 0, -1 for n == 0, -3 when out_cap < counts[5] (nothing written). */
int of_extract_features(const float* xyz, size_t n, size_t stride_floats, const of_params* P, float* out4,
                        size_t out_cap, size_t* counts) {
  for (int i = 0; i < 6; i++) counts[i] = 0;
  if (n == 0) return -1;
  const size_t cr = (size_t)P->curvature_region;
  const int R = P->n_feature_regions;
  const float factor = (float)(P->n_rings - 1) / (P->upper_deg - P->lower_deg);
  /* ---- arrangePCLInScanLines */
  const float* p0 = xyz;
  const float* pl = xyz + (n - 1) * stride_floats;
  float startOri = -of_atan2(p0[1], p0[0]);
  float endOri = -of_atan2(pl[1], pl[0]) + 2 * (float)OF_PI;
  if (endOri - startOri > 3 * OF_PI) endOri -= 2 * OF_PI;
  else if (endOri - startOri < OF_PI) endOri += 2 * OF_PI;
  int halfPassed = 0;
  of_cloud* scans = (of_cloud*)calloc((size_t)P->n_rings, sizeof(of_cloud));
  for (size_t i = 0; i < n; i++) {
    const float* q = xyz + i * stride_floats;
    of_pt point;
    point.x = q[1]; point.y = q[2]; point.z = q[0];
    if (!isfinite(point.x) || !isfinite(point.y) || !isfinite(point.z)) continue;
    if (point.x * point.x + point.y * point.y + point.z * point.z < 0.0001) continue;
    float angle = of_atan(point.y / sqrtf(point.x * point.x + point.z * point.z));
    int scanID = (int)(((angle * 180 / OF_PI) - P->lower_deg) * factor + 0.5);
    if (scanID >= P->n_rings || scanID < 0) continue;
    float ori = -of_atan2(point.x, point.z);
    if (!halfPassed) {
      if (ori < startOri - OF_PI / 2) ori += 2 * OF_PI;
      else if (ori > startOri + OF_PI * 3 / 2) ori -= 2 * OF_PI;
      if (ori - startOri > OF_PI) halfPassed = 1;
    } else {
      ori += 2 * OF_PI;
      if (ori < endOri - OF_PI * 3 / 2) ori += 2 * OF_PI;
      else if (ori > endOri + OF_PI / 2) ori -= 2 * OF_PI;
    }
    float relTime = P->scan_period * (ori - startOri) / (endOri - startOri);
    point.intensity = scanID + relTime;
    push(&scans[scanID], point);
  }
  of_cloud cloud = {0, 0, 0};
  size_t* first = (size_t*)malloc((size_t)P->n_rings * sizeof(size_t));
  size_t* last = (size_t*)malloc((size_t)P->n_rings * sizeof(size_t));
  size_t cloudSizeScans = 0;
  for (int r = 0; r < P->n_rings; r++) {
    append(&cloud, &scans[r]);
    first[r] = cloudSizeScans;
    cloudSizeScans += scans[r].n;
    last[r] = cloudSizeScans > 0 ? cloudSizeScans - 1 : 0;
  }
  /* ---- extractFeatures */
  of_cloud sharp = {0, 0, 0}, less_sharp = {0, 0, 0}, flat = {0, 0, 0}, less_flat = {0, 0, 0};
  int* picked = (int*)malloc((cloud.n + 1) * sizeof(int));
  float* curv = (float*)malloc((cloud.n + 1) * sizeof(float));
  size_t* sortIdx = (size_t*)malloc((cloud.n + 1) * sizeof(size_t));
  int* label = (int*)malloc((cloud.n + 1) * sizeof(int));
  for (int r = 0; r < P->n_rings; r++) {
    const size_t S = first[r], E = last[r];
    if (E <= S + 2 * cr) continue;
    of_cloud lf_scan = {0, 0, 0};
    /* setScanBuffersFor */
    for (size_t i = 0; i <= E - S; i++) picked[i] = 0;
    for (size_t i = S + cr; i < E - cr; i++) {
      const of_pt* prev = &cloud.p[i - 1]; const of_pt* pt = &cloud.p[i]; const of_pt* next = &cloud.p[i + 1];
      float diffNext = sq_diff(next, pt);
      if (diffNext > 0.1) {
        float depth1 = pt_dist(pt), depth2 = pt_dist(next);
        if (depth1 > depth2) {
          float wd = sqrtf(sq_diff_w(next, pt, depth2 / depth1)) / depth2;
          if (wd < 0.1) {
            for (size_t k = 0; k < cr + 1; k++) picked[i - S - cr + k] = 1;
            continue;
          }
        } else {
          float wd = sqrtf(sq_diff_w(pt, next, depth1 / depth2)) / depth1;
          if (wd < 0.1) for (size_t k = 0; k < cr + 1; k++) picked[i - S + 1 + k] = 1;
        }
      }
      float diffPrevious = sq_diff(pt, prev);
      float dis = pt_sqdist(pt);
      if (diffNext > 0.0002 * dis && diffPrevious > 0.0002 * dis) picked[i - S] = 1;
    }
    for (int j = 0; j < R; j++) {
      size_t sp = ((S + cr) * (size_t)(R - j) + (E - cr) * (size_t)j) / (size_t)R;
      size_t ep = ((S + cr) * (size_t)(R - 1 - j) + (E - cr) * (size_t)(j + 1)) / (size_t)R - 1;
      if (ep <= sp) continue;
      size_t m = ep - sp + 1;
      /* setRegionBuffersFor */
      float w = -2 * (int)cr;
      for (size_t i = sp, ri = 0; i <= ep; i++, ri++) {
        float dX = w * cloud.p[i].x, dY = w * cloud.p[i].y, dZ = w * cloud.p[i].z;
        for (size_t k = 1; k <= cr; k++) {
          dX += cloud.p[i + k].x + cloud.p[i - k].x;
          dY += cloud.p[i + k].y + cloud.p[i - k].y;
          dZ += cloud.p[i + k].z + cloud.p[i - k].z;
        }
        curv[ri] = dX * dX + dY * dY + dZ * dZ;
        sortIdx[ri] = i;
        label[ri] = SURFACE_LESS_FLAT;
      }
      for (size_t i = 1; i < m; i++)
        for (size_t k = i; k >= 1; k--)
          if (curv[sortIdx[k] - sp] < curv[sortIdx[k - 1] - sp]) { size_t t = sortIdx[k]; sortIdx[k] = sortIdx[k - 1]; sortIdx[k - 1] = t; }
      /* corners */
      int largest = 0;
      for (size_t k = m; k > 0 && largest < P->max_corner_less_sharp;) {
        size_t idx = sortIdx[--k], si = idx - S, ri = idx - sp;
        if (picked[si] == 0 && curv[ri] > P->curvature_threshold) {
          largest++;
          if (largest <= P->max_corner_sharp) { label[ri] = CORNER_SHARP; push(&sharp, cloud.p[idx]); }
          else label[ri] = CORNER_LESS_SHARP;
          push(&less_sharp, cloud.p[idx]);
          /* markAsPicked */
          picked[si] = 1;
          for (size_t a = 1; a <= cr; a++) { if (sq_diff(&cloud.p[idx + a], &cloud.p[idx + a - 1]) > 0.05) break; picked[si + a] = 1; }
          for (size_t a = 1; a <= cr; a++) { if (sq_diff(&cloud.p[idx - a], &cloud.p[idx - a + 1]) > 0.05) break; picked[si - a] = 1; }
        }
      }
      /* flat */
      int smallest = 0;
      for (size_t k = 0; k < m && smallest < P->max_surface_flat; k++) {
        size_t idx = sortIdx[k], si = idx - S, ri = idx - sp;
        if (picked[si] == 0 && curv[ri] < P->curvature_threshold) {
          smallest++;
          label[ri] = SURFACE_FLAT;
          push(&flat, cloud.p[idx]);
          picked[si] = 1;
          for (size_t a = 1; a <= cr; a++) { if (sq_diff(&cloud.p[idx + a], &cloud.p[idx + a - 1]) > 0.05) break; picked[si + a] = 1; }
          for (size_t a = 1; a <= cr; a++) { if (sq_diff(&cloud.p[idx - a], &cloud.p[idx - a + 1]) > 0.05) break; picked[si - a] = 1; }
        }
      }
      for (size_t k = 0; k < m; k++)
        if (label[k] <= SURFACE_LESS_FLAT) push(&lf_scan, cloud.p[sp + k]);
    }
    voxel_grid(&lf_scan, P->less_flat_leaf, &less_flat);
    free(lf_scan.p);
  }
  counts[0] = cloud.n; counts[1] = sharp.n; counts[2] = less_sharp.n; counts[3] = flat.n; counts[4] = less_flat.n;
  counts[5] = sharp.n + less_sharp.n + flat.n + less_flat.n;
  int status = 0;
  if (counts[5] > out_cap) {
    status = -3;
  } else {
    float I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Ry[9], Rz[9], A[9], M[9];
    float theta = (float)(OF_PI / 2);
    angle_axis(theta, 1, Ry);
    angle_axis(theta, 2, Rz);
    matmul3(I, Ry, A);
    matmul3(A, Rz, M);
    const of_cloud* parts[4] = {&sharp, &less_sharp, &flat, &less_flat};
    size_t o = 0;
    for (int c = 0; c < 4; c++)
      for (size_t i = 0; i < parts[c]->n; i++, o++) {
        const of_pt* q = &parts[c]->p[i];
        /* PCL 1.10 Transformer::se3: m0*x + (m1*y + (m2*z + t)), t = 0 */
        for (int d = 0; d < 3; d++) out4[4 * o + d] = M[3 * d] * q->x + (M[3 * d + 1] * q->y + (M[3 * d + 2] * q->z + 0.0f));
        out4[4 * o + 3] = q->intensity;
      }
  }
  for (int r = 0; r < P->n_rings; r++) free(scans[r].p);
  free(scans); free(first); free(last); free(cloud.p); free(picked); free(curv); free(sortIdx); free(label);
  free(sharp.p); free(less_sharp.p); free(flat.p); free(less_flat.p);
  return status;
}
