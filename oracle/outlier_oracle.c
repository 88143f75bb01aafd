/* outlier_oracle.c -- TEST INFRASTRUCTURE ONLY (see lb_oracle.h): CPU restatement of the two PCL outlier filters LOCUS
 * can switch on (SURVEY 8f row f5):
 *   pcl::StatisticalOutlierRemoval<PointF>  point_cloud_filter/src/PointCloudFilter.cc:126-133 (filtering/outlier_filter,
 *                                           outlier_knn 10, outlier_std 1.0), run in the lidar callback (locus/src/Locus.cc:450)
 *   pcl::RadiusOutlierRemoval<PointF>       PointCloudFilter.cc:135-143 (filtering/radius_filter 0.15 m, 3) and the three
 *                                           callbacks of point_cloud_merger/src/PointCloudMerger.cc:112-117,139-144,169-174
 *                                           (merging/b_use_radius_filter, 0.1 m, 3) on the full-resolution merged cloud
 *
 * The arithmetic lives in PCL, which is NOT vendored in the reference (de-facto ROS Noetic version PCL 1.10.0).  This
 * file restates applyFilterIndices of filters/impl/statistical_outlier_removal.hpp and radius_outlier_removal.hpp:
 *
 *   StatisticalOutlierRemoval (mean_k, std_mul, negative):
 *     per point: nearestKSearch(mean_k + 1) (the point itself included, FLANN sorted results);
 *                dist_sum (double) += sqrt(nn_dists[k]) for k = 1..mean_k ("k = 0 is the query point");
 *                distances[i] = (float)(dist_sum / mean_k)
 *     then serially in input order: sum += distances[i]; sq_sum += distances[i] * distances[i]   (double sums, float product)
 *     mean = sum / n; variance = (sq_sum - sum * sum / n) / (n - 1); stddev = sqrt(variance);
 *     threshold = mean + std_mul * stddev
 *     removed iff distances[i] > threshold (negative: distances[i] <= threshold), the float compared in double.
 *     PCL writes an unqualified sqrt on a float; whether that is sqrtf or sqrt(double) depends on the headers in scope.
 *     Pinned here (and on the GPU): sqrtf.  n == 1 divides 0 by 0: the threshold is NaN, no comparison holds and every
 *     point is kept (the C ABI refuses n < mean_k + 1 before that, so only og_sor_threshold can show it).
 *   RadiusOutlierRemoval (radius, min_neighbors, negative), two branches on input->is_dense:
 *     dense:     k = nearestKSearch(min_neighbors + 1); inlier iff k == min_neighbors + 1 and
 *                !(radius * radius (double) < nn_dists[k - 1] (float))
 *     not dense: k = radiusSearch(radius) = every point with d2 < float(radius * radius) (FLANN's strict compare);
 *                inlier iff k > min_neighbors
 *     kept iff inlier (negative: iff not).  Both count the point itself.  radius == 0: PCL logs an error and outputs
 *     nothing; the wrapper here refuses radius <= 0.
 * Output of both: ascending indices of the kept points (PCL's output order).
 *
 * PARITY UNPINNED: the reference holds no outlier-filter test and PCL cannot be built here.  The neighbour order among
 * equidistant points (FLANN) is taken as ascending index, like the rest of this oracle.  Serial, no OpenMP: the
 * statistics are serial sums anyway, and the timed CPU baseline of tools/bench_outliers.py is this code.
 */
#include <math.h>
#include <stdlib.h>

#include "lb_oracle.h"

/* the statistics and the flag pass of StatisticalOutlierRemoval from the per-point distances; stats3 (nullable) =
 * {mean, stddev, threshold}; kept (capacity n) = ascending kept indices; returns their number */
int og_sor_threshold(const float* distances, int n, double std_mul, int negative, int* kept, double* stats3) {
  double sum = 0.0, sq_sum = 0.0;
  for (int i = 0; i < n; i++) {
    sum += distances[i];
    sq_sum += (double)(distances[i] * distances[i]);
  }
  double mean = sum / (double)n;
  double variance = (sq_sum - sum * sum / (double)n) / ((double)n - 1.0);
  double stddev = sqrt(variance);
  double threshold = mean + std_mul * stddev;
  if (stats3) { stats3[0] = mean; stats3[1] = stddev; stats3[2] = threshold; }
  int m = 0;
  for (int i = 0; i < n; i++) {
    double d = (double)distances[i];
    int removed = negative ? (d <= threshold) : (d > threshold);
    if (!removed) kept[m++] = i;
  }
  return m;
}

/* pts: n points, stride_f floats apart.  mean_dist (nullable, n floats), stats3 (nullable, 3 doubles).  Returns the
 * number of kept points, -1 when mean_k < 1 or n < mean_k + 1 (the C ABI refuses those), -2 on allocation failure. */
int og_statistical_outlier_removal(const float* pts, int n, int stride_f, int mean_k, double std_mul, int negative,
                                   int* kept, float* mean_dist, double* stats3) {
  if (mean_k < 1 || n < mean_k + 1) return -1;
  og_kdtree* tree = og_kdtree_build(pts, n, stride_f);
  float* dist = (float*)malloc(sizeof(float) * (size_t)n);
  int* idx = (int*)malloc(sizeof(int) * (size_t)(mean_k + 1));
  float* d2 = (float*)malloc(sizeof(float) * (size_t)(mean_k + 1));
  int m = -2;
  if (tree && dist && idx && d2) {
    for (int i = 0; i < n; i++) {
      og_kdtree_knn(tree, pts + (size_t)i * stride_f, mean_k + 1, idx, d2);
      double dist_sum = 0.0;
      for (int k = 1; k < mean_k + 1; k++) dist_sum += sqrtf(d2[k]);
      dist[i] = (float)(dist_sum / mean_k);
    }
    if (mean_dist) for (int i = 0; i < n; i++) mean_dist[i] = dist[i];
    m = og_sor_threshold(dist, n, std_mul, negative, kept, stats3);
  }
  if (tree) og_kdtree_free(tree);
  free(dist); free(idx); free(d2);
  return m;
}

/* dense selects PCL's is_dense branch (k-NN form) over the radius-search branch.  Returns the number of kept points,
 * -1 when radius <= 0 or min_neighbors < 0, -2 on allocation failure. */
int og_radius_outlier_removal(const float* pts, int n, int stride_f, double radius, int min_neighbors, int dense, int negative,
                              int* kept) {
  if (!(radius > 0.0) || min_neighbors < 0) return -1;
  og_kdtree* tree = og_kdtree_build(pts, n, stride_f);
  const int mk = min_neighbors < n ? min_neighbors + 1 : n + 1;    /* nearestKSearch returns at most n anyway */
  int* idx = (int*)malloc(sizeof(int) * (size_t)(n > mk ? n : mk));
  float* d2 = (float*)malloc(sizeof(float) * (size_t)(n > mk ? n : mk));
  int m = -2;
  if (tree && idx && d2) {
    const double nn_dists_max = radius * radius;
    const float r2f = (float)(radius * radius);
    m = 0;
    for (int i = 0; i < n; i++) {
      const float* p = pts + (size_t)i * stride_f;
      int inlier;
      if (dense) {
        int k = og_kdtree_knn(tree, p, mk, idx, d2);
        inlier = (k == min_neighbors + 1) && !(nn_dists_max < d2[k - 1]);
      } else {
        int k = og_kdtree_radius(tree, p, r2f, idx, d2, n);
        inlier = k > min_neighbors;
      }
      if (inlier != (negative != 0)) kept[m++] = i;
    }
  }
  if (tree) og_kdtree_free(tree);
  free(idx); free(d2);
  return m;
}
