/*
 * locus_b200.h -- C ABI of the H100 (sm_90a) GICP scan matcher and VoxelGrid
 * front-end that drops in behind LOCUS's registration and filter seams.
 *
 * Plain C, plain pointers and sizes; no C++/torch/PCL types cross this
 * boundary and no exception ever does: every function returns an lb_status
 * (0 = OK, < 0 = error; lb_last_error_string() gives the text).  On any error
 * the handle keeps its previous state (the last good pose stays valid), which
 * is how the reference behaves on solver failure (gicp.hpp:542-547).
 *
 * Reference interfaces each entry point replaces (paths relative to the
 * LOCUS repository):
 *
 *   lb_gicp_create/destroy        make_shared<MultithreadedGeneralizedIterativeClosestPoint>
 *                                 point_cloud_odometry/src/PointCloudOdometry.cc:142-146
 *                                 point_cloud_localization/src/PointCloudLocalization.cc:229-232
 *   lb_gicp_set_params            setTransformationEpsilon / setMaxCorrespondenceDistance /
 *                                 setMaximumIterations / setRANSACIterations /
 *                                 setMaximumOptimizerIterations / setNumThreads /
 *                                 enableTimingOutput / RecomputeTarget|SourceCovariance /
 *                                 setEuclideanFitnessEpsilon
 *                                 PointCloudOdometry.cc:147-155, PointCloudLocalization.cc:234-245,
 *                                 multithreaded_gicp/include/multithreaded_gicp/gicp.h:111-143,264-298
 *   lb_gicp_set_source            icp_->setInputSource()   PointCloudOdometry.cc:265,
 *                                 PointCloudLocalization.cc:306 (gicp.h:162-179)
 *   lb_gicp_set_target            icp_->setInputTarget()   PointCloudOdometry.cc:266,
 *                                 PointCloudLocalization.cc:307 (gicp.h:196-200)
 *   lb_gicp_align                 icp_->align() + getFinalTransformation() + hasConverged()
 *                                 PointCloudOdometry.cc:267-269, PointCloudLocalization.cc:309-313
 *                                 (computeTransformation, gicp.hpp:405-617)
 *   lb_gicp_transform_source      the `output` cloud of align() (gicp.hpp:586) and
 *                                 pcl::transformPointCloudWithNormals, PointCloudLocalization.cc:325
 *   lb_gicp_nn_target             icp_->getSearchMethodTarget()->nearestKSearch(pt, 1, ..)
 *                                 PointCloudLocalization.cc:327-336
 *   lb_gicp_fitness               icp_->getFitnessScore()
 *                                 point_cloud_odometry/test/test_point_cloud_odometry.cpp:298
 *   lb_gicp_point2plane_information   normalizePCloud + ComputeAp_ForPoint2PlaneICP
 *                                 point_cloud_localization/src/utils.cc:106-128, PointCloudLocalization.cc:694-750
 *   lb_gicp_compute_normals       NormalComputation::filter, k-NN mode (pcl::NormalEstimationOMP)
 *                                 point_cloud_filter/src/normal_computation.cc:26-59
 *   lb_gicp_compute_normals_radius   the same nodelet in its radius mode + removeNaNNormalsFromPointCloud
 *                                 normal_computation.cc:53-57,73-77
 *   lb_gicp_statistical_outlier_removal   pcl::StatisticalOutlierRemoval<PointF>  point_cloud_filter/src/
 *                                 PointCloudFilter.cc:126-133 (filtering/outlier_filter, run from locus/src/Locus.cc:450)
 *   lb_gicp_radius_outlier_removal   pcl::RadiusOutlierRemoval<PointF>  PointCloudFilter.cc:135-143 and
 *                                 point_cloud_merger/src/PointCloudMerger.cc:112-117,139-144,169-174
 *   lb_voxel_create/destroy       pcl::VoxelGrid<pcl::PCLPointCloud2> impl_
 *                                 point_cloud_filter/include/point_cloud_filter/custom_voxel_grid.h:25
 *   lb_voxel_set_leaf_size        impl_.setLeafSize()      custom_voxel_grid.cc:62-73, 97-101
 *   lb_voxel_set_filter_limits    impl_.setFilterFieldName/Limits/LimitsNegative  custom_voxel_grid.cc:103-134
 *   lb_voxel_filter               impl_.setInputCloud + setIndices + filter()     custom_voxel_grid.cc:76-87
 *   lb_voxel_extract_features     the `filtering/extract_features` branch of PointCloudFilter::Filter
 *                                 point_cloud_filter/src/PointCloudFilter.cc:144-173 (run from locus/src/Locus.cc:450)
 *   lb_ndt_*                      pclomp::NormalDistributionsTransform behind `registration_method: ndt`
 *                                 PointCloudOdometry.cc:182-195, PointCloudLocalization.cc:267-280 (section NDT below)
 *   lb_odometry_submit/next       the per-scan chain of the lidar callback: filtered scan -> odometry_.SetLidar()
 *                                 -> odometry_.UpdateEstimate()   locus/src/Locus.cc:451-453,
 *                                 PointCloudOdometry.cc:221-230 (SetLidar), 237-247 (UpdateEstimate: first scan
 *                                 only stored; afterwards reference_ = previous query_), 249-274 (UpdateICP)
 *
 * Threading: a handle is used from one thread at a time (the reference calls
 * the seam from the dedicated lidar spinner thread, locus/src/Locus.cc:63-69,
 * and CustomVoxelGrid::filter holds mutex_, custom_voxel_grid.cc:79).  One
 * handle owns one CUDA stream; independent scan streams use independent
 * handles (one per GPU in the multi-GPU mode).
 *
 * Ownership: input buffers are borrowed for the duration of the call only;
 * the library owns all device memory.  `mem` says where a buffer lives.
 */
#ifndef LOCUS_B200_H_
#define LOCUS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB_VERSION 100

typedef enum lb_status {
  LB_OK = 0,
  LB_ERR_INVALID_ARG = -1,
  LB_ERR_CUDA = -2,
  LB_ERR_NO_DEVICE = -3,
  LB_ERR_EMPTY_SOURCE = -4,       /* gicp.h:164-171: empty source cloud -> error, state untouched */
  LB_ERR_NO_TARGET = -5,
  LB_ERR_TOO_FEW_POINTS = -6,     /* gicp.hpp:72-79: k_correspondences > cloud size */
  LB_ERR_VOXEL_OVERFLOW = -7,     /* leaf size too small: int32 voxel index would overflow */
  LB_ERR_CAPACITY = -8,           /* output buffer too small */
  LB_ERR_UNSUPPORTED = -9,
  LB_ERR_NO_ALIGN = -10           /* result requested before any successful align() */
} lb_status;

typedef enum lb_mem { LB_MEM_HOST = 0, LB_MEM_DEVICE = 1 } lb_mem;
typedef enum lb_optimizer { LB_OPT_BFGS = 0, LB_OPT_GAUSS_NEWTON = 1 } lb_optimizer;
/* STREAM_ORDERED (default): one outer iteration = three launches on the handle's stream -- the correspondence search as
 * full-occupancy grids (candidates staged through shared memory with TMA bulk copies, the undecided queries of the
 * whole cloud queued and finished by a second grid), then the inner solve as a cooperative grid (leader warp + worker
 * warps per CTA, grid-wide all-reduce through L2) -- with the loop state resident in device memory and a few
 * iterations enqueued ahead of the host (kernels after convergence return at once).
 * PERSISTENT: the whole of align() as ONE cooperative kernel (the default of round 1; 10 % slower per align and 16 %
 * slower in the pipeline).  HOST_DRIVEN sequences one launch per objective evaluation from the host.
 * PERSISTENT_CLUSTER runs the inner solve inside one 16-CTA thread-block cluster (all-reduce pushed through
 * distributed shared memory; sources <= 45056 points, falls back to PERSISTENT otherwise).
 * All four run the same device functions with the same reduction shape: identical bits. */
typedef enum lb_execution { LB_EXEC_PERSISTENT = 0, LB_EXEC_HOST_DRIVEN = 1, LB_EXEC_PERSISTENT_CLUSTER = 2,
                            LB_EXEC_STREAM_ORDERED = 3 } lb_execution;

#define LB_NO_NORMALS ((ptrdiff_t)-1)

int lb_version(void);
const char* lb_last_error_string(void);
const char* lb_status_string(int status);
int lb_device_count(int* n);

/* ------------------------------------------------------------------ GICP */
typedef struct lb_gicp lb_gicp;

typedef struct lb_gicp_params {
  /* values and defaults: gicp.h:111-127 (SURVEY.md Appendix E) */
  int k_correspondences;                /* 20   setCorrespondenceRandomness */
  double gicp_epsilon;                  /* 1e-3 */
  double rotation_epsilon;              /* 2e-3 setRotationEpsilon */
  double transformation_epsilon;        /* 5e-4 setTransformationEpsilon */
  double max_correspondence_distance;   /* 5.0  setMaxCorrespondenceDistance */
  int max_iterations;                   /* 200  setMaximumIterations */
  int max_optimizer_iterations;         /* 20   setMaximumOptimizerIterations */
  /* 1: k-NN + SVD covariances (gicp.hpp:85-154).  0: from normals
   * (gicp.hpp:81-82) -- needs normals in the cloud, else falls back to k-NN. */
  int recompute_source_covariance;      /* reference default 0; here 1 (normals are optional) */
  int recompute_target_covariance;
  int optimizer;                        /* lb_optimizer; LB_OPT_BFGS = reference-exact */
  int execution;                        /* lb_execution; LB_EXEC_STREAM_ORDERED by default */
  /* accepted for interface compatibility, no effect on the GPU path */
  double euclidean_fitness_epsilon;     /* setEuclideanFitnessEpsilon (unused by gicp.hpp too) */
  int ransac_iterations;                /* setRANSACIterations(0) */
  int num_threads;                      /* setNumThreads */
  int enable_timing_output;             /* enableTimingOutput: spans are always in lb_gicp_result */
  float index_cell_size;                /* voxel-hash cell size in metres; 0 = automatic (a pure function of the cloud) */
  int align_points_per_cta;             /* source points per CTA of the align solve kernel (any execution); 0 = 512 (lowest latency
                                           of one align: ~60 SMs for a 30k-point scan).  Larger values (1024, 2048) use
                                           fewer SMs per align for longer: more aligns fit on the GPU at once, which is
                                           what lb_odometry's workers want.  Changes the shape of the reduction, i.e. the
                                           last bits of the pose, not the algorithm. */
} lb_gicp_params;

typedef struct lb_gicp_result {
  float final_transformation[16];  /* row-major 4x4 = previous_transformation_ * guess (gicp.hpp:583) */
  int converged;                   /* hasConverged(): delta < 1 OR iteration cap (gicp.hpp:566-568) */
  int iterations;                  /* nr_iterations_ */
  int n_correspondences;           /* of the last outer iteration */
  double delta;                    /* last convergence ratio (gicp.hpp:526-541) */
  int n_objective_evals;           /* fused f+gradient passes */
  int n_inner_iterations;
  /* CUDA-event spans, same three spans the reference times (gicp.hpp:588-616) */
  float t_covariances_ms;
  float t_iterations_ms;
  float t_total_ms;
  int status;
  /* previous_transformation_ / transformation_ of pcl::Registration after align(): the guess-free increment the loop
   * converged to (final_transformation = transformation * guess, gicp.hpp:583); getLastIncrementalTransformation() */
  float transformation[16];
} lb_gicp_result;

int lb_gicp_default_params(lb_gicp_params* p);
int lb_gicp_create(int device, lb_gicp** h);
/* same, but work is enqueued on the caller's cudaStream_t (so the caller can
 * bracket it with its own CUDA events) */
int lb_gicp_create_on_stream(int device, void* cuda_stream, lb_gicp** h);
int lb_gicp_destroy(lb_gicp* h);
int lb_gicp_set_params(lb_gicp* h, const lb_gicp_params* p);
int lb_gicp_get_params(lb_gicp* h, lb_gicp_params* p);

/* pts: n points, `stride` bytes apart; float32 x,y,z at byte offset xyz_off;
 * float32 normal_x,y,z at normal_off (LB_NO_NORMALS if absent).
 * Builds the voxel-hash index of the cloud and (lazily, in align) its
 * covariances.  Invalidates previous covariances like gicp.h:177-178,196-200. */
int lb_gicp_set_source(lb_gicp* h, const void* pts, size_t n, size_t stride, size_t xyz_off,
                       ptrdiff_t normal_off, int mem);
int lb_gicp_set_target(lb_gicp* h, const void* pts, size_t n, size_t stride, size_t xyz_off,
                       ptrdiff_t normal_off, int mem, uint64_t* generation /* nullable */);
/* Optional: pre-size the handle for clouds of up to max_points points (its current clouds, its scratch, and
 * `spare_clouds` spare cloud objects, which set_source / set_target rotate through), so that a stream in steady state
 * performs no device allocation -- an allocation synchronises the whole device and stalls every other handle working on
 * it.  lb_odometry does this for its workers. */
int lb_gicp_reserve(lb_gicp* h, size_t max_points, int spare_clouds);
/* scan-to-scan odometry (PointCloudOdometry.cc:243-244 copies the last scan into
 * reference_): re-use the current source's index and covariances as the next
 * target instead of rebuilding them. */
int lb_gicp_promote_source_to_target(lb_gicp* h);

/* Prepared clouds shared between handles.  In scan-to-scan odometry every filtered scan is the source of one
 * registration and the target of the next (PointCloudOdometry.cc:243-244: copyPointCloud(*query_, *reference_)).  The
 * reference recomputes the target's kd-tree and covariances anyway (setInputTarget clears them, gicp.h:196-200);
 * these entry points let a caller that runs registrations on several handles (lb_odometry's workers) compute each
 * scan's index + covariances once: the handle that has the scan as its SOURCE prepares it and shares it, the handle
 * that needs it as TARGET adopts it.  Same bits as rebuilding it (the index is a pure function of the cloud).
 *   lb_gicp_prepare_source   enqueue index + covariances of the current source now (align would do it lazily)
 *   lb_gicp_share_source     a new reference to the prepared source (release it with lb_cloud_release)
 *   lb_gicp_set_target_cloud adopt a shared cloud as target (no copy; this handle's stream waits for its preparation)
 *   lb_gicp_set_source_cloud adopt a shared cloud as source, likewise (lb_locus: scan k's cloud is odometry source k,
 *                            odometry target k+1 and localization source k)
 * A shared cloud is immutable: a handle that still holds it and gets new data switches to another object.  The
 * handles must sit on the same device and use the same covariance parameters. */
typedef struct lb_cloud lb_cloud;
int lb_gicp_prepare_source(lb_gicp* h);
int lb_gicp_share_source(lb_gicp* h, lb_cloud** out);
int lb_gicp_set_target_cloud(lb_gicp* h, lb_cloud* cloud);
int lb_gicp_set_source_cloud(lb_gicp* h, lb_cloud* cloud);
int lb_cloud_release(lb_cloud* cloud);

/* guess: row-major 4x4 float, NULL = identity (the callers pass none). */
int lb_gicp_align(lb_gicp* h, const float* guess, lb_gicp_result* out);

/* out_pts[i] = T * source[i] (and rotated normals if normal_off >= 0), in the
 * source's original order and layout.  T NULL = final transformation. */
int lb_gicp_transform_source(lb_gicp* h, const float* T, void* out_pts, size_t stride, size_t xyz_off,
                             ptrdiff_t normal_off, int mem);
/* exact 1-NN of n query points in the current target: original target index
 * and float32 squared distance. */
int lb_gicp_nn_target(lb_gicp* h, const void* xyz, size_t n, size_t stride, int32_t* idx, float* d2, int mem);
/* pcl::Registration::getFitnessScore(max_range) for transform T (NULL = final). */
int lb_gicp_fitness(lb_gicp* h, const float* T, double max_range, double* score);
/* SURVEY 8f row f1 -- the step right after align() in PointCloudLocalization::MeasurementUpdate:
 * normalizePCloud (point_cloud_localization/src/utils.cc:106-128) followed by ComputeAp_ForPoint2PlaneICP
 * (PointCloudLocalization.cc:694-750): Ap = sum_i H_i' H_i, H_i = [a_i x n_i, n_i], a_i = (normalised) query point,
 * n_i = normal of reference point correspondences[i] (rotated by T's rotation when T != NULL), NaN rows skipped.
 * query: n points (xyz at q_xyz_off); reference: n_ref points (normal at r_normal_off); correspondences: n int32
 * indices into reference.  Ap36: 36 doubles row-major (host).  All buffers host or all device (`mem`). */
int lb_gicp_point2plane_information(lb_gicp* h, const void* query, size_t n, size_t q_stride, size_t q_xyz_off,
                                    const void* reference, size_t n_ref, size_t r_stride, size_t r_normal_off,
                                    const int32_t* correspondences, const float* T, int normalize, double* Ap36, int mem);
/* SURVEY 8f row f1, completed -- the ICP covariance LOCUS's shipped localization computes after every align
 * (point_cloud_localization/config/parameters.yaml: compute_icp_covariance true, icp_covariance_method 1,
 * icp_max_covariance 0.01): PointCloudLocalization.cc:325-336 (1-NN of every aligned point) and :398-421, :469-541
 * (ComputePoint2PlaneICPCovariance).  For the handle's source q (caller order) and its target:
 *   1. aligned = T q (T NULL = the final transformation), float, as lb_gicp_transform_source;
 *   2. corr[i] = exact 1-NN of aligned[i] in the target, no distance gate, ties -> lowest index (nearestKSearch(pt, 1));
 *      or the caller's `correspondences` (n_source int32 target indices, host or device: `mem`) -- then T is not used;
 *   3. a_i = normalizePCloud(q)[i] (float sums in point order); n_i = the target's normal of corr[i] (the submap's
 *      stored normal when the target is a submap), rotated by `normal_rotation` (3x3 row-major float, NULL = none) in
 *      float as transformPointCloudWithNormals rotates normals;
 *   4. Ap = sum H^T H, H = [a_i x n_i, n_i], rows where a_i or n_i has a NaN skipped (:723-750).  A target point without
 *      a normal is such a row; a target without normals gives Ap = 0;
 *   5-9. cov = 0.05^2 Ap^-1, Eigen's LDLT clamp to [1e-12, max_covariance] with the reference's pivot-permuted rebuild,
 *      the NaN fallbacks and the condition number s0 / s5: locus_b200/csrc/icp_cov.h, which states the Eigen readings.
 * One stream sequence on the handle's stream (existing transform / 1-NN / normalize / Ap kernels) with one host
 * synchronisation.  The first search of a target cloud adds one more: the density probe that picks the 1-NN kernel, as in
 * lb_gicp_nn_target.  A submap target is a new cloud after every change of the map, so in lb_locus the first scan after
 * a keyframe insert or crop pays two synchronisations here, every other scan one.
 * Errors: no source LB_ERR_EMPTY_SOURCE; no target LB_ERR_NO_TARGET; T and correspondences both NULL before any align
 * LB_ERR_NO_ALIGN; a correspondence out of range, or max_covariance not finite or <= 0, LB_ERR_INVALID_ARG.  The
 * handle's clouds, index, covariances and last align result are never changed.  A submap target must be unchanged
 * since lb_gicp_set_target_submap (LB_ERR_INVALID_ARG otherwise). */
#define LB_ICPCOV_CLAMPED 1   /* step 7 clamped a pivot and rebuilt cov */
#define LB_ICPCOV_D_NAN 2     /* step 6: the LDLT pivots had a NaN -> cov = max I, no condition number */
#define LB_ICPCOV_COV_NAN 4   /* step 8: cov had a NaN -> max on the diagonal */
typedef struct lb_icp_covariance {
  double Ap[36];            /* row-major */
  double covariance[36];    /* row-major: icp_covariance_ */
  double condition_number;  /* NaN when step 6 returned early */
  int flags;                /* LB_ICPCOV_* */
  size_t n_query, n_used;   /* query points; rows that entered Ap */
} lb_icp_covariance;
int lb_gicp_icp_covariance(lb_gicp* h, const float* T, const int32_t* correspondences, int mem, const float* normal_rotation,
                           double max_covariance, lb_icp_covariance* out);
/* SURVEY 8f row f2 -- the step right before the path: point_cloud_filter::NormalComputation::filter in its k-NN
 * mode (point_cloud_filter/src/normal_computation.cc:26-59; norm_est_ = pcl::NormalEstimationOMP<PointXYZI, Normal>,
 * normal_computation.h:38; k = normal_search_knn, cfg/NormalComputation.cfg:15).  Per point of the cloud currently set
 * as source (which = 0) or target (which = 1): the k nearest neighbours (itself included) -> PCL's float32
 * mean/covariance -> eigenvector of the smallest eigenvalue (PCL eigen33) -> flipped towards `viewpoint` (NULL = the
 * origin, what fromROSMsg leaves in sensor_origin_).  out4: n x (normal_x, normal_y, normal_z, curvature) float32 in
 * the caller's point order, host or device.  3 <= k <= 20.  (Radius mode: lb_gicp_compute_normals_radius.) */
int lb_gicp_compute_normals(lb_gicp* h, int which, int k, const float* viewpoint, float* out4, int mem);
/* The same normals, written into the cloud itself instead of a caller buffer: the NormalComputation nodelet in front of
 * the registration (locus/launch/locus.launch:177-181).  Afterwards the source (which = 0) or target (1) has normals,
 * exactly as if it had been uploaded with those normals at normal_off, and its covariances are invalidated: with
 * recompute_source/target_covariance = 0 the next prepare_source / align takes them from the normals (gicp.hpp:81-82).
 * A prepared source shared from here carries the normals, and lb_gicp_transform_source returns them rotated.  Errors as
 * lb_gicp_compute_normals (3 <= k <= 20, at least k points), and the cloud is left as it was.  A cloud shared with
 * another handle is refused (LB_ERR_INVALID_ARG): it is immutable. */
int lb_gicp_estimate_normals(lb_gicp* h, int which, int k, const float* viewpoint);
/* The nodelet's radius mode (normal_computation.cc:73-77, norm_est_.setRadiusSearch(normal_search_radius)) together
 * with the NaN-normal removal that follows it (:53-57, pcl::removeNaNNormalsFromPointCloud).  Neighbourhood of a point =
 * every point with squared distance < float(radius^2) (FLANN's strict compare), itself included, taken in ascending
 * distance order; fewer than three neighbours -> NaN normal and curvature (pcl::computePointNormal).  out4: n x 4 as
 * above (NaN rows included); valid_idx (nullable, capacity n): ascending indices of the points whose normal is finite,
 * i.e. the points of the nodelet's output cloud; n_valid (nullable): their number.  LB_ERR_CAPACITY when a neighbourhood
 * exceeds 2048 points. */
int lb_gicp_compute_normals_radius(lb_gicp* h, int which, double radius, const float* viewpoint, float* out4,
                                   int32_t* valid_idx, size_t* n_valid, int mem);
/* SURVEY 8f row f5 -- the outlier filters of point_cloud_filter (PointCloudFilter.cc:126-143) and point_cloud_merger
 * (PointCloudMerger.cc:112-117,139-144,169-174), i.e. pcl::StatisticalOutlierRemoval / pcl::RadiusOutlierRemoval
 * (applyFilterIndices of filters/impl/statistical_outlier_removal.hpp and radius_outlier_removal.hpp, PCL 1.10), on the cloud currently set as source (which = 0)
 * or target (which = 1).  Those clouds are dense (lb_gicp_set_source refuses non-finite points).  Output: kept_idx
 * (capacity n) = ascending indices of the points the filter keeps, PCL's output order; *n_kept = their number.  All
 * buffers host or all device (`mem`).  The handle's clouds, index and covariances stay as they were.
 *
 * Statistical: per point the mean_k + 1 nearest neighbours (itself included, ascending (d2, index));
 *   distance = (float)(sum of sqrtf(d2) over neighbours 1..mean_k, in double, / mean_k).  sqrtf is the pinned reading of
 *   PCL's unqualified sqrt on a float.  Then, serially in input order, sum += distance and sq_sum += distance * distance
 *   (a float product) in double; mean = sum / n, variance = (sq_sum - sum * sum / n) / (n - 1), stddev = sqrt(variance),
 *   threshold = mean + std_mul * stddev.  Removed iff distance > threshold (negative: distance <= threshold).  A NaN
 *   threshold removes nothing (PCL's n == 1 case, which mean_k >= 1 already refuses).  mean_dist (nullable): n floats,
 *   the per-point distance; stats3 (nullable): {mean, stddev, threshold}.  1 <= mean_k <= 19 (LB_ERR_UNSUPPORTED above);
 *   n < mean_k + 1 -> LB_ERR_TOO_FEW_POINTS.
 * Radius: `dense` selects PCL's branch on input->is_dense.  dense = 1: nearestKSearch(min_neighbors + 1), inlier iff that
 *   many points came back and !(r^2 (double) < d2 of the last) -- i.e. at least min_neighbors + 1 points with
 *   (double)d2 <= r^2.  dense = 0: radiusSearch, inlier iff more than min_neighbors points have d2 < float(r^2)
 *   (FLANN's strict compare).  Both count the point itself.  negative keeps the outliers instead.  radius <= 0 ->
 *   LB_ERR_INVALID_ARG (PCL logs an error and outputs nothing for radius 0).  min_neighbors = 0 keeps every point
 *   (with dense = 0, as long as float(r^2) > 0). */
int lb_gicp_statistical_outlier_removal(lb_gicp* h, int which, int mean_k, double std_mul, int negative,
                                        int32_t* kept_idx, size_t* n_kept, float* mean_dist, double* stats3, int mem);
int lb_gicp_radius_outlier_removal(lb_gicp* h, int which, double radius, int min_neighbors, int dense, int negative,
                                   int32_t* kept_idx, size_t* n_kept, int mem);
/* covariances used by the last align, n x 9 doubles row-major, original point order. which: 0 source, 1 target */
int lb_gicp_get_covariances(lb_gicp* h, int which, double* out9, size_t capacity_points);
/* number of points currently indexed. which: 0 source, 1 target */
int lb_gicp_cloud_size(lb_gicp* h, int which, size_t* n);
/* kernels launched by this handle since creation (bench.py reports it) */
int lb_gicp_launch_count(lb_gicp* h, uint64_t* n);
/* CUDA-event duration (ms, averaged per launch) of a named kernel class since the last reset:
 * "nn_corr", "objective", "knn_cov", "align_persistent" (the iteration part of align() in any execution mode),
 * "loop_nn" (search grids), "loop_solve", "index_build", "nn_query". */
int lb_gicp_kernel_time(lb_gicp* h, const char* name, float* ms_avg, uint64_t* launches);
/* enable_timing: 0 off; 1 event timers of every kernel class plus the align kernel's cycle counters;
 * 2 only the event pair around the align kernel (cheap enough for a throughput run) */
int lb_gicp_reset_kernel_times(lb_gicp* h, int enable_timing);

/* ------------------------------------------------------------- VoxelGrid */
typedef struct lb_voxel lb_voxel;

/* sensor_msgs/PointField datatypes */
enum { LB_INT8 = 1, LB_UINT8 = 2, LB_INT16 = 3, LB_UINT16 = 4, LB_INT32 = 5, LB_UINT32 = 6,
       LB_FLOAT32 = 7, LB_FLOAT64 = 8 };

typedef struct lb_field {
  char name[32];
  uint32_t offset;
  uint8_t datatype;
  uint32_t count;
} lb_field;

int lb_voxel_create(int device, lb_voxel** h);
int lb_voxel_create_on_stream(int device, void* cuda_stream, lb_voxel** h);
int lb_voxel_destroy(lb_voxel* h);
int lb_voxel_set_leaf_size(lb_voxel* h, float lx, float ly, float lz);
int lb_voxel_get_leaf_size(lb_voxel* h, float* leaf3);
/* field_name NULL or "" = no filter field.  Defaults: none, [-FLT_MAX, FLT_MAX], not negative. */
int lb_voxel_set_filter_limits(lb_voxel* h, const char* field_name, double limit_min, double limit_max, int negative);
/* SURVEY 8f row f4 -- the BodyFilter nodelet that runs right before the voxel grid
 * (point_cloud_filter/src/body_filter.cc:28-56: pcl::CropBox<PointXYZI>, setMin/setMax from cfg/BodyFilter.cfg,
 * setRotation((0, 0, rotation)), setNegative(true)) folded into the filter's load predicate: points inside the box
 * (rotated by rotation_z about z) are removed before voxelisation.  enabled = 0 restores the plain VoxelGrid. */
int lb_voxel_set_body_filter(lb_voxel* h, int enabled, const float* min3, const float* max3, float rotation_z);
int lb_voxel_set_min_points_per_voxel(lb_voxel* h, int min_points);
int lb_voxel_set_downsample_all_data(lb_voxel* h, int all);

/* data: n_pts points of point_step bytes described by `fields` (must contain
 * FLOAT32 x, y, z).  indices: accepted for signature compatibility with
 * pcl_ros::Filter::filter(); pcl::VoxelGrid<PCLPointCloud2> ignores them and
 * so does this call.  out: capacity out_capacity_pts points of point_step
 * bytes; *n_out = number of voxels written (ascending voxel index).
 * out_voxel_idx (nullable, host or device like out): int32 PCL leaf index of
 * each output point. */
int lb_voxel_filter(lb_voxel* h, const uint8_t* data, size_t n_pts, uint32_t point_step,
                    const lb_field* fields, int n_fields, const int32_t* indices, size_t n_indices,
                    uint8_t* out, size_t out_capacity_pts, size_t* n_out, int32_t* out_voxel_idx,
                    int mem_in, int mem_out);
/* SURVEY 8f row f4, the rest of the front end folded into the filter's loads.
 * lb_voxel_set_input_passthrough: what each lidar's pcl/PassThrough nodelet does before everything else
 *   (locus/launch/locus.launch:90-133: filter_field_name z, limits [-100, 100], output_frame base_link): points that
 *   are not finite or whose field lies outside [min, max] (inside, when negative) are dropped -- tested on the RAW
 *   value, in the sensor frame, before the input's transform is applied.  field_name NULL or "" = off (default).
 * lb_voxel_filter_merged: 1..3 input clouds treated as one, in the order a, b, c -- the concatenation
 *   point_cloud_merger performs (point_cloud_merger/src/PointCloudMerger.cc:150-178: a + (b + c)); `transform`
 *   (row-major 4x4 float, NULL = identity) is the sensor -> base_link transform the PassThrough nodelet applies to its
 *   output (pcl_ros::transformPointCloud: Eigen Matrix4f * Vector4f per point).  Then, on the transformed
 *   coordinates: the BodyFilter box, the VoxelGrid limits and the grid itself, exactly as lb_voxel_filter.  Needs the
 *   x, y, z, intensity layout (four averaged FLOAT32 fields) when more than one input or a transform is given.
 *   The merger's optional filters (off in the shipped config) are not part of this call: its radius-outlier filter is
 *   lb_gicp_radius_outlier_removal on the merged cloud; its random sampler (seeded with time(nullptr)) has no GPU form. */
typedef struct lb_voxel_input {
  const uint8_t* data;        /* n_pts points of point_step bytes (host or device: mem_in) */
  size_t n_pts;
  const float* transform;     /* 16 floats, row-major; NULL = identity */
} lb_voxel_input;
int lb_voxel_set_input_passthrough(lb_voxel* h, const char* field_name, double limit_min, double limit_max, int negative);
int lb_voxel_filter_merged(lb_voxel* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step,
                           const lb_field* fields, int n_fields, uint8_t* out, size_t out_capacity_pts, size_t* n_out,
                           int32_t* out_voxel_idx, int mem_in, int mem_out);
/* SURVEY 8f row f6 -- LOAM-style feature extraction of the point-cloud filter (PointCloudFilter.cc:144-173,
 * arrangePCLInScanLines + extractFeatures :179-515): scan-ring arrangement, curvature, per-region sharp / less-sharp /
 * flat picks, a VoxelGrid of each ring's less-flat points, then the fixed rotation of Filter().  Semantics:
 * locus_b200/csrc/features.h.  Defaults (lb_features_default_params) are the reference's hard-coded values
 * (PointCloudFilter.h:79-96): 16 rings over [-15, 15] deg, scan period 0.1, curvature region 5, 6 regions, at most 2
 * sharp / 20 less-sharp / 4 flat points per region, curvature threshold 0.1, less-flat leaf 0.2. */
typedef struct lb_features_params {
  int n_rings;                    /* 1..128 */
  float lower_deg, upper_deg;     /* finite, lower < upper */
  float scan_period;
  int curvature_region;           /* 1..32 */
  int n_feature_regions;          /* 1..1024 */
  int max_corner_sharp, max_corner_less_sharp, max_surface_flat;   /* >= 0 */
  float curvature_threshold;
  float less_flat_leaf;           /* > 0 */
} lb_features_params;
/* n_less_sharp includes the sharp points, which the output holds twice, as the reference's does */
typedef struct lb_features_result {
  size_t n_arranged, n_sharp, n_less_sharp, n_flat, n_less_flat, n_out;
} lb_features_result;
int lb_features_default_params(lb_features_params* p);
/* pts: n points of `stride` bytes with FLOAT32 x, y, z at xyz_off (host or device: mem_in).  out4: n_out points of
 * four floats x, y, z, intensity (host or device: mem_out; a device buffer 16-byte aligned), in the order sharp,
 * less-sharp, flat, less-flat.  n == 0 -> LB_ERR_EMPTY_SOURCE (the reference reads point 0 unconditionally); invalid
 * params -> LB_ERR_INVALID_ARG; out_capacity < n_out -> LB_ERR_CAPACITY with r->n_out the size needed and nothing
 * written.  The handle's VoxelGrid settings are neither read nor changed. */
int lb_voxel_extract_features(lb_voxel* h, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem_in,
                              const lb_features_params* p, float* out4, size_t out_capacity, lb_features_result* r,
                              int mem_out);
int lb_voxel_launch_count(lb_voxel* h, uint64_t* n);
int lb_voxel_kernel_time(lb_voxel* h, float* ms_total_last_call);
/* CUDA-event duration per call (first launch .. result available), averaged over the calls since the last reset */
int lb_voxel_kernel_time_avg(lb_voxel* h, float* ms_avg, uint64_t* calls, int reset);

/* ------------------------------------------------- resident rolling submap (SURVEY 8f row f3)
 * The local map LOCUS keeps in its external point_cloud_mapper object, resident in HBM, in the fixed frame:
 *   lb_submap_insert      mapper_->InsertPoints(cloud, incremental)   locus/src/Locus.cc:464-465,531-532: a point enters
 *                         the map iff no map point occupies its voxel (edge = `resolution`) yet; points are taken in
 *                         input order, so within one call the first point of a voxel wins
 *   lb_submap_neighbors   mapper_->ApproxNearestNeighbors(scan, neighbors)   Locus.cc:479-483: for every query point
 *                         the nearest map point (EXACT here; ties -> lowest map index)
 *   lb_submap_crop_box    mapper_->Refresh(current_pose)   Locus.cc:536-537, lo_settings.yaml:58 box_filter_size: keeps
 *                         the points with |p - centre| <= half_size on every axis (pcl::CropBox bounds are inclusive)
 *   lb_gicp_set_target_submap   the map itself as the registration target (BASELINE configs[2]): its voxel-hash index
 *                         is rebuilt only after the map changed, and the k-NN covariance of a map point is computed
 *                         once -- by the first registration after its insertion, from the map as it is then -- and
 *                         cached until the point leaves the window.  (The reference recomputes every target
 *                         covariance for every scan: setInputTarget clears them, gicp.h:196-200.)
 * The mapper package is not vendored in the reference tree; its octree anchoring and the "approximate" of its
 * nearest-neighbour search are therefore unpinned: voxels are world-anchored here (floor(p / resolution)).
 * oracle/submap_oracle.py restates these semantics for the tests.  Map indices are insertion-order positions; they
 * shift when a crop removes points.  One handle is used from one thread at a time. */
typedef struct lb_submap lb_submap;
int lb_submap_create(int device, float resolution, lb_submap** out);
int lb_submap_destroy(lb_submap* m);
int lb_submap_clear(lb_submap* m);
/* pts: n points (float32 x,y,z at xyz_off, `stride` bytes apart), fixed frame.  n_inserted (nullable): points added.
 * inserted_xyz (nullable): the added points, n_inserted x 3 float32, input order (capacity n; host or device like pts):
 * the `incremental_points` output of InsertPoints.  Non-finite points are skipped. */
int lb_submap_insert(lb_submap* m, const void* pts, size_t n, size_t stride, size_t xyz_off, int mem, size_t* n_inserted,
                     float* inserted_xyz);
/* lb_submap_insert for points with normals (float32 x,y,z at normal_off, fixed frame): the winning point of a voxel
 * keeps its normal, and crops keep points and normals paired (Locus.cc:530-532 inserts the keyframe with its normals).
 * Points inserted by lb_submap_insert have none. */
int lb_submap_insert_with_normals(lb_submap* m, const void* pts, size_t n, size_t stride, size_t xyz_off, size_t normal_off,
                                  int mem, size_t* n_inserted, float* inserted_xyz);
int lb_submap_crop_box(lb_submap* m, const float* center3, float half_size, size_t* n_removed /* nullable */);
int lb_submap_size(lb_submap* m, size_t* n);
/* changes whenever the point set changed (insert that added points, crop that removed points, clear) */
int lb_submap_generation(lb_submap* m, uint64_t* generation);
/* the map's points, insertion order, n x 3 float32 */
int lb_submap_points(lb_submap* m, float* xyz_out, size_t capacity_points, int mem);
/* the map's normals, insertion order, n x 3 float32; NaN for points inserted without a normal */
int lb_submap_normals(lb_submap* m, float* xyz_out, size_t capacity_points, int mem);
/* neighbors_xyz (nullable): n x 3 float32, the nearest map point of every query; idx / d2 (nullable): its map index and
 * float32 squared distance.  All buffers host or all device (`mem`). */
int lb_submap_neighbors(lb_submap* m, const void* query, size_t n, size_t stride, size_t xyz_off, float* neighbors_xyz,
                        int32_t* idx, float* d2, int mem);
int lb_submap_launch_count(lb_submap* m, uint64_t* n);
/* the submap as target of `h` (same device; k_correspondences <= 20).  Call again after the map changed; while it is
 * unchanged the call only checks the generation.  Uses h's k_correspondences / gicp_epsilon for the covariances.
 * With h's recompute_target_covariance = 0 and a normal on every map point, the covariances come from the stored
 * normals instead (as for an uploaded cloud with normals), rebuilt only when the map or gicp_epsilon changed; otherwise
 * the k-NN covariance cache is used. */
int lb_gicp_set_target_submap(lb_gicp* h, lb_submap* m);

/* ------------------------------------------------------------------ NDT (SURVEY 8f row f4)
 * LOCUS's alternative registration method (`registration_method: ndt`, registration_settings.h:3-12): the OpenMP NDT
 * fork multithreaded_gicp/include/multithreaded_ndt/ndt_omp{.h,_impl.hpp} + voxel_grid_covariance_omp{.h,_impl.hpp},
 * set up at PointCloudOdometry.cc:182-195 and PointCloudLocalization.cc:267-280 and then driven through the same
 * icp_->setInputSource / setInputTarget / align / getFinalTransformation calls as GICP.
 *
 *   lb_ndt_create/destroy     make_shared<pclomp::NormalDistributionsTransform<PointF, PointF>>
 *   lb_ndt_set_params         setTransformationEpsilon / setMaximumIterations / setResolution / setStepSize /
 *                             setOulierRatio / setNeighborhoodSearchMethod (ndt_omp.h:124-196) and the voxel grid's
 *                             setMinPointPerVoxel / setCovEigValueInflationRatio (voxel_grid_covariance_omp.h:203-236)
 *   lb_ndt_set_source         icp_->setInputSource()
 *   lb_ndt_set_target         icp_->setInputTarget() -> init() (ndt_omp.h:116-119,257-262): the target's voxel Gaussians
 *   lb_ndt_align              icp_->align() + getFinalTransformation() + hasConverged() + getTransformationProbability()
 *                             (computeTransformation, ndt_omp_impl.hpp:100-208)
 *   lb_ndt_target_voxels      getTargetCells().getLeaves() restricted to the searchable voxels (voxel_centroids_ order)
 *   lb_ndt_derivatives        computeDerivatives / computeHessian at a given pose (ndt_omp_impl.hpp:221-343,641-718)
 *
 * Semantics kept: non-finite target points are skipped; a source with a non-finite point is refused (previous source
 * kept); a target whose int32 voxel index would overflow is refused (previous target kept); voxels with fewer than
 * min_points_per_voxel points are not searchable; a voxel whose covariance fails the eigenvalue / inverse check stays in
 * the radius search with nr_points = -1 exactly as in the reference (voxel_grid_covariance_omp_impl.hpp:326-355). */
typedef struct lb_ndt lb_ndt;

typedef struct lb_ndt_params {
  float resolution;                 /* 1.0   voxel side and neighbour radius (ndt_omp_impl.hpp:50) */
  double step_size;                 /* 0.1   More-Thuente maximum step (:51) */
  double outlier_ratio;             /* 0.55  (:52) */
  double transformation_epsilon;    /* 0.1   (:93); LOCUS passes icp_tf_epsilon / tf_epsilon */
  int max_iterations;               /* 35    (:94); LOCUS passes icp_iterations / iterations */
  int min_points_per_voxel;         /* 6     voxel_grid_covariance_omp.h:186 */
  double min_covar_eigvalue_mult;   /* 0.01  voxel_grid_covariance_omp.h:187 */
  int search_method;                /* 0 KDTREE (default, :96), 1 DIRECT26, 2 DIRECT7, 3 DIRECT1 (pclomp::NeighborSearchMethod values) */
  /* accepted for interface compatibility (PointCloudOdometry.cc:189,191-193), no effect -- as in the reference's NDT */
  double max_correspondence_distance;
  int ransac_iterations;
  int num_threads;
  int enable_timing_output;
} lb_ndt_params;

typedef struct lb_ndt_result {
  float final_transformation[16];   /* row-major 4x4 */
  int converged;
  int nr_iterations;
  int n_evaluations;                /* computeDerivatives passes */
  int n_target_voxels;              /* searchable voxels of the target */
  double trans_probability;         /* score / source points (ndt_omp_impl.hpp:207) */
  double pose[6];                   /* x y z roll pitch yaw of the last iterate */
  double t_total_s;
} lb_ndt_result;

void lb_ndt_default_params(lb_ndt_params* p);
int lb_ndt_create(int device, lb_ndt** h);
int lb_ndt_create_on_stream(int device, void* cuda_stream, lb_ndt** h);
int lb_ndt_destroy(lb_ndt* h);
int lb_ndt_set_params(lb_ndt* h, const lb_ndt_params* p);
int lb_ndt_set_source(lb_ndt* h, const void* pts, size_t n, size_t stride_bytes, size_t xyz_offset_bytes, int mem);
int lb_ndt_set_target(lb_ndt* h, const void* pts, size_t n, size_t stride_bytes, size_t xyz_offset_bytes, int mem);
/* The resident submap's current points as the target (the NDT counterpart of lb_gicp_set_target_submap; the map on the
 * handle's device).  The points are gathered device to device into the handle's target, with no host copy; the voxel
 * Gaussians are built lazily by the next align / derivatives / target_voxels, exactly as after lb_ndt_set_target of the
 * same points (lb_submap_points order).  While the map's generation is unchanged a repeated call does no device work,
 * so the Gaussians are rebuilt only after a keyframe insert or a crop.  After the map changed, align / derivatives /
 * target_voxels refuse with LB_ERR_INVALID_ARG until the target is set again; the handle stays usable.  An empty map is
 * LB_ERR_NO_TARGET, a map on another device LB_ERR_INVALID_ARG; the previous target is kept on any refusal. */
int lb_ndt_set_target_submap(lb_ndt* h, lb_submap* m);
/* guess16: row-major 4x4 float, NULL = identity (what LOCUS passes).  Blocking. */
int lb_ndt_align(lb_ndt* h, const float* guess16, lb_ndt_result* result);
/* host output buffers of `capacity` voxels each (any may be NULL); *n_voxels = searchable voxels, ascending voxel index */
int lb_ndt_target_voxels(lb_ndt* h, size_t capacity, size_t* n_voxels, int32_t* leaf_idx, int32_t* nr_points, double* mean3,
                         double* icov9, float* centroid3);
/* sums over the source transformed by T16 (row-major 4x4), angle derivatives taken at pose6.  compute_hessian: 0 / 1 = the
 * float path without / with the Hessian, 2 = the double-precision Hessian pass the line search ends with (score and
 * gradient come back as 0). */
int lb_ndt_derivatives(lb_ndt* h, const float* T16, const double* pose6, int compute_hessian, double* score, double* gradient6,
                       double* hessian36);
int lb_ndt_launch_count(lb_ndt* h, uint64_t* n);

/* ------------------------------------------------- scan-to-scan odometry pipeline
 * One robot's lidar stream, scans submitted in order: VoxelGrid(scan k) -> GICP(source = filtered k, target =
 * filtered k-1), i.e. what Locus.cc:451-453 + PointCloudOdometry::UpdateEstimate do per scan.  Results are
 * identical to calling lb_voxel_filter / lb_gicp_set_source / lb_gicp_set_target / lb_gicp_align per scan; what
 * the pipeline adds is overlap: a voxel stage (one host thread, one CUDA stream) and `depth` registration workers
 * (one host thread, one lb_gicp handle and stream each).  Scan k+1 is filtered and indexed while scan k is still in
 * its align kernels -- latency-bound cooperative grids that occupy a fraction of the SMs -- and up to `depth`
 * aligns are in flight at once.  Registration k does not depend on the pose of registration k-1 (the caller's
 * prior, if any, comes from IMU/odometry: PointCloudOdometry.cc:252-262), so the overlap changes no result.
 * In the reference the voxel filter already runs in its own nodelet thread ahead of the odometry thread.
 *
 * Threading: submit/next/drain are called from one thread (the lidar callback).  A submitted scan buffer (and the
 * optional filtered_out buffer) must stay valid until its result has been returned by lb_odometry_next. */
typedef struct lb_odometry lb_odometry;

typedef struct lb_odometry_result {
  uint64_t ticket;          /* 0-based submission number */
  int status;               /* lb_status of the stages of this scan */
  int has_pose;             /* 0 for the first scan (UpdateEstimate only stores it) or when a stage failed */
  size_t n_filtered;        /* points after VoxelGrid */
  lb_gicp_result gicp;      /* as lb_gicp_align (valid when has_pose).  Under LB_REG_NDT all zero except
                               final_transformation, converged, iterations (= ndt.nr_iterations) and status, which carry
                               the NDT align's values, so that a caller reading the pose needs no branch */
  char error[160];          /* message when status != LB_OK */
  lb_ndt_result ndt;        /* as lb_ndt_align under LB_REG_NDT (valid when has_pose); zeros under LB_REG_GICP */
} lb_odometry_result;

/* the registration method of a pipeline (`registration_method: gicp | ndt`, PointCloudOdometry.cc:182-195,
 * PointCloudLocalization.cc:267-280) */
typedef enum lb_registration { LB_REG_GICP = 0, LB_REG_NDT = 1 } lb_registration;

/* depth: registration workers (1..16).  max_points / max_point_step size the ring of filtered clouds. */
int lb_odometry_create(int device, int depth, size_t max_points, uint32_t max_point_step, lb_odometry** out);
int lb_odometry_destroy(lb_odometry* h);
/* the pipeline's VoxelGrid handle: configure leaf / limits on it before the first submit */
lb_voxel* lb_odometry_voxel(lb_odometry* h);
/* registration worker i's handle (0 <= i < depth): read-only use for counters / kernel times while idle */
lb_gicp* lb_odometry_gicp(lb_odometry* h, int i);
int lb_odometry_depth(lb_odometry* h);
/* applied to every worker's lb_gicp handle (call while the pipeline is idle) */
int lb_odometry_set_gicp_params(lb_odometry* h, const lb_gicp_params* p);
/* Cloud sharing (ON by default).  on != 0: every filtered scan's index + covariances are computed once, by the worker
 * that registers it as source, and adopted as target by the worker of the next scan (lb_gicp_share_source /
 * lb_gicp_set_target_cloud) instead of being rebuilt there.  Same poses, bit for bit (the index is a pure function of
 * the cloud).  on == 0: both clouds are rebuilt for every registration, which is what the reference's callers make
 * the reference do (setInputTarget clears the target's covariances, gicp.h:196-200).  Call while the pipeline is idle,
 * before the first scan. */
int lb_odometry_set_cloud_sharing(lb_odometry* h, int on);
/* Normals stage (OFF by default; k = 0).  3 <= k <= 20: the worker that prepares scan k's cloud gives it its k-NN
 * normals (lb_gicp_estimate_normals, viewpoint NULL = the origin) before its index and covariances are built, so odometry
 * source k, odometry target k+1 and lb_locus's localization source k all carry them; without cloud sharing the target
 * gets its normals the same way.  Covariances come from them where the gicp params say recompute_*_covariance = 0.
 * Call while the pipeline is idle, before the first scan. */
int lb_odometry_set_normals(lb_odometry* h, int k, const float* viewpoint);
/* Registration method (LB_REG_GICP by default).  LB_REG_NDT: every worker owns an lb_ndt handle (own stream) and
 * registration k is lb_ndt_set_source(filtered k) + lb_ndt_set_target(filtered k-1) + lb_ndt_align(prior), i.e. what the
 * blocking lb_ndt_* calls give; `ndt` (validated as lb_ndt_set_params does) is applied to every worker.  Cloud sharing is
 * a GICP concept and is ignored under NDT; the normals stage has no consumer there, so NDT together with normals k > 0 is
 * refused (LB_ERR_UNSUPPORTED) whichever of the two calls comes second.  Call while the pipeline is idle; a method
 * change after the first scan is refused (LB_ERR_UNSUPPORTED).  ndt may be NULL with LB_REG_GICP.  Any refusal leaves
 * the previous setting in place. */
int lb_odometry_set_registration(lb_odometry* h, int method, const lb_ndt_params* ndt);
/* scan: n_pts points of point_step bytes described by fields (as lb_voxel_filter); xyz must be FLOAT32 fields.
 * guess: row-major 4x4 prior handed to align() (NULL = identity).  filtered_out (nullable): host (LB_MEM_HOST) or
 * device buffer of at least n_pts * point_step bytes that receives the filtered cloud.  Blocks while 2*depth+2 scans
 * are already in flight.  *ticket (nullable) = the submission number. */
int lb_odometry_submit(lb_odometry* h, const uint8_t* scan, size_t n_pts, uint32_t point_step, const lb_field* fields,
                       int n_fields, int mem, const float* guess, uint8_t* filtered_out, int mem_filtered,
                       uint64_t* ticket);
/* One scan of a robot with several lidars: the stage-V work of the front-end nodes in LOCUS's multi-lidar launch (one
 * pcl/PassThrough per lidar, point_cloud_merger, BodyFilter, VoxelGrid) as one lb_voxel_filter_merged call on the
 * pipeline's voxel handle, in place of lb_voxel_filter.  Everything after the VoxelGrid is that of lb_odometry_submit;
 * the filtered scan (and, with lb_locus, the keyframe the map receives) is the merged one.
 *   Order: inputs[0 .. n_inputs-1] are merged in the order given, as lb_voxel_filter_merged does.  Inside a voxel the
 *     points are summed in merged order, so the order changes the centroids' bits: pass the merger's alive_keys_ order
 *     (PointCloudMerger.cc:191-250; a lidar that failed and came back is last).
 *   Varying count: n_inputs (1..3) may change from one scan to the next, and an input may have n_pts = 0.  A scan whose
 *     inputs are all empty filters to nothing and changes no state, as an empty scan does.
 *   Lifetimes: every input's data must stay valid until the scan's result is returned (as `scan` above).  The
 *     transforms (row-major 4x4 float, sensor -> base_link; NULL = identity) are copied here, so they may live on the
 *     caller's stack.
 *   Settings: PassThrough, BodyFilter, limits and leaf come from the pipeline's voxel handle (lb_odometry_voxel /
 *     lb_locus_voxel), as for one cloud; lb_locus's adaptive voxelization retunes on the merged filtered count.
 *   Refused here (no ticket taken, pending unchanged): n_inputs outside 1..3, inputs NULL, data NULL with n_pts > 0
 *     (LB_ERR_INVALID_ARG); sum of n_pts > max_points or point_step > max_point_step (LB_ERR_CAPACITY).
 *   What lb_voxel_filter_merged itself refuses (a layout other than x, y, z, intensity with more than one input or with
 *     a transform: LB_ERR_UNSUPPORTED) comes back as the scan's result status and changes no state, like any failed
 *     VoxelGrid.
 *   filtered_out (nullable) must hold sum(n_pts) * point_step bytes. */
int lb_odometry_submit_merged(lb_odometry* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step,
                              const lb_field* fields, int n_fields, int mem, const float* guess,
                              uint8_t* filtered_out, int mem_filtered, uint64_t* ticket);
/* next result in submission order.  block != 0: wait for it; block == 0: returns 1 when it is not ready yet.
 * Returns LB_ERR_NO_ALIGN when every submitted scan has already been returned. */
int lb_odometry_next(lb_odometry* h, lb_odometry_result* r, int block);
/* scans submitted but not yet returned by lb_odometry_next */
int lb_odometry_pending(lb_odometry* h, size_t* n);
/* kernels launched by all stages since creation */
int lb_odometry_launch_count(lb_odometry* h, uint64_t* n);
/* host wall-clock accounting since creation, to see which stage bounds the throughput:
 * out6 = { scans filtered, VoxelGrid stage busy s, its wait s (for a scan or a free ring slot),
 *          scans registered, registration workers busy s (summed over workers), their wait s (for a filtered scan) } */
int lb_odometry_stage_times(lb_odometry* h, double* out6);

/* ------------------------------------------------- the whole lidar callback as one pipeline
 * Locus::LidarCallback from raw scan to integrated pose and updated map (locus/src/Locus.cc:450-543): VoxelGrid ->
 * scan-to-scan odometry (PointCloudOdometry::UpdateEstimate) -> MotionUpdate -> scan-to-submap GICP
 * (PointCloudLocalization::MeasurementUpdate) -> keyframe test -> InsertPoints -> Refresh.  The lb_odometry pipeline
 * runs the first two stages; a third stage (one host thread, one lb_gicp handle bound to the caller's lb_submap) takes
 * the scans strictly in order and localizes them.  Each filtered scan's index and covariances are built once and shared
 * by odometry source k, odometry target k+1 and localization source k.  The rolling submap stands in for the external
 * mapper's neighbours as the localization target (the semantics of lb_gicp_set_target_submap).  Pose semantics and
 * what is unpinned: locus_b200/csrc/lo_pose.h and DESIGN.md.
 *
 * Threading and buffers as lb_odometry: submit / next from one thread; a submitted scan stays valid until its result
 * is returned.  The submap belongs to the caller but must not be used by anybody else while scans are in flight. */
typedef struct lb_locus lb_locus;

typedef struct lb_locus_thresholds {
  int enabled;               /* transform_thresholding */
  double max_translation;    /* metres, |t| <= max_translation */
  double max_rotation;       /* radians, |ToEulerZYX| <= max_rotation */
} lb_locus_thresholds;

/* The front end LOCUS ships in front of its callback; all 0 = off (lb_locus_default_params).  Shipped values:
 * normals_k = 20 (NormalComputation nodelet, locus.launch:177-181, NormalComputation.cfg:13,15), adaptive_voxelization
 * = 1 and points_to_process = 3000 (lo_settings.yaml:84-85). */
typedef struct lb_locus_front_end {
  int normals_k;              /* 0 = off; 3..20: every filtered scan gets its k-NN normals (lb_odometry_set_normals),
                                 keyframes enter the map with their normals rotated into the fixed frame */
  float viewpoint[3];         /* the normals' viewpoint, sensor frame (the origin in LOCUS) */
  int adaptive_voxelization;  /* b_adaptive_input_voxelization: retune the VoxelGrid leaf after every filtered scan,
                                 Locus.cc:780-810; the new leaf applies to the next scan */
  int points_to_process;      /* points_to_process_in_callback: the filtered point count the leaf aims at (> 0) */
} lb_locus_front_end;

/* The ICP covariance of the localization (lb_gicp_icp_covariance against the submap after every align); off by default.
 * Shipped values: enabled = 1, max_covariance = 0.01 (point_cloud_localization/config/parameters.yaml:6,8,10). */
typedef struct lb_locus_icp_covariance {
  int enabled;
  double max_covariance;     /* icp_max_covariance, finite and > 0 */
} lb_locus_icp_covariance;

typedef struct lb_locus_params {
  lb_gicp_params odometry;               /* k_correspondences, gicp_epsilon and index_cell_size must equal the */
  lb_gicp_params localization;           /* localization's: the shared clouds serve both registrations; so must the
                                            odometry's two recompute_*_covariance and the localization's
                                            recompute_source_covariance (one prepared cloud is all three) */
  lb_locus_thresholds odometry_thresholds;       /* point_cloud_odometry icp/transform_thresholding, max_* */
  lb_locus_thresholds localization_thresholds;   /* point_cloud_localization localization/transform_thresholding, max_* */
  double translation_threshold_kf;       /* keyframe when |t| of PoseDelta(last keyframe, pose) exceeds it ... */
  double rotation_threshold_kf;          /* ... or its 2 acos(q.w) does */
  int add_keyframes;                     /* b_add_keyframes_enabled */
  int refresh_every;                     /* >= 1: keyframes per Refresh (map_publishment/meters) */
  int msw;                               /* b_enable_msw: Refresh crops the map to the window */
  float window_half_size;                /* > 0: crop box centre = pose translation, +- this on every axis */
  int prior_map;                         /* b_run_with_gt_point_cloud: localize the first scan against the caller's map */
  double initial_pose[16];               /* row-major; L and the last keyframe before the first scan */
  lb_locus_front_end front_end;          /* normals and adaptive input voxelization (off by default) */
  lb_locus_icp_covariance icp_covariance;   /* the localization's ICP covariance (off by default) */
  /* registration_method of each package (LB_REG_GICP by default; fixed after the first scan).  Odometry NDT registers
   * filtered k against filtered k-1 with odometry_ndt; the scan's GICP cloud is still prepared and shared for the
   * localization stage (keyframe transform, ICP covariance, GICP localization), with the `odometry` GICP params.
   * Localization NDT aligns the scan's filtered points against the submap's points (lb_ndt_set_target_submap) with
   * localization_ndt; the ICP covariance, when enabled, is computed on the NDT pose against the submap.  An NDT params
   * block is validated (as lb_ndt_set_params) only when its method is NDT.  Defaults: lb_ndt_default_params with
   * transformation_epsilon / max_iterations of the packages' parameters.yaml: odometry 1e-3 / 20, localization 1e-5 / 20. */
  int odometry_method, localization_method;
  lb_ndt_params odometry_ndt, localization_ndt;
} lb_locus_params;

typedef struct lb_locus_result {
  uint64_t ticket;
  int status;                      /* lb_status of the scan's first failing stage */
  char error[160];
  size_t n_filtered;
  int has_odometry;                /* 0 for the first scan and the scan after a failed one (no odometry target) */
  lb_gicp_result odometry;
  int odometry_accepted;           /* the increment passed the odometry thresholds (O moved) */
  int has_localization;
  lb_gicp_result localization;
  int correction_accepted;         /* the localization correction passed its thresholds */
  double odometry_pose[16];        /* O_k, row-major, after this scan */
  double incremental[16];          /* I_k: what localization received (also when the odometry thresholds discarded it) */
  double pose[16];                 /* L_k: the integrated localization estimate */
  int keyframe;                    /* the scan was inserted into the map (the first scan or a keyframe) */
  size_t n_inserted, n_removed;    /* map points added by the insert / removed by the crop of this scan */
  size_t map_size;                 /* after this scan */
  float leaf_size;                 /* the VoxelGrid x leaf this scan was filtered with */
  /* icp_covariance enabled: the covariance LOCUS publishes in the odometry message's pose.covariance (Locus.cc:510-511),
   * computed after the localization align and before the keyframe insert, with T = the align's final transformation,
   * against the submap, the map's normals rotated by the float rotation of P^-1 (P = the align's guess).  Zeros when
   * the scan was not localized (the first scan without prior_map: PublishPoseNoUpdate, PointCloudLocalization.cc:580-587) */
  int has_icp_covariance;
  double icp_covariance[36];
  double condition_number;         /* the last one computed (Locus.cc:547-548), kept over a scan that took the NaN fallback;
                                      NaN until the first one is computed (the first scan without prior_map, or a run of
                                      fallbacks from the start: the reference publishes an uninitialised value there);
                                      0 when icp_covariance is off */
  int icp_covariance_flags;        /* LB_ICPCOV_* */
  /* the NDT aligns' results under LB_REG_NDT (zeros under GICP); `odometry` / `localization` then carry their
   * final_transformation, converged, iterations and status as in lb_odometry_result */
  lb_ndt_result odometry_ndt, localization_ndt;
} lb_locus_result;

/* the reference's shipped values: locus/config/lo_settings.yaml, point_cloud_odometry/config/parameters.yaml,
 * point_cloud_localization/config/parameters.yaml; odometry align_points_per_cta = 1024 (DESIGN.md, SM budget) */
int lb_locus_default_params(lb_locus_params* p);
/* depth: odometry workers (1..16); `map` on `device`, owned by the caller and outliving the handle */
int lb_locus_create(int device, int depth, size_t max_points, uint32_t max_point_step, lb_submap* map, lb_locus** out);
/* joins every stage; scans still in flight are dropped */
int lb_locus_destroy(lb_locus* h);
lb_voxel* lb_locus_voxel(lb_locus* h);
/* refused while scans are in flight, when the two gicp params disagree on the shared clouds, when front_end is out of
 * range, when normals_k or a registration method changes after the first scan, and when the NDT params of a method set
 * to NDT are invalid; the previous parameters stay in place */
int lb_locus_set_params(lb_locus* h, const lb_locus_params* p);
/* same arguments and blocking rule as lb_odometry_submit; guess = the odometry prior */
int lb_locus_submit(lb_locus* h, const uint8_t* scan, size_t n_pts, uint32_t point_step, const lb_field* fields,
                    int n_fields, int mem, const float* guess, uint8_t* filtered_out, int mem_filtered, uint64_t* ticket);
/* same arguments and rules as lb_odometry_submit_merged (order, varying lidar count, lifetimes, copied transforms,
 * refusals): one scan of 1..3 lidars merged in the VoxelGrid stage; the keyframe inserted is the merged filtered scan */
int lb_locus_submit_merged(lb_locus* h, const lb_voxel_input* inputs, int n_inputs, uint32_t point_step,
                           const lb_field* fields, int n_fields, int mem, const float* guess, uint8_t* filtered_out,
                           int mem_filtered, uint64_t* ticket);
int lb_locus_next(lb_locus* h, lb_locus_result* r, int block);
int lb_locus_pending(lb_locus* h, size_t* n);
/* out9 = the six values of lb_odometry_stage_times, then { scans localized, localization stage busy s, its wait s } */
int lb_locus_stage_times(lb_locus* h, double* out9);

#ifdef __cplusplus
}
#endif
#endif /* LOCUS_B200_H_ */
