/*
 * cupoch_b200.h -- C ABI of the H100-native ICP / kNN / voxel-grid engine.
 *
 * This is the drop-in boundary for cupoch's hot path (SURVEY.md section 8b).
 * cupoch has no FFI/plugin registry: its boundary is the public C++ headers
 * (and the pybind11 module built on them).  Each entry point below names the
 * reference interface it replaces; include/cupoch/ holds the header-compatible
 * C++ facade that forwards to these symbols, cupoch_b200/ the Python mirror,
 * and INTEGRATION.md the binding a cupoch maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers + sizes, no torch / thrust / Eigen types.
 *   - all data pointers are DEVICE pointers unless the name starts with h_;
 *     they are borrowed for the duration of the call and never retained
 *     (contexts keep private re-packed copies), outputs are caller-allocated.
 *   - points / normals / colors: packed float32 xyz, 12-byte stride (the
 *     layout of cupoch's device_vector<Eigen::Vector3f>, pointcloud.h:259-262).
 *   - covariances: 9 float32 per point; cov_col_major=1 for Eigen's default
 *     column-major Matrix3f (pointcloud.h:262), 0 for row-major (numpy).
 *   - 4x4 transforms: float32[16], ROW-major.  (Eigen::Matrix4f is column-major:
 *     the facade transposes 16 floats on the host.)
 *   - sizes are 64-bit; indices are int32 like the reference.
 *   - return value: 0 = CPHB_OK, <0 = error (message via cphb_last_error()).
 *     Nothing here calls exit() (the reference's cudaSafeCall does,
 *     platform.cu:60-67).
 *   - stream: a cudaStream_t passed as void* (NULL = default stream).  Calls
 *     are asynchronous on that stream unless they return host values, in which
 *     case they synchronise the stream before returning (documented per call).
 */
#ifndef CUPOCH_B200_H
#define CUPOCH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CPHB_VERSION 100 /* 0.1.0 */

enum cphb_status {
    CPHB_OK = 0,
    CPHB_ERR_INVALID = -1,  /* bad argument (the reference logs and continues / returns -1) */
    CPHB_ERR_CUDA = -2,     /* CUDA runtime error */
    CPHB_ERR_NO_DEVICE = -3,
    CPHB_ERR_NCCL = -4,
    CPHB_ERR_UNSUPPORTED = -5
};

/* registration::TransformationEstimationType, transformation_estimation.h:40-47 */
enum cphb_estimation {
    CPHB_EST_UNSPECIFIED = 0,
    CPHB_EST_POINT_TO_POINT = 1,
    CPHB_EST_POINT_TO_PLANE = 2,
    CPHB_EST_SYMMETRIC = 3,
    CPHB_EST_COLORED_ICP = 4,
    CPHB_EST_GENERALIZED_ICP = 5
};

int cphb_version(void);
const char *cphb_last_error(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
uint64_t cphb_launch_count(void);
/* cudaGetDeviceCount / properties without torch */
int cphb_device_count(void);
int cphb_set_device(int device);

/* ------------------------------------------------------------------------ *
 * Spatial index  (replaces knn::KDTreeFlann + the vendored FLANN CUDA kd-tree,
 * kdtree_flann.h:43-124, kdtree_flann.inl:125-144, kdtree_cuda_builder.h)
 * ------------------------------------------------------------------------ */
typedef struct cphb_index cphb_index;

/* KDTreeFlann::SetRawData (kdtree_flann.inl:125-144).  Like the reference the
 * index owns a private re-packed copy of the points: xyz may be freed after
 * the call returns (the call is stream-ordered; no host sync). n may be 0. */
int cphb_index_create(const float *xyz, size_t n, void *stream, cphb_index **out);
void cphb_index_destroy(cphb_index *index);
size_t cphb_index_size(const cphb_index *index);

/* KDTreeFlann::SearchRadius(query, radius, max_nn, indices, distance2)
 * (kdtree_flann.h:66-72, .inl:97-122; result set result_set.h:372-474):
 * for each query the <= max_nn nearest points with d2 < radius*radius (strict,
 * radius squared in float), ascending by (d2, index).  idx / d2 are
 * [n_query * max_nn]; unfilled slots idx=-1, d2=+inf.  1 <= max_nn <= 100
 * (NUM_MAX_NN, kdtree_search_param.h:26) else CPHB_ERR_INVALID (reference: -1).
 * h_count (optional, host): number of filled slots = the reference's return
 * value; requesting it synchronises the stream. */
int cphb_search_radius(const cphb_index *index, const float *query, size_t n_query,
                       float radius, int max_nn, int32_t *idx, float *d2,
                       int64_t *h_count, void *stream);
/* KDTreeFlann::SearchKNN (kdtree_flann.h:60-65, .inl:70-95). */
int cphb_search_knn(const cphb_index *index, const float *query, size_t n_query,
                    int knn, int32_t *idx, float *d2, int64_t *h_count, void *stream);
/* north_star's name for the same operation (SURVEY.md section 0). */
int cphb_search_hybrid(const cphb_index *index, const float *query, size_t n_query,
                       float radius, int max_nn, int32_t *idx, float *d2,
                       int64_t *h_count, void *stream);

/* ------------------------------------------------------------------------ *
 * geometry::PointCloud operations (pointcloud.h)
 * ------------------------------------------------------------------------ */
typedef struct cphb_cloud {
    const float *points;         /* n x 3 */
    const float *normals;        /* n x 3 or NULL  (HasNormals, pointcloud.h:82-94) */
    const float *colors;         /* n x 3 or NULL */
    const float *covariances;    /* n x 9 or NULL */
    const float *color_gradient; /* n x 3 or NULL (PointCloudForColoredICP, colored_icp.cu:36-40) */
    size_t n;
    int cov_col_major;
} cphb_cloud;

/* PointCloud::Transform (pointcloud.cu:293-299): in place p<-Rp+t, n<-Rn,
 * C<-R C R^T; any of normals/covariances may be NULL. */
int cphb_transform(float *points, float *normals, float *covariances, int cov_col_major,
                   size_t n, const float h_T[16], void *stream);
/* PointCloud::GetMinBound / GetMaxBound (eigen.inl:197-221). Synchronises. */
int cphb_min_max_bound(const float *points, size_t n, float h_min[3], float h_max[3], void *stream);

/* PointCloud::VoxelDownSample (down_sample.cu:170-273).  normals / colors in
 * and out may be NULL (together).  out_* must hold n elements; *h_n_out gets
 * the voxel count (synchronises).  Output order: lexicographic by voxel
 * (x,y,z) like the reference's sort.  voxel<=0 or voxel*INT_MAX < extent
 * return CPHB_OK with *h_n_out = 0 (the reference warns and returns an empty
 * cloud). */
int cphb_voxel_down_sample(const float *points, const float *normals, const float *colors,
                           size_t n, float voxel_size, float *out_points, float *out_normals,
                           float *out_colors, size_t *h_n_out, void *stream);

/* The same with a caller-supplied grid origin (every component <= the cloud's minimum): several ranks can
 * down-sample disjoint parts of one cloud on one common grid (cupoch_b200.distributed.voxel_down_sample). */
int cphb_voxel_down_sample_origin(const float *points, const float *normals, const float *colors,
                                  size_t n, float voxel_size, const float h_origin[3], float *out_points,
                                  float *out_normals, float *out_colors, size_t *h_n_out, void *stream);
/* Batched VoxelGrid::GetVoxel (voxelgrid.cu:338-341): out_indices (device, n x 3 int32) =
 * floor((p - origin) / voxel_size), the key arithmetic of every voxel kernel in this library. */
int cphb_voxel_indices(const float *points, size_t n, float voxel_size, const float h_origin[3],
                       int32_t *out_indices, void *stream);

/* PointCloud::EstimateNormals (estimate_normals.cu:82-127).  knn>0: KNN search
 * (k includes the point itself, default 30); knn<=0: radius + max_nn. */
int cphb_estimate_normals(const float *points, size_t n, int knn, float radius, int max_nn,
                          float *out_normals, void *stream);
/* Multi-GPU building block: the normals of points [first, first + count) only (out_normals holds count rows),
 * neighbours searched in the whole cloud.  Ranks estimate disjoint blocks and all-gather them; the union equals
 * cphb_estimate_normals bit for bit (same search, same per-point arithmetic). */
int cphb_estimate_normals_range(const float *points, size_t n, int knn, float radius, int max_nn, size_t first,
                                size_t count, float *out_normals, void *stream);
/* InitializePointCloudForGeneralizedICP covariance step (generalized_icp.cu:53-60). */
int cphb_covariances_from_normals(const float *normals, size_t n, float epsilon,
                                  float *out_cov, int cov_col_major, void *stream);
/* InitializePointCloudForColoredICP (colored_icp.cu:120-148): radius search
 * (radius, max_nn) + per-point intensity-gradient fit. */
int cphb_color_gradient(const float *points, const float *normals, const float *colors, size_t n,
                        float radius, int max_nn, float *out_gradient, void *stream);

/* VoxelGrid::CreateFromPointCloudWithinBounds (voxelgrid_factory.cu:164-219): grid index
 * floor((p - min_bound) / voxel_size) per point (negative below the bound, as in the reference), one voxel per
 * distinct index in lexicographic (x, y, z) order, colour = mean colour of its points ((1,1,1) when colors is
 * NULL).  out_keys (device, n x 3 int32) / out_colors (device, n x 3 float) must hold n rows; *h_n_out = voxel
 * count (synchronises).  For VoxelGrid::CreateFromPointCloud pass the cloud's bounds widened by half a voxel
 * (:221-228).  voxel_size <= 0 or voxel_size * INT_MAX < extent give an empty grid. */
int cphb_voxel_grid_from_point_cloud(const float *points, const float *colors, size_t n, float voxel_size,
                                     const float h_min_bound[3], const float h_max_bound[3], int32_t *out_keys,
                                     float *out_colors, size_t *h_n_out, void *stream);

/* PointCloud::RemoveRadiusOutliers (down_sample.cu:317-354): search the cloud against itself with
 * (radius, nb_points + 1) and keep the points all of whose slots are filled (more than nb_points neighbours
 * inside the radius, the point itself included).  indices_out (device, n int32) receives the ascending indices
 * of the kept points, *h_n_out their number (synchronises).  As in the reference a negative radius acts as
 * |radius| and radius == 0 keeps nothing; nb_points + 1 > 100 (NUM_MAX_NN) is CPHB_ERR_INVALID. */
int cphb_remove_radius_outliers(const float *points, size_t n, int nb_points, float radius,
                                int32_t *indices_out, size_t *h_n_out, void *stream);
/* PointCloud::RemoveStatisticalOutliers (down_sample.cu:356-438): per point the mean of the squared distances
 * to its nb_neighbors nearest points (itself included), cloud mean and Bessel-corrected standard deviation of
 * those means, keep 0 < mean_i < cloud mean + std_ratio * std.  h_stats (optional) = {cloud mean, std,
 * threshold}.  Outputs as above. */
int cphb_remove_statistical_outliers(const float *points, size_t n, int nb_neighbors, float std_ratio,
                                     int32_t *indices_out, size_t *h_n_out, float h_stats[3], void *stream);
/* PointCloud::GaussianFilter (pointcloud.cu:56-106,387-433): radius search of the cloud against itself
 * (search_radius, num_max_search_points <= 100), every row replaced by the exp(-0.5 d2 / sigma2)-weighted mean of
 * its neighbours' rows.  normals / colors in and out may be NULL (together); outputs hold n rows; *h_n_out = n, or
 * 0 for illegal parameters (the reference returns an empty cloud).  Synchronises. */
int cphb_gaussian_filter(const float *points, const float *normals, const float *colors, size_t n,
                         float search_radius, float sigma2, int num_max_search_points, float *out_points,
                         float *out_normals, float *out_colors, size_t *h_n_out, void *stream);
/* PointCloud::SelectByIndex (down_sample.cu:40-127, invert = false): out row t = in row indices[t].
 * normals / colors in and out may be NULL (together). */
int cphb_select_by_index(const float *points, const float *normals, const float *colors, size_t n,
                         const int32_t *indices, size_t n_indices, float *out_points, float *out_normals,
                         float *out_colors, void *stream);
/* Region selection (boundingvolume.cu:38-101,221-244,413-425; pointcloud.cu:38-53,105-121): indices_out (device, n
 * int32) receives the ascending indices of the points the test keeps, *h_n_out their number (synchronises).
 *   aabb:   kept unless p[a] < h_min[a] or p[a] > h_max[a] for some axis a (inclusive; a NaN coordinate is kept).
 *           PassThroughFilter(axis, lo, hi) is this test with lo / hi on that axis and -inf / +inf on the others.
 *   obb:    h_box_points = OrientedBoundingBox::GetBoxPoints() (8 x xyz); the reference's six determinant plane tests,
 *           either sign pattern (DESIGN.md fixes the determinant's expansion order).
 *   finite: removed when (remove_nan and a coordinate is NaN) or (remove_infinite and a coordinate is infinite).
 * n > 2^31-1: CPHB_ERR_INVALID. */
int cphb_aabb_point_indices(const float *points, size_t n, const float h_min[3], const float h_max[3],
                            int32_t *indices_out, size_t *h_n_out, void *stream);
int cphb_obb_point_indices(const float *points, size_t n, const float h_box_points[24], int32_t *indices_out,
                           size_t *h_n_out, void *stream);
int cphb_finite_point_indices(const float *points, size_t n, int remove_nan, int remove_infinite, int32_t *indices_out,
                              size_t *h_n_out, void *stream);
/* OrientedBoundingBox::CreateFromPoints (boundingvolume.cu:219-269): mean and centred covariance summed in double in
 * the tiled order of DESIGN.md's arithmetic contract, a double symmetric eigensolve, axes sorted by descending
 * eigenvalue, each axis signed so its largest-magnitude component (the first among equal ones) is positive; the
 * extent and centre come from the float32 bounds of the points transformed by [R^T | -R^T mean].  h_R is row-major.
 * n == 0: the zero box with R = I.  Synchronises. */
int cphb_oriented_bounding_box(const float *points, size_t n, float h_center[3], float h_R[9], float h_extent[3],
                               void *stream);
/* PointCloud::UniformDownSample (down_sample.cu:275-300): out row t = in row t * every_k for t < n / every_k (rounded
 * down; *h_n_out gets that count).  normals / colors in and out may be NULL (together).  every_k == 0:
 * CPHB_ERR_INVALID.  Asynchronous. */
int cphb_uniform_down_sample(const float *points, const float *normals, const float *colors, size_t n, size_t every_k,
                             float *out_points, float *out_normals, float *out_colors, size_t *h_n_out, void *stream);
/* PointCloud::NormalizeNormals (pointcloud.cu:282-285): in place, n /= sqrt(|n|^2) where |n|^2 > 0.  Asynchronous. */
int cphb_normalize_normals(float *normals, size_t n, void *stream);
/* PointCloud::OrientNormalsToAlignWithDirection (estimate_normals.cu:66-78,129-141): in place, a zero normal becomes
 * h_reference, a normal with n . h_reference < 0 is negated.  Asynchronous. */
int cphb_orient_normals(float *normals, size_t n, const float h_reference[3], void *stream);
/* PointCloud::SegmentPlane (segmentation.cu:187-267): RANSAC plane [a,b,c,d] with |dot3(abc, p) + d| <
 * distance_threshold inliers.  h_seeds (host, num_iterations ints) are the seeds the reference draws with rand(),
 * one per iteration; iteration t samples d_cards[0..2] after a stable sort of d_cards by thrust's random_functor(
 * h_seeds[t], n) keys, cumulative over t.  All hypotheses are scored in one pass; the best (fitness >, or == with
 * "inlier_rmse" <) defines the final inliers (ascending, into inliers_out, device, room for n), which are refitted
 * (GetPlaneFromPoints) into h_plane.  Sums over points / inliers follow the order of DESIGN.md's arithmetic
 * contract (tiles of 1024 consecutive elements summed sequentially in double, then the tiles in order).
 * ransac_n < 3 or n < ransac_n: zero plane, no inliers (the reference logs an error).  Optional outputs (NULL to
 * skip): h_best_iteration (-1 if no hypothesis won), h_fitness_rmse = the winner's {fitness, inlier_rmse},
 * h_phase_ms = CUDA-event times of {sampling, scoring + selection, final inliers + refit}.  num_iterations < 0 or
 * n > 2^31-1: CPHB_ERR_INVALID.  Synchronises. */
int cphb_segment_plane(const float *points, size_t n, float distance_threshold, int ransac_n, int num_iterations,
                       const int32_t *h_seeds, float h_plane[4], int32_t *inliers_out, size_t *h_n_out,
                       int32_t *h_best_iteration, float h_fitness_rmse[2], float h_phase_ms[3], void *stream);
/* PointCloud::FarthestPointDownSample (pointcloud.cu:122-139,301-338): indices_out (device, num_samples int32)
 * receives the farthest-point sequence: index 0 first, then at every step the point whose squared distance (dist2,
 * DESIGN.md arithmetic contract) to the nearest point selected so far is largest, the smallest index among equal
 * distances.  Running distances start at +inf and are updated with fminf, so a NaN distance never replaces one.  Any
 * num_samples >= 1 runs the loop, num_samples >= n included (on a finite cloud, once every distinct point is taken the
 * sequence repeats index 0; the front ends return an empty cloud for 0 and a copy for n).  d2_out (device, n floats, optional) receives
 * every point's final running distance: its squared distance to the nearest selected point.  One cooperative launch
 * for the whole loop; asynchronous on the stream (no host synchronisation).  n == 0 with num_samples > 0, or
 * n > 2^31-1: CPHB_ERR_INVALID. */
int cphb_farthest_point_down_sample(const float *points, size_t n, size_t num_samples, int32_t *indices_out,
                                    float *d2_out, void *stream);
/* geometry::keypoint::ComputeISSKeypoints (keypoint.h:54-60, iss_keypoints.cu:108-172): Intrinsic Shape Signature
 * keypoints.  salient_radius == 0 or non_max_radius == 0 replaces BOTH by 6 and 4 times the resolution sqrtf(sum of
 * the cloud's 2-NN squared distances / (float)n), the sum taken in DESIGN.md's tiled order.  A point's saliency is the
 * smallest eigenvalue of its neighbourhood covariance (radius search (salient_radius, max_neighbors), the point
 * itself included), as FastEigen3x3 returns it (normalised by the covariance's largest coefficient); it is -1 when
 * fewer than min_neighbors points are listed, when every covariance coefficient is within 1e-5 of 0 (absolute), or
 * unless lambda2 / lambda3 < gamma_21 and lambda1 / lambda2 < gamma_32.  A point is a keypoint (mask_out[i] = 1) iff
 * its saliency is >= 0 and no point of its (non_max_radius, max_neighbors) list has a strictly larger one.
 * mask_out: device, n bytes.  Optional (NULL to skip): indices_out (device, n int32) gets the ascending keypoint
 * indices, saliency_out (device, n floats) every saliency, h_radii the two radii used.  *h_n_out = keypoint count.
 * max_neighbors in [0, 256] (0: no keypoints), else CPHB_ERR_INVALID; a negative radius acts as its absolute value;
 * n == 0 gives 0 keypoints.  One index serves every search; no [n][max_neighbors] table is built.  Synchronises. */
int cphb_compute_iss_keypoints(const float *points, size_t n, float salient_radius, float non_max_radius,
                               float gamma_21, float gamma_32, int min_neighbors, int max_neighbors, uint8_t *mask_out,
                               int32_t *indices_out, size_t *h_n_out, float *saliency_out, float h_radii[2],
                               void *stream);

/* ------------------------------------------------------------------------ *
 * registration  (registration.h:35-91, transformation_estimation.h:36-143,
 * generalized_icp.h, colored_icp.h)
 * ------------------------------------------------------------------------ */
typedef struct cphb_icp_params {
    int estimation;               /* enum cphb_estimation */
    float max_correspondence_distance;
    float relative_fitness;       /* ICPConvergenceCriteria, registration.h:35-49 */
    float relative_rmse;
    int max_iteration;
    float det_thresh;             /* PointToPlane / Symmetric / Colored: 1e-6; ignored for GICP */
    float lambda_geometric;       /* Colored ICP, default 0.968 */
    int flags;                    /* reserved, ignored (keeps the struct layout) */
    /* Multi-GPU: with shard_world > 1 every rank passes the FULL source; the library orders it along the
     * Hilbert curve and keeps the shard_rank-th contiguous block of that order (a spatially compact
     * shard at full density).  correspondence indices stay global.  0/0 or 1 = no library-side sharding
     * (a caller may still pass its own shard together with a communicator). */
    int shard_rank;
    int shard_world;
} cphb_icp_params;

typedef struct cphb_icp_result {
    float transformation[16];     /* row-major */
    float fitness;
    float inlier_rmse;
    int64_t n_correspondences;    /* global count (all ranks) */
    int64_t n_local_correspondences; /* pairs written to corr_out by this rank (== global on one GPU) */
    int iterations;               /* updates applied */
    int converged;
    float loop_ms;                /* device time of the launch loop (CUDA events on `stream`) */
    int loop_launches;            /* kernels launched inside that region */
} cphb_icp_result;

typedef struct cphb_icp cphb_icp;
typedef struct cphb_comm cphb_comm; /* multi-GPU communicator, see the end of this header */

/* Build the per-call state of RegistrationICP (registration.cu:146-147): the
 * spatial index over target.points and a Hilbert-ordered working copy of the
 * source.  Nothing of either cloud is retained: the target points live in the
 * index, the target attributes the estimator reads (normals, colour
 * intensity, colour gradient, covariances) are copied into index order, the
 * source into its working copy -- both clouds may be freed or overwritten
 * as soon as this call's work on `stream` has completed. */
int cphb_icp_create(const cphb_cloud *source, const cphb_cloud *target,
                    const cphb_icp_params *params, void *stream, cphb_icp **out);
void cphb_icp_destroy(cphb_icp *icp);

/* Run the loop of RegistrationICP (registration.cu:148-172) from init.  One
 * fused kernel per iteration, no host round trip inside the loop.
 * comm: NULL (single GPU) or a communicator whose ranks each hold a contiguous
 * shard of the source; the 32 partial sums are exchanged once per iteration
 * (NCCL all-reduce, or the peer-memory exchange fused into the reduce kernel).  corr_out (device, optional): 2*source.n int32 receiving the
 * final correspondence set (i, j) ascending in i (local shard indices).
 * Synchronises the stream before returning h_result. */
int cphb_icp_run(cphb_icp *icp, const float h_init[16], cphb_comm *comm,
                 cphb_icp_result *h_result, int32_t *corr_out, void *stream);

/* Debug / test hook: one GetRegistrationResultAndCorrespondences +
 * ComputeJTJandJTr step at pose h_T applied to the pristine source:
 * h_sums[32] doubles = 21 JTJ upper | 6 JTr | sum r^2 | sum d^2 | count | 0 0
 * (P2P: sum s(3) sum t(3) sum s t^T(9) ... | sum d^2 | count); corr_index
 * (device, optional, source.n int32): matched target index per source point
 * or -1.  Synchronises. */
int cphb_icp_step(cphb_icp *icp, const float h_T[16], double h_sums[32],
                  int32_t *corr_index, void *stream);

/* One-shot registration::RegistrationICP / RegistrationGeneralizedICP /
 * RegistrationColoredICP on device-resident clouds.  For GICP the clouds must
 * carry covariances, for Colored ICP the target must carry color_gradient
 * (use cphb_covariances_from_normals / cphb_color_gradient, as the reference's
 * Initialize* helpers do). */
int cphb_registration_icp(const cphb_cloud *source, const cphb_cloud *target,
                          const float h_init[16], const cphb_icp_params *params,
                          cphb_comm *comm, cphb_icp_result *h_result, int32_t *corr_out,
                          void *stream);

/* The same from HOST buffers (every pointer of the two clouds is a host pointer, pinned for full speed): the
 * uploads are issued on a separate stream in the order the loop first needs them (target points, source, target
 * attributes) and overlap the index build and the source ordering.  h_corr_out (optional, host, 2 * source.n
 * int32) receives the (i, j) pairs.  Complete on return. */
int cphb_registration_icp_host(const cphb_cloud *h_source, const cphb_cloud *h_target,
                               const float h_init[16], const cphb_icp_params *params, cphb_comm *comm,
                               cphb_icp_result *h_result, int32_t *h_corr_out, void *stream);

/* TransformationEstimation*::ComputeTransformation / ComputeRMSE on an explicit correspondence list
 * (transformation_estimation.h:49-77; corr = device (i, j) pairs).  Synchronise. */
int cphb_compute_transformation(int estimation, const cphb_cloud *source, const cphb_cloud *target,
                                const int32_t *corr, size_t n_corr, const cphb_icp_params *params,
                                float h_T[16], void *stream);
int cphb_compute_rmse(int estimation, const cphb_cloud *source, const cphb_cloud *target,
                      const int32_t *corr, size_t n_corr, const cphb_icp_params *params,
                      float *h_rmse, void *stream);
/* registration::Kabsch(model, target[, corres]) (kabsch.h:30-49); corr NULL pairs i<->i. */
int cphb_kabsch(const float *model, size_t n_model, const float *target, const int32_t *corr,
                size_t n_corr, float h_T[16], void *stream);

/* registration::KabschWeighted(model, target, weight) (kabsch.h:46-49, kabsch.cu:138-201; FilterReg's M-step,
 * filterreg.cu:80): weighted centres, H = sum w^2 (m - mc)(t - tc)^T / sum w^2, R = V diag(1,1,det(UV)) U^T. */
int cphb_kabsch_weighted(const float *model, const float *target, const float *weight, size_t n,
                         float h_T[16], void *stream);

/* The other users of the normal-equation reducer (SURVEY 8f rank 3), on EXPLICIT rows: J [n][num_j][6] and r [n][num_j]
 * float32, device.  utility::ComputeJTJandJTr<Matrix6f, Vector6f, NumJ> (eigen.inl:120-145; RGB-D odometry,
 * odometry.cu:618): h_sums[32] = 21 JTJ upper | 6 JTr | sum r^2 | 0... */
int cphb_compute_jtj_jtr(const float *J, const float *r, size_t n, int num_j, double h_sums[32], void *stream);
/* utility::ComputeWeightedJTJandJTr (eigen.inl:147-195) with the Student-t weights of the RGB-D odometry
 * (odometry.cu:633-648, :688): w_sum = sum_i r2_i (nu + 1) / (nu + r2_i / sigma2), w_i = (nu + 1) / (nu + r2_i / w_sum),
 * h_sums = sums of w_i * (JTJ_i, JTr_i, r2_i) laid out as above; *h_w_sum = w_sum (the caller's next sigma2). */
int cphb_compute_weighted_jtj_jtr(const float *J, const float *r, size_t n, int num_j, float sigma2, float nu,
                                  double h_sums[32], float *h_w_sum, void *stream);

/* registration::ComputeFPFHFeature(input, search_param) (feature.h, fpfh.cu:192-229): out_features [n][33] float32.
 * knn > 0: KDTreeSearchParamKNN(knn); else KDTreeSearchParamRadius(radius, max_nn).  Normals are required. */
int cphb_compute_fpfh_feature(const float *points, const float *normals, size_t n, int knn, float radius,
                              int max_nn, float *out_features, void *stream);

/* registration::ComputeSHOTFeature(input, radius, search_param) (feature.h:62-66, shot.cu:222-255):
   knn > 0 -> KDTreeSearchParamKNN(knn), else KDTreeSearchParamRadius(search_radius, max_nn).
   out_features [n][352] float32, one row per point.  `radius` is the descriptor's support (frame weights radius - d,
   shells at radius / 4, / 2, * 3 / 4), independent of the search.  Normals are required; a point's row is all zero
   when fewer than 5 other points are listed.  knn <= 100 and 0 <= max_nn <= 256, else CPHB_ERR_INVALID; n == 0 is a
   no-op.  One index serves one fused kernel; no [n][k] table is built.  Synchronises. */
int cphb_compute_shot_feature(const float *points, const float *normals, size_t n, float radius,
                              int knn, float search_radius, int max_nn, float *out_features, void *stream);

/* geometry::PointCloud::ClusterDBSCAN(eps, min_points, print_progress, max_edges) (pointcloud.h:195-199,
 * pointcloud_cluster.cu:84-179): labels_out (device, n int32), -1 = noise; *h_n_clusters (optional) = cluster ids
 * handed out.  max_edges in [1, 255] (reference default NUM_MAX_NN = 100). */
int cphb_cluster_dbscan(const float *points, size_t n, float eps, int min_points, int max_edges,
                        int32_t *labels_out, int *h_n_clusters, void *stream);

/* ------------------------------------------------------------------------ *
 * geometry::OccupancyGrid (occupancygrid.h:74-147, occupancygrid.cu): a dense
 * resolution^3 log-odds grid.  Cells are float prob_log (NaN = unknown); voxel
 * (x, y, z) of the grid covers origin + (x - resolution/2 .. +1) * voxel_size.
 * ------------------------------------------------------------------------ */
typedef struct cphb_occgrid cphb_occgrid;
typedef struct cphb_occgrid_params { /* occupancygrid.h:139-143 (defaults -2.0, 3.5, 0.85, -0.4, 0.0) */
    float clamping_thres_min, clamping_thres_max, prob_hit_log, prob_miss_log, occ_prob_thres_log;
} cphb_occgrid_params;
void cphb_occgrid_default_params(cphb_occgrid_params *p);
/* OccupancyGrid(voxel_size, resolution = 512, origin = 0) (occupancygrid.cu:289-297); the grid owns its device memory */
int cphb_occgrid_create(float voxel_size, int resolution, const float origin[3], void *stream, cphb_occgrid **out);
void cphb_occgrid_destroy(cphb_occgrid *grid);
int cphb_occgrid_clear(cphb_occgrid *grid, void *stream);                       /* Clear (:310-315) */
int cphb_occgrid_set_params(cphb_occgrid *grid, const cphb_occgrid_params *p);  /* the public members :139-143 */
int cphb_occgrid_set_geometry(cphb_occgrid *grid, float voxel_size, const float origin[3]); /* voxel_size_ / origin_ */
const float *cphb_occgrid_data(const cphb_occgrid *grid);                       /* device prob_log[resolution^3], borrowed */
int cphb_occgrid_resolution(const cphb_occgrid *grid);
/* OccupancyGrid::Insert(points, viewpoint, max_range = -1) (occupancygrid.cu:462-526): every voxel crossed by a ray
 * viewpoint -> point gets prob_miss_log once, every voxel holding a point within max_range gets prob_hit_log once
 * (occupied wins), both clamped.  points: device, packed xyz. */
int cphb_occgrid_insert(cphb_occgrid *grid, const float *points, size_t n, const float viewpoint[3], float max_range,
                        void *stream);
/* AddVoxels(voxels, occupied) (:579-600): device [n][3] int32 grid indices inside the grid; AddVoxel (:554-577): one
 * host index, range-checked (CPHB_ERR_INVALID outside, where the reference logs an error). */
int cphb_occgrid_add_voxels(cphb_occgrid *grid, const int32_t *voxels, size_t n, int occupied, void *stream);
int cphb_occgrid_add_voxel(cphb_occgrid *grid, const int32_t voxel[3], int occupied, void *stream);
/* SetFreeArea(min_bound, max_bound) (:415-460): adds prob_miss_log to every cell of the (clipped) box and REPLACES the
 * grid's bound box by it, as the reference does. */
int cphb_occgrid_set_free_area(cphb_occgrid *grid, const float min_bound[3], const float max_bound[3], void *stream);
/* min_bound_ / max_bound_ (grid indices; GetMinBound / GetMaxBound :317-333 convert them to coordinates) */
int cphb_occgrid_bounds(const cphb_occgrid *grid, int32_t h_min[3], int32_t h_max[3], void *stream);
/* ExtractKnownVoxels / ExtractFreeVoxels / ExtractOccupiedVoxels (:358-408): which = 0 / 1 / 2.  Voxels of the bound
 * box that satisfy the predicate, in box order; out_index (device [capacity][3], the voxel's stored grid_index_) and
 * out_prob (device [capacity]) may be null; *h_count = number of matching voxels (call with capacity 0 to size). */
int cphb_occgrid_extract(const cphb_occgrid *grid, int which, int32_t *out_index, float *out_prob, size_t capacity,
                         size_t *h_count, void *stream);
/* GetVoxel(point) (:351-356, densegrid.inl:137-146): *h_known = inside the grid and not NaN */
int cphb_occgrid_get_voxel(const cphb_occgrid *grid, const float point[3], int *h_known, float *h_prob_log,
                           int32_t h_grid_index[3], void *stream);
/* the five probability parameters cphb_occgrid_set_params last set (the defaults before that) */
int cphb_occgrid_get_params(const cphb_occgrid *grid, cphb_occgrid_params *p);

/* ------------------------------------------------------------------------ *
 * geometry::VoxelGrid operations (voxelgrid.cu, voxelgrid_factory.cu).  A grid is
 * keys [n][3] int32 + colors [n][3] float32 (device) with voxel_size and origin.
 * CreateDense, merge and carving leave keys lexicographically sorted and unique
 * when their inputs are; every lookup also accepts unsorted, repeated keys.
 * Lookups and merges need a key span below 2^21 on each axis (CPHB_ERR_INVALID).
 * ------------------------------------------------------------------------ */
/* VoxelGrid::CreateDense (voxelgrid_factory.cu:134-162): counts int(roundf(extent / voxel_size)) per axis, keys
 * (w, h, d) in lexicographic order, every colour (1, 1, 1).  *h_n = the voxel count; the keys and colours are written
 * only when capacity >= it (call with capacity 0 to size).  voxel_size <= 0 or non-finite, a negative, non-finite or
 * >= 2^31 count, or a total whose keys and colours do not fit a size_t byte count: CPHB_ERR_INVALID. */
int cphb_voxel_grid_create_dense(float voxel_size, float width, float height, float depth, int32_t *out_keys,
                                 float *out_colors, size_t capacity, size_t *h_n, void *stream);
/* VoxelGrid::CheckIfIncluded (voxelgrid.cu:365-376): out[i] = 1 when the cell floor((q_i - origin) / voxel_size) of
 * query i is one of the keys.  Non-finite queries and cells outside the int range give 0.  queries [nq][3] float32,
 * out [nq] uint8 (device).  Synchronises. */
int cphb_voxel_grid_check_if_included(const int32_t *keys, size_t n, float voxel_size, const float h_origin[3],
                                      const float *queries, size_t nq, uint8_t *out, void *stream);
/* whether key h_key is one of the keys (GetVoxelCenterCoordinate's find, voxelgrid.cu:343-354).  Synchronises. */
int cphb_voxel_grid_has_key(const int32_t *keys, size_t n, const int32_t h_key[3], int *h_found, void *stream);
/* VoxelGrid::CarveDepthMap / CarveSilhouette (voxelgrid.cu:45-123,378-430): a voxel is kept when one of its 8
 * corners projects, through h_extrinsic (4x4 row-major) and h_intrinsic (3x3 row-major), inside the image with
 * sampled value d > 0 and z >= d, or outside the image while keep_outside is set.  Only a 1-channel float32 image is
 * sampled (bilinear, FloatValueAt of image.h:240-270); any other kind is outside everywhere, and image may then be
 * NULL.  A corner with z == 0 or a non-finite u or v is outside.  The survivors keep their order in out_keys /
 * out_colors (n rows); *h_n_out = their number (synchronises).  width or height < 2: CPHB_ERR_INVALID. */
int cphb_voxel_grid_carve(const int32_t *keys, const float *colors, size_t n, float voxel_size, const float h_origin[3],
                          const void *image, int width, int height, int num_of_channels, int bytes_per_channel,
                          const float h_intrinsic[9], const float h_extrinsic[16], int keep_outside, int32_t *out_keys,
                          float *out_colors, size_t *h_n_out, void *stream);
/* VoxelGrid::operator+= (average = 1, voxelgrid.cu:235-286) and AddVoxels (average = 0, :288-319): a's voxels then
 * b's, stable-sorted by key; each run of equal keys becomes one voxel whose colour is the run's colours summed left to
 * right in float and divided by the run length (average = 1), or the run's first colour (average = 0).  Outputs hold
 * na + nb rows; *h_n_out = the voxel count (synchronises).  na + nb > 2^31-1: CPHB_ERR_INVALID. */
int cphb_voxel_grid_merge(const int32_t *keys_a, const float *colors_a, size_t na, const int32_t *keys_b,
                          const float *colors_b, size_t nb, int average, int32_t *out_keys, float *out_colors,
                          size_t *h_n_out, void *stream);
/* PaintUniformColor (indices NULL) and PaintIndexedColor (voxelgrid.cu:321-336): colors[i] = h_color for every i, or
 * for every i in indices [m] int64.  An index outside [0, n) is CPHB_ERR_INVALID and nothing is painted. */
int cphb_voxel_grid_paint(float *colors, size_t n, const int64_t *indices, size_t m, const float h_color[3], void *stream);
/* VoxelGrid::SelectByIndex (voxelgrid.cu:432-475): invert = 0: out row t = row indices[t] (m rows); invert = 1: the
 * rows not among indices, ascending (repeated indices are allowed).  An index outside [0, n) is CPHB_ERR_INVALID.
 * Outputs hold m (invert = 0) or n (invert = 1) rows; *h_n_out = rows written (synchronises). */
int cphb_voxel_grid_select_by_index(const int32_t *keys, const float *colors, size_t n, const int64_t *indices, size_t m,
                                    int invert, int32_t *out_keys, float *out_colors, size_t *h_n_out, void *stream);
/* VoxelGrid::CreateFromOccupancyGrid (voxelgrid_factory.cu:283-305): keys = the occupied cells' grid indices in
 * ExtractOccupiedVoxels order, colours (0, 0, 1); h_origin = grid origin - (resolution / 2) * voxel_size, so every
 * voxel covers the cell it came from.  PointCloud::CreateFromOccupancyGrid (pointcloud_factory.cu:239-256,418-430):
 * point = (cell + (float)(-(resolution / 2) + 0.5)) * voxel_size + origin, colour (0, 0, 1).  *h_count = the occupied
 * count; rows are written only when capacity >= it (capacity 0 sizes).  Synchronises. */
int cphb_voxel_grid_from_occgrid(const cphb_occgrid *grid, int32_t *out_keys, float *out_colors, size_t capacity,
                                 size_t *h_count, float h_origin[3], void *stream);
/* VoxelGrid::CreateFromTriangleMeshWithinBounds (voxelgrid_factory.cu:229-272, DESIGN section 4 item 25): origin =
 * h_min_bound, n_a = int(roundf((max_a - min_a) / voxel_size)) cells per axis.  Key k (0 <= k_a < n_a) is a voxel when
 * Akenine-Moeller's triangle/box overlap test, in IEEE float32, says some triangle meets the closed cell of centre
 * ((float)k + 0.5f) * voxel_size + origin and half size 0.5f * voxel_size.  A triangle with a non-finite vertex
 * meets no cell.  Keys are unique and in lexicographic order, colours (1, 1, 1).  vertices [n_vertices][3] float32,
 * triangles [n_triangles][3] int32 (device).  *h_n = the voxel count; keys and colours are written only when capacity
 * >= it (capacity 0 sizes; the sizing call does the same work).  A vertex index outside [0, n_vertices), a voxel size
 * that is not positive and finite, non-finite bounds, or a count that is negative or >= 2^21 on an axis:
 * CPHB_ERR_INVALID.  Synchronises. */
int cphb_voxel_grid_from_triangle_mesh(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                       float voxel_size, const float h_min_bound[3], const float h_max_bound[3], int32_t *out_keys,
                                       float *out_colors, size_t capacity, size_t *h_n, void *stream);
int cphb_point_cloud_from_occgrid(const cphb_occgrid *grid, float *out_points, float *out_colors, size_t capacity,
                                  size_t *h_count, void *stream);

/* ------------------------------------------------------------------------ *
 * geometry::DistanceTransform (distancetransform.h, distancetransform.cu): a
 * dense resolution^3 grid, cell (x, y, z) at linear index (x * res + y) * res + z
 * and centred on origin like the OccupancyGrid.  Each cell holds its nearest
 * site and the distance to it: nearest is u32 x << 20 | y << 10 | z with bit 30
 * = DistanceVoxel::NotSite, distance is float32 |nearest - cell| * voxel_size.
 * Among equidistant sites the lexicographically smallest (x, y, z) is taken.  A
 * fresh grid, and every cell Reconstruct adds, is nearest (0,0,0), NotSite,
 * distance 0.  1 <= resolution <= 1024, else CPHB_ERR_INVALID.  The compute
 * calls are stream-ordered (no host synchronisation) and start from an empty
 * site set: a clear, a stamp and three sweeps, whatever the resolution.
 * ------------------------------------------------------------------------ */
typedef struct cphb_dt cphb_dt;
/* DistanceTransform(voxel_size, resolution = 512, origin = 0) (distancetransform.cu:293-301) */
int cphb_dt_create(float voxel_size, int resolution, const float origin[3], void *stream, cphb_dt **out);
void cphb_dt_destroy(cphb_dt *dt);
/* Reconstruct (densegrid.inl:128-134): the linear prefix of the old cells is kept, distances are not rescaled */
int cphb_dt_reconstruct(cphb_dt *dt, float voxel_size, int resolution, void *stream);
int cphb_dt_set_geometry(cphb_dt *dt, float voxel_size, const float origin[3]); /* voxel_size_ / origin_ */
/* ComputeEDT (with_distance = 1) / ComputeVoronoiDiagram (0, every distance 0) of device [n][3] int32 grid indices;
 * indices outside the grid are ignored.  No site at all: every nearest is (0,0,0) with NotSite, its distance
 * |cell| * voxel_size (0 for the Voronoi diagram). */
int cphb_dt_compute_sites(cphb_dt *dt, const int32_t *cells, size_t n, int with_distance, void *stream);
/* the same from VoxelGrid keys (device [n][3] int32): cell = floor(((key * vs + vg_origin) - origin) / vs) + res / 2
 * with vs the transform's voxel size, each operation rounded on its own (distancetransform.cu:254-260).
 * |voxel_size - vg_voxel_size| > FLT_EPSILON: CPHB_ERR_INVALID and the grid is left unchanged. */
int cphb_dt_compute_voxel_grid(cphb_dt *dt, const int32_t *keys, size_t n, float vg_voxel_size, const float vg_origin[3],
                               int with_distance, void *stream);
/* CreateFromOccupancyGrid (distancetransform_factory.cu:40-62): a new transform with the grid's voxel size,
 * resolution and origin, and the EDT of its occupied cells (!isnan(p) && p > occ_prob_thres_log) */
int cphb_dt_from_occgrid(const cphb_occgrid *grid, void *stream, cphb_dt **out);
/* GetDistances (:421-435): out[i] = distance of cell floor(((q - origin) + (0.5 * vs) * res) / vs); 0 for a query
 * outside the grid or with a NaN coordinate.  points, out: device. */
int cphb_dt_get_distances(const cphb_dt *dt, const float *points, size_t n, float *out, void *stream);
/* GetVoxel (densegrid.inl:137-155): cell floor((point - origin) / vs) + res / 2.  Outside the grid or NaN:
 * *h_found = 0 and the default voxel.  h_state: 0, or 2 (NotSite).  Synchronises. */
int cphb_dt_get_voxel(const cphb_dt *dt, const float point[3], int *h_found, int32_t h_nearest[3], int *h_state,
                      float *h_distance, void *stream);
const float *cphb_dt_distance_data(const cphb_dt *dt);   /* device distance[res^3], borrowed */
const uint32_t *cphb_dt_nearest_data(const cphb_dt *dt); /* device nearest[res^3] (packed as above), borrowed */

/* ------------------------------------------------------------------------ *
 * integration::UniformTSDFVolume (integration/uniform_tsdfvolume.cu) and the RGB-D conversion it reads
 * (geometry/rgbdimage_factory.cu, image.cu, image_factory.cu).  A volume owns a dense resolution^3 grid on the device:
 * a float2 {tsdf, weight} plane and, by color_type (0 NoColor, 1 RGB8, 2 Gray32), 3, 1 or 0 float colour planes.
 * Voxel idx = x res^2 + y res + z; its centre is origin + vl (k - res / 2) + vl / 2, vl = length / resolution.
 * Images and outputs are device buffers, borrowed; the outputs are caller-allocated.  Matrices are row-major:
 * the 3x3 intrinsic [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] and the 4x4 world-to-camera extrinsic.
 * ------------------------------------------------------------------------ */
typedef struct cphb_tsdf cphb_tsdf;
/* CreateFromColorAndDepth's image conversion, [height * width] float32 out.  to_depth: ConvertDepthToFloatImage of a
 * 1-channel image -- raw value (x 1/255 for 8-bit) / (float)(int)depth_scale, 0 where it is >= (float)(int)depth_trunc;
 * depth_scale < 1 (which truncates to 0) or a non-finite one is CPHB_ERR_INVALID.  Otherwise CreateFloatImage(WEIGHTED)
 * of a 1- or 3-channel image (x 1/255 for 8-bit).  bytes_per_channel 1, 2 or 4 (uint8, uint16, float32).  Asynchronous. */
int cphb_rgbd_convert(const void *src, int width, int height, int channels, int bytes_per_channel, int to_depth, float depth_scale,
                      float depth_trunc, float *out, void *stream);
/* UniformTSDFVolume(length, resolution, sdf_trunc, color_type, origin): every voxel tsdf 0, weight 0, colour (1, 1, 1).
 * resolution outside [2, 1290] (the voxel count must fit int32), a length or sdf_trunc that is not positive and finite,
 * or an unknown color_type: CPHB_ERR_INVALID.  origin may be NULL (zero). */
int cphb_tsdf_create(float length, int resolution, float sdf_trunc, int color_type, const float origin[3], void *stream,
                     cphb_tsdf **out);
void cphb_tsdf_destroy(cphb_tsdf *volume);
/* Reset: every voxel back to the initial state (the reference empties the grid instead).  Asynchronous. */
int cphb_tsdf_reset(cphb_tsdf *volume, void *stream);
/* borrowed device planes: tw [res^3][2] float32 (tsdf, weight), col [planes][res^3] float32 (NULL for NoColor) */
int cphb_tsdf_data(const cphb_tsdf *volume, float **tw, float **col);
/* Integrate(RGBDImage, intrinsic, extrinsic) (uniform_tsdfvolume.cu:670-701, integrate_functor.h:84-139).  depth:
 * 1-channel float32 metres; color: uint8 RGB for RGB8, 1-channel float32 for Gray32, unread (may be NULL) for
 * NoColor.  The reference's format checks -- and the depth and colour sizes against the intrinsic's width x height --
 * fail with CPHB_ERR_INVALID.  Asynchronous. */
int cphb_tsdf_integrate(cphb_tsdf *volume, const float *depth, int depth_width, int depth_height, int depth_channels,
                        int depth_bytes_per_channel, const void *color, int color_width, int color_height, int color_channels,
                        int color_bytes_per_channel, int width, int height, const float h_intrinsic[9], const float h_extrinsic[16],
                        void *stream);
/* ExtractPointCloud (uniform_tsdfvolume.cu:85-156, 703-737): one row per zero crossing between interior band voxels,
 * in (x, y, z, axis) order; points, normals and (unless NoColor) colours [count][3].  *h_count = the number of rows;
 * they are written only when capacity >= it (capacity 0 sizes).  Synchronises. */
int cphb_tsdf_extract_points(const cphb_tsdf *volume, float *points, float *normals, float *colors, size_t capacity, size_t *h_count,
                             void *stream);
/* ExtractVoxelPointCloud / ExtractVoxelGrid (uniform_tsdfvolume.cu:352-408, 840-895): the band voxels in index order;
 * keys [count][3] int32 grid indices and points [count][3] voxel centres (either may be NULL), colours
 * [count][3] = (tsdf + 1) / 2.  Sizing as cphb_tsdf_extract_points.  Synchronises. */
int cphb_tsdf_extract_voxels(const cphb_tsdf *volume, int32_t *keys, float *points, float *colors, size_t capacity, size_t *h_count,
                             void *stream);
/* Raycast(intrinsic, extrinsic, sdf_trunc, project_valid_depth_only) (uniform_tsdfvolume.cu:509-639, 924-951): one ray
 * per pixel of the width x height image, entering the grid where the ray meets the box of cells [0, res - 1).  Points, normals and colours
 * [rows][3]; capacity must be >= width * height.  project_valid_depth_only: only the hit rows, in pixel order; otherwise
 * every pixel's row, NaN for a miss.  *h_count = rows written.  sdf_trunc not positive and finite: CPHB_ERR_INVALID.
 * Synchronises. */
int cphb_tsdf_raycast(const cphb_tsdf *volume, int width, int height, const float h_intrinsic[9], const float h_extrinsic[16],
                      float sdf_trunc, int project_valid_depth_only, float *points, float *normals, float *colors, size_t capacity,
                      size_t *h_count, void *stream);
/* ExtractTriangleMesh: welded marching cubes (DESIGN section 4 item 19).  One vertex per crossed grid edge of a valid
 * cube (all 8 corner weights nonzero), in (x, y, z, axis) order of the edge's origin voxel: vertices [n_vertices][3]
 * and, unless NoColor, colours [n_vertices][3]; triangles [n_triangles][3] int32 vertex indices, cube by cube in cube
 * index order, then table order, oriented so that (v1 - v0) x (v2 - v0) points from negative to positive tsdf.
 * *h_n_vertices / *h_n_triangles are the counts; the rows are written only when both capacities hold them (0 sizes).
 * A vertex count past INT32_MAX is CPHB_ERR_INVALID.  Synchronises. */
int cphb_tsdf_extract_mesh(const cphb_tsdf *volume, float *vertices, float *colors, int32_t *triangles, size_t vertex_capacity,
                           size_t triangle_capacity, size_t *h_n_vertices, size_t *h_n_triangles, void *stream);

/* ------------------------------------------------------------------------ *
 * integration::ScalableTSDFVolume (integration/scalable_tsdfvolume.cu): 16^3-voxel units allocated on demand near
 * observed surfaces.  Unit key floor(p / U), U = voxel_length * 16, each axis in [-2^20, 2^20).  Voxel (x, y, z) of the
 * unit with key k has the centre fma(vl, (x, y, z), vl / 2) + k * U and index x * 256 + y * 16 + z in its slot.  Units
 * are kept in slots in the order the frames first touched them, ascending key within a frame (the packed key: each
 * axis + 2^20 in 21 bits, x highest); the extractions go in slot order, voxel index, axis.  map_size is the pool's
 * first capacity, which doubles as needed.  Conventions as cphb_tsdf_*.
 * ------------------------------------------------------------------------ */
typedef struct cphb_stsdf cphb_stsdf;
/* ScalableTSDFVolume(voxel_length, sdf_trunc, color_type, depth_sampling_stride, map_size).  A voxel_length or
 * sdf_trunc that is not positive and finite, sdf_trunc over 64 units, an unknown color_type, a stride or map_size
 * below 1: CPHB_ERR_INVALID. */
int cphb_stsdf_create(float voxel_length, float sdf_trunc, int color_type, int depth_sampling_stride, int map_size, void *stream,
                      cphb_stsdf **out);
void cphb_stsdf_destroy(cphb_stsdf *volume);
/* Reset: no unit allocated.  Asynchronous. */
int cphb_stsdf_reset(cphb_stsdf *volume, void *stream);
/* Integrate(RGBDImage, intrinsic, extrinsic): the units within sdf_trunc of the frame's strided depth points
 * (cphb_depth_to_points' projection, every depth_sampling_stride-th pixel) are allocated, then every allocated voxel
 * is updated as cphb_tsdf_integrate updates a voxel.  The image rules of cphb_tsdf_integrate; a singular extrinsic, a
 * unit key out of range or more than 524287 units (the voxel count must fit int32) is CPHB_ERR_INVALID, and a failed
 * allocation CPHB_ERR_CUDA; a call that fails leaves the volume as it was.  Synchronises. */
int cphb_stsdf_integrate(cphb_stsdf *volume, const float *depth, int depth_width, int depth_height, int depth_channels,
                         int depth_bytes_per_channel, const void *color, int color_width, int color_height, int color_channels,
                         int color_bytes_per_channel, int width, int height, const float h_intrinsic[9], const float h_extrinsic[16],
                         void *stream);
/* ExtractPointCloud: one row per zero crossing between a band voxel and its +1 neighbour on an axis (across unit
 * faces; a missing unit counts as weight 0); points, normals (GetNormalAt) and, unless NoColor, colours.  Sizing as
 * cphb_tsdf_extract_points.  Synchronises. */
int cphb_stsdf_extract_points(const cphb_stsdf *volume, float *points, float *normals, float *colors, size_t capacity, size_t *h_count,
                              void *stream);
/* ExtractVoxelPointCloud: every band voxel's centre, colour (tsdf + 1) / 2.  Sizing as above.  Synchronises. */
int cphb_stsdf_extract_voxels(const cphb_stsdf *volume, float *points, float *colors, size_t capacity, size_t *h_count, void *stream);
/* borrowed device state: the unit count, keys [units] packed, tw [units][4096][2] float32 and col
 * [units][planes][4096] float32 (NULL for NoColor) */
int cphb_stsdf_data(const cphb_stsdf *volume, size_t *h_units, uint64_t **keys, float **tw, float **col);
/* the unit count, the pool's capacity in units and the device bytes of the pool and its table */
int cphb_stsdf_info(const cphb_stsdf *volume, size_t *h_units, size_t *h_capacity, size_t *h_device_bytes);

/* ------------------------------------------------------------------------ *
 * TriangleMesh normals, edge list, filters, area and sampling (geometry/trianglemesh.cu), on device arrays: vertices
 * [n_vertices][3] float32, triangles [n_triangles][3] int32.  A vertex index outside [0, n_vertices) is
 * CPHB_ERR_INVALID.  Synchronise.
 * ------------------------------------------------------------------------ */
/* ComputeTriangleNormals: (v1 - v0) x (v2 - v0) per triangle, normalised (NormalizeNormals' rule) when asked */
int cphb_mesh_triangle_normals(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles, int normalized,
                               float *triangle_normals, void *stream);
/* ComputeVertexNormals' sum: vertex v's normal is the sum of its triangles' normals in ascending (triangle, corner)
 * order, normalised when asked; a vertex in no triangle gets 0, so the rows stay aligned with the vertices */
int cphb_mesh_vertex_normals(const int32_t *triangles, size_t n_triangles, const float *triangle_normals, size_t n_vertices,
                             int normalized, float *vertex_normals, void *stream);
/* ComputeEdgeList: the 6 directed edges (a, b), (b, a) of every triangle edge, sorted lexicographically and unique, as
 * edges [n_edges][2] int32 (a triangle with a repeated vertex gives the self-edge (a, a)).  *h_n_edges is the count; the
 * rows are written only when capacity >= it (capacity 0 sizes; 6 n_triangles always holds them).  More than 2^31 - 1
 * directed edges (6 n_triangles) or vertices is CPHB_ERR_INVALID. */
int cphb_mesh_edge_list(const int32_t *triangles, size_t n_triangles, size_t n_vertices, int32_t *edges, size_t capacity,
                        size_t *h_n_edges, void *stream);
/* FilterSharpen / FilterSmoothSimple / FilterSmoothLaplacian / FilterSmoothTaubin over a sorted edge list (as
 * cphb_mesh_edge_list gives it; an index outside [0, n_vertices) or a pair out of order is CPHB_ERR_INVALID).  Each
 * attribute given (vertices, normals, colours [n_vertices][3], NULL when absent) is filtered into its output when its
 * bit is set in filter_mask (1 vertices, 2 normals, 4 colours) and number_of_iterations > 0, and copied to it otherwise.
 * Per pass, vertex v with N > 0 neighbours nb (its row of the edge list, summed left to right):
 *   Sharpen   prv + strength * (prv * N - sum(prev[nb]))
 *   Simple    (prv + sum(prev[nb])) / (float)(1.0 + N)
 *   Laplacian prv + lambda * (sum(w * prev[nb]) / sum(w) - prv),  w = (float)(1.0 / (|v - nb| + 1e-12)) from the input
 *   Taubin    Laplacian with lambda, then with mu, per iteration
 * and a vertex without neighbours keeps its value.  strength_or_lambda is the strength (Sharpen) or lambda; mu is read by
 * Taubin only.  Outputs must not alias inputs. */
#define CPHB_MESH_SHARPEN 0
#define CPHB_MESH_SIMPLE 1
#define CPHB_MESH_LAPLACIAN 2
#define CPHB_MESH_TAUBIN 3
int cphb_mesh_filter(int kind, int number_of_iterations, float strength_or_lambda, float mu, const int32_t *edges, size_t n_edges,
                     size_t n_vertices, const float *vertices, const float *normals, const float *colors, int filter_mask,
                     float *out_vertices, float *out_normals, float *out_colors, void *stream);
/* GetSurfaceArea: per triangle 0.5 |(p0 - p1) x (p0 - p2)| in float32, written to triangle_areas [n_triangles] when it
 * is not NULL; *h_area = their float64 sum in the fixed order of the engine's reductions, rounded to float32. */
int cphb_mesh_surface_area(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                           float *triangle_areas, float *h_area, void *stream);
/* SamplePointsUniformly: exactly number_of_points points [n][3]; triangle i gets the points [b_i, b_i+1) with
 * b_i+1 = llrint(cdf_i n) from a fixed-order float64 scan of the triangle areas (b_0 = 0, the last = n).  Point p uses
 * draws 2p + 1 and 2p + 2 of thrust::default_random_engine with its default seed, mapped by
 * uniform_real_distribution<float>(0, 1): a = 1 - sqrt(r1), b = sqrt(r1) (1 - r2), c = sqrt(r1) r2.  normals (may be
 * NULL): triangle_normals[i] when triangle_normals is given, else the interpolated vertex_normals; colors (may be NULL):
 * the interpolated vertex_colors.  number_of_points 0 or above CPHB_MESH_MAX_SAMPLES (the draws must stay inside the
 * generator's period 2^31 - 2), no triangles, a bad index, or a total area that is not positive and finite is
 * CPHB_ERR_INVALID. */
#define CPHB_MESH_MAX_SAMPLES 1073741823u
int cphb_mesh_sample_points_uniformly(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                      const float *vertex_normals, const float *triangle_normals, const float *vertex_colors,
                                      size_t number_of_points, float *points, float *normals, float *colors, void *stream);

/* ------------------------------------------------------------------------ *
 * TriangleMesh cleanup, operator+= and GetSelfIntersectingTriangles (geometry/trianglemesh.cu:903-1141, DESIGN section 4
 * item 26), on device arrays.  Every entry first checks each vertex index against [0, n_vertices) (CPHB_ERR_INVALID
 * when one is outside) and rejects more than 2^31 - 1 vertices or triangles.  Outputs are separate buffers as large as
 * the inputs; optional attributes (normals, colours, triangle normals) are NULL when absent.  Synchronise.
 * ------------------------------------------------------------------------ */
/* RemoveDuplicatedVertices: the distinct positions (IEEE ==, so -0 == +0) in lexicographic (x, y, z) order, each with
 * the attributes of its lowest original index; a vertex with a NaN coordinate merges with nothing and goes after the
 * others, in original order.  Triangles are remapped (order kept).  *h_n_vertices = the new count. */
int cphb_mesh_remove_duplicated_vertices(const float *vertices, const float *vertex_normals, const float *vertex_colors, size_t n_vertices,
                                         const int32_t *triangles, size_t n_triangles, float *out_vertices, float *out_normals,
                                         float *out_colors, int32_t *out_triangles, size_t *h_n_vertices, void *stream);
/* RemoveDuplicatedTriangles: each triangle rotated so its smallest index is first (orientation kept), sorted
 * lexicographically (stable) and the first of each run kept, with its triangle normal.  *h_n_triangles = the count. */
int cphb_mesh_remove_duplicated_triangles(const int32_t *triangles, const float *triangle_normals, size_t n_triangles, size_t n_vertices,
                                          int32_t *out_triangles, float *out_triangle_normals, size_t *h_n_triangles, void *stream);
/* RemoveUnreferencedVertices: stable compaction of the vertices some triangle references (with their normals and
 * colours); triangles are remapped.  *h_n_vertices = the count. */
int cphb_mesh_remove_unreferenced_vertices(const float *vertices, const float *vertex_normals, const float *vertex_colors, size_t n_vertices,
                                           const int32_t *triangles, size_t n_triangles, float *out_vertices, float *out_normals,
                                           float *out_colors, int32_t *out_triangles, size_t *h_n_vertices, void *stream);
/* RemoveDegenerateTriangles: stable compaction of the triangles with three distinct indices, with their normals.
 * *h_n_triangles = the count. */
int cphb_mesh_remove_degenerate_triangles(const int32_t *triangles, const float *triangle_normals, size_t n_triangles, size_t n_vertices,
                                          int32_t *out_triangles, float *out_triangle_normals, size_t *h_n_triangles, void *stream);
/* operator+='s triangles: out [n_triangles_a + n_triangles_b][3] = a, then b shifted by n_vertices_a */
int cphb_mesh_append_triangles(const int32_t *triangles_a, size_t n_triangles_a, size_t n_vertices_a, const int32_t *triangles_b,
                               size_t n_triangles_b, size_t n_vertices_b, int32_t *out_triangles, void *stream);
/* GetSelfIntersectingTriangles: every pair (i, j), i < j, of triangles that share no vertex index, whose vertices are
 * all finite, whose closed float32 boxes overlap, and which the reference's TriangleTriangle3d (mean / sigma
 * normalisation, then Moller's NoDivTriTriIsect with its epsilon test) says intersect; pairs [n][2] int32 in ascending
 * (i, j) order.  *h_n_pairs is the count; the pairs are written only when capacity >= it (capacity 0 sizes).
 * *h_n_candidates (may be NULL) = the box-overlapping pairs the predicate was evaluated on.  Memory grows with the
 * triangles, the grid's candidate pairs (the pairs of triangles sharing a grid cell) and the hits; the candidate pairs
 * reach n_triangles^2 / 2 only when every triangle falls into one cell (DESIGN section 4 item 26). */
int cphb_mesh_self_intersecting_triangles(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                          int32_t *pairs, size_t capacity, size_t *h_n_pairs, size_t *h_n_candidates, void *stream);

/* ------------------------------------------------------------------------ *
 * PointCloud::CreateFromDepthImage / CreateFromRGBDImage (geometry/pointcloud_factory.cu:43-200, 329-373).  Images are
 * device buffers, row-major; outputs are caller-allocated device [rows][3] float32.
 * ------------------------------------------------------------------------ */
/* The point of every stride-th pixel of every stride-th row, (width / stride) x (height / stride) samples in pixel
 * order.  depth: 1 channel, uint16 (bytes 2: raw / (float)(int)depth_scale, 0 where that is >= (float)(int)depth_trunc,
 * as cphb_rgbd_convert's to_depth) or float32 metres (bytes 4, taken as it is; depth_scale and depth_trunc unread).
 * A sample has a point when d > 0, d < depth_cutoff if depth_cutoff > 0, and the point is finite:
 * x = ((col - cx) d) / fx, y = ((row - cy) d) / fy, z = d, moved by the camera pose extrinsic^-1 (inverted in float64,
 * rounded to float32; extrinsic row-major world-to-camera).  color (may be NULL): uint8 RGB (colour c / 255) or 1-channel
 * float32 (grey g as (g, g, g)), the depth's size.  compute_normals: the structured normal of a sample from its
 * left / right / up / down neighbouring samples ((left - right) x (up - down), a neighbour without a point counting as
 * zero, normalised and turned to z <= 0); a sample on a border row or column, or with a zero cross product, gets 0.
 * project_valid_depth_only: only the samples with a point, in pixel order; otherwise one row per sample, NaN in
 * every attribute where there is no point.  *h_count = the number of rows; they are written only when capacity >= it
 * (capacity 0 sizes).  CPHB_ERR_INVALID: an unsupported image format, images of different sizes, stride < 1, a NaN
 * depth_cutoff, a depth_scale / depth_trunc outside cphb_rgbd_convert's range for uint16 depth, a singular extrinsic.
 * Synchronises. */
int cphb_depth_to_points(const void *depth, int width, int height, int depth_channels, int depth_bytes_per_channel, float depth_scale,
                         float depth_trunc, int stride, const void *color, int color_width, int color_height, int color_channels,
                         int color_bytes_per_channel, const float h_intrinsic[9], const float h_extrinsic[16], float depth_cutoff,
                         int compute_normals, int project_valid_depth_only, float *points, float *normals, float *colors,
                         size_t capacity, size_t *h_count, void *stream);

/* ------------------------------------------------------------------------ *
 * collision::ComputeIntersection (collision.h:36-160, collision.cu:1137-1231)
 * between VoxelGrids, OccupancyGrids and primitives.  Every grid element is an
 * integer key k with the box [k * vs + origin, (k + 1) * vs + origin]: a
 * VoxelGrid key as stored, an OccupancyGrid cell (x, y, z) as k = (x, y, z) -
 * resolution / 2.  An OccupancyGrid's elements are its occupied cells
 * (!isnan(p) && p > occ_prob_thres_log, inside its bound box, as
 * cphb_occgrid_extract(which = 2) lists them: ascending linear index) and an
 * element's index is its linear cell index x * res^2 + y * res + z.
 * ------------------------------------------------------------------------ */
enum { /* collision::Primitive::PrimitiveType */
    CPHB_PRIM_UNSPECIFIED = 0,
    CPHB_PRIM_BOX = 1,
    CPHB_PRIM_SPHERE = 2,
    CPHB_PRIM_CAPSULE = 3,
    CPHB_PRIM_CYLINDER = 4 /* never collides (the reference's default branch) */
};
typedef struct cphb_primitive { /* primitives.h:30-160: Box, Sphere, Capsule, Cylinder */
    int32_t type;               /* CPHB_PRIM_* */
    float transform[16];        /* row-major 4x4; a Capsule's axis is its third column */
    float lengths[3];           /* Box */
    float radius;               /* Sphere, Capsule, Cylinder */
    float height;               /* Capsule, Cylinder */
} cphb_primitive;
enum { /* CollisionResult::CollisionType */
    CPHB_COLL_PRIMITIVES = 1,
    CPHB_COLL_VOXEL_GRID = 2,
    CPHB_COLL_OCCUPANCY_GRID = 3
};
typedef struct cphb_coll_operand {
    int32_t kind;                      /* CPHB_COLL_* */
    const int32_t *keys;               /* VOXEL_GRID: device [n][3] voxels_keys_ (any order, duplicates allowed) */
    size_t n;                          /* VOXEL_GRID: keys; PRIMITIVES: primitives */
    float voxel_size, origin[3];       /* VOXEL_GRID */
    const cphb_occgrid *occ;           /* OCCUPANCY_GRID (its own voxel size, origin and threshold) */
    const cphb_primitive *primitives;  /* PRIMITIVES: device [n] */
} cphb_coll_operand;
/* ComputeIntersection(a, b, margin): a is the target, b the query.  Every query element that collides with some
 * target element gives one pair (smallest colliding index in a, index in b), in ascending query order, written to
 * pairs_out (device [capacity][2] int32); *h_count = the number of pairs (capacity 0 sizes the output).  Grid
 * against grid: the query box widened by margin overlaps the target box (inclusive).  Primitive against grid element
 * (centre (k + 0.5) * vs + origin, half size vs / 2): Box = separating axes with margin added to the half size,
 * Sphere and Capsule with radius + margin.  An empty operand gives no pairs.  CPHB_ERR_INVALID: a pair the reference
 * does not offer (OccupancyGrid x OccupancyGrid, primitives x primitives), a non-finite margin, a VoxelGrid with keys
 * or any OccupancyGrid whose voxel size is not positive and finite, or VoxelGrid target keys spanning 2^21 or more
 * on an axis.  Synchronises. */
int cphb_compute_intersection(const cphb_coll_operand *a, const cphb_coll_operand *b, float margin, int32_t *pairs_out,
                              size_t capacity, size_t *h_count, void *stream);

/* registration::EvaluateRegistration (registration.cu:106-119). */
int cphb_evaluate_registration(const cphb_cloud *source, const cphb_cloud *target,
                               float max_correspondence_distance, const float h_T[16],
                               cphb_icp_result *h_result, int32_t *corr_out, void *stream);

/* ------------------------------------------------------------------------ *
 * Host-buffer convenience used by bench.py's e2e leg and the Python mirror:
 * thin wrappers that cudaMalloc/cudaMemcpyAsync around the calls above.
 * ------------------------------------------------------------------------ */
/* utility::InitializeAllocator(PoolAllocation, initial_pool_size, ...) (device_vector.cu:28-69): pre-reserve
 * physical memory in the stream-ordered pool that every allocation of this library comes from, so that no call
 * on the hot path ever has to grow the pool (a growth step costs tens of milliseconds). */
int cphb_reserve_pool(size_t bytes);
void *cphb_malloc(size_t bytes);              /* pool allocation on the default stream, NULL on failure */
void cphb_free(void *p);
void *cphb_malloc_host(size_t bytes);         /* pinned */
void cphb_free_host(void *p);
int cphb_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
int cphb_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream);
int cphb_memset(void *dst, int value, size_t bytes, void *stream);
int cphb_stream_synchronize(void *stream);
int cphb_memcpy_d2d(void *dst, const void *src, size_t bytes, void *stream);
/* CUDA events on `stream` (bench.py times the hot path on the device, not by wall clock) */
void *cphb_event_create(void);
void cphb_event_destroy(void *event);
int cphb_event_record(void *event, void *stream);
int cphb_event_elapsed_ms(void *start, void *stop, float *h_ms); /* synchronises on stop */
/* ------------------------------------------------------------------------ *
 * Multi-GPU communicator (one process per GPU, one node).  Two kinds:
 *  NCCL: rank 0 calls cphb_nccl_unique_id, the 128 bytes reach every rank by any means
 *        (torch.distributed broadcast, MPI, a file), every rank calls cphb_comm_nccl_create.
 *  P2P : every rank calls cphb_comm_p2p_create (allocates a mailbox in its HBM and returns a 64-byte
 *        CUDA IPC handle), the handles are all-gathered in rank order by any means, every rank calls
 *        cphb_comm_p2p_connect.  The per-iteration exchange is then fused into the ICP reduce kernel:
 *        NVLink stores into the peers' mailboxes + flags, no collective library on the path.
 * ------------------------------------------------------------------------ */
int cphb_nccl_unique_id(char h_id[128]);
int cphb_comm_nccl_create(const char h_id[128], int world_size, int rank, cphb_comm **out);
int cphb_comm_p2p_create(int world_size, int rank, char h_handle[64], cphb_comm **out);
int cphb_comm_p2p_connect(cphb_comm *comm, const char *h_handles /* world_size * 64 bytes */);
int cphb_comm_destroy(cphb_comm *comm);
/* in-place sum over ranks of <= 32 doubles (device buffer); what the ICP loop uses, exposed for tests */
int cphb_comm_allreduce_f64(cphb_comm *comm, double *buf, int count, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CUPOCH_B200_H */
