// crop.cu -- region selection and point-cloud cleanup (SURVEY 8f rank 10):
//   AxisAlignedBoundingBox / OrientedBoundingBox::GetPointIndicesWithinBoundingBox   boundingvolume.cu:38-101,176-244,413-425
//   OrientedBoundingBox::CreateFromPoints                                            boundingvolume.cu:219-269
//   PointCloud::PassThroughFilter / RemoveNoneFinitePoints                           pointcloud.cu:36-53,105-121,359-385,436-460
//   PointCloud::UniformDownSample                                                    down_sample.cu:275-300
//   PointCloud::NormalizeNormals / OrientNormalsToAlignWithDirection                 pointcloud.cu:282-285, estimate_normals.cu:66-78,129-141
//
// Every region selection is one flag kernel (crop_flag_kernel<Predicate>: packed xyz staged through shared memory, one
// keep byte per point) followed by the shared stable compaction (cphb_compact_flags); the front ends gather the kept
// rows with cphb_select_by_index.  PassThroughFilter is the AABB predicate with +-inf on the other two axes.
//
// Arithmetic (DESIGN.md arithmetic contract; oracle/crop.c restates it):
//   OBB test_plane(a, b, c, x) = det[b - a | c - a | x - a], expanded along the first row in Eigen's order
//     u0 (v1 w2 - w1 v2) - v0 (u1 w2 - w1 u2) + w0 (u1 v2 - v1 u2), every minor a det2, then two FMAs;
//   OBB creation: mean and centred second moments summed in double over tiles of CROP_TILE consecutive points (each
//     tile sequentially from 0.0, then the tiles in order: the SegmentPlane order), a double symmetric eigensolve on the
//     host, then the reference's float32 transform (dot3 + t) and min/max bound;
//   normals: |n|^2 = dot3(n, n), n . ref = dot3(n, ref), IEEE sqrt and division.
#include <math.h>
#include <string.h>

#include "cphb_internal.cuh"

#define CROP_BLOCK 256
#define CROP_TILE 1024  // summation tile of the OBB moments (the SegmentPlane order)

// reduce.cu: one-sided Jacobi SVD in double, A = U diag(sv) V^T; for a symmetric positive semi-definite A the columns
// of V are its eigenvectors and sv its eigenvalues
void cphb_host_svd3(const double *A, double *U, double *sv, double *V);

// ---- predicates ---------------------------------------------------------------------------------------------------
// check_within_axis_aligned_bounding_box_functor (boundingvolume.cu:82-101): inclusive bounds; a NaN coordinate
// compares false both ways, so NaN points are kept.  pass_through_filter_functor (pointcloud.cu:105-121) is the same
// test with lo/hi on one axis and -inf/+inf on the others.
struct AabbPredicate {
    float lo[3], hi[3];
    __device__ __forceinline__ bool operator()(float x, float y, float z) const {
        return !(x < lo[0] || x > hi[0] || y < lo[1] || y > hi[1] || z < lo[2] || z > hi[2]);
    }
};

// check_within_oriented_bounding_box_functor (boundingvolume.cu:38-79): six plane tests over the box points, either
// sign pattern
__device__ __forceinline__ float obb_test_plane(const float *a, const float *b, const float *c, float x, float y, float z) {
    const float u0 = __fsub_rn(b[0], a[0]), u1 = __fsub_rn(b[1], a[1]), u2 = __fsub_rn(b[2], a[2]);
    const float v0 = __fsub_rn(c[0], a[0]), v1 = __fsub_rn(c[1], a[1]), v2 = __fsub_rn(c[2], a[2]);
    const float w0 = __fsub_rn(x, a[0]), w1 = __fsub_rn(y, a[1]), w2 = __fsub_rn(z, a[2]);
    const float m0 = det2(v1, w2, w1, v2), m1 = det2(u1, w2, w1, u2), m2 = det2(u1, v2, v1, u2);
    return __fmaf_rn(w0, m2, __fmaf_rn(-v0, m1, __fmul_rn(u0, m0)));
}
struct ObbPredicate {
    float b[8][3];
    __device__ __forceinline__ bool operator()(float x, float y, float z) const {
        const float d0 = obb_test_plane(b[0], b[1], b[3], x, y, z);
        const float d1 = obb_test_plane(b[0], b[5], b[3], x, y, z);
        const float d2 = obb_test_plane(b[2], b[5], b[7], x, y, z);
        const float d3 = obb_test_plane(b[1], b[4], b[7], x, y, z);
        const float d4 = obb_test_plane(b[3], b[4], b[5], x, y, z);
        const float d5 = obb_test_plane(b[0], b[1], b[7], x, y, z);
        return (d0 <= 0.f && d1 >= 0.f && d2 <= 0.f && d3 >= 0.f && d4 <= 0.f && d5 >= 0.f) ||
               (d0 >= 0.f && d1 <= 0.f && d2 >= 0.f && d3 <= 0.f && d4 >= 0.f && d5 <= 0.f);
    }
};

// check_nan_functor (pointcloud.cu:38-53), negated: keep what is not removed
struct FinitePredicate {
    int remove_nan, remove_infinite;
    __device__ __forceinline__ bool operator()(float x, float y, float z) const {
        const bool is_nan = remove_nan && (isnan(x) || isnan(y) || isnan(z));
        const bool is_inf = remove_infinite && (isinf(x) || isinf(y) || isinf(z));
        return !(is_nan || is_inf);
    }
};

// one keep byte per point; the block's 256 packed points are read as 768 consecutive floats
template <class P>
__global__ void __launch_bounds__(CROP_BLOCK) crop_flag_kernel(const float *__restrict__ pts, size_t n, P pred,
                                                               uint8_t *__restrict__ keep) {
    __shared__ float s_p[3 * CROP_BLOCK];
    const size_t base = blockIdx.x * (size_t)CROP_BLOCK;
    const int cnt = (int)min((size_t)CROP_BLOCK, n - base);
    for (int k = threadIdx.x; k < 3 * cnt; k += CROP_BLOCK) s_p[k] = pts[3 * base + k];
    __syncthreads();
    const int t = threadIdx.x;
    if (t < cnt) keep[base + t] = pred(s_p[3 * t], s_p[3 * t + 1], s_p[3 * t + 2]) ? 1 : 0;
}

template <class P>
static int point_indices(const float *points, size_t n, const P &pred, int32_t *indices_out, size_t *h_n_out,
                         cudaStream_t s, const char *who) {
    if (!h_n_out) {
        cphb_set_error("%s: null argument", who);
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    if (n == 0) return CPHB_OK;
    if (!points || !indices_out) {
        cphb_set_error("%s: null argument", who);
        return CPHB_ERR_INVALID;
    }
    if (n > 0x7fffffffull) {
        cphb_set_error("%s: n = %zu exceeds the int32 index range", who, n);
        return CPHB_ERR_INVALID;
    }
    cphb_scratch sc(s);
    uint8_t *keep = nullptr;
    int rc = sc.alloc(&keep, n);
    if (rc) return rc;
    CPHB_LAUNCH(crop_flag_kernel<P>, (unsigned)((n + CROP_BLOCK - 1) / CROP_BLOCK), CROP_BLOCK, 0, s, points, n, pred, keep);
    return cphb_compact_flags(keep, n, indices_out, h_n_out, s);  // synchronises
}

extern "C" int cphb_aabb_point_indices(const float *points, size_t n, const float h_min[3], const float h_max[3],
                                       int32_t *indices_out, size_t *h_n_out, void *stream) {
    if (!h_min || !h_max) {
        cphb_set_error("cphb_aabb_point_indices: null argument");
        return CPHB_ERR_INVALID;
    }
    AabbPredicate p;
    for (int a = 0; a < 3; ++a) { p.lo[a] = h_min[a]; p.hi[a] = h_max[a]; }
    return point_indices(points, n, p, indices_out, h_n_out, (cudaStream_t)stream, "cphb_aabb_point_indices");
}

extern "C" int cphb_obb_point_indices(const float *points, size_t n, const float h_box_points[24], int32_t *indices_out,
                                      size_t *h_n_out, void *stream) {
    if (!h_box_points) {
        cphb_set_error("cphb_obb_point_indices: null argument");
        return CPHB_ERR_INVALID;
    }
    ObbPredicate p;
    memcpy(p.b, h_box_points, sizeof(p.b));
    return point_indices(points, n, p, indices_out, h_n_out, (cudaStream_t)stream, "cphb_obb_point_indices");
}

extern "C" int cphb_finite_point_indices(const float *points, size_t n, int remove_nan, int remove_infinite,
                                         int32_t *indices_out, size_t *h_n_out, void *stream) {
    FinitePredicate p = {remove_nan ? 1 : 0, remove_infinite ? 1 : 0};
    return point_indices(points, n, p, indices_out, h_n_out, (cudaStream_t)stream, "cphb_finite_point_indices");
}

// ---- OrientedBoundingBox::CreateFromPoints --------------------------------------------------------------------------
// one block per tile: the tile's points are staged coalesced, then thread j sums component j sequentially in double.
// pass 0: the coordinates; pass 1: the six second moments of (double)p - mean, products and sums in double.
__global__ void __launch_bounds__(128) obb_moment_tile_kernel(const float *__restrict__ pts, size_t n, int pass,
                                                              const double *__restrict__ mean, double *__restrict__ partial) {
    __shared__ float s_p[3 * CROP_TILE];
    const size_t base = blockIdx.x * (size_t)CROP_TILE;
    const int cnt = (int)min((size_t)CROP_TILE, n - base);
    for (int k = threadIdx.x; k < 3 * cnt; k += blockDim.x) s_p[k] = pts[3 * base + k];
    __syncthreads();
    const int j = threadIdx.x;
    if (pass == 0) {
        if (j >= 3) return;
        double s = 0.0;
        for (int i = 0; i < cnt; ++i) s = __dadd_rn(s, (double)s_p[3 * i + j]);
        partial[6 * blockIdx.x + j] = s;
        return;
    }
    if (j >= 6) return;
    const int a = j < 3 ? 0 : (j < 5 ? 1 : 2), b = j < 3 ? j : (j < 5 ? j - 2 : 2);  // (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
    const double ma = mean[a], mb = mean[b];
    double s = 0.0;
    for (int i = 0; i < cnt; ++i)
        s = __dadd_rn(s, __dmul_rn(__dsub_rn((double)s_p[3 * i + a], ma), __dsub_rn((double)s_p[3 * i + b], mb)));
    partial[6 * blockIdx.x + j] = s;
}

// lane j adds component j over the tiles in order; pass 0 then turns the sums into the mean (out[0..2]), pass 1 writes
// the second-moment sums (out[3..8])
__global__ void __launch_bounds__(32) obb_moment_final_kernel(const double *__restrict__ partial, size_t n_tiles, size_t n,
                                                              int pass, double *out) {
    const int j = threadIdx.x;
    if (j >= (pass == 0 ? 3 : 6)) return;
    double s = 0.0;
#pragma unroll 16
    for (size_t t = 0; t < n_tiles; ++t) s = __dadd_rn(s, partial[6 * t + j]);  // unrolled: the loads overlap, the sum order stays
    if (pass == 0) out[j] = __ddiv_rn(s, (double)n);
    else out[3 + j] = s;
}

// host float32 dot with the device's operation order (dot3)
static float host_dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0));
}

extern "C" int cphb_oriented_bounding_box(const float *points, size_t n, float h_center[3], float h_R[9], float h_extent[3],
                                          void *stream) {
    if (!h_center || !h_R || !h_extent || (n && !points)) {
        cphb_set_error("cphb_oriented_bounding_box: null argument");
        return CPHB_ERR_INVALID;
    }
    for (int k = 0; k < 9; ++k) h_R[k] = (k % 4 == 0) ? 1.f : 0.f;
    for (int a = 0; a < 3; ++a) h_center[a] = h_extent[a] = 0.f;
    if (n == 0) return CPHB_OK;  // the reference divides by zero here; the zero box with R = I instead
    cudaStream_t s = (cudaStream_t)stream;
    const size_t n_tiles = (n + CROP_TILE - 1) / CROP_TILE;
    if (n_tiles > 0x7fffffffull) {
        cphb_set_error("cphb_oriented_bounding_box: n = %zu is too large", n);
        return CPHB_ERR_INVALID;
    }
    cphb_scratch sc(s);
    double *partial = nullptr, *mom = nullptr;
    float *tp = nullptr;
    int rc = sc.alloc(&partial, 6 * n_tiles);
    if (!rc) rc = sc.alloc(&mom, 9);
    if (!rc) rc = sc.alloc(&tp, 3 * n);
    if (rc) return rc;
    for (int pass = 0; pass < 2; ++pass) {
        CPHB_LAUNCH(obb_moment_tile_kernel, (unsigned)n_tiles, 128, 0, s, points, n, pass, mom, partial);
        CPHB_LAUNCH(obb_moment_final_kernel, 1, 32, 0, s, partial, n_tiles, n, pass, mom);
    }
    double h[9];
    rc = cphb_read_back(h, mom, sizeof(h), s, "cphb_oriented_bounding_box");
    if (rc) return rc;
    // cov /= n (symmetric, row-major), then its eigenvectors, each normalised
    const double nd = (double)n;
    const double c00 = h[3] / nd, c01 = h[4] / nd, c02 = h[5] / nd, c11 = h[6] / nd, c12 = h[7] / nd, c22 = h[8] / nd;
    const double cov[9] = {c00, c01, c02, c01, c11, c12, c02, c12, c22};
    double U[9], ev[3], V[9];
    cphb_host_svd3(cov, U, ev, V);
    for (int c = 0; c < 3; ++c) {
        const double nn = sqrt(V[c] * V[c] + V[3 + c] * V[3 + c] + V[6 + c] * V[6 + c]);
        for (int r = 0; r < 3; ++r) V[3 * r + c] /= nn;
    }
    // the reference's swaps (:242-253): eigenvalues descending
    const int sw[3][2] = {{1, 0}, {2, 0}, {2, 1}};
    for (int k = 0; k < 3; ++k) {
        const int a = sw[k][0], b = sw[k][1];
        if (ev[a] > ev[b]) {
            double t = ev[a]; ev[a] = ev[b]; ev[b] = t;
            for (int r = 0; r < 3; ++r) { t = V[3 * r + a]; V[3 * r + a] = V[3 * r + b]; V[3 * r + b] = t; }
        }
    }
    // sign: each column's largest-magnitude component (the first among equal magnitudes) is positive
    float R[9];
    for (int c = 0; c < 3; ++c) {
        int big = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(V[3 * r + c]) > fabs(V[3 * big + c])) big = r;
        const double sg = V[3 * big + c] < 0.0 ? -1.0 : 1.0;
        for (int r = 0; r < 3; ++r) R[3 * r + c] = (float)(sg * V[3 * r + c]);
    }
    // trans = [R^T | -R^T mean] in float32, the points transformed as PointCloud::Transform does, then their bounds
    const float mean[3] = {(float)h[0], (float)h[1], (float)h[2]};
    float T[16] = {0.f};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = R[3 * j + i];
        T[4 * i + 3] = -host_dot3(R[i], R[3 + i], R[6 + i], mean[0], mean[1], mean[2]);
    }
    T[15] = 1.f;
    CPHB_CUDA(cudaMemcpyAsync(tp, points, sizeof(float) * 3 * n, cudaMemcpyDeviceToDevice, s));
    rc = cphb_transform(tp, nullptr, nullptr, 0, n, T, s);
    float mn[3], mx[3];
    if (!rc) rc = cphb_min_max_bound(tp, n, mn, mx, s);  // synchronises
    if (rc) return rc;
    float c[3];
    for (int a = 0; a < 3; ++a) {
        c[a] = (mn[a] + mx[a]) * 0.5f;  // AxisAlignedBoundingBox::GetCenter
        h_extent[a] = mx[a] - mn[a];    // GetExtent
    }
    for (int i = 0; i < 3; ++i) h_center[i] = host_dot3(R[3 * i], R[3 * i + 1], R[3 * i + 2], c[0], c[1], c[2]) + mean[i];
    memcpy(h_R, R, sizeof(R));
    return CPHB_OK;
}

// ---- UniformDownSample and the normal operations --------------------------------------------------------------------
__global__ void __launch_bounds__(256) uniform_gather_kernel(const float *__restrict__ pts, const float *__restrict__ nrm,
                                                             const float *__restrict__ col, size_t m, size_t k, float *o_pts,
                                                             float *o_nrm, float *o_col) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    const size_t i = t * k;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        o_pts[3 * t + c] = pts[3 * i + c];
        if (nrm) o_nrm[3 * t + c] = nrm[3 * i + c];
        if (col) o_col[3 * t + c] = col[3 * i + c];
    }
}

extern "C" int cphb_uniform_down_sample(const float *points, const float *normals, const float *colors, size_t n,
                                        size_t every_k, float *out_points, float *out_normals, float *out_colors,
                                        size_t *h_n_out, void *stream) {
    if (!h_n_out) {
        cphb_set_error("cphb_uniform_down_sample: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    if (every_k == 0) {
        cphb_set_error("cphb_uniform_down_sample: every_k_points must be >= 1");
        return CPHB_ERR_INVALID;
    }
    const size_t m = n / every_k;
    if (m == 0) return CPHB_OK;
    if (!points || !out_points || (normals && !out_normals) || (colors && !out_colors)) {
        cphb_set_error("cphb_uniform_down_sample: null argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(uniform_gather_kernel, (unsigned)((m + 255) / 256), 256, 0, (cudaStream_t)stream, points, normals, colors, m,
                every_k, out_points, out_normals, out_colors);
    CPHB_CHECK_LAUNCH();
    *h_n_out = m;
    return CPHB_OK;
}

// Eigen's normalize(): n /= sqrt(|n|^2) when |n|^2 > 0
__global__ void __launch_bounds__(256) normalize_normals_kernel(float *nrm, size_t n) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v[3] = {nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]};
    if (!cphb_normalize3(v)) return;
    nrm[3 * i] = v[0];
    nrm[3 * i + 1] = v[1];
    nrm[3 * i + 2] = v[2];
}

// align_normals_direction_functor (estimate_normals.cu:66-78): a zero normal becomes the reference, one pointing away
// from it is negated
__global__ void __launch_bounds__(256) orient_normals_kernel(float *nrm, size_t n, float r0, float r1, float r2) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = nrm[3 * i], y = nrm[3 * i + 1], z = nrm[3 * i + 2];
    if (dot3(x, y, z, x, y, z) == 0.f) {
        nrm[3 * i] = r0;
        nrm[3 * i + 1] = r1;
        nrm[3 * i + 2] = r2;
    } else if (dot3(x, y, z, r0, r1, r2) < 0.f) {
        nrm[3 * i] = -x;
        nrm[3 * i + 1] = -y;
        nrm[3 * i + 2] = -z;
    }
}

extern "C" int cphb_normalize_normals(float *normals, size_t n, void *stream) {
    if (n == 0) return CPHB_OK;
    if (!normals) {
        cphb_set_error("cphb_normalize_normals: null argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(normalize_normals_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, normals, n);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

extern "C" int cphb_orient_normals(float *normals, size_t n, const float h_reference[3], void *stream) {
    if (!h_reference) {
        cphb_set_error("cphb_orient_normals: null argument");
        return CPHB_ERR_INVALID;
    }
    if (n == 0) return CPHB_OK;
    if (!normals) {
        cphb_set_error("cphb_orient_normals: null argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(orient_normals_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, normals, n, h_reference[0],
                h_reference[1], h_reference[2]);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}
