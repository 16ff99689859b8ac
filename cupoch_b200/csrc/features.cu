// features.cu -- per-point neighbourhood features that sit immediately before
// the ICP loop: EstimateNormals (estimate_normals.cu:38-127), the GICP
// covariance initialisation (generalized_icp.cu:18-61) and the Colored-ICP
// intensity-gradient fit (colored_icp.cu:73-148).  EstimateNormals is ONE
// kernel (k-best search + cumulants + eigen-solve); the gradient fit is one
// search (search.cu) + one kernel; the reference uses a search + reduce_by_key
// over n*k cumulant tuples + a transform.
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "cphb_eigen3.cuh"
#include "cphb_internal.cuh"
#include "fused_neighbourhood.cuh"
#include "cphb_searchk.cuh"

// ComputeNormal (estimate_normals.cu:38-54): covariance E[xx^T] - E[x]E[x]^T in float32, eigenvector of the smallest
// eigenvalue, (0,0,1) with fewer than 3 neighbours or a zero / NaN vector
__device__ __forceinline__ void normal_from_cumulants(const double (&cum)[9], int cnt, float &nx, float &ny, float &nz) {
    nx = 0.f; ny = 0.f; nz = 1.f;
    if (cnt < 3) return;
    float cov[9];
    covariance_from_cumulants(cum, cnt, cov);
    float e[3], V[9];
    fast_eigen3x3(cov, e, V);
    int mi = 0;
    if (e[1] < e[mi]) mi = 1;
    if (e[2] < e[mi]) mi = 2;
    nx = V[mi]; ny = V[3 + mi]; nz = V[6 + mi];
    const float nn = sqrtf(dot3(nx, ny, nz, nx, ny, nz));
    if (nn == 0.0f || nn != nn) { nx = 0.f; ny = 0.f; nz = 1.f; }
}

__global__ void __launch_bounds__(256) fill_normals_kernel(float *out, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) { out[3 * i] = 0.f; out[3 * i + 1] = 0.f; out[3 * i + 2] = 1.f; }
}

// two-pass form (search result [n][k] in HBM, then this kernel): kept as the A/B partner of the fused kernel below
// (CPHB_NORMALS_UNFUSED=1) -- the two must agree bit for bit (tests/test_gpu_geometry.py)
__global__ void __launch_bounds__(128) normals_kernel(const float *__restrict__ pts, size_t n,
                                                      const int32_t *__restrict__ nbr, int k, float *out) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    double cum[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int cnt = 0;
    for (int j = 0; j < k; ++j) {
        int id = nbr[i * k + j];
        if (id < 0) continue;
        cumulant_add(cum, pts[3 * (size_t)id], pts[3 * (size_t)id + 1], pts[3 * (size_t)id + 2]);
        ++cnt;
    }
    float nx, ny, nz;
    normal_from_cumulants(cum, cnt, nx, ny, nz);
    out[3 * i] = nx; out[3 * i + 1] = ny; out[3 * i + 2] = nz;
}

// EstimateNormals in ONE kernel (SURVEY 8f rank 1; estimate_normals.cu:82-127 + geometry_functor.h:35-55): the warp's
// k-best search (lists in shared memory) is followed, in the same kernel, by the 9 cumulants over each lane's list in
// list order and the 3x3 eigen-solve -- the [n][k] index / distance table (8 k bytes per point written and read back,
// 2.4 GB at 10 M x k = 30) never exists.  Query order: fused_query_setup (fused_neighbourhood.cuh).
template <int TOP>
__global__ void normals_fused_kernel(IndexView ix, const float *__restrict__ pts, size_t first, size_t count,
                                     const uint32_t *__restrict__ perm, int self_order, float r2, int k, float *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem[];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, pts, first, count, perm, self_order, r2, k, pos);
    fused_query_search<TOP>(ix, w);
    if (!w.valid) return;
    double cum[9];
    int cnt;
    list_cumulants(w, k, init, pts, cum, cnt);
    float nx, ny, nz;
    normal_from_cumulants(cum, cnt, nx, ny, nz);
    out[3 * pos] = nx; out[3 * pos + 1] = ny; out[3 * pos + 2] = nz;
}

// k limits as the search entry points have them: SearchKNN rejects knn > NUM_MAX_NN = 100 (kdtree_flann.cu:52-54),
// SearchRadius is bounded by what one warp's lists can hold in shared memory (search.cu)
static int normals_impl(const float *points, size_t n, int knn, float radius, int max_nn, size_t first, size_t count,
                        float *out_normals, cudaStream_t s) {
    const int k = (knn > 0) ? knn : max_nn;
    if (k <= 0) {  // estimate_normals.cu:102-106
        CPHB_LAUNCH(fill_normals_kernel, (unsigned)((count + 255) / 256), 256, 0, s, out_normals, count);
        CPHB_CHECK_LAUNCH();
        return CPHB_OK;
    }
    if ((knn > 0 && k > 100) || k > 256) {
        cphb_set_error("search: k=%d outside [0,%d]", k, knn > 0 ? 100 : 256);
        return CPHB_ERR_INVALID;
    }
    // either form builds one fresh index of the whole cloud, as the reference builds a fresh tree (:86-87)
    if (getenv("CPHB_NORMALS_UNFUSED")) {  // A/B hook (read per call): the two-pass form, identical results
        cphb_nbr_table t;
        int rc = cphb_nbr_table_create(points, n, first, count, knn, radius, max_nn, &t, s);
        if (!rc) {
            CPHB_LAUNCH(normals_kernel, (unsigned)((count + 127) / 128), 128, 0, s, points, count, t.idx, k, out_normals);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) { cphb_set_error("normals_kernel: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
        }
        return cphb_nbr_table_release(&t, rc, s);
    }
    // fused: the queries [first, first + count) against the index of the whole cloud -- the whole cloud in index order,
    // a block in its own Hilbert order
    const float r2 = (knn > 0) ? INFINITY : radius * radius;  // kdtree_flann.inl:120
    const bool self_order = (first == 0 && count == n);
    cphb_index *ix = nullptr;
    cphb_scratch sc(s);
    uint32_t *perm = nullptr;
    int rc = cphb_index_create(points, n, s, &ix);
    if (!rc && !self_order && count > 32) {
        rc = sc.alloc(&perm, count);
        if (!rc) rc = cphb_hilbert_order_n(points + 3 * first, count, perm, ix->bounds, 1, count < n ? count : n, s);
    }
    if (!rc) {
        const size_t lanes = self_order ? (size_t)ix->v.n_leaves * CPHB_LEAF : count;
        rc = launch_fused(ix, normals_fused_kernel<3>, normals_fused_kernel<5>, lanes, k, s, points, first, count, perm,
                          self_order ? 1 : 0, r2, k, out_normals);
    }
    sc.release();
    const cudaError_t e = cudaStreamSynchronize(s);
    cphb_index_destroy(ix);
    if (!rc && e != cudaSuccess) { cphb_set_error("normals_fused_kernel: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
    return rc;
}

extern "C" int cphb_estimate_normals(const float *points, size_t n, int knn, float radius, int max_nn,
                                     float *out_normals, void *stream) {
    if (n == 0) return CPHB_OK;
    if (!points || !out_normals) {
        cphb_set_error("cphb_estimate_normals: null argument");
        return CPHB_ERR_INVALID;
    }
    return normals_impl(points, n, knn, radius, max_nn, 0, n, out_normals, (cudaStream_t)stream);
}

// Multi-GPU building block (DESIGN.md section 6): normals of the points [first, first + count) only, neighbours taken
// from the whole cloud.  Every rank indexes the full cloud and estimates its own block; the blocks are then
// all-gathered (cupoch_b200.distributed.estimate_normals).  Same kernel as cphb_estimate_normals (its queries in the
// block's own Hilbert order instead of index order): identical per-point arithmetic, identical results.
extern "C" int cphb_estimate_normals_range(const float *points, size_t n, int knn, float radius, int max_nn, size_t first,
                                           size_t count, float *out_normals, void *stream) {
    if (count == 0) return CPHB_OK;
    if (!points || !out_normals || first > n || count > n - first) {
        cphb_set_error("cphb_estimate_normals_range: invalid argument");
        return CPHB_ERR_INVALID;
    }
    return normals_impl(points, n, knn, radius, max_nn, first, count, out_normals, (cudaStream_t)stream);
}

// GetRotationFromE1ToX + Rx*diag(eps,1,1)*Rx^T (generalized_icp.cu:18-30,53-60)
__global__ void __launch_bounds__(256) cov_from_normals_kernel(const float *__restrict__ nrm, size_t n, float eps,
                                                               float *out, int col_major) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x[3] = {nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]};
    float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    const float c = x[0];
    if (!(c < -0.99f)) {
        const float v[3] = {0.f, -x[2], x[1]};
        const float sv[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
        float ss[9];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b)
                ss[3 * a + b] = dot3(sv[3 * a], sv[3 * a + 1], sv[3 * a + 2], sv[b], sv[3 + b], sv[6 + b]);
        const float factor = 1 / (1 + c);
#pragma unroll
        for (int a = 0; a < 9; ++a) R[a] = __fmaf_rn(ss[a], factor, R[a] + sv[a]);
    }
    const float cd[3] = {eps, 1.f, 1.f};
    float tmp[9], C[9];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) tmp[3 * a + b] = R[3 * a + b] * cd[b];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
            C[3 * a + b] = dot3(tmp[3 * a], tmp[3 * a + 1], tmp[3 * a + 2], R[3 * b], R[3 * b + 1], R[3 * b + 2]);
    float *o = out + 9 * i;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) o[col_major ? 3 * b + a : 3 * a + b] = C[3 * a + b];
}

extern "C" int cphb_covariances_from_normals(const float *normals, size_t n, float epsilon, float *out_cov,
                                             int cov_col_major, void *stream) {
    if (n == 0) return CPHB_OK;
    if (!normals || !out_cov) {
        cphb_set_error("cphb_covariances_from_normals: null argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(cov_from_normals_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, normals, n, epsilon, out_cov,
                cov_col_major);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// compute_color_gradient_functor (colored_icp.cu:73-118): slot 0 of the neighbour row is skipped
__global__ void __launch_bounds__(128) color_gradient_kernel(const float *__restrict__ pts, const float *__restrict__ nrm,
                                                             const float *__restrict__ col, size_t n,
                                                             const int32_t *__restrict__ nbr, int k, float *out) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float vt[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    const float nt[3] = {nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]};
    const float it = intensity(col[3 * i], col[3 * i + 1], col[3 * i + 2]);
    float AtA[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, Atb[3] = {0, 0, 0};
    int nn = 0;
    for (int j = 1; j < k; ++j) {
        const int a = nbr[i * k + j];
        if (a < 0) continue;
        const float va[3] = {pts[3 * (size_t)a], pts[3 * (size_t)a + 1], pts[3 * (size_t)a + 2]};
        const float s = dot3(va[0] - vt[0], va[1] - vt[1], va[2] - vt[2], nt[0], nt[1], nt[2]);
        float vtmp[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) vtmp[c] = __fmaf_rn(-s, nt[c], va[c]) - vt[c];
        const float di = intensity(col[3 * (size_t)a], col[3 * (size_t)a + 1], col[3 * (size_t)a + 2]) - it;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int c = 0; c < 3; ++c) AtA[3 * r + c] = __fmaf_rn(vtmp[r], vtmp[c], AtA[3 * r + c]);
            Atb[r] = __fmaf_rn(di, vtmp[r], Atb[r]);
        }
        ++nn;
    }
    float o[3] = {0.f, 0.f, 0.f};
    if (nn >= 4) {
        const float w = (float)((nn - 1) * (nn - 1));
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float wn = w * nt[r];
#pragma unroll
            for (int c = 0; c < 3; ++c) AtA[3 * r + c] = __fmaf_rn(wn, nt[c], AtA[3 * r + c]);
        }
        AtA[0] += 1.0e-6f; AtA[4] += 1.0e-6f; AtA[8] += 1.0e-6f;
        float inv[9];
        inverse3x3(AtA, inv);
#pragma unroll
        for (int r = 0; r < 3; ++r) o[r] = dot3(inv[3 * r], inv[3 * r + 1], inv[3 * r + 2], Atb[0], Atb[1], Atb[2]);
    }
    out[3 * i] = o[0]; out[3 * i + 1] = o[1]; out[3 * i + 2] = o[2];
}

extern "C" int cphb_color_gradient(const float *points, const float *normals, const float *colors, size_t n,
                                   float radius, int max_nn, float *out_gradient, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return CPHB_OK;
    if (!points || !normals || !colors || !out_gradient || max_nn < 1 || max_nn > 100) {
        cphb_set_error("cphb_color_gradient: invalid argument");
        return CPHB_ERR_INVALID;
    }
    cphb_nbr_table t;
    int rc = cphb_nbr_table_create(points, n, 0, n, 0, radius, max_nn, &t, s);
    if (!rc) {
        CPHB_LAUNCH(color_gradient_kernel, (unsigned)((n + 127) / 128), 128, 0, s, points, normals, colors, n, t.idx, max_nn,
                    out_gradient);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { cphb_set_error("color_gradient_kernel: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
    }
    return cphb_nbr_table_release(&t, rc, s);
}
