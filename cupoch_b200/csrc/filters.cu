// filters.cu -- kNN consumers on the point cloud (SURVEY 8f, rank 4): PointCloud::RemoveRadiusOutliers,
// RemoveStatisticalOutliers (down_sample.cu:317-438) and SelectByIndex (down_sample.cu:40-127).
//
// Both filters are "search the cloud against itself, reduce every row of the result, keep the rows that pass":
// the search is the library's own exact k-NN / radius search (search.cu), the per-row reduction and the
// stable compaction of the surviving indices are the small kernels below.  The reference materialises the
// [n][k] result, runs a thrust::reduce_by_key over it and a copy_if; here the row reduction reads each row
// once and the keep-flags are compacted with one count / scan / write pass.
//
// Arithmetic (the CPU restatement used by the tests follows the same contract): per-point mean of the k squared
// distances and both cloud statistics are accumulated in float64 and rounded to float32 once (thrust's float reductions have no
// specified order; float64 is the limit of every order); the scalar formulas (mean, Bessel-corrected standard
// deviation, threshold) are evaluated in unfused float32 in the reference's order.
#include <float.h>
#include <math.h>

#include "cphb_internal.cuh"

#define FLT_BLOCK 1024

// ---- per-row reductions ---------------------------------------------------
// keep[i] = (number of valid slots of row i) > nb_points   (down_sample.cu:333-349)
__global__ void __launch_bounds__(256) radius_keep_kernel(const int32_t *__restrict__ idx, size_t n, int k, int nb_points,
                                                          uint8_t *__restrict__ keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int cnt = 0;
    for (int j = 0; j < k; ++j) cnt += idx[i * k + j] >= 0;
    keep[i] = cnt > nb_points ? 1 : 0;
}

// avg[i] = mean of the valid squared distances of row i, -1 if none   (down_sample.cu:379-405)
__global__ void __launch_bounds__(256) row_mean_kernel(const float *__restrict__ d2, size_t n, int k, float *__restrict__ avg) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    int c = 0;
    for (int j = 0; j < k; ++j) {
        const float d = d2[i * k + j];
        if (isinf(d) || d < 0.f) continue;
        s += (double)d;
        ++c;
    }
    avg[i] = (c > 0) ? __fdiv_rn((float)s, (float)c) : -1.0f;
}

// ---- cloud statistics: fixed-order two-stage sums --------------------------
// block partials {a, b} are added in block order by one final block; `scalars` (4 floats on the device) carries
// mean, std, threshold and the valid count from pass to pass, so the host never has to look at them
__device__ __forceinline__ double block_sum(double v, double *s_w) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(CPHB_FULL, v, o);
    if (lane_id() == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) {
        t = s_w[threadIdx.x];  // FLT_BLOCK / 32 == 32 warps
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(CPHB_FULL, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0 (whole first warp)
}

// pass 0: partial[b] = {sum of valid avg, count};  pass 1 (mean known): partial[b] = {sum of squared deviations, 0}
__global__ void __launch_bounds__(FLT_BLOCK) stat_partial_kernel(const float *__restrict__ avg, size_t n, int pass,
                                                                 const float *__restrict__ scalars, double *partial) {
    __shared__ double s_w[32];
    const size_t i = blockIdx.x * (size_t)FLT_BLOCK + threadIdx.x;
    double a = 0.0, b = 0.0;
    if (i < n) {
        const float x = avg[i];
        if (pass == 0) {
            if (x >= 0.f) { a = (double)x; b = 1.0; }
        } else if (x > 0.f) {
            const float e = __fsub_rn(x, scalars[0]);
            a = (double)__fmul_rn(e, e);
        }
    }
    const double sa = block_sum(a, s_w);
    const double sb = block_sum(b, s_w);
    if (threadIdx.x == 0) {
        partial[2 * (size_t)blockIdx.x] = sa;
        partial[2 * (size_t)blockIdx.x + 1] = sb;
    }
}

// one block: adds the partials in block order, then the reference's scalar formulas (down_sample.cu:418-430)
// scalars: [0] mean, [1] std, [2] threshold, [3] valid count (as float bits of an unsigned via __uint_as_float)
__global__ void __launch_bounds__(FLT_BLOCK) stat_final_kernel(const double *__restrict__ partial, unsigned nb, int pass,
                                                               float std_ratio, float *scalars) {
    __shared__ double s_w[32];
    double a = 0.0, b = 0.0;
    for (unsigned i = threadIdx.x; i < nb; i += FLT_BLOCK) {  // fixed assignment, fixed order per thread
        a += partial[2 * (size_t)i];
        b += partial[2 * (size_t)i + 1];
    }
    const double sa = block_sum(a, s_w);
    const double sb = block_sum(b, s_w);
    if (threadIdx.x != 0) return;
    if (pass == 0) {
        const unsigned valid = (unsigned)sb;
        float mean = (float)sa;
        mean = valid ? __fdiv_rn(mean, (float)valid) : 0.f;
        scalars[0] = mean;
        scalars[3] = __uint_as_float(valid);
    } else {
        const unsigned valid = __float_as_uint(scalars[3]);
        const float sq = (float)sa;
        const float std_dev = sqrtf(__fdiv_rn(sq, (float)(valid - 1u)));  // valid == 1: x / 0, as the reference
        scalars[1] = std_dev;
        scalars[2] = __fadd_rn(scalars[0], __fmul_rn(std_ratio, std_dev));
    }
}

// keep[i] = 0 < avg[i] < threshold   (check_distance_threshold_functor, down_sample.cu:92-100)
__global__ void __launch_bounds__(256) stat_keep_kernel(const float *__restrict__ avg, size_t n, const float *__restrict__ scalars,
                                                        uint8_t *__restrict__ keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = avg[i];
    const bool any_valid = __float_as_uint(scalars[3]) != 0u;  // no valid distance at all: empty result (:414-417)
    keep[i] = (any_valid && x > 0.f && x < scalars[2]) ? 1 : 0;
}

// ---- stable compaction of the indices whose flag is set ---------------------
__global__ void __launch_bounds__(FLT_BLOCK) keep_count_kernel(const uint8_t *__restrict__ keep, size_t n, unsigned *block_counts) {
    const size_t i = blockIdx.x * (size_t)FLT_BLOCK + threadIdx.x;
    const unsigned c = block_flag_count(i < n && keep[i]);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}
// exclusive scan of the block counts in place (one block), total to *total.  The one copy of this step: every block
// compaction of the engine (this file's, VoxelDownSample's dense path, ICP's correspondence list) launches it through
// cphb_scan_block_counts.
__global__ void __launch_bounds__(FLT_BLOCK) keep_scan_kernel(unsigned *block_counts, unsigned nb, unsigned *total) {
    __shared__ unsigned s_w[32];
    __shared__ unsigned s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (unsigned base = 0; base < nb; base += FLT_BLOCK) {
        const unsigned i = base + threadIdx.x;
        const unsigned v = i < nb ? block_counts[i] : 0u;
        unsigned x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(CPHB_FULL, x, o);
            if (lane_id() >= o) x += y;
        }
        if (lane_id() == 31) s_w[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            const unsigned ws = s_w[threadIdx.x];
            unsigned z = ws;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned y = __shfl_up_sync(CPHB_FULL, z, o);
                if (lane_id() >= o) z += y;
            }
            s_w[threadIdx.x] = z - ws;
        }
        __syncthreads();
        const unsigned excl = x - v + s_w[threadIdx.x >> 5] + s_carry;
        if (i < nb) block_counts[i] = excl;
        __syncthreads();
        if (threadIdx.x == FLT_BLOCK - 1) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_carry;
}
__global__ void __launch_bounds__(FLT_BLOCK) keep_write_kernel(const uint8_t *__restrict__ keep, size_t n,
                                                               const unsigned *__restrict__ block_offsets, int32_t *out) {
    const size_t i = blockIdx.x * (size_t)FLT_BLOCK + threadIdx.x;
    const bool v = i < n && keep[i];
    const unsigned r = block_flag_rank(v);
    if (v) out[block_offsets[blockIdx.x] + r] = (int32_t)i;
}

void cphb_scan_block_counts(unsigned *counts, unsigned nb, unsigned *total, cudaStream_t s) {
    CPHB_LAUNCH(keep_scan_kernel, 1, FLT_BLOCK, 0, s, counts, nb, total);
}

// keep flags -> ascending indices in indices_out, count to *h_n_out (synchronises)
int cphb_compact_flags(const uint8_t *keep, size_t n, int32_t *indices_out, size_t *h_n_out, cudaStream_t s) {
    const unsigned nb = (unsigned)((n + FLT_BLOCK - 1) / FLT_BLOCK);
    cphb_scratch sc(s);
    unsigned *counts = nullptr, *total = nullptr;
    int rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (rc) return rc;
    CPHB_LAUNCH(keep_count_kernel, nb, FLT_BLOCK, 0, s, keep, n, counts);
    cphb_scan_block_counts(counts, nb, total, s);
    CPHB_LAUNCH(keep_write_kernel, nb, FLT_BLOCK, 0, s, keep, n, counts, indices_out);
    unsigned h = 0;
    rc = cphb_read_back(&h, total, sizeof(h), s, "cphb_compact_flags");
    if (!rc) *h_n_out = h;
    return rc;
}

// ---- the C ABI --------------------------------------------------------------
extern "C" int cphb_remove_radius_outliers(const float *points, size_t n, int nb_points, float radius, int32_t *indices_out,
                                           size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out) {
        cphb_set_error("cphb_remove_radius_outliers: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    // the reference logs nb_points < 1 / radius <= 0 and carries on (down_sample.cu:319-323); radius == 0 then
    // matches nothing (strict d2 < 0) and a negative radius acts as |radius| (the search squares it)
    if (n == 0 || radius == 0.f || nb_points < 0) return CPHB_OK;
    if (!points || !indices_out) {
        cphb_set_error("cphb_remove_radius_outliers: null argument");
        return CPHB_ERR_INVALID;
    }
    if (nb_points + 1 > 100) {  // KDTreeFlann's NUM_MAX_NN (kdtree_flann.cu:46-48): the reference's search returns -1
        cphb_set_error("cphb_remove_radius_outliers: nb_points + 1 = %d exceeds NUM_MAX_NN (100)", nb_points + 1);
        return CPHB_ERR_INVALID;
    }
    const int k = nb_points + 1;
    cphb_nbr_table t;
    cphb_scratch sc(s);
    uint8_t *keep = nullptr;
    int rc = cphb_nbr_table_create(points, n, 0, n, 0, radius, k, &t, s);  // the reference builds a fresh tree too (:324-325)
    if (!rc) rc = sc.alloc(&keep, n);
    if (!rc) {
        CPHB_LAUNCH(radius_keep_kernel, (unsigned)((n + 255) / 256), 256, 0, s, t.idx, n, k, nb_points, keep);
        rc = cphb_compact_flags(keep, n, indices_out, h_n_out, s);
    }
    sc.release();
    return cphb_nbr_table_release(&t, rc, s);
}

extern "C" int cphb_remove_statistical_outliers(const float *points, size_t n, int nb_neighbors, float std_ratio,
                                                int32_t *indices_out, size_t *h_n_out, float h_stats[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out) {
        cphb_set_error("cphb_remove_statistical_outliers: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    if (h_stats) h_stats[0] = h_stats[1] = h_stats[2] = 0.f;
    if (n == 0 || nb_neighbors < 1) return CPHB_OK;  // empty cloud -> empty result (:363-366); nb < 1: no neighbours
    if (!points || !indices_out) {
        cphb_set_error("cphb_remove_statistical_outliers: null argument");
        return CPHB_ERR_INVALID;
    }
    if (nb_neighbors > 100) {
        cphb_set_error("cphb_remove_statistical_outliers: nb_neighbors = %d exceeds NUM_MAX_NN (100)", nb_neighbors);
        return CPHB_ERR_INVALID;
    }
    const int k = nb_neighbors;
    const unsigned nb = (unsigned)((n + FLT_BLOCK - 1) / FLT_BLOCK);
    cphb_nbr_table t;
    cphb_scratch sc(s);
    float *avg = nullptr, *scalars = nullptr;
    double *partial = nullptr;
    uint8_t *keep = nullptr;
    int rc = cphb_nbr_table_create(points, n, 0, n, k, 0.f, 0, &t, s);
    if (!rc) rc = sc.alloc(&avg, n);
    if (!rc) rc = sc.alloc(&scalars, 4);
    if (!rc) rc = sc.alloc(&partial, 2 * (size_t)nb);
    if (!rc) rc = sc.alloc(&keep, n);
    if (!rc) {
        const unsigned g256 = (unsigned)((n + 255) / 256);
        CPHB_LAUNCH(row_mean_kernel, g256, 256, 0, s, t.d2, n, k, avg);
        CPHB_LAUNCH(stat_partial_kernel, nb, FLT_BLOCK, 0, s, avg, n, 0, scalars, partial);
        CPHB_LAUNCH(stat_final_kernel, 1, FLT_BLOCK, 0, s, partial, nb, 0, std_ratio, scalars);
        CPHB_LAUNCH(stat_partial_kernel, nb, FLT_BLOCK, 0, s, avg, n, 1, scalars, partial);
        CPHB_LAUNCH(stat_final_kernel, 1, FLT_BLOCK, 0, s, partial, nb, 1, std_ratio, scalars);
        CPHB_LAUNCH(stat_keep_kernel, g256, 256, 0, s, avg, n, scalars, keep);
        rc = cphb_compact_flags(keep, n, indices_out, h_n_out, s);
        if (!rc && h_stats) rc = cphb_read_back(h_stats, scalars, sizeof(float) * 3, s, "cphb_remove_statistical_outliers");
    }
    sc.release();
    return cphb_nbr_table_release(&t, rc, s);
}

// PointCloud::GaussianFilter (pointcloud.cu:56-106,387-433): weighted mean of the neighbours found by a radius search
// of the cloud against itself; weight = exp(-0.5 * d2 / sigma2) evaluated in double and rounded to float (the
// reference's literal 0.5 promotes the expression), sequential float32 sums in slot order, one division per component
__global__ void __launch_bounds__(128) gaussian_filter_kernel(const float *__restrict__ pts, const float *__restrict__ nrm,
                                                              const float *__restrict__ col, size_t n,
                                                              const int32_t *__restrict__ idx, const float *__restrict__ d2, int k,
                                                              float sigma2, float *o_pts, float *o_nrm, float *o_col) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float tw = 0.f, rp[3] = {0.f, 0.f, 0.f}, rn[3] = {0.f, 0.f, 0.f}, rc[3] = {0.f, 0.f, 0.f};
    for (int s = 0; s < k; ++s) {
        const int j = idx[i * k + s];
        if (j < 0) continue;
        const float w = (float)exp(-0.5 * (double)d2[i * k + s] / (double)sigma2);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            rp[a] = __fadd_rn(rp[a], __fmul_rn(w, pts[3 * (size_t)j + a]));
            if (nrm) rn[a] = __fadd_rn(rn[a], __fmul_rn(w, nrm[3 * (size_t)j + a]));
            if (col) rc[a] = __fadd_rn(rc[a], __fmul_rn(w, col[3 * (size_t)j + a]));
        }
        tw = __fadd_rn(tw, w);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        o_pts[3 * i + a] = __fdiv_rn(rp[a], tw);
        if (nrm) o_nrm[3 * i + a] = __fdiv_rn(rn[a], tw);
        if (col) o_col[3 * i + a] = __fdiv_rn(rc[a], tw);
    }
}

extern "C" int cphb_gaussian_filter(const float *points, const float *normals, const float *colors, size_t n, float search_radius,
                                    float sigma2, int num_max_search_points, float *out_points, float *out_normals,
                                    float *out_colors, size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out) {
        cphb_set_error("cphb_gaussian_filter: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    // pointcloud.cu:390-395: illegal parameters are logged and an empty cloud is returned
    if (search_radius <= 0.f || sigma2 <= 0.f || num_max_search_points <= 0 || n == 0) return CPHB_OK;
    if (!points || !out_points || (normals && !out_normals) || (colors && !out_colors)) {
        cphb_set_error("cphb_gaussian_filter: null argument");
        return CPHB_ERR_INVALID;
    }
    if (num_max_search_points > 100) {
        cphb_set_error("cphb_gaussian_filter: num_max_search_points = %d exceeds NUM_MAX_NN (100)", num_max_search_points);
        return CPHB_ERR_INVALID;
    }
    const int k = num_max_search_points;
    cphb_nbr_table t;
    int rc = cphb_nbr_table_create(points, n, 0, n, 0, search_radius, k, &t, s);
    if (!rc) {
        CPHB_LAUNCH(gaussian_filter_kernel, (unsigned)((n + 127) / 128), 128, 0, s, points, normals, colors, n, t.idx, t.d2, k,
                    sigma2, out_points, out_normals, out_colors);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { cphb_set_error("gaussian_filter_kernel: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
    }
    rc = cphb_nbr_table_release(&t, rc, s);
    if (!rc) *h_n_out = n;
    return rc;
}

// PointCloud::SelectByIndex (down_sample.cu:40-127): gather of the rows named by indices, in the order given
__global__ void __launch_bounds__(256) select_rows_kernel(const float *__restrict__ points, const float *__restrict__ normals,
                                                          const float *__restrict__ colors, size_t n,
                                                          const int32_t *__restrict__ indices, size_t m, float *o_points,
                                                          float *o_normals, float *o_colors) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    const size_t i = (size_t)indices[t];
    if (i >= n) return;  // out-of-range index: row left untouched (the reference would read out of bounds)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        o_points[3 * t + c] = points[3 * i + c];
        if (normals) o_normals[3 * t + c] = normals[3 * i + c];
        if (colors) o_colors[3 * t + c] = colors[3 * i + c];
    }
}

extern "C" int cphb_select_by_index(const float *points, const float *normals, const float *colors, size_t n,
                                    const int32_t *indices, size_t n_indices, float *out_points, float *out_normals,
                                    float *out_colors, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n_indices == 0) return CPHB_OK;
    if (!points || !indices || !out_points || (normals && !out_normals) || (colors && !out_colors)) {
        cphb_set_error("cphb_select_by_index: null argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(select_rows_kernel, (unsigned)((n_indices + 255) / 256), 256, 0, s, points, normals, colors, n, indices,
                n_indices, out_points, out_normals, out_colors);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}
