// iss.cu -- geometry::keypoint::ComputeISSKeypoints (iss_keypoints.cu:108-172): Intrinsic Shape Signature keypoints.
//
// The reference runs two radius searches into [n][max_nn] index / distance tables (max_nn = 100 by default), a
// reduce_by_key over n * max_nn cumulant tuples, and for automatic radii a kNN-2 search plus a blocking
// thrust::reduce.  Here one index serves every search, and each search is fused with the work that consumes it
// (fused_neighbourhood.cuh, as EstimateNormals does): no [n][k] table exists.
//   radii      (only when salient_radius == 0 || non_max_radius == 0, :124-132) iss_knn2_kernel writes every point's
//              slot-1 d2 of a kNN-2 search; iss_tile_sum_kernel + iss_radii_kernel add them in the fixed tiled order
//              and write {6, 4} * sqrtf(sum / (float)n) to the device radii -- no host round trip;
//   saliency   iss_saliency_kernel: radius search (salient_radius, max_neighbors), cumulants, covariance, isZero,
//              FastEigen3x3Val, the ratio tests -> saliency[n] (:133-156);
//   suppression iss_suppress_kernel: radius search (non_max_radius, max_neighbors) of the points with saliency >= 0
//              only, each compared with its listed neighbours' saliency as the list is read -> mask[n] (:158-166);
//   output     the shared compaction of the mask into ascending indices (SelectByMask, down_sample.cu:131-167).
// Every search takes its queries in index order (self_order of fused_query_setup).
//
// Arithmetic (DESIGN.md arithmetic contract; oracle/iss.c restates it):
//   - resolution sum: tiles of ISS_TILE consecutive slot-1 d2 (original order) summed sequentially in double from 0,
//     then the tile sums in tile order, rounded to float once; resolution = sqrtf(sum / (float)n), IEEE;
//   - covariance: EstimateNormals' (float64 cumulants, cum / (float)count, explicit FMAs);
//   - isZero: Eigen's DenseBase::isZero() with dummy_precision<float>() = 1e-5, i.e. isMuchSmallerThan(c, 1, 1e-5) =
//     |c| <= 1 * 1e-5 for every coefficient -- an ABSOLUTE threshold (Eigen/src/Core/Fuzzy.h, MathFunctions.h);
//   - FastEigen3x3Val (eigenvalue.inl:164-170): (min, ((e0 + e1) + e2) - min - max, max) of FastEigen3x3's eigenvalues,
//     min / max as Eigen's minCoeff / maxCoeff visitors (first strict improvement); the eigenvalues are those of
//     A / max_coeff in the general branch (not scaled back), so the saliency is normalised per point;
//   - the ratio tests divide with IEEE division (the reference's --use_fast_math divides approximately).
#include <math.h>

#include "cphb_eigen3.cuh"
#include "cphb_internal.cuh"
#include "fused_neighbourhood.cuh"

#define ISS_TILE 1024        // resolution-sum tile (the SegmentPlane order)
#define ISS_MAX_NN 256       // the radius search's own limit (search.cu CPHB_RADIUS_MAX_NN)
#define ISS_ZERO_PREC 1e-5f  // Eigen::NumTraits<float>::dummy_precision()

// kNN-2 of every indexed point: its slot-1 squared distance (+inf when the cloud has one point)
template <int TOP>
__global__ void iss_knn2_kernel(IndexView ix, const float *__restrict__ pts, float *__restrict__ d2_1) {
    extern __shared__ __align__(16) unsigned char smem[];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, pts, 0, 0, nullptr, 1, INFINITY, 2, pos);
    fused_query_search<TOP>(ix, w);
    if (!w.valid) return;
    const unsigned long long key = w.list[32];
    d2_1[pos] = key < init ? __uint_as_float((unsigned)(key >> 32)) : INFINITY;
}

__global__ void __launch_bounds__(128) iss_tile_sum_kernel(const float *__restrict__ d2_1, size_t n, double *__restrict__ partial) {
    const size_t tile = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t base = tile * ISS_TILE;
    if (base >= n) return;
    const size_t end = min(base + ISS_TILE, n);
    double s = 0.0;
    for (size_t i = base; i < end; ++i) s = __dadd_rn(s, (double)d2_1[i]);
    partial[tile] = s;
}

// ComputeModelResolution (:37-49) and the radii (:125-127)
__global__ void iss_radii_kernel(const double *__restrict__ partial, size_t n_tiles, size_t n, float *__restrict__ radii) {
    if (threadIdx.x != 0) return;
    double s = 0.0;
    for (size_t t = 0; t < n_tiles; ++t) s = __dadd_rn(s, partial[t]);
    const float resolution = __fsqrt_rn(__fdiv_rn((float)s, (float)n));
    radii[0] = __fmul_rn(6.f, resolution);
    radii[1] = __fmul_rn(4.f, resolution);
}

// compute_third_eigen_values_functor + ComputeThirdEigenValue (:51-81)
__device__ __forceinline__ float iss_saliency(const double (&cum)[9], int cnt, int min_neighbors, float gamma_21, float gamma_32) {
    if (cnt < min_neighbors) return -1.f;
    float cov[9];
    covariance_from_cumulants(cum, cnt, cov);
    bool zero = true;
#pragma unroll
    for (int a = 0; a < 9; ++a) zero = zero && fabsf(cov[a]) <= ISS_ZERO_PREC;
    if (zero) return -1.f;  // the (-1, -1, -1) the reference returns fails e[2] > 0
    float e[3], V[9];
    fast_eigen3x3(cov, e, V);
    float mn = e[0], mx = e[0];
    if (e[1] < mn) mn = e[1];
    if (e[2] < mn) mn = e[2];
    if (e[1] > mx) mx = e[1];
    if (e[2] > mx) mx = e[2];
    const float mid = __fsub_rn(__fsub_rn(__fadd_rn(__fadd_rn(e[0], e[1]), e[2]), mn), mx);
    return (mx > 0.f && __fdiv_rn(mid, mx) < gamma_21 && __fdiv_rn(mn, mid) < gamma_32) ? mn : -1.f;
}

template <int TOP>
__global__ void iss_saliency_kernel(IndexView ix, const float *__restrict__ pts, const float *__restrict__ radii, int k,
                                    int min_neighbors, float gamma_21, float gamma_32, float *__restrict__ saliency) {
    extern __shared__ __align__(16) unsigned char smem[];
    const float r = radii[0];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, pts, 0, 0, nullptr, 1, __fmul_rn(r, r), k, pos);
    fused_query_search<TOP>(ix, w);
    if (!w.valid) return;
    double cum[9];
    int cnt;
    list_cumulants(w, k, init, pts, cum, cnt);
    saliency[pos] = iss_saliency(cum, cnt, min_neighbors, gamma_21, gamma_32);
}

// is_local_maxima_functor (:83-101): saliency >= 0 and no listed neighbour strictly more salient.  Points that cannot
// be keypoints (saliency < 0) take no part in the search.
template <int TOP>
__global__ void iss_suppress_kernel(IndexView ix, const float *__restrict__ pts, const float *__restrict__ radii, int k,
                                    const float *__restrict__ saliency, uint8_t *__restrict__ mask) {
    extern __shared__ __align__(16) unsigned char smem[];
    const float r = radii[1];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, pts, 0, 0, nullptr, 1, __fmul_rn(r, r), k, pos);
    const bool real = w.valid;
    const float q = real ? saliency[pos] : -1.f;
    w.valid = real && !(q < 0.f);
    fused_query_search<TOP>(ix, w);
    if (!real) return;
    bool keep = w.valid;
    for (int j = 0; keep && j < k; ++j) {
        const unsigned long long key = w.list[j * 32];
        if (!(key < init)) break;
        if (q < saliency[(unsigned)(key & 0xffffffffull)]) keep = false;
    }
    mask[pos] = keep ? 1 : 0;
}

__global__ void __launch_bounds__(256) iss_fill_kernel(float *__restrict__ saliency, uint8_t *__restrict__ mask, size_t n) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    saliency[i] = -1.f;
    mask[i] = 0;
}

extern "C" int cphb_compute_iss_keypoints(const float *points, size_t n, float salient_radius, float non_max_radius,
                                          float gamma_21, float gamma_32, int min_neighbors, int max_neighbors,
                                          uint8_t *mask_out, int32_t *indices_out, size_t *h_n_out, float *saliency_out,
                                          float h_radii[2], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out) {
        cphb_set_error("cphb_compute_iss_keypoints: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    if (max_neighbors < 0 || max_neighbors > ISS_MAX_NN || n > (size_t)INT32_MAX) {
        cphb_set_error("cphb_compute_iss_keypoints: max_neighbors = %d, n = %zu (need 0 <= max_neighbors <= %d, n <= 2^31-1)",
                       max_neighbors, n, ISS_MAX_NN);
        return CPHB_ERR_INVALID;
    }
    const bool automatic = salient_radius == 0.f || non_max_radius == 0.f;  // :124: both are replaced
    if (h_radii) {
        h_radii[0] = salient_radius;
        h_radii[1] = non_max_radius;
    }
    if (n == 0) return CPHB_OK;  // :117-120
    if (!points || !mask_out) {
        cphb_set_error("cphb_compute_iss_keypoints: null argument");
        return CPHB_ERR_INVALID;
    }
    const int k = max_neighbors;
    const size_t n_tiles = (n + ISS_TILE - 1) / ISS_TILE;
    cphb_index *ix = nullptr;
    // the stand-ins for the caller's saliency / index buffers go back to the pool after the other scratch: the order in
    // which the next call gets these blocks back is measurable at 10 M points
    cphb_scratch sc(s), stand_in(s);
    float *radii = nullptr, *d2_1 = nullptr, *sal = saliency_out;
    double *partial = nullptr;
    int32_t *idx = indices_out;
    int rc = cphb_index_create(points, n, s, &ix);
    const size_t lanes = rc ? 0 : (size_t)ix->v.n_leaves * CPHB_LEAF;  // every search: the indexed points in index order
    if (!rc) rc = sc.alloc(&radii, 2);
    if (!rc && !sal) rc = stand_in.alloc(&sal, n);
    if (!rc && !idx) rc = stand_in.alloc(&idx, n);
    if (!rc && automatic) {
        rc = sc.alloc(&d2_1, n);
        if (!rc) rc = sc.alloc(&partial, n_tiles);
        if (!rc) rc = launch_fused(ix, iss_knn2_kernel<3>, iss_knn2_kernel<5>, lanes, 2, s, points, d2_1);
        if (!rc) {
            CPHB_LAUNCH(iss_tile_sum_kernel, (unsigned)((n_tiles + 127) / 128), 128, 0, s, d2_1, n, partial);
            CPHB_LAUNCH(iss_radii_kernel, 1, 32, 0, s, partial, n_tiles, n, radii);
            CPHB_CHECK_LAUNCH();
        }
    } else if (!rc) {
        const float given[2] = {salient_radius, non_max_radius};  // pageable: staged before the call returns
        const cudaError_t e = cudaMemcpyAsync(radii, given, sizeof(given), cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) {
            cphb_set_error("cphb_compute_iss_keypoints: %s", cudaGetErrorString(e));
            rc = CPHB_ERR_CUDA;
        }
    }
    if (!rc && k == 0) {  // no neighbour is ever listed, not even the point itself: nothing is salient
        CPHB_LAUNCH(iss_fill_kernel, (unsigned)((n + 255) / 256), 256, 0, s, sal, mask_out, n);
        CPHB_CHECK_LAUNCH();
    } else if (!rc) {
        rc = launch_fused(ix, iss_saliency_kernel<3>, iss_saliency_kernel<5>, lanes, k, s, points, (const float *)radii, k,
                          min_neighbors, gamma_21, gamma_32, sal);
        if (!rc)
            rc = launch_fused(ix, iss_suppress_kernel<3>, iss_suppress_kernel<5>, lanes, k, s, points, (const float *)radii,
                              k, (const float *)sal, mask_out);
    }
    if (!rc) rc = cphb_compact_flags(mask_out, n, idx, h_n_out, s);  // synchronises
    if (!rc && h_radii && automatic) rc = cphb_read_back(h_radii, radii, 2 * sizeof(float), s, "cphb_compute_iss_keypoints");
    sc.release();
    stand_in.release();
    cudaStreamSynchronize(s);
    if (ix) cphb_index_destroy(ix);
    return rc;
}
