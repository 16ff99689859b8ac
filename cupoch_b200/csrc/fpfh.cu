// fpfh.cu -- registration::ComputeFPFHFeature (fpfh.cu:34-229): an index client (SURVEY 8f rank 4).
//   k-NN / radius neighbours of every point (the library's own search) -> SPFH (11 + 11 + 11 bin histogram of the pair
//   features of a point with each neighbour) -> FPFH (distance-weighted sum of the neighbours' SPFH + the point's own).
// Arithmetic contract: float32 pair features in the reference's operation order; the three transcendental calls
// (acos for the frame choice, atan2 for the first angle) are the deterministic float64 routines of cphb_eigen3.cuh,
// rounded once to float32 -- the oracle uses the same specification, so histograms are bit-exact; histogram
// increments are float32 additions in neighbour order (nearest first), exactly as the reference's sequential loops.
#include <math.h>

#include "cphb_internal.cuh"
#include "cphb_eigen3.cuh"

// ComputePairFeatures (fpfh.cu:34-69)
__device__ void pair_features(const float *p1, const float *n1, const float *p2, const float *n2, float (&f)[4]) {
    float d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
    f[0] = f[1] = f[2] = 0.f;
    f[3] = sqrtf(dot3(d[0], d[1], d[2], d[0], d[1], d[2]));
    if (f[3] == 0.f) { f[3] = 0.f; return; }
    float a[3] = {n1[0], n1[1], n1[2]}, b[3] = {n2[0], n2[1], n2[2]};
    const float angle1 = __fdiv_rn(dot3(a[0], a[1], a[2], d[0], d[1], d[2]), f[3]);
    const float angle2 = __fdiv_rn(dot3(b[0], b[1], b[2], d[0], d[1], d[2]), f[3]);
    // acos(|x|) is NaN beyond 1 (an un-normalised normal): the comparison is then false, as in the reference
    const float c1 = fabsf(angle1), c2 = fabsf(angle2);
    const bool swap = (c1 <= 1.f && c2 <= 1.f) && (det_acosf(c1) > det_acosf(c2));
    if (swap) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { const float t = a[k]; a[k] = b[k]; b[k] = t; d[k] = -d[k]; }
        f[2] = -angle2;
    } else {
        f[2] = angle1;
    }
    float v[3];
    cross3(d, a, v);
    const float vn = sqrtf(dot3(v[0], v[1], v[2], v[0], v[1], v[2]));
    if (vn == 0.f) { f[0] = f[1] = f[2] = f[3] = 0.f; return; }
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = __fdiv_rn(v[k], vn);
    float w[3];
    cross3(a, v, w);
    f[1] = dot3(v[0], v[1], v[2], b[0], b[1], b[2]);
    f[0] = det_atan2f(dot3(w[0], w[1], w[2], b[0], b[1], b[2]), dot3(a[0], a[1], a[2], b[0], b[1], b[2]));
}

__device__ __forceinline__ int hist_bin(double x) {
    int h = (int)floor(x);
    return h < 0 ? 0 : (h >= 11 ? 10 : h);
}
// compute_spfh_functor (fpfh.cu:71-112)
__global__ void __launch_bounds__(128) spfh_kernel(const float *__restrict__ pts, const float *__restrict__ nrm, size_t n,
                                                   const int32_t *__restrict__ idx, int k, float *spfh) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ft[33];
#pragma unroll
    for (int j = 0; j < 33; ++j) ft[j] = 0.f;
    int cnt = 0;
    for (int q = 0; q < k; ++q) cnt += idx[i * k + q] >= 0;
    const float hist_incr = (float)(100.0 / (double)(float)(cnt - 1));
    for (int q = 0; q < k; ++q) {
        const int32_t j = idx[i * k + q];
        if (j < 0 || (size_t)j == i) continue;
        float pf[4];
        pair_features(pts + 3 * i, nrm + 3 * i, pts + 3 * (size_t)j, nrm + 3 * (size_t)j, pf);
        const double PI = 3.14159265358979323846;
        ft[hist_bin(11.0 * ((double)pf[0] + PI) / (2.0 * PI))] += hist_incr;
        ft[11 + hist_bin(11.0 * ((double)pf[1] + 1.0) * 0.5)] += hist_incr;
        ft[22 + hist_bin(11.0 * ((double)pf[2] + 1.0) * 0.5)] += hist_incr;
    }
    for (int j = 0; j < 33; ++j) spfh[i * 33 + j] = ft[j];
}
// compute_fpfh_functor (fpfh.cu:147-190)
__global__ void __launch_bounds__(128) fpfh_kernel(const float *__restrict__ spfh, size_t n, const int32_t *__restrict__ idx,
                                                   const float *__restrict__ d2, int k, float *out) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ft[33];
#pragma unroll
    for (int j = 0; j < 33; ++j) ft[j] = 0.f;
    float sum[3] = {0.f, 0.f, 0.f};
    for (int q = 0; q < k; ++q) {
        const int32_t nb = idx[i * k + q];
        if (nb < 0 || (size_t)nb == i) continue;
        const float dist = d2[i * k + q];
        if (dist == 0.f) continue;
        for (int j = 0; j < 33; ++j) {
            const float val = __fdiv_rn(spfh[(size_t)nb * 33 + j], dist);
            sum[j / 11] = __fadd_rn(sum[j / 11], val);
            ft[j] = __fadd_rn(ft[j], val);
        }
    }
    for (int j = 0; j < 3; ++j)
        if (sum[j] != 0.f) sum[j] = (float)(100.0 / (double)sum[j]);
    for (int j = 0; j < 33; ++j) out[i * 33 + j] = __fadd_rn(__fmul_rn(ft[j], sum[j / 11]), spfh[i * 33 + j]);
}

// knn > 0: KDTreeSearchParamKNN(knn); else KDTreeSearchParamRadius(radius, max_nn).  out_features: [n][33] float32.
extern "C" int cphb_compute_fpfh_feature(const float *points, const float *normals, size_t n, int knn, float radius, int max_nn,
                                         float *out_features, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return CPHB_OK;
    if (!points || !normals || !out_features) {
        cphb_set_error("cphb_compute_fpfh_feature: null argument (the reference requires normals)");
        return CPHB_ERR_INVALID;
    }
    const int k = (knn > 0) ? knn : max_nn;
    if (k <= 0 || k > 100) {
        cphb_set_error("cphb_compute_fpfh_feature: neighbour count %d outside [1, 100]", k);
        return CPHB_ERR_INVALID;
    }
    cphb_nbr_table t;
    cphb_scratch sc(s);
    float *spfh = nullptr;
    int rc = cphb_nbr_table_create(points, n, 0, n, knn, radius, max_nn, &t, s);
    if (!rc) rc = sc.alloc(&spfh, n * 33);
    if (!rc) {
        CPHB_LAUNCH(spfh_kernel, (unsigned)((n + 127) / 128), 128, 0, s, points, normals, n, t.idx, k, spfh);
        CPHB_LAUNCH(fpfh_kernel, (unsigned)((n + 127) / 128), 128, 0, s, spfh, n, t.idx, t.d2, k, out_features);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { cphb_set_error("fpfh kernels: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
    }
    sc.release();
    return cphb_nbr_table_release(&t, rc, s);
}
