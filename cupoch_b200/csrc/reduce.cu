// reduce.cu -- the other users of the normal-equation reducer (SURVEY 8f rank 3):
//   utility::ComputeJTJandJTr<Matrix6f, Vector6f, NumJ>        eigen.inl:120-145  (RGB-D odometry, odometry.cu:618)
//   utility::ComputeWeightedJTJandJTr<.., NumJ>                eigen.inl:147-195  (odometry.cu:688, Student-t weights :633-648)
//   registration::KabschWeighted                               kabsch.cu:138-201  (FilterReg, filterreg.cu:80)
// on EXPLICIT rows / weights: the callers' row functors (RGB-D Jacobians, FilterReg's E-step) are outside the hot path
// this library replaces; what they share with ICP is this reduction, so it is exported on its own.
//
// Arithmetic contract (DESIGN.md): every per-element quantity is computed in float32 with the reference's operations in
// the reference's order; sums over elements are float64 accumulations of those float32 values in a FIXED order (thread ->
// block -> grid), rounded once -- the limit of every order thrust could choose, reproducible run to run.
#include <math.h>
#include <string.h>

#include "cphb_internal.cuh"
#include "cphb_eigen3.cuh"
#include "sum_values.cuh"

// ---------------------------------------------------------------------------------------------------------------------
// ComputeJTJandJTr / ComputeWeightedJTJandJTr on explicit rows
// ---------------------------------------------------------------------------------------------------------------------
// multiple_jtj_jtr_functor (eigen.inl:48-70): per element, over its num_j rows IN ORDER, float32:
//   JTJ_private += J_j J_j^T ; JTr_private += J_j r_j ; r2_private += r_j r_j       (28 values: 21 upper | 6 | 1)
__device__ __forceinline__ void private_sums(const float *J, const float *r, size_t i, int num_j, float (&v)[28]) {
#pragma unroll
    for (int k = 0; k < 28; ++k) v[k] = 0.f;
    for (int j = 0; j < num_j; ++j) {
        const float *row = J + ((size_t)i * num_j + j) * 6;
        const float x[6] = {row[0], row[1], row[2], row[3], row[4], row[5]};
        const float rr = r[(size_t)i * num_j + j];
        int p = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = a; b < 6; ++b) { v[p] = __fadd_rn(v[p], __fmul_rn(x[a], x[b])); ++p; }
#pragma unroll
        for (int a = 0; a < 6; ++a) v[21 + a] = __fadd_rn(v[21 + a], __fmul_rn(x[a], rr));
        v[27] = __fadd_rn(v[27], __fmul_rn(rr, rr));
    }
}
struct JtjRows {
    const float *J, *r;
    int num_j;
    __device__ void operator()(size_t i, float (&v)[28]) const { private_sums(J, r, i, num_j, v); }
};
// weight_reduce_functor (odometry.cu:633-640): r2 * (nu + 1.0) / (nu + r2 / sigma2) -- the 1.0 literal makes the product
// and the quotient double precision in the reference, the denominator stays float
struct WeightReduce {
    const float *J, *r;
    int num_j;
    float sigma2, nu;
    __device__ void operator()(size_t i, float (&v)[1]) const {
        float p[28];
        private_sums(J, r, i, num_j, p);
        const float r2 = p[27];
        const float den = __fadd_rn(nu, __fdiv_rn(r2, sigma2));
        v[0] = (float)(((double)r2 * ((double)nu + 1.0)) / (double)den);
    }
};
// calc_weights_functor (odometry.cu:642-648): w = (nu + 1) / (nu + r2 / w_sum); then w * (JTJ_i, JTr_i, r2_i) in float32
struct WeightedRows {
    const float *J, *r;
    int num_j;
    float nu, w_sum;
    __device__ void operator()(size_t i, float (&v)[28]) const {
        private_sums(J, r, i, num_j, v);
        const float w = __fdiv_rn(__fadd_rn(nu, 1.f), __fadd_rn(nu, __fdiv_rn(v[27], w_sum)));
#pragma unroll
        for (int k = 0; k < 28; ++k) v[k] = __fmul_rn(v[k], w);
    }
};

static void fill32(const double v[28], double h_sums[32]) {
    for (int k = 0; k < 32; ++k) h_sums[k] = (k < 28) ? v[k] : 0.0;
}

extern "C" int cphb_compute_jtj_jtr(const float *J, const float *r, size_t n, int num_j, double h_sums[32], void *stream) {
    if (!h_sums || (n && (!J || !r)) || num_j < 1 || num_j > 16) {
        cphb_set_error("cphb_compute_jtj_jtr: invalid argument");
        return CPHB_ERR_INVALID;
    }
    double v[28];
    JtjRows f = {J, r, num_j};
    int rc = sum_values<28>(f, n, v, (cudaStream_t)stream);
    fill32(v, h_sums);
    return rc;
}

extern "C" int cphb_compute_weighted_jtj_jtr(const float *J, const float *r, size_t n, int num_j, float sigma2, float nu,
                                             double h_sums[32], float *h_w_sum, void *stream) {
    if (!h_sums || !h_w_sum || (n && (!J || !r)) || num_j < 1 || num_j > 16) {
        cphb_set_error("cphb_compute_weighted_jtj_jtr: invalid argument");
        return CPHB_ERR_INVALID;
    }
    double ws[1];
    WeightReduce f1 = {J, r, num_j, sigma2, nu};
    int rc = sum_values<1>(f1, n, ws, (cudaStream_t)stream);
    if (rc) return rc;
    *h_w_sum = (float)ws[0];
    double v[28];
    WeightedRows f2 = {J, r, num_j, nu, *h_w_sum};
    rc = sum_values<28>(f2, n, v, (cudaStream_t)stream);
    fill32(v, h_sums);
    return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
// KabschWeighted (kabsch.cu:138-201)
// ---------------------------------------------------------------------------------------------------------------------
struct WeightedCenters {  // sum w | sum m w (3) | sum t w (3) | sum w w
    const float *m, *t, *w;
    __device__ void operator()(size_t i, float (&v)[8]) const {
        const float wi = w[i];
        v[0] = wi;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            v[1 + a] = __fmul_rn(m[3 * i + a], wi);
            v[4 + a] = __fmul_rn(t[3 * i + a], wi);
        }
        v[7] = __fmul_rn(wi, wi);
    }
};
struct WeightedH {  // ((w * w) * cx_a) * cy_b, row-major a, b (Eigen: scalar * vector, then outer product)
    const float *m, *t, *w;
    float mc[3], tc[3];
    __device__ void operator()(size_t i, float (&v)[9]) const {
        const float wi = w[i], ww = __fmul_rn(wi, wi);
        float cx[3], cy[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            cx[a] = __fmul_rn(ww, __fsub_rn(m[3 * i + a], mc[a]));
            cy[a] = __fsub_rn(t[3 * i + a], tc[a]);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) v[3 * a + b] = __fmul_rn(cx[a], cy[b]);
    }
};

// host-side epilogue shared with the oracle's specification: R = V diag(1, 1, det(U V)) U^T of the SVD of H, t = tc - R mc
void cphb_kabsch_rotation_from_h(const double H[9], double R[9]);

extern "C" int cphb_kabsch_weighted(const float *model, const float *target, const float *weight, size_t n, float h_T[16],
                                    void *stream) {
    if (!h_T || (n && (!model || !target || !weight))) {
        cphb_set_error("cphb_kabsch_weighted: null argument");
        return CPHB_ERR_INVALID;
    }
    for (int i = 0; i < 16; ++i) h_T[i] = (i % 5 == 0) ? 1.f : 0.f;
    if (n == 0) return CPHB_OK;
    cudaStream_t s = (cudaStream_t)stream;
    double c[8];
    WeightedCenters f1 = {model, target, weight};
    int rc = sum_values<8>(f1, n, c, s);
    if (rc) return rc;
    const float total_weight = (float)c[0];
    const float divided_by = 1.0f / total_weight;
    WeightedH f2;
    f2.m = model; f2.t = target; f2.w = weight;
    for (int a = 0; a < 3; ++a) {
        f2.mc[a] = (float)c[1 + a] * divided_by;
        f2.tc[a] = (float)c[4 + a] * divided_by;
    }
    const float h_weight = (float)c[7];
    double hs[9];
    rc = sum_values<9>(f2, n, hs, s);
    if (rc) return rc;
    double H[9], R[9];
    for (int k = 0; k < 9; ++k) H[k] = (double)((float)hs[k] / h_weight);
    cphb_kabsch_rotation_from_h(H, R);
    for (int i = 0; i < 3; ++i) {
        float Rf[3] = {(float)R[3 * i], (float)R[3 * i + 1], (float)R[3 * i + 2]};
        for (int j = 0; j < 3; ++j) h_T[4 * i + j] = Rf[j];
        // tr.block<3,1>(0,3) = target_center - R * model_center (float32, sequential k sum)
        h_T[4 * i + 3] = f2.tc[i] - ((Rf[0] * f2.mc[0] + Rf[1] * f2.mc[1]) + Rf[2] * f2.mc[2]);
    }
    return CPHB_OK;
}

// one-sided Jacobi SVD (double) on the host -- the same algorithm as svd3 in icp_solve.cuh (stands in for
// Eigen::JacobiSVD<Matrix3f>; R = V diag(1,1,det(UV)) U^T is unique whatever the SVD's sign / ordering conventions).
// Also the symmetric eigensolver of OrientedBoundingBox::CreateFromPoints (crop.cu).
void cphb_host_svd3(const double *A, double *U, double *sv, double *V) {
    double B[9];
    for (int i = 0; i < 9; ++i) { B[i] = A[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < 3; ++i) {
                    al += B[3 * i + p] * B[3 * i + p];
                    be += B[3 * i + q] * B[3 * i + q];
                    ga += B[3 * i + p] * B[3 * i + q];
                }
                if (fabs(ga) <= 1e-300 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
                off += fabs(ga);
                double zeta = (be - al) / (2.0 * ga);
                double t = ((zeta >= 0) ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < 3; ++i) {
                    double bp = B[3 * i + p], bq = B[3 * i + q];
                    B[3 * i + p] = c * bp - sn * bq;
                    B[3 * i + q] = sn * bp + c * bq;
                    double vp = V[3 * i + p], vq = V[3 * i + q];
                    V[3 * i + p] = c * vp - sn * vq;
                    V[3 * i + q] = sn * vp + c * vq;
                }
            }
        if (off == 0) break;
    }
    for (int j = 0; j < 3; ++j) {
        double nn = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
        sv[j] = nn;
        for (int i = 0; i < 3; ++i) U[3 * i + j] = (nn > 0) ? B[3 * i + j] / nn : 0.0;
    }
    for (int j = 0; j < 3; ++j)
        if (sv[j] == 0) {
            int a = (j + 1) % 3, b = (j + 2) % 3;
            if (sv[a] > 0 && sv[b] > 0) {
                U[j] = U[3 + a] * U[6 + b] - U[6 + a] * U[3 + b];
                U[3 + j] = U[6 + a] * U[b] - U[a] * U[6 + b];
                U[6 + j] = U[a] * U[3 + b] - U[3 + a] * U[b];
            }
        }
}
void cphb_kabsch_rotation_from_h(const double H[9], double R[9]) {
    double U[9], sv[3], V[9], UV[9];
    cphb_host_svd3(H, U, sv, V);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) UV[3 * i + j] = U[3 * i] * V[j] + U[3 * i + 1] * V[3 + j] + U[3 * i + 2] * V[6 + j];
    double dd = UV[0] * (UV[4] * UV[8] - UV[5] * UV[7]) - UV[1] * (UV[3] * UV[8] - UV[5] * UV[6]) +
                UV[2] * (UV[3] * UV[7] - UV[4] * UV[6]);
    double ss[3] = {1.0, 1.0, dd};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double r = 0;
            for (int k = 0; k < 3; ++k) r += V[3 * i + k] * ss[k] * U[3 * j + k];
            R[3 * i + j] = r;
        }
}
