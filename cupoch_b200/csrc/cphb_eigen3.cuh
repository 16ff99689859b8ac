// cphb_eigen3.cuh -- small fixed-size float32 linear algebra shared by icp.cu and
// features.cu: cross products, the analytic symmetric 3x3 eigen-solver
// (eigenvalue.inl:30-178), SqrtMatrix3x3 and Eigen's cofactor 3x3 inverse; the deterministic acos / cos / atan2
// (det_acosf, det_cosf, det_atan2f) that iss.cu, fpfh.cu and shot.cu use as well.
// Translation units including this must be compiled with -fmad=false.
#pragma once
#include "cphb_internal.cuh"

// ===========================================================================
// small host-order float helpers (never fused: this TU is built -fmad=false)
// ===========================================================================
__device__ __forceinline__ void cross3(const float *a, const float *b, float *o) {
    o[0] = det2(a[1], b[2], a[2], b[1]);
    o[1] = det2(a[2], b[0], a[0], b[2]);
    o[2] = det2(a[0], b[1], a[1], b[0]);
}
__device__ __forceinline__ float intensity(float r, float g, float b) {  // colored_icp.cu:176-181
    return (float)((double)(r + g + b) / 3.0);
}

// ---- eigenvalue.inl:30-178 (FastEigen3x3 / SqrtMatrix3x3), row-major A ------
__device__ __forceinline__ float signf_(float x) { return x / fabsf(x); }
static __device__ void eigvec0(const float *A, float e0, float *out) {
    float r0[3] = {A[0] - e0, A[1], A[2]};
    float r1[3] = {A[1], A[4] - e0, A[5]};
    float r2[3] = {A[2], A[5], A[8] - e0};
    float rx[3][3];
    cross3(r0, r1, rx[0]);
    cross3(r0, r2, rx[1]);
    cross3(r1, r2, rx[2]);
    float d0 = dot3(rx[0][0], rx[0][1], rx[0][2], rx[0][0], rx[0][1], rx[0][2]);
    float d1 = dot3(rx[1][0], rx[1][1], rx[1][2], rx[1][0], rx[1][1], rx[1][2]);
    float d2 = dot3(rx[2][0], rx[2][1], rx[2][2], rx[2][0], rx[2][1], rx[2][2]);
    float dm = d0;
    float v0 = rx[0][0], v1 = rx[0][1], v2 = rx[0][2];
    if (d1 > dm) { dm = d1; v0 = rx[1][0]; v1 = rx[1][1]; v2 = rx[1][2]; }
    if (d2 > dm) { dm = d2; v0 = rx[2][0]; v1 = rx[2][1]; v2 = rx[2][2]; }
    float s = sqrtf(dm);
    out[0] = v0 / s; out[1] = v1 / s; out[2] = v2 / s;
}
static __device__ void eigvec1(const float *A, const float *e0v, float e1, float *out) {
    float mx = fmaxf(fabsf(e0v[0]), fabsf(e0v[1]));
    float inv_len = 1 / sqrtf(__fmaf_rn(e0v[2], e0v[2], mx * mx));
    float U[3], V[3];
    if (fabsf(e0v[0]) > fabsf(e0v[1])) { U[0] = -e0v[2]; U[1] = 0; U[2] = e0v[0]; }
    else { U[0] = 0; U[1] = e0v[2]; U[2] = -e0v[1]; }
    U[0] *= inv_len; U[1] *= inv_len; U[2] *= inv_len;
    cross3(e0v, U, V);
    float AU[3] = {dot3(A[0], A[1], A[2], U[0], U[1], U[2]), dot3(A[1], A[4], A[5], U[0], U[1], U[2]),
                   dot3(A[2], A[5], A[8], U[0], U[1], U[2])};
    float AV[3] = {dot3(A[0], A[1], A[2], V[0], V[1], V[2]), dot3(A[1], A[4], A[5], V[0], V[1], V[2]),
                   dot3(A[2], A[5], A[8], V[0], V[1], V[2])};
    float m00 = dot3(U[0], U[1], U[2], AU[0], AU[1], AU[2]) - e1;
    float m01 = dot3(U[0], U[1], U[2], AV[0], AV[1], AV[2]);
    float m11 = dot3(V[0], V[1], V[2], AV[0], AV[1], AV[2]) - e1;
    float a00 = fabsf(m00), a01 = fabsf(m01), a11 = fabsf(m11);
    float mac0 = fmaxf(a00, a11);
    float mac = fmaxf(mac0, a01);
    float coef2 = fminf(mac0, a01) / fmaxf(mac, 1.0e-6f);
    float coef1 = 1.0f / sqrtf(__fmaf_rn(coef2, coef2, 1.0f));
    float cu, cv;
    if (a00 >= a11) {
        coef2 *= coef1 * signf_(m00) * signf_(m01);
        if (mac0 >= a01) { cu = coef2; cv = coef1; } else { cu = coef1; cv = coef2; }
    } else {
        coef2 *= coef1 * signf_(m11) * signf_(m01);
        if (mac0 >= a01) { cu = coef1; cv = coef2; } else { cu = coef2; cv = coef1; }
    }
    for (int i = 0; i < 3; ++i) out[i] = __fmaf_rn(cu, U[i], -(cv * V[i]));
}
// ---- deterministic acos / cos (specification: oracle/oracle.c "deterministic acos / cos"; tables from
// tools/gen_trig_coeffs.py).  float64 Horner with explicit fma, IEEE sqrt/add/mul, one rounding to float32: the same bits
// on the host oracle and on the device, unlike acosf / cosf (libm vs libdevice differ in the last ulp).
namespace dt {
static __device__ const double DT_ASIN[26] = {
    0x1.0000000000000p+0,
    0x1.5555555555555p-3,
    0x1.3333333333333p-4,
    0x1.6db6db6db6db7p-5,
    0x1.f1c71c71c71c7p-6,
    0x1.6e8ba2e8ba2e9p-6,
    0x1.1c4ec4ec4ec4fp-6,
    0x1.c99999999999ap-7,
    0x1.7a87878787878p-7,
    0x1.3fde50d79435ep-7,
    0x1.12ef3cf3cf3cfp-7,
    0x1.df3bd37a6f4dfp-8,
    0x1.a6863d70a3d71p-8,
    0x1.782dda12f684cp-8,
    0x1.51ba308d3dcb1p-8,
    0x1.31683bdef7bdfp-8,
    0x1.15ee9d45d1746p-8,
    0x1.fcaf8fb6db6dbp-9,
    0x1.d3d2a8e0dd67dp-9,
    0x1.b026f57b13b14p-9,
    0x1.90cb77f60c7cep-9,
    0x1.750de64d7d05fp-9,
    0x1.5c5f56efaaaabp-9,
    0x1.464c0950f7d47p-9,
    0x1.3275586c5f2f0p-9,
    0x1.208d3570ae5a6p-9,
};
static __device__ const double DT_COS[12] = {
    0x1.0000000000000p+0,
    -0x1.0000000000000p-1,
    0x1.5555555555555p-5,
    -0x1.6c16c16c16c17p-10,
    0x1.a01a01a01a01ap-16,
    -0x1.27e4fb7789f5cp-22,
    0x1.1eed8eff8d898p-29,
    -0x1.93974a8c07c9dp-37,
    0x1.ae7f3e733b81fp-45,
    -0x1.6827863b97d97p-53,
    0x1.e542ba4020225p-62,
    -0x1.0ce396db7f853p-70,
};
static __device__ const double DT_SIN[12] = {
    0x1.0000000000000p+0,
    -0x1.5555555555555p-3,
    0x1.1111111111111p-7,
    -0x1.a01a01a01a01ap-13,
    0x1.71de3a556c734p-19,
    -0x1.ae64567f544e4p-26,
    0x1.6124613a86d09p-33,
    -0x1.ae7f3e733b81fp-41,
    0x1.952c77030ad4ap-49,
    -0x1.2f49b46814157p-57,
    0x1.71b8ef6dcf572p-66,
    -0x1.761b41316381ap-75,
};
constexpr double PI = 0x1.921fb54442d18p+1, PI_2 = 0x1.921fb54442d18p+0, PI_4 = 0x1.921fb54442d18p-1;
__device__ __forceinline__ double asin_p(double z) {
    const double z2 = __dmul_rn(z, z);
    double p = DT_ASIN[25];
#pragma unroll
    for (int k = 24; k >= 0; --k) p = fma(p, z2, DT_ASIN[k]);
    return __dmul_rn(z, p);
}
__device__ __forceinline__ double cos_p(double u) {
    const double u2 = __dmul_rn(u, u);
    double p = DT_COS[11];
#pragma unroll
    for (int k = 10; k >= 0; --k) p = fma(p, u2, DT_COS[k]);
    return p;
}
__device__ __forceinline__ double sin_p(double u) {
    const double u2 = __dmul_rn(u, u);
    double p = DT_SIN[11];
#pragma unroll
    for (int k = 10; k >= 0; --k) p = fma(p, u2, DT_SIN[k]);
    return __dmul_rn(u, p);
}
}  // namespace dt
static __device__ float det_acosf(float xf) {  // xf in [-1, 1]
    const double x = (double)xf;
    double r;
    if (x > 0.5) r = __dmul_rn(2.0, dt::asin_p(sqrt(__dmul_rn(__dsub_rn(1.0, x), 0.5))));
    else if (x < -0.5) r = __dsub_rn(dt::PI, __dmul_rn(2.0, dt::asin_p(sqrt(__dmul_rn(__dadd_rn(1.0, x), 0.5)))));
    else r = __dsub_rn(dt::PI_2, dt::asin_p(x));
    return (float)r;
}
// deterministic atan2f (fpfh.cu, shot.cu): float64, IEEE add / mul / div / sqrt only.  atan(t), t >= 0: two half-angle
// reductions t <- t / (1 + sqrt(1 + t^2)) (atan t = 2 atan of that) bring t below 0.2, then 13 Taylor terms (error < 1e-17).
__device__ __forceinline__ double dt_atan_pos(double t) {
    int doubled = 0;
    for (int k = 0; k < 3; ++k) {
        if (t > 0.2) {
            t = __ddiv_rn(t, __dadd_rn(1.0, sqrt(__dadd_rn(1.0, __dmul_rn(t, t)))));
            ++doubled;
        }
    }
    const double t2 = __dmul_rn(t, t);
    double p = 1.0 / 25.0;
#pragma unroll
    for (int k = 11; k >= 0; --k) p = __dsub_rn(1.0 / (double)(2 * k + 1), __dmul_rn(t2, p));
    double a = __dmul_rn(t, p);
    for (int k = 0; k < doubled; ++k) a = __dmul_rn(2.0, a);
    return a;
}
static __device__ float det_atan2f(float yf, float xf) {
    const double y = (double)yf, x = (double)xf;
    const double PI = 0x1.921fb54442d18p+1, PI_2 = 0x1.921fb54442d18p+0;
    if (x == 0.0 && y == 0.0) return copysignf((signbit(xf) ? (float)PI : 0.f), yf);
    const double ay = fabs(y), ax = fabs(x);
    double a;  // angle of (ax, ay) in [0, pi/2]
    if (ay <= ax) a = dt_atan_pos(__ddiv_rn(ay, ax));
    else a = __dsub_rn(PI_2, dt_atan_pos(__ddiv_rn(ax, ay)));
    if (x < 0.0) a = __dsub_rn(PI, a);
    return (float)(signbit(y) ? -a : a);  // atan2(-0, x < 0) = -pi, not +pi
}
static __device__ float det_cosf(float yf) {  // yf in [0, 2 pi]
    double y = (double)yf;
    if (y > dt::PI) y = __dsub_rn(__dmul_rn(2.0, dt::PI), y);
    double r;
    if (y <= dt::PI_4) r = dt::cos_p(y);
    else if (y <= __dmul_rn(3.0, dt::PI_4)) r = -dt::sin_p(__dsub_rn(y, dt::PI_2));
    else r = -dt::cos_p(__dsub_rn(dt::PI, y));
    return (float)r;
}
static __device__ void fast_eigen3x3(const float *Ain, float *eval, float *evec) {
    float A[9];
    float mc = Ain[0];
#pragma unroll
    for (int i = 0; i < 9; ++i) { A[i] = Ain[i]; if (Ain[i] > mc) mc = Ain[i]; }
    if (mc == 0) {
        eval[0] = eval[1] = eval[2] = 0;
#pragma unroll
        for (int i = 0; i < 9; ++i) evec[i] = (i % 4 == 0) ? 1.f : 0.f;
        return;
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) A[i] /= mc;
    float norm = __fmaf_rn(A[5], A[5], __fmaf_rn(A[2], A[2], A[1] * A[1]));
    if (norm > 0) {
        float q = (A[0] + A[4] + A[8]) / 3;
        float b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
        float p = sqrtf(__fmaf_rn(norm, 2.f, __fmaf_rn(b22, b22, __fmaf_rn(b11, b11, b00 * b00))) / 6);
        float c00 = det2(b11, b22, A[5], A[5]);
        float c01 = det2(A[1], b22, A[5], A[2]);
        float c02 = det2(A[1], A[5], b11, A[2]);
        float det = __fmaf_rn(A[2], c02, __fmaf_rn(-A[1], c01, b00 * c00)) / (p * p * p);
        float half_det = det * 0.5f;
        half_det = fminf(fmaxf(half_det, -1.0f), 1.0f);
        float angle = det_acosf(half_det) / (float)3;
        const float two_thirds_pi = 2.09439510239319549f;
        float beta2 = det_cosf(angle) * 2;
        float beta0 = det_cosf(angle + two_thirds_pi) * 2;
        float beta1 = -(beta0 + beta2);
        eval[0] = __fmaf_rn(p, beta0, q);
        eval[1] = __fmaf_rn(p, beta1, q);
        eval[2] = __fmaf_rn(p, beta2, q);
        float c0[3], c1[3], c2[3];
        if (half_det >= 0) {
            eigvec0(A, eval[2], c2);
            eigvec1(A, c2, eval[1], c1);
            cross3(c1, c2, c0);
        } else {
            eigvec0(A, eval[0], c0);
            eigvec1(A, c0, eval[1], c1);
            cross3(c0, c1, c2);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) { evec[3 * r] = c0[r]; evec[3 * r + 1] = c1[r]; evec[3 * r + 2] = c2[r]; }
    } else {
        eval[0] = Ain[0]; eval[1] = Ain[4]; eval[2] = Ain[8];
#pragma unroll
        for (int i = 0; i < 9; ++i) evec[i] = (i % 4 == 0) ? 1.f : 0.f;
    }
}
static __device__ void sqrt_matrix3x3(const float *A, float *W) {
    float e[3], V[9], VD[9];
    fast_eigen3x3(A, e, V);
    float s[3] = {sqrtf(e[0]), sqrtf(e[1]), sqrtf(e[2])};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) VD[3 * i + k] = V[3 * i + k] * s[k];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            W[3 * i + j] = dot3(VD[3 * i], VD[3 * i + 1], VD[3 * i + 2], V[3 * j], V[3 * j + 1], V[3 * j + 2]);
}
static __device__ void inverse3x3(const float *m, float *inv) {
    float cof[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            cof[3 * i + j] = det2(m[3 * i1 + j1], m[3 * i2 + j2], m[3 * i1 + j2], m[3 * i2 + j1]);
        }
    float det = dot3(cof[0], cof[3], cof[6], m[0], m[3], m[6]);
    float invdet = 1.0f / det;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) inv[3 * i + j] = cof[3 * j + i] * invdet;
}

