// C glue around the reference's NoDivTriTriIsect (third_party/tomasakeninemoeller/opttritri.h, #included as it lies in
// the checkout): ref_tritri(p, q) = intersection_test::TriangleTriangle3d(p0, p1, p2, q0, q1, q2)
// (intersection_test.inl:47-69).  Only the normalisation is restated here, in float32 in Eigen's evaluation order:
// mu = (p0 + p1 + p2 + q0 + q1 + q2) / 6, sigma = sqrt(sum of the six squared deviations / 5) + 1e-12, x' = (x - mu) / sigma.
#define __host__
#define __device__
#include <math.h>

#include <tomasakeninemoeller/opttritri.h>

extern "C" int ref_tritri(const float *p, const float *q) {
    float mu[3], sg[3], pm[9], qm[9];
    for (int k = 0; k < 3; ++k) {
        mu[k] = (p[k] + p[3 + k] + p[6 + k] + q[k] + q[3 + k] + q[6 + k]) / 6.0f;
        float s = 0.0f;
        for (int j = 0; j < 6; ++j) {
            const float x = (j < 3 ? p[3 * j + k] : q[3 * (j - 3) + k]) - mu[k];
            s = j == 0 ? x * x : s + x * x;
        }
        sg[k] = sqrtf(s / 5.0f) + 1e-12f;
        for (int j = 0; j < 3; ++j) {
            pm[3 * j + k] = (p[3 * j + k] - mu[k]) / sg[k];
            qm[3 * j + k] = (q[3 * j + k] - mu[k]) / sg[k];
        }
    }
    return NoDivTriTriIsect(pm, pm + 3, pm + 6, qm, qm + 3, qm + 6) != 0;
}

extern "C" void ref_tritri_many(const float *p, const float *q, long long n, unsigned char *out) {
    for (long long i = 0; i < n; ++i) out[i] = (unsigned char)ref_tritri(p + 9 * i, q + 9 * i);
}
