/*
 * crop.c -- CPU restatement of cupoch's bounding-box selection and point-cloud cleanup (SURVEY 8f rank 10).
 * TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and tools/bench_ops.py through crop_py.py, never by the
 * product.  Built by oracle.build() (oracle/__init__.py): -ffp-contract=off, no -ffast-math, OpenMP.
 *
 * oracle.c is compiled into this translation unit (the #include below) for its dot3f / det2f conventions and its
 * one-sided Jacobi svd3, which serves as the symmetric eigensolver.  The arithmetic is DESIGN.md's arithmetic
 * contract; see also csrc/crop.cu.
 */
#include "oracle.c"

#define CROP_TILE 1024 /* moment-sum tile (the SegmentPlane order) */

void orc_crop_aabb(const float *pts, int n, const float lo[3], const float hi[3], uint8_t *keep);
void orc_crop_obb(const float *pts, int n, const float box[24], uint8_t *keep);
void orc_crop_finite(const float *pts, int n, int remove_nan, int remove_infinite, uint8_t *keep);
void orc_obb_create(const float *pts, int n, float center[3], float R[9], float extent[3]);
int orc_uniform_down_sample(int n, int every_k, int32_t *rows);
void orc_normalize_normals(float *nrm, int n);
void orc_orient_normals(float *nrm, int n, const float ref[3]);

/* check_within_axis_aligned_bounding_box_functor (geometry/boundingvolume.cu:82-101): dropped only when a coordinate is
 * below its min or above its max, so NaN coordinates are kept; PassThroughFilter (pointcloud.cu:105-121) is this test
 * with +-inf on the two other axes */
void orc_crop_aabb(const float *pts, int n, const float lo[3], const float hi[3], uint8_t *keep) {
#pragma omp parallel for
    for (int i = 0; i < n; ++i) {
        const float *p = pts + 3 * (size_t)i;
        int out = 0;
        for (int a = 0; a < 3; ++a)
            if (p[a] < lo[a] || p[a] > hi[a]) out = 1;
        keep[i] = (uint8_t)!out;
    }
}

/* test_plane (boundingvolume.cu:43-50): det[b - a | c - a | x - a], Eigen's first-row expansion
 * u0 (v1 w2 - w1 v2) - v0 (u1 w2 - w1 u2) + w0 (u1 v2 - v1 u2) with det2f minors and two fmaf */
static float test_plane(const float *a, const float *b, const float *c, const float *x) {
    const float u0 = b[0] - a[0], u1 = b[1] - a[1], u2 = b[2] - a[2];
    const float v0 = c[0] - a[0], v1 = c[1] - a[1], v2 = c[2] - a[2];
    const float w0 = x[0] - a[0], w1 = x[1] - a[1], w2 = x[2] - a[2];
    const float m0 = det2f(v1, w2, w1, v2), m1 = det2f(u1, w2, w1, u2), m2 = det2f(u1, v2, v1, u2);
    return fmaf(w0, m2, fmaf(-v0, m1, u0 * m0));
}

/* check_within_oriented_bounding_box_functor (boundingvolume.cu:51-79): the six plane tests over GetBoxPoints(), either
 * sign pattern */
void orc_crop_obb(const float *pts, int n, const float box[24], uint8_t *keep) {
    const float *b0 = box, *b1 = box + 3, *b2 = box + 6, *b3 = box + 9, *b4 = box + 12, *b5 = box + 15, *b7 = box + 21;
#pragma omp parallel for
    for (int i = 0; i < n; ++i) {
        const float *p = pts + 3 * (size_t)i;
        const float d0 = test_plane(b0, b1, b3, p), d1 = test_plane(b0, b5, b3, p), d2 = test_plane(b2, b5, b7, p);
        const float d3 = test_plane(b1, b4, b7, p), d4 = test_plane(b3, b4, b5, p), d5 = test_plane(b0, b1, b7, p);
        keep[i] = (uint8_t)((d0 <= 0 && d1 >= 0 && d2 <= 0 && d3 >= 0 && d4 <= 0 && d5 >= 0) ||
                            (d0 >= 0 && d1 <= 0 && d2 >= 0 && d3 <= 0 && d4 >= 0 && d5 <= 0));
    }
}

/* check_nan_functor (pointcloud.cu:38-53), negated */
void orc_crop_finite(const float *pts, int n, int remove_nan, int remove_infinite, uint8_t *keep) {
#pragma omp parallel for
    for (int i = 0; i < n; ++i) {
        const float *p = pts + 3 * (size_t)i;
        const int is_nan = remove_nan && (isnan(p[0]) || isnan(p[1]) || isnan(p[2]));
        const int is_inf = remove_infinite && (isinf(p[0]) || isinf(p[1]) || isinf(p[2]));
        keep[i] = (uint8_t)!(is_nan || is_inf);
    }
}

/* the order-preserving float -> uint map of the min/max bound (NaN with the sign bit clear above +inf, set below -inf) */
static uint32_t ord_f(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
static float f_ord(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

/* OrientedBoundingBox::CreateFromPoints (boundingvolume.cu:219-269), as DESIGN.md restates it:
 *   mean: coordinates summed in double over tiles of CROP_TILE points (each tile from 0.0 in order, then the tiles in
 *         order), divided by n in double;
 *   cov:  the six products ((double)p_a - mean_a) * ((double)p_b - mean_b) summed the same way, divided by n;
 *   axes: svd3's V (eigenvectors of the symmetric cov), each column normalised, the reference's three swaps (:242-253)
 *         by eigenvalue, then each column signed so its largest-magnitude component (first among equals) is positive;
 *   box:  p' = dot3f(R^T row, p) + t with t = -dot3f(R^T row, mean_f) in float32, its ordered min/max, centre
 *         (min + max) * 0.5f, extent max - min, center = dot3f(R row, centre) + mean_f.
 * n == 0 gives the zero box with R = I. */
void orc_obb_create(const float *pts, int n, float center[3], float R[9], float extent[3]) {
    for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.f : 0.f;
    for (int a = 0; a < 3; ++a) center[a] = extent[a] = 0.f;
    if (n <= 0) return;
    double S[3] = {0, 0, 0};
    for (int base = 0; base < n; base += CROP_TILE) {
        const int end = base + CROP_TILE < n ? base + CROP_TILE : n;
        double t[3] = {0, 0, 0};
        for (int i = base; i < end; ++i)
            for (int a = 0; a < 3; ++a) t[a] += (double)pts[3 * (size_t)i + a];
        for (int a = 0; a < 3; ++a) S[a] += t[a];
    }
    double mean[3];
    for (int a = 0; a < 3; ++a) mean[a] = S[a] / (double)n;
    static const int PA[6] = {0, 0, 0, 1, 1, 2}, PB[6] = {0, 1, 2, 1, 2, 2};
    double M[6] = {0, 0, 0, 0, 0, 0};
    for (int base = 0; base < n; base += CROP_TILE) {
        const int end = base + CROP_TILE < n ? base + CROP_TILE : n;
        double t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = base; i < end; ++i) {
            const float *p = pts + 3 * (size_t)i;
            for (int j = 0; j < 6; ++j) t[j] += ((double)p[PA[j]] - mean[PA[j]]) * ((double)p[PB[j]] - mean[PB[j]]);
        }
        for (int j = 0; j < 6; ++j) M[j] += t[j];
    }
    const double nd = (double)n;
    const double c00 = M[0] / nd, c01 = M[1] / nd, c02 = M[2] / nd, c11 = M[3] / nd, c12 = M[4] / nd, c22 = M[5] / nd;
    const double cov[9] = {c00, c01, c02, c01, c11, c12, c02, c12, c22};
    double U[9], ev[3], V[9];
    svd3(cov, U, ev, V);
    for (int c = 0; c < 3; ++c) {
        const double nn = sqrt(V[c] * V[c] + V[3 + c] * V[3 + c] + V[6 + c] * V[6 + c]);
        for (int r = 0; r < 3; ++r) V[3 * r + c] /= nn;
    }
    static const int SW[3][2] = {{1, 0}, {2, 0}, {2, 1}};
    for (int k = 0; k < 3; ++k) {
        const int a = SW[k][0], b = SW[k][1];
        if (ev[a] > ev[b]) {
            double t = ev[a];
            ev[a] = ev[b];
            ev[b] = t;
            for (int r = 0; r < 3; ++r) {
                t = V[3 * r + a];
                V[3 * r + a] = V[3 * r + b];
                V[3 * r + b] = t;
            }
        }
    }
    for (int c = 0; c < 3; ++c) {
        int big = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(V[3 * r + c]) > fabs(V[3 * big + c])) big = r;
        const double sg = V[3 * big + c] < 0.0 ? -1.0 : 1.0;
        for (int r = 0; r < 3; ++r) R[3 * r + c] = (float)(sg * V[3 * r + c]);
    }
    const float mf[3] = {(float)mean[0], (float)mean[1], (float)mean[2]};
    float t[3];
    for (int i = 0; i < 3; ++i) t[i] = -dot3f(R[i], R[3 + i], R[6 + i], mf[0], mf[1], mf[2]);
    uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0, 0, 0};
    for (int k = 0; k < n; ++k) {
        const float *p = pts + 3 * (size_t)k;
        for (int i = 0; i < 3; ++i) {
            const uint32_t o = ord_f(dot3f(R[i], R[3 + i], R[6 + i], p[0], p[1], p[2]) + t[i]);
            if (o < lo[i]) lo[i] = o;
            if (o > hi[i]) hi[i] = o;
        }
    }
    float c[3];
    for (int a = 0; a < 3; ++a) {
        const float mn = f_ord(lo[a]), mx = f_ord(hi[a]);
        c[a] = (mn + mx) * 0.5f;
        extent[a] = mx - mn;
    }
    for (int i = 0; i < 3; ++i) center[i] = dot3f(R[3 * i], R[3 * i + 1], R[3 * i + 2], c[0], c[1], c[2]) + mf[i];
}

/* UniformDownSample (down_sample.cu:275-300): rows 0, k, 2k, ... -- n / k of them, rounded down (the reference sizes
 * its output so but copies ceil(n / k)); k < 1 gives -1 */
int orc_uniform_down_sample(int n, int every_k, int32_t *rows) {
    if (every_k < 1) return -1;
    const int m = n / every_k;
    for (int t = 0; t < m; ++t) rows[t] = t * every_k;
    return m;
}

/* NormalizeNormals (pointcloud.cu:282-285): Eigen's normalize(), n /= sqrtf(|n|^2) when |n|^2 > 0 */
void orc_normalize_normals(float *nrm, int n) {
#pragma omp parallel for
    for (int i = 0; i < n; ++i) {
        float *v = nrm + 3 * (size_t)i;
        const float n2 = dot3f(v[0], v[1], v[2], v[0], v[1], v[2]);
        if (!(n2 > 0.f)) continue;
        const float l = sqrtf(n2);
        for (int a = 0; a < 3; ++a) v[a] = v[a] / l;
    }
}

/* align_normals_direction_functor (estimate_normals.cu:66-78): a zero normal becomes ref; n . ref < 0 negates n */
void orc_orient_normals(float *nrm, int n, const float ref[3]) {
#pragma omp parallel for
    for (int i = 0; i < n; ++i) {
        float *v = nrm + 3 * (size_t)i;
        if (dot3f(v[0], v[1], v[2], v[0], v[1], v[2]) == 0.f) {
            for (int a = 0; a < 3; ++a) v[a] = ref[a];
        } else if (dot3f(v[0], v[1], v[2], ref[0], ref[1], ref[2]) < 0.f) {
            for (int a = 0; a < 3; ++a) v[a] = -v[a];
        }
    }
}
