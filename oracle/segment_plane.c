/*
 * segment_plane.c -- CPU restatement of cupoch's PointCloud::SegmentPlane (geometry/segmentation.cu:36-267).
 * TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and tools/bench_ops.py through segment_plane_py.py,
 * never by the product.  Built by segment_plane_py.build() with oracle/Makefile's flags: -ffp-contract=off (no
 * implicit FMA; the one fused multiply-add, dot3f, is explicit) and no -ffast-math.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* SegmentPlane with the T seeds the reference draws from rand(): plane [a,b,c,d] of the refit, idx [n] the ascending
 * final inliers (*m of them), *best the winning iteration (-1 if none), fr = {fitness, inlier_rmse} of the winner.
 * ransac_n < 3 or n < ransac_n: zero plane, no inliers.  Returns 0, -1 for T < 0.  Its sampler: the n keys
 * random_functor(seed, n) tabulates, and the T samples (3 indices each) of the sort chain. */
int orc_segment_plane(const float *pts, int n, float thr, int ransac_n, int T, const int32_t *seeds, float plane[4],
                      int32_t *idx, int *m_out, int *best_out, float fr[2]);
void orc_ransac_keys(int32_t seed, int n, int32_t *keys);
void orc_ransac_samples(int n, int T, const int32_t *seeds, int32_t *samples);

/* the arithmetic contract's device-code dot product (oracle.c, DESIGN.md) */
static inline float dot3f(float a0, float a1, float a2, float b0, float b1, float b2) {
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0));
}

/* Summation order (DESIGN.md arithmetic contract): every sum over points or over inliers is taken over tiles of
 * SEG_TILE consecutive elements, each tile summed sequentially in double from 0.0, then the tile sums added in tile
 * order.  The refit's determinant step cancels badly for axis-aligned planes, so the order is part of the answer. */
#define SEG_TILE 1024
#define LCG_A 48271u      /* thrust::minstd_rand = default_random_engine (thrust/random.h) */
#define LCG_M 2147483647u /* 2^31 - 1 */

static inline uint32_t lcg_mulmod(uint32_t x, uint32_t y) {
    const uint64_t p = (uint64_t)x * y;
    uint64_t r = (p & LCG_M) + (p >> 31);
    r = (r & LCG_M) + (r >> 31);
    return (uint32_t)(r >= LCG_M ? r - LCG_M : r);
}

/* random_functor (segmentation.cu:38-48) at positions 0..n-1: default_random_engine(seed) -- the int seed converted
 * to the engine's uint32_t, reduced mod m, 0 -> 1 (linear_congruential_engine.inl seed()) --, discard(p), one draw u,
 * uniform_int_distribution<int>(0, n-1), which goes through uniform_real_distribution<double>(0, (n-1) + 1):
 * (u - min) / (1 + max - min) * ((n-1) + 1 - 0) + 0, truncated to int (uniform_{int,real}_distribution.inl). */
void orc_ransac_keys(int32_t seed, int n, int32_t *keys) {
    uint32_t x = (uint32_t)seed % LCG_M;
    if (x == 0) x = 1;
    const double span = (double)(n - 1) + 1.0;
    for (int p = 0; p < n; ++p) {
        x = lcg_mulmod(x, LCG_A);
        keys[p] = (int32_t)(((double)(x - 1u) / 2147483646.0) * span + 0.0);
    }
}

/* segmentation.cu:214-229: d_cards = 0..n-1 once, then per iteration tabulate the keys and stable-sort d_cards by them
 * (thrust's radix sort of int keys is stable); the sample is d_cards[0..2].  Keys lie in [0, n): a counting sort. */
void orc_ransac_samples(int n, int T, const int32_t *seeds, int32_t *samples) {
    int32_t *cards = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    int32_t *tmp = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    int32_t *keys = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    int32_t *start = (int32_t *)malloc(sizeof(int32_t) * ((size_t)n + 1));
    for (int i = 0; i < n; ++i) cards[i] = i;
    for (int t = 0; t < T; ++t) {
        orc_ransac_keys(seeds[t], n, keys);
        memset(start, 0, sizeof(int32_t) * ((size_t)n + 1));
        for (int p = 0; p < n; ++p) ++start[keys[p] + 1];
        for (int k = 0; k < n; ++k) start[k + 1] += start[k];
        for (int p = 0; p < n; ++p) tmp[start[keys[p]]++] = cards[p];
        int32_t *sw = cards;
        cards = tmp;
        tmp = sw;
        for (int k = 0; k < 3; ++k) samples[3 * (size_t)t + k] = cards[k];
    }
    free(cards);
    free(tmp);
    free(keys);
    free(start);
}

/* ComputeTrianglePlane (segmentation.cu:60-74), host code compiled without FMA: unfused float32, Eigen's cross
 * product, norm = sqrtf((x*x + y*y) + z*z), per-component division, d = -((a*x + b*y) + c*z). */
static void seg_triangle_plane(const float *p0, const float *p1, const float *p2, float pl[4]) {
    const float e0[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
    const float e1[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
    float a = e0[1] * e1[2] - e0[2] * e1[1];
    float b = e0[2] * e1[0] - e0[0] * e1[2];
    float c = e0[0] * e1[1] - e0[1] * e1[0];
    const float norm = sqrtf((a * a + b * b) + c * c);
    if (norm == 0.f) { pl[0] = pl[1] = pl[2] = pl[3] = 0.f; return; }
    a /= norm; b /= norm; c /= norm;
    pl[0] = a; pl[1] = b; pl[2] = c;
    pl[3] = -((a * p0[0] + b * p0[1]) + c * p0[2]);
}

/* compute_distance_functor (:50-58), device code: |plane . (x, y, z, 1)| with the contract's dot3 */
static inline float seg_dist(const float pl[4], const float *p) {
    return fabsf(dot3f(pl[0], pl[1], pl[2], p[0], p[1], p[2]) + pl[3]);
}

/* SegmentPlane (:187-267) with the caller's T seeds (the reference draws seed_t = rand() in iteration t).
 * EvaluateRANSACBasedOnDistance (:94-128): strict dist < thr; fitness = (float)count / (float)n; "inlier_rmse" =
 * (float)(double sum of the inlier distances) / sqrtf((float)count) -- a sum of distances, mirrored as written.
 * Selection: fitness >, or == with rmse <, starting from (0, 0).  Final inliers against the best plane (the zero
 * plane if none won: every finite point), then GetPlaneFromPoints (:135-185): centroid and six second moments as
 * tiled double sums rounded once, the rest unfused float32 host arithmetic.  Returns 0, or -1 for T < 0. */
int orc_segment_plane(const float *pts, int n, float thr, int ransac_n, int T, const int32_t *seeds, float plane[4],
                      int32_t *idx, int *m_out, int *best_out, float fr[2]) {
    plane[0] = plane[1] = plane[2] = plane[3] = 0.f;
    *m_out = 0;
    *best_out = -1;
    fr[0] = fr[1] = 0.f;
    if (T < 0) return -1;
    if (ransac_n < 3 || n < ransac_n) return 0; /* :204-212: logged, zero plane, no inliers */
    int32_t *samples = (int32_t *)malloc(sizeof(int32_t) * 3 * (size_t)(T > 0 ? T : 1));
    orc_ransac_samples(n, T, seeds, samples);
    float best_pl[4] = {0.f, 0.f, 0.f, 0.f}, best_fit = 0.f, best_rmse = 0.f;
    int best = -1;
    for (int t = 0; t < T; ++t) {
        float pl[4];
        const int32_t *s = samples + 3 * (size_t)t;
        seg_triangle_plane(pts + 3 * (size_t)s[0], pts + 3 * (size_t)s[1], pts + 3 * (size_t)s[2], pl);
        if (pl[0] == 0.f && pl[1] == 0.f && pl[2] == 0.f && pl[3] == 0.f) continue; /* isZero(0) */
        long cnt = 0;
        double sum = 0.0;
        for (int base = 0; base < n; base += SEG_TILE) {
            const int end = base + SEG_TILE < n ? base + SEG_TILE : n;
            long c = 0;
            double ts = 0.0;
            for (int i = base; i < end; ++i) {
                const float d = seg_dist(pl, pts + 3 * (size_t)i);
                if (d < thr) { ++c; ts += (double)d; }
            }
            cnt += c;
            sum += ts;
        }
        const float fit = cnt ? (float)cnt / (float)n : 0.f;
        const float rmse = cnt ? (float)sum / sqrtf((float)cnt) : 0.f;
        if (fit > best_fit || (fit == best_fit && rmse < best_rmse)) {
            best_fit = fit; best_rmse = rmse; best = t;
            memcpy(best_pl, pl, sizeof(best_pl));
        }
    }
    free(samples);
    int m = 0;
    for (int i = 0; i < n; ++i)
        if (seg_dist(best_pl, pts + 3 * (size_t)i) < thr) idx[m++] = i;
    /* GetPlaneFromPoints */
    double S[6] = {0, 0, 0, 0, 0, 0};
    for (int base = 0; base < m; base += SEG_TILE) {
        const int end = base + SEG_TILE < m ? base + SEG_TILE : m;
        double ts[3] = {0, 0, 0};
        for (int k = base; k < end; ++k)
            for (int a = 0; a < 3; ++a) ts[a] += (double)pts[3 * (size_t)idx[k] + a];
        for (int a = 0; a < 3; ++a) S[a] += ts[a];
    }
    float cen[3];
    for (int a = 0; a < 3; ++a) cen[a] = (float)S[a] / (float)m; /* m == 0: NaN, unused (zero moments below) */
    double M[6] = {0, 0, 0, 0, 0, 0};
    for (int base = 0; base < m; base += SEG_TILE) {
        const int end = base + SEG_TILE < m ? base + SEG_TILE : m;
        double ts[6] = {0, 0, 0, 0, 0, 0};
        for (int k = base; k < end; ++k) {
            const float *p = pts + 3 * (size_t)idx[k];
            const float r0 = p[0] - cen[0], r1 = p[1] - cen[1], r2 = p[2] - cen[2];
            const float prod[6] = {r0 * r0, r0 * r1, r0 * r2, r1 * r1, r1 * r2, r2 * r2};
            for (int j = 0; j < 6; ++j) ts[j] += (double)prod[j];
        }
        for (int j = 0; j < 6; ++j) M[j] += ts[j];
    }
    float mu[6];
    for (int j = 0; j < 6; ++j) mu[j] = (float)M[j];
    const float det_x = mu[3] * mu[5] - mu[4] * mu[4];
    const float det_y = mu[0] * mu[5] - mu[2] * mu[2];
    const float det_z = mu[0] * mu[3] - mu[1] * mu[1];
    float abc[3];
    if (det_x > det_y && det_x > det_z) {
        abc[0] = det_x; abc[1] = mu[2] * mu[4] - mu[1] * mu[5]; abc[2] = mu[1] * mu[4] - mu[2] * mu[3];
    } else if (det_y > det_z) {
        abc[0] = mu[2] * mu[4] - mu[1] * mu[5]; abc[1] = det_y; abc[2] = mu[1] * mu[2] - mu[4] * mu[0];
    } else {
        abc[0] = mu[1] * mu[4] - mu[2] * mu[3]; abc[1] = mu[1] * mu[2] - mu[4] * mu[0]; abc[2] = det_z;
    }
    const float norm = sqrtf((abc[0] * abc[0] + abc[1] * abc[1]) + abc[2] * abc[2]);
    if (norm != 0.f) {
        for (int a = 0; a < 3; ++a) plane[a] = abc[a] / norm;
        plane[3] = -((plane[0] * cen[0] + plane[1] * cen[1]) + plane[2] * cen[2]);
    }
    *m_out = m;
    *best_out = best;
    fr[0] = best_fit;
    fr[1] = best_rmse;
    return 0;
}
