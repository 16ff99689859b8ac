/*
 * iss.c -- CPU restatement of cupoch's geometry::keypoint::ComputeISSKeypoints (geometry/iss_keypoints.cu:37-172).
 * TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and tools/bench_ops.py through iss_py.py, never by the
 * product.  Built by oracle.build() (oracle/__init__.py): -ffp-contract=off, no -ffast-math, OpenMP.
 *
 * oracle.c is compiled into this translation unit (the #include below), so the kd-tree search with its result set and
 * tie rule (kd_search_rec, rset_*) and the FastEigen3x3 restatement (fast_eigen3x3, static there) are the oracle's
 * own code, unchanged.  The per-point arithmetic is DESIGN.md's arithmetic contract; see also csrc/iss.cu.
 */
#include "oracle.c"

#define ISS_TILE 1024        /* resolution-sum tile (the SegmentPlane order) */
#define ISS_MAX_NN 256       /* the radius search's limit */
#define ISS_ZERO_PREC 1e-5f  /* Eigen::NumTraits<float>::dummy_precision() */

int orc_iss_keypoints(const float *pts, int n, float salient_radius, float non_max_radius, float gamma_21, float gamma_32,
                      int min_neighbors, int max_neighbors, uint8_t *mask, float *saliency, float radii[2]);

/* ComputeModelResolution (:37-49): kNN-2 of every point, slot-1 d2 summed over tiles of ISS_TILE consecutive points
 * (each sequentially in double from 0, then the tiles in order), rounded to float once; sqrtf(sum / (float)n) */
static float iss_resolution(const orc_kdtree *t, const float *pts, int n) {
    float *d = (float *)malloc(sizeof(float) * (size_t)n);
#pragma omp parallel for schedule(dynamic, 256)
    for (int q = 0; q < n; ++q) {
        int32_t idx[2];
        float d2[2];
        rset s;
        rset_init(&s, 2, -1.0f, idx, d2);
        kd_search_rec(t, 0, pts + 3 * (size_t)q, &s);
        d[q] = d2[1]; /* +inf for a one-point cloud */
    }
    double sum = 0.0;
    for (int base = 0; base < n; base += ISS_TILE) {
        const int end = base + ISS_TILE < n ? base + ISS_TILE : n;
        double ts = 0.0;
        for (int i = base; i < end; ++i) ts += (double)d[i];
        sum += ts;
    }
    free(d);
    return sqrtf((float)sum / (float)n);
}

/* KDTreeFlann::SearchRadius(q, radius, k) of one query: the <= k nearest with d2 < radius * radius (float), ascending by
 * (d2, index), unfilled slots -1.  A negative radius acts as |radius| (the search squares it); radius * radius == 0 or
 * NaN lists nothing (strict d2 < r2).  (rset_init reads radius <= 0 as "no radius", so the radius goes in as |r|.) */
static void iss_list(const orc_kdtree *t, const float *q, int k, float radius, int32_t *idx, float *d2) {
    for (int j = 0; j < k; ++j) idx[j] = -1;
    if (k == 0 || !(radius * radius > 0.0f)) return;
    rset s;
    rset_init(&s, k, fabsf(radius), idx, d2);
    kd_search_rec(t, 0, q, &s);
}

/* compute_third_eigen_values_functor + ComputeThirdEigenValue (:51-81): the cumulants as orc_normals_from_neighbors forms
 * them, the covariance, Eigen's isZero() (|c| <= 1e-5 for every coefficient: absolute), FastEigen3x3Val (eigenvalue.inl
 * :164-170; minCoeff / maxCoeff keep the first strict improvement), the ratio tests */
static float iss_saliency(const float *pts, const int32_t *idx, int k, int min_neighbors, float gamma_21, float gamma_32) {
    double cum[9] = {0};
    int cnt = 0;
    for (int j = 0; j < k; ++j) {
        if (idx[j] < 0) continue;
        const float *p = pts + 3 * (size_t)idx[j];
        cum[0] += p[0]; cum[1] += p[1]; cum[2] += p[2];
        cum[3] += (double)p[0] * p[0]; cum[4] += (double)p[0] * p[1];
        cum[5] += (double)p[0] * p[2]; cum[6] += (double)p[1] * p[1];
        cum[7] += (double)p[1] * p[2]; cum[8] += (double)p[2] * p[2];
        ++cnt;
    }
    if (cnt < min_neighbors) return -1.0f;
    float cov[9];
    covariance_from_cumulants(cum, cnt, cov); /* cnt == 0: NaN, which fails every test below */
    int zero = 1;
    for (int a = 0; a < 9; ++a) zero = zero && fabsf(cov[a]) <= ISS_ZERO_PREC;
    if (zero) return -1.0f;
    float e[3], V[9];
    fast_eigen3x3(cov, e, V);
    float mn = e[0], mx = e[0];
    if (e[1] < mn) mn = e[1];
    if (e[2] < mn) mn = e[2];
    if (e[1] > mx) mx = e[1];
    if (e[2] > mx) mx = e[2];
    const float mid = ((e[0] + e[1]) + e[2] - mn) - mx;
    return (mx > 0.0f && mid / mx < gamma_21 && mn / mid < gamma_32) ? mn : -1.0f;
}

/* ComputeISSKeypoints (:108-172) -> the keypoint count; mask[n], saliency[n] and the radii used.  n <= 0: 0 keypoints,
 * radii as given; max_neighbors outside [0, ISS_MAX_NN]: -1. */
int orc_iss_keypoints(const float *pts, int n, float salient_radius, float non_max_radius, float gamma_21, float gamma_32,
                      int min_neighbors, int max_neighbors, uint8_t *mask, float *saliency, float radii[2]) {
    radii[0] = salient_radius;
    radii[1] = non_max_radius;
    if (max_neighbors < 0 || max_neighbors > ISS_MAX_NN) return -1;
    if (n <= 0) return 0;
    orc_kdtree *t = orc_kdtree_build(pts, n);
    if (salient_radius == 0.0f || non_max_radius == 0.0f) { /* :124: both are replaced */
        const float resolution = iss_resolution(t, pts, n);
        radii[0] = 6 * resolution;
        radii[1] = 4 * resolution;
    }
    const int k = max_neighbors;
#pragma omp parallel for schedule(dynamic, 256)
    for (int i = 0; i < n; ++i) {
        int32_t idx[ISS_MAX_NN];
        float d2[ISS_MAX_NN];
        iss_list(t, pts + 3 * (size_t)i, k, radii[0], idx, d2);
        saliency[i] = iss_saliency(pts, idx, k, min_neighbors, gamma_21, gamma_32);
    }
    int count = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : count)
    for (int i = 0; i < n; ++i) { /* is_local_maxima_functor (:83-101) */
        const float q = saliency[i];
        int keep = !(q < 0.0f);
        if (keep) {
            int32_t idx[ISS_MAX_NN];
            float d2[ISS_MAX_NN];
            iss_list(t, pts + 3 * (size_t)i, k, radii[1], idx, d2);
            for (int j = 0; j < k && keep; ++j)
                if (idx[j] >= 0 && q < saliency[idx[j]]) keep = 0;
        }
        mask[i] = (uint8_t)keep;
        count += keep;
    }
    orc_kdtree_free(t);
    return count;
}
