/*
 * shot.c -- CPU restatement of cupoch's registration::ComputeSHOTFeature (registration/shot.cu:33-255).
 * TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and tools/bench_ops.py through shot_py.py, never by the
 * product.  Built by oracle.build() (oracle/__init__.py): -ffp-contract=off, no -ffast-math, OpenMP.
 *
 * oracle.c is compiled into this translation unit (the #include below), so the kd-tree search with its result set and
 * tie rule (kd_search_rec, rset_*), the FastEigen3x3 restatement (fast_eigen3x3) and the deterministic det_acosf /
 * det_atan2f are the oracle's own code, unchanged.  The per-point arithmetic is DESIGN.md's arithmetic contract; see
 * also csrc/shot.cu.
 */
#include "oracle.c"

#define SHOT_DIM 352
#define SHOT_BINS 10
#define SHOT_MIN_NB 5
#define SHOT_SECTORS 32
#define SHOT_KNN_MAX 100
#define SHOT_RADIUS_MAX 256

static const float PST_RAD_45 = 0.78539816339744830961566084581988f;
static const float PST_RAD_90 = 1.5707963267948966192313216916398f;
static const float PST_RAD_135 = 2.3561944901923449288469825374596f;
static const float PST_RAD_PI_7_8 = 2.7488935718910690836548129603691f;

int orc_shot_neighbours(const float *pts, int n, int knn, float search_radius, int max_nn, int32_t *idx, float *d2);
int orc_compute_shot_feature(const float *pts, const float *nrm, int n, float radius, int knn, float search_radius,
                             int max_nn, float *out);

/* min(max(v, lo), hi) with a float v and double bounds: double fmax / fmin (NaN loses), rounded to float */
static float clamp_d(float v, double lo, double hi) { return (float)fmin(fmax((double)v, lo), hi); }

/* the search the reference runs (shot.cu:233-245): knn > 0 -> KNN(knn), else Radius(search_radius, max_nn); the <= k
 * nearest with d2 < r2 ascending by (d2, index), unfilled slots -1.  r2 = search_radius * search_radius (float); r2 == 0
 * or NaN lists nothing. */
static void shot_list(const orc_kdtree *t, const float *q, int knn, float search_radius, int k, int32_t *idx, float *d2) {
    for (int j = 0; j < k; ++j) { idx[j] = -1; d2[j] = INFINITY; }
    if (k == 0) return;
    if (knn <= 0 && !(search_radius * search_radius > 0.0f)) return;
    rset s;
    rset_init(&s, k, knn > 0 ? -1.0f : fabsf(search_radius), idx, d2);
    kd_search_rec(t, 0, q, &s);
}

static int shot_k(int knn, int max_nn) {
    if (knn > 0) return knn <= SHOT_KNN_MAX ? knn : -1;
    return (max_nn >= 0 && max_nn <= SHOT_RADIUS_MAX) ? max_nn : -1;
}

/* the neighbour tables [n][k] the descriptor reads (k as shot_k); -1 for illegal arguments, else k */
int orc_shot_neighbours(const float *pts, int n, int knn, float search_radius, int max_nn, int32_t *idx, float *d2) {
    const int k = shot_k(knn, max_nn);
    if (k < 0) return -1;
    if (n <= 0 || k == 0) return k;
    orc_kdtree *t = orc_kdtree_build(pts, n);
#pragma omp parallel for schedule(dynamic, 256)
    for (int i = 0; i < n; ++i)
        shot_list(t, pts + 3 * (size_t)i, knn, search_radius, k, idx + (size_t)i * k, d2 + (size_t)i * k);
    orc_kdtree_free(t);
    return k;
}

/* compute_shot_lrf (:63-98): x, y, z axes; returns n_nb */
static int shot_lrf(const float *pts, int i, const int32_t *idx, const float *d2, int k, float radius, float X[3],
                    float Y[3], float Z[3]) {
    const float *pi = pts + 3 * (size_t)i;
    float cov[9] = {0};
    float w_total = 0.0f;
    int n_nb = 0;
    for (int j = 0; j < k; ++j) {
        const int id = idx[j];
        if (id < 0 || id == i) continue;
        const float *pj = pts + 3 * (size_t)id;
        const float q[3] = {pj[0] - pi[0], pj[1] - pi[1], pj[2] - pi[2]};
        const float w = radius - sqrtf(d2[j]);
        for (int a = 0; a < 3; ++a) {
            const float wq = w * q[a];
            for (int b = 0; b < 3; ++b) cov[3 * a + b] = cov[3 * a + b] + wq * q[b];
        }
        w_total = w_total + w;
        n_nb += 1;
    }
    for (int a = 0; a < 9; ++a) cov[a] = cov[a] / w_total;
    float e[3], V[9];
    fast_eigen3x3(cov, e, V);
    int mn = 0, mx = 0; /* Eigen minCoeff / maxCoeff: first strict improvement */
    for (int c = 1; c < 3; ++c) {
        if (e[c] < e[mn]) mn = c;
        if (e[c] > e[mx]) mx = c;
    }
    for (int r = 0; r < 3; ++r) { Z[r] = V[3 * r + mn]; X[r] = V[3 * r + mx]; }
    int n_px = 0, n_pz = 0;
    for (int j = 0; j < k; ++j) {
        const int id = idx[j];
        if (id < 0 || id == i) continue;
        const float *pj = pts + 3 * (size_t)id;
        const float q[3] = {pj[0] - pi[0], pj[1] - pi[1], pj[2] - pi[2]};
        n_px += dot3f(q[0], q[1], q[2], X[0], X[1], X[2]) >= 0.0f;
        n_pz += dot3f(q[0], q[1], q[2], Z[0], Z[1], Z[2]) >= 0.0f;
    }
    if (n_px < n_nb - n_px) for (int r = 0; r < 3; ++r) X[r] = -X[r];
    if (n_pz < n_nb - n_pz) for (int r = 0; r < 3; ++r) Z[r] = -Z[r];
    cross3(Z, X, Y);
    return n_nb;
}

/* compute_shot_functor::operator() (:100-218) of point i over its list */
static void shot_point(const float *pts, const float *nrm, int i, const int32_t *idx, const float *d2, int k, float radius,
                       float *ft) {
    for (int b = 0; b < SHOT_DIM; ++b) ft[b] = 0.0f;
    float X[3], Y[3], Z[3];
    const int n_nb = shot_lrf(pts, i, idx, d2, k, radius, X, Y, Z);
    if (n_nb < SHOT_MIN_NB) return;
    const float r12 = (float)((double)radius * 0.5), r34 = (float)((double)radius * 3.0 / 4.0);
    const float r14 = (float)((double)radius * 0.25);
    const float *pi = pts + 3 * (size_t)i, *ni = nrm + 3 * (size_t)i;
    for (int j = 0; j < k; ++j) {
        const int id = idx[j];
        if (id < 0 || id == i) continue;
        const float *pj = pts + 3 * (size_t)id;
        const float q[3] = {pj[0] - pi[0], pj[1] - pi[1], pj[2] - pi[2]};
        const float dist = sqrtf(d2[j]);
        if (dist == 0.0f) continue;
        const float cos_desc = clamp_d(dot3f(Z[0], Z[1], Z[2], ni[0], ni[1], ni[2]), -1.0, 1.0); /* the point's OWN normal */
        float bindist = (float)(((1.0 + (double)cos_desc) * SHOT_BINS) / 2.0);
        float x = dot3f(q[0], q[1], q[2], X[0], X[1], X[2]);
        float y = dot3f(q[0], q[1], q[2], Y[0], Y[1], Y[2]);
        float z = dot3f(q[0], q[1], q[2], Z[0], Z[1], Z[2]);
        if ((double)fabsf(x) < 1.0e-30) x = 0.0f;
        if ((double)fabsf(y) < 1.0e-30) y = 0.0f;
        if ((double)fabsf(z) < 1.0e-30) z = 0.0f;
        const int bit4 = (y > 0 || (y == 0.0f && x < 0)) ? 1 : 0;
        const int bit3 = (x > 0 || (x == 0.0f && y > 0)) ? !bit4 : bit4;
        int desc = ((bit4 << 3) + (bit3 << 2)) << 1;
        if (x * y > 0 || x == 0.0f) desc += (fabsf(x) >= fabsf(y)) ? 0 : 4;
        else desc += (fabsf(x) > fabsf(y)) ? 4 : 0;
        desc += z > 0 ? 1 : 0;
        desc += (dist > r12) ? 2 : 0;
        /* ceilf / floorf of a double argument take it as float */
        const int step = (bindist < 0.0) ? (int)ceilf((float)((double)bindist - 0.5)) : (int)floorf((float)((double)bindist + 0.5));
        const int vol = desc * (SHOT_BINS + 1);
        bindist = bindist - (float)step;
        float iw = 1.0f - fabsf(bindist);
        if (bindist > 0) ft[vol + ((step + 1) % SHOT_BINS)] += bindist;
        else ft[vol + ((step - 1 + SHOT_BINS) % SHOT_BINS)] += -bindist;
        if (dist > r12) {
            const float rd = (dist - r34) / r12;
            if (dist > r34) {
                iw += 1.0f - rd;
            } else {
                iw += 1.0f + rd;
                ft[(desc - 2) * (SHOT_BINS + 1) + step] -= rd;
            }
        } else {
            const float rd = (dist - r14) / r12;
            if (dist < r14) {
                iw += 1.0f + rd;
            } else {
                iw += 1.0f - rd;
                ft[(desc + 2) * (SHOT_BINS + 1) + step] += rd;
            }
        }
        const float inc = det_acosf(clamp_d(z / dist, -1.0, 1.0));
        if (inc > PST_RAD_90 || ((double)fabsf(inc - PST_RAD_90) < 1e-30 && z <= 0)) {
            const float d = (inc - PST_RAD_135) / PST_RAD_90;
            if (inc > PST_RAD_135) {
                iw += 1.0f - d;
            } else {
                iw += 1.0f + d;
                ft[(desc + 1) * (SHOT_BINS + 1) + step] -= d;
            }
        } else {
            const float d = (inc - PST_RAD_45) / PST_RAD_90;
            if (inc < PST_RAD_45) {
                iw += 1.0f + d;
            } else {
                iw += 1.0f - d;
                ft[(desc - 1) * (SHOT_BINS + 1) + step] += d;
            }
        }
        if (y != 0.0f || x != 0.0f) {
            const float az = det_atan2f(y, x);
            const int sel = desc >> 2;
            const float span = PST_RAD_45, start = -PST_RAD_PI_7_8;
            const float ad = clamp_d((az - (start + span * (float)sel)) / span, -0.5, 0.5);
            if (ad > 0) {
                iw += 1.0f - ad;
                ft[((desc + 4) % SHOT_SECTORS) * (SHOT_BINS + 1) + step] += ad;
            } else {
                iw += 1.0f + ad;
                ft[((desc - 4 + SHOT_SECTORS) % SHOT_SECTORS) * (SHOT_BINS + 1) + step] -= ad;
            }
        }
        ft[vol + step] += iw;
    }
    float sq = ft[0] * ft[0]; /* Eigen's norm: linear redux in bin order */
    for (int b = 1; b < SHOT_DIM; ++b) sq = sq + ft[b] * ft[b];
    const float norm = sqrtf(sq);
    if (norm > 0)
        for (int b = 0; b < SHOT_DIM; ++b) ft[b] = ft[b] / norm;
}

/* ComputeSHOTFeature (:222-255): out [n][352].  Returns 0, or -1 for knn > 100 or max_nn outside [0, 256] (knn <= 0
 * selects the radius search).  The normals are required. */
int orc_compute_shot_feature(const float *pts, const float *nrm, int n, float radius, int knn, float search_radius,
                             int max_nn, float *out) {
    const int k = shot_k(knn, max_nn);
    if (k < 0) return -1;
    if (n <= 0) return 0;
    if (k == 0) {
        memset(out, 0, sizeof(float) * (size_t)n * SHOT_DIM);
        return 0;
    }
    orc_kdtree *t = orc_kdtree_build(pts, n);
#pragma omp parallel for schedule(dynamic, 256)
    for (int i = 0; i < n; ++i) {
        int32_t idx[SHOT_RADIUS_MAX];
        float d2[SHOT_RADIUS_MAX];
        shot_list(t, pts + 3 * (size_t)i, knn, search_radius, k, idx, d2);
        shot_point(pts, nrm, i, idx, d2, k, radius, out + (size_t)i * SHOT_DIM);
    }
    orc_kdtree_free(t);
    return 0;
}

/* the descriptor of every point over caller-given tables [n][k] (tests restate the arithmetic on the same lists) */
void orc_shot_from_neighbours(const float *pts, const float *nrm, int n, const int32_t *idx, const float *d2, int k,
                              float radius, float *out) {
#pragma omp parallel for schedule(dynamic, 256)
    for (int i = 0; i < n; ++i)
        shot_point(pts, nrm, i, idx + (size_t)i * k, d2 + (size_t)i * k, k, radius, out + (size_t)i * SHOT_DIM);
}
