/*
 * oracle.c -- CPU restatement of cupoch's ICP / kNN / voxel-grid hot path.
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  Built by oracle.build()
 * (oracle/__init__.py).  Compile flags matter: -ffp-contract=off (no implicit
 * FMA; every fused multiply-add below is an explicit fmaf) and no -ffast-math.
 *
 * Arithmetic conventions (shared with the CUDA product by specification, not
 * by code):
 *   dot3(a,b)   = fmaf(a2,b2, fmaf(a1,b1, a0*b0))        device-code dots
 *   a*b - c*d   = fmaf(a,b, -(c*d))                      device-code 2x2 dets
 *   host-code (6x6 solve, se3 exp, 4x4 compose) uses NO fma.
 *   Reductions over correspondences accumulate exact float*float products in
 *   double and round once to float (the reference's thrust float order is
 *   unspecified; see DESIGN.md "parity hazards").
 */
#include "oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
/* bench.py sets the thread count explicitly (torchrun exports OMP_NUM_THREADS=1, which would silently turn the
 * "all host cores" baseline into a single-thread one) */
void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n <= 0) n = omp_get_num_procs();
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

static inline float dot3f(float a0, float a1, float a2, float b0, float b1,
                          float b2) {
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0));
}
static inline float det2f(float a, float b, float c, float d) {
    return fmaf(a, b, -(c * d));
}
/* flann kdtree_cuda_3d_index.cu:211-228 + cutil_math.h:1127-1130: dot(d,d) on
 * float4 with w=0, FMA-contracted under --use_fast_math. */
static inline float dist2f(const float *a, const float *b) {
    float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return fmaf(dz, dz, fmaf(dx, dx, dy * dy));
}

/* ======================================================================== */
/* result set: k best by (d2, idx), strict d2 < r2                           */
/* result_set.h:372-474 (KnnRadiusResultSet): insert needs strict '<';       */
/* unfilled slots idx=-1 / d2=+inf (:447-459).                               */
/* ======================================================================== */
typedef struct {
    int k, count;
    float r2; /* +inf when no radius */
    int32_t *idx;
    float *d2;
} rset;

static inline void rset_init(rset *s, int k, float radius, int32_t *idx,
                             float *d2) {
    s->k = k;
    s->count = 0;
    s->r2 = (radius > 0.0f) ? radius * radius : INFINITY;
    s->idx = idx;
    s->d2 = d2;
    for (int i = 0; i < k; ++i) {
        idx[i] = -1;
        d2[i] = INFINITY;
    }
}
static inline int before(float da, int ia, float db, int ib) {
    return (da < db) || (da == db && ia < ib);
}
/* bound for pruning: a subtree whose min distance is > this cannot matter */
static inline float rset_bound(const rset *s) {
    return (s->count < s->k) ? s->r2 : s->d2[s->k - 1];
}
static inline void rset_insert(rset *s, float d, int i) {
    if (!(d < s->r2)) return;
    if (s->count == s->k) {
        if (!before(d, i, s->d2[s->k - 1], s->idx[s->k - 1])) return;
    } else {
        s->count++;
    }
    int p = s->count - 1;
    while (p > 0 && before(d, i, s->d2[p - 1], s->idx[p - 1])) {
        s->d2[p] = s->d2[p - 1];
        s->idx[p] = s->idx[p - 1];
        --p;
    }
    s->d2[p] = d;
    s->idx[p] = i;
}

long orc_search_bruteforce(const float *tgt, int m, const float *qry, int n,
                           int k, float radius, int32_t *idx, float *d2) {
    long total = 0;
#pragma omp parallel for schedule(static) reduction(+ : total)
    for (int q = 0; q < n; ++q) {
        rset s;
        rset_init(&s, k, radius, idx + (size_t)q * k, d2 + (size_t)q * k);
        for (int j = 0; j < m; ++j) rset_insert(&s, dist2f(qry + 3 * q, tgt + 3 * j), j);
        total += s.count;
    }
    return total;
}

/* ======================================================================== */
/* kd-tree (exact; same result set / tie rule as brute force).  Stands in    */
/* for the vendored FLANN CUDA kd-tree (kdtree_cuda_3d_index.cu:52-129):     */
/* that search is exact (prune test mindistsq <= worstDist, :117), so only   */
/* the arithmetic and the tie rule are mirrored, not the traversal.          */
/* ======================================================================== */
#define KD_LEAF 12
typedef struct {
    float split;
    int axis;        /* -1 = leaf */
    int left, right; /* children, or [begin,end) for leaves */
} kdnode;
struct orc_kdtree {
    int m, n_nodes, cap;
    kdnode *nodes;
    float *pts; /* reordered xyz */
    int32_t *ids;
};

static int kd_new(orc_kdtree *t) {
    if (t->n_nodes == t->cap) {
        t->cap = t->cap ? 2 * t->cap : 1024;
        t->nodes = (kdnode *)realloc(t->nodes, sizeof(kdnode) * t->cap);
    }
    return t->n_nodes++;
}
static void kd_swap(orc_kdtree *t, int a, int b) {
    if (a == b) return;
    float tmp[3];
    memcpy(tmp, t->pts + 3 * a, 12);
    memcpy(t->pts + 3 * a, t->pts + 3 * b, 12);
    memcpy(t->pts + 3 * b, tmp, 12);
    int32_t ti = t->ids[a];
    t->ids[a] = t->ids[b];
    t->ids[b] = ti;
}
static void kd_select(orc_kdtree *t, int lo, int hi, int nth, int ax) {
    /* quickselect on [lo,hi) so that element nth is in sorted position */
    while (hi - lo > 1) {
        int mid = lo + (hi - lo) / 2;
        float a = t->pts[3 * lo + ax], b = t->pts[3 * mid + ax],
              c = t->pts[3 * (hi - 1) + ax];
        int pi = (a < b) ? ((b < c) ? mid : ((a < c) ? hi - 1 : lo))
                         : ((a < c) ? lo : ((b < c) ? hi - 1 : mid));
        float pv = t->pts[3 * pi + ax];
        int i = lo, j = hi - 1;
        while (i <= j) {
            while (t->pts[3 * i + ax] < pv) ++i;
            while (t->pts[3 * j + ax] > pv) --j;
            if (i <= j) {
                kd_swap(t, i, j);
                ++i;
                --j;
            }
        }
        if (nth <= j)
            hi = j + 1;
        else if (nth >= i)
            lo = i;
        else
            return;
    }
}
static int kd_build_rec(orc_kdtree *t, int lo, int hi) {
    int id = kd_new(t);
    if (hi - lo <= KD_LEAF) {
        t->nodes[id].axis = -1;
        t->nodes[id].left = lo;
        t->nodes[id].right = hi;
        t->nodes[id].split = 0.f;
        return id;
    }
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = lo; i < hi; ++i)
        for (int a = 0; a < 3; ++a) {
            float v = t->pts[3 * i + a];
            if (v < mn[a]) mn[a] = v;
            if (v > mx[a]) mx[a] = v;
        }
    int ax = 0;
    if (mx[1] - mn[1] > mx[ax] - mn[ax]) ax = 1;
    if (mx[2] - mn[2] > mx[ax] - mn[ax]) ax = 2;
    int mid = lo + (hi - lo) / 2;
    kd_select(t, lo, hi, mid, ax);
    float split = t->pts[3 * mid + ax];
    int l = kd_build_rec(t, lo, mid);
    int r = kd_build_rec(t, mid, hi);
    t->nodes[id].axis = ax;
    t->nodes[id].split = split;
    t->nodes[id].left = l;
    t->nodes[id].right = r;
    return id;
}
orc_kdtree *orc_kdtree_build(const float *tgt, int m) {
    orc_kdtree *t = (orc_kdtree *)calloc(1, sizeof(*t));
    t->m = m;
    t->pts = (float *)malloc(sizeof(float) * 3 * (m > 0 ? m : 1));
    t->ids = (int32_t *)malloc(sizeof(int32_t) * (m > 0 ? m : 1));
    memcpy(t->pts, tgt, sizeof(float) * 3 * m);
    for (int i = 0; i < m; ++i) t->ids[i] = i;
    if (m > 0) kd_build_rec(t, 0, m);
    return t;
}
void orc_kdtree_free(orc_kdtree *t) {
    if (!t) return;
    free(t->nodes);
    free(t->pts);
    free(t->ids);
    free(t);
}
static void kd_search_rec(const orc_kdtree *t, int id, const float *q, rset *s) {
    const kdnode *nd = &t->nodes[id];
    if (nd->axis < 0) {
        for (int i = nd->left; i < nd->right; ++i)
            rset_insert(s, dist2f(q, t->pts + 3 * i), t->ids[i]);
        return;
    }
    float diff = q[nd->axis] - nd->split;
    int near = (diff < 0.f) ? nd->left : nd->right;
    int far = (diff < 0.f) ? nd->right : nd->left;
    kd_search_rec(t, near, q, s);
    /* plane distance is a lower bound for the far side; '<=' keeps ties */
    if (diff * diff <= rset_bound(s)) kd_search_rec(t, far, q, s);
}
long orc_kdtree_search(const orc_kdtree *t, const float *qry, int n, int k,
                       float radius, int32_t *idx, float *d2) {
    long total = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : total)
    for (int q = 0; q < n; ++q) {
        rset s;
        rset_init(&s, k, radius, idx + (size_t)q * k, d2 + (size_t)q * k);
        if (t->m > 0) kd_search_rec(t, 0, qry + 3 * q, &s);
        total += s.count;
    }
    return total;
}

/* ======================================================================== */
/* geometry                                                                  */
/* ======================================================================== */
/* geometry_utils.cu:34-43 transform_points_functor: R*p + t (Eigen lazy      */
/* 3x3*3x1 = sequential k sum, contracted; then + t).                         */
void orc_transform_points(float *p, int n, const float T[16]) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
        p[3 * i + 0] = dot3f(T[0], T[1], T[2], x, y, z) + T[3];
        p[3 * i + 1] = dot3f(T[4], T[5], T[6], x, y, z) + T[7];
        p[3 * i + 2] = dot3f(T[8], T[9], T[10], x, y, z) + T[11];
    }
}
/* geometry_utils.cu:45-53 transform_normals_functor: n <- R n, no renormalise */
void orc_transform_normals(float *nr, int n, const float T[16]) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        float x = nr[3 * i], y = nr[3 * i + 1], z = nr[3 * i + 2];
        nr[3 * i + 0] = dot3f(T[0], T[1], T[2], x, y, z);
        nr[3 * i + 1] = dot3f(T[4], T[5], T[6], x, y, z);
        nr[3 * i + 2] = dot3f(T[8], T[9], T[10], x, y, z);
    }
}
/* geometry_utils.cu:257-265: C <- (R*C)*R^T */
static void rot_cov(const float T[16], float *C) {
    float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    float tmp[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            tmp[3 * i + j] = dot3f(R[3 * i], R[3 * i + 1], R[3 * i + 2], C[j], C[3 + j], C[6 + j]);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            C[3 * i + j] = dot3f(tmp[3 * i], tmp[3 * i + 1], tmp[3 * i + 2], R[3 * j], R[3 * j + 1], R[3 * j + 2]);
}
void orc_rotate_covariances(float *cov, int n, const float T[16]) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) rot_cov(T, cov + 9 * (size_t)i);
}
/* eigen.inl:197-221 ComputeMinBound/MaxBound: element-wise min/max */
void orc_min_bound(const float *p, int n, float out[3]) {
    out[0] = out[1] = out[2] = 0.f;
    if (n <= 0) return;
    memcpy(out, p, 12);
    for (int i = 1; i < n; ++i)
        for (int a = 0; a < 3; ++a)
            if (p[3 * i + a] < out[a]) out[a] = p[3 * i + a];
}
void orc_max_bound(const float *p, int n, float out[3]) {
    out[0] = out[1] = out[2] = 0.f;
    if (n <= 0) return;
    memcpy(out, p, 12);
    for (int i = 1; i < n; ++i)
        for (int a = 0; a < 3; ++a)
            if (p[3 * i + a] > out[a]) out[a] = p[3 * i + a];
}

/* ======================================================================== */
/* VoxelDownSample  down_sample.cu:170-273, key :64-75, normalise :78-90,    */
/* order = lexicographic (x,y,z) helper.h:113-121                             */
/* ======================================================================== */
typedef struct {
    int32_t k[3];
    int32_t i;
} vkey;
static int vkey_cmp(const void *a, const void *b) {
    const vkey *x = (const vkey *)a, *y = (const vkey *)b;
    for (int c = 0; c < 3; ++c)
        if (x->k[c] != y->k[c]) return x->k[c] < y->k[c] ? -1 : 1;
    return (x->i < y->i) ? -1 : (x->i > y->i);
}
/* origin == NULL: the reference's own origin (:180); otherwise a caller-supplied common grid origin (the sharded
 * down-sample of tests/test_distributed_gloo.py) */
int orc_voxel_down_sample_origin(const float *pts, const float *nrm, const float *col,
                                 int n, float voxel, const float *origin, float *out_pts, float *out_nrm,
                                 float *out_col) {
    if (voxel <= 0.0f || n <= 0) return 0;
    float mn[3], mx[3], org[3];
    orc_min_bound(pts, n, mn);
    orc_max_bound(pts, n, mx);
    float ext = 0.f;
    for (int a = 0; a < 3; ++a) {
        org[a] = origin ? origin[a] : mn[a] - voxel * 0.5f;            /* :180 */
        float hi = mx[a] + voxel * 0.5f;          /* :181 */
        if (hi - org[a] > ext) ext = hi - org[a];
    }
    if (voxel * (float)2147483647 < ext) return 0; /* :183-187 */
    vkey *keys = (vkey *)malloc(sizeof(vkey) * n);
    for (int i = 0; i < n; ++i) {
        for (int a = 0; a < 3; ++a)
            keys[i].k[a] = (int32_t)floorf((pts[3 * i + a] - org[a]) / voxel);
        keys[i].i = i;
    }
    qsort(keys, n, sizeof(vkey), vkey_cmp);
    int n_out = 0;
    for (int b = 0; b < n;) {
        int e = b;
        double sp[3] = {0, 0, 0}, sn[3] = {0, 0, 0}, sc[3] = {0, 0, 0};
        while (e < n && keys[e].k[0] == keys[b].k[0] && keys[e].k[1] == keys[b].k[1] &&
               keys[e].k[2] == keys[b].k[2]) {
            int i = keys[e].i;
            for (int a = 0; a < 3; ++a) {
                sp[a] += pts[3 * i + a];
                if (nrm) sn[a] += nrm[3 * i + a];
                if (col) sc[a] += col[3 * i + a];
            }
            ++e;
        }
        float cnt = (float)(e - b);
        for (int a = 0; a < 3; ++a) out_pts[3 * n_out + a] = (float)sp[a] / cnt;
        if (col)
            for (int a = 0; a < 3; ++a) out_col[3 * n_out + a] = (float)sc[a] / cnt;
        if (nrm) {
            float v[3];
            for (int a = 0; a < 3; ++a) v[a] = (float)sn[a] / cnt;
            /* Eigen normalize(): v / sqrt(squaredNorm) when norm > 0 */
            float nn = sqrtf(dot3f(v[0], v[1], v[2], v[0], v[1], v[2]));
            for (int a = 0; a < 3; ++a) out_nrm[3 * n_out + a] = (nn > 0.f) ? v[a] / nn : v[a];
        }
        ++n_out;
        b = e;
    }
    free(keys);
    return n_out;
}
int orc_voxel_down_sample(const float *pts, const float *nrm, const float *col,
                          int n, float voxel, float *out_pts, float *out_nrm,
                          float *out_col) {
    return orc_voxel_down_sample_origin(pts, nrm, col, n, voxel, NULL, out_pts, out_nrm, out_col);
}

/* ======================================================================== */
/* VoxelGrid::CreateFromPointCloudWithinBounds  voxelgrid_factory.cu:164-219   */
/* key = floor((p - min_bound) / voxel) (:73-76, negative for points below the  */
/* bound: the reference does not clip); voxels sorted lexicographically,        */
/* colour = mean of the points' colours (sum / count), (1,1,1) without colours  */
/* (Voxel's default, voxelgrid.h:61).  voxel <= 0 and "voxel too small" are only */
/* logged by the reference; here they return an empty grid.                     */
/* ======================================================================== */
int orc_voxel_grid_from_point_cloud(const float *pts, const float *col, int n, float voxel, const float min_bound[3],
                                    const float max_bound[3], int32_t *out_keys, float *out_col) {
    if (voxel <= 0.0f || n <= 0) return 0;
    float ext = 0.f;
    for (int a = 0; a < 3; ++a)
        if (max_bound[a] - min_bound[a] > ext) ext = max_bound[a] - min_bound[a];
    if (voxel * (float)2147483647 < ext) return 0; /* :174-177 */
    vkey *keys = (vkey *)malloc(sizeof(vkey) * n);
    for (int i = 0; i < n; ++i) {
        for (int a = 0; a < 3; ++a) keys[i].k[a] = (int32_t)floorf((pts[3 * i + a] - min_bound[a]) / voxel);
        keys[i].i = i;
    }
    qsort(keys, n, sizeof(vkey), vkey_cmp);
    int n_out = 0;
    for (int b = 0; b < n;) {
        int e = b;
        double sc[3] = {0, 0, 0};
        while (e < n && keys[e].k[0] == keys[b].k[0] && keys[e].k[1] == keys[b].k[1] && keys[e].k[2] == keys[b].k[2]) {
            if (col)
                for (int a = 0; a < 3; ++a) sc[a] += col[3 * keys[e].i + a];
            ++e;
        }
        const float cnt = (float)(e - b);
        for (int a = 0; a < 3; ++a) {
            out_keys[3 * n_out + a] = keys[b].k[a];
            out_col[3 * n_out + a] = col ? (float)sc[a] / cnt : 1.0f;
        }
        ++n_out;
        b = e;
    }
    free(keys);
    return n_out;
}

/* ======================================================================== */
/* symmetric 3x3 eigen solver   eigenvalue.inl:30-178                         */
/* m is ROW-major 3x3; only the entries the reference reads are read.        */
/* ======================================================================== */
static inline float signf_(float x) { return x / fabsf(x); }
static void cross3(const float *a, const float *b, float *o) {
    o[0] = det2f(a[1], b[2], a[2], b[1]);
    o[1] = det2f(a[2], b[0], a[0], b[2]);
    o[2] = det2f(a[0], b[1], a[1], b[0]);
}
static void eigvec0(const float *A, float e0, float *out) { /* :32-50 */
    float r0[3] = {A[0] - e0, A[1], A[2]};
    float r1[3] = {A[1], A[4] - e0, A[5]};
    float r2[3] = {A[2], A[5], A[8] - e0};
    float rx[3][3];
    cross3(r0, r1, rx[0]);
    cross3(r0, r2, rx[1]);
    cross3(r1, r2, rx[2]);
    float d[3];
    for (int i = 0; i < 3; ++i) d[i] = dot3f(rx[i][0], rx[i][1], rx[i][2], rx[i][0], rx[i][1], rx[i][2]);
    int im = 0;
    if (d[1] > d[im]) im = 1;
    if (d[2] > d[im]) im = 2;
    float s = sqrtf(d[im]);
    for (int i = 0; i < 3; ++i) out[i] = rx[im][i] / s;
}
static void eigvec1(const float *A, const float *e0v, float e1, float *out) { /* :52-91 */
    float mx = fmaxf(fabsf(e0v[0]), fabsf(e0v[1]));
    float inv_len = 1 / sqrtf(fmaf(e0v[2], e0v[2], mx * mx));
    float U[3], V[3];
    if (fabsf(e0v[0]) > fabsf(e0v[1])) {
        U[0] = -e0v[2]; U[1] = 0; U[2] = e0v[0];
    } else {
        U[0] = 0; U[1] = e0v[2]; U[2] = -e0v[1];
    }
    for (int i = 0; i < 3; ++i) U[i] *= inv_len;
    cross3(e0v, U, V);
    float AU[3] = {dot3f(A[0], A[1], A[2], U[0], U[1], U[2]),
                   dot3f(A[1], A[4], A[5], U[0], U[1], U[2]),
                   dot3f(A[2], A[5], A[8], U[0], U[1], U[2])};
    float AV[3] = {dot3f(A[0], A[1], A[2], V[0], V[1], V[2]),
                   dot3f(A[1], A[4], A[5], V[0], V[1], V[2]),
                   dot3f(A[2], A[5], A[8], V[0], V[1], V[2])};
    float m00 = dot3f(U[0], U[1], U[2], AU[0], AU[1], AU[2]) - e1;
    float m01 = dot3f(U[0], U[1], U[2], AV[0], AV[1], AV[2]);
    float m11 = dot3f(V[0], V[1], V[2], AV[0], AV[1], AV[2]) - e1;
    float a00 = fabsf(m00), a01 = fabsf(m01), a11 = fabsf(m11);
    float mac0 = fmaxf(a00, a11);
    float mac = fmaxf(mac0, a01);
    float coef2 = fminf(mac0, a01) / fmaxf(mac, 1.0e-6f);
    float coef1 = 1.0f / sqrtf(fmaf(coef2, coef2, 1.0f));
    float cu, cv;
    if (a00 >= a11) {
        coef2 *= coef1 * signf_(m00) * signf_(m01);
        if (mac0 >= a01) { cu = coef2; cv = coef1; } else { cu = coef1; cv = coef2; }
    } else {
        coef2 *= coef1 * signf_(m11) * signf_(m01);
        if (mac0 >= a01) { cu = coef1; cv = coef2; } else { cu = coef2; cv = coef1; }
    }
    for (int i = 0; i < 3; ++i) out[i] = fmaf(cu, U[i], -(cv * V[i]));
}
/* ---- deterministic acos / cos for FastEigen3x3 ------------------------------------------------------------
 * The reference evaluates acosf / cosf of CUDA's --use_fast_math library (eigenvalue.inl:120-123); libm and libdevice
 * differ from it and from each other in the last ulp, which is enough to flip a near-tie of the GICP search after 30
 * iterations.  Product and oracle therefore share a SPECIFICATION (not code; the kernel side is
 * cupoch_b200/csrc/cphb_eigen3.cuh): float64 Taylor polynomials evaluated by Horner with explicit fma, IEEE
 * sqrt / add / mul only, result rounded once to float32 (error < 1e-16 before the rounding, i.e. correctly rounded
 * except in astronomically rare cases).  Tables: tools/gen_trig_coeffs.py (exact rationals -> nearest double).
 *   asin_p(z), |z| <= 0.5   = z * sum_{k<26} DT_ASIN[k] z^2k
 *   acos(x) = pi/2 - asin_p(x)                     |x| <= 0.5
 *           = 2 asin_p(sqrt((1 - x)/2))            x > 0.5
 *           = pi - 2 asin_p(sqrt((1 + x)/2))       x < -0.5
 *   cos(y), 0 <= y <= 2 pi:  y > pi -> y = 2 pi - y;  y <= pi/4: cos_p(y);  y <= 3pi/4: -sin_p(y - pi/2);
 *                            else -cos_p(pi - y)     (cos_p / sin_p: 12 Taylor terms on |u| <= pi/4) */
static const double DT_ASIN[26] = {
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
static const double DT_COS[12] = {
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
static const double DT_SIN[12] = {
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
#define DT_PI 0x1.921fb54442d18p+1
#define DT_PI_2 0x1.921fb54442d18p+0
#define DT_PI_4 0x1.921fb54442d18p-1
static double dt_asin_p(double z) {
    const double z2 = z * z;
    double p = DT_ASIN[25];
    for (int k = 24; k >= 0; --k) p = fma(p, z2, DT_ASIN[k]);
    return z * p;
}
static double dt_cos_p(double u) {
    const double u2 = u * u;
    double p = DT_COS[11];
    for (int k = 10; k >= 0; --k) p = fma(p, u2, DT_COS[k]);
    return p;
}
static double dt_sin_p(double u) {
    const double u2 = u * u;
    double p = DT_SIN[11];
    for (int k = 10; k >= 0; --k) p = fma(p, u2, DT_SIN[k]);
    return u * p;
}
static float det_acosf(float xf) { /* xf in [-1, 1] */
    const double x = (double)xf;
    double r;
    if (x > 0.5) r = 2.0 * dt_asin_p(sqrt((1.0 - x) * 0.5));
    else if (x < -0.5) r = DT_PI - 2.0 * dt_asin_p(sqrt((1.0 + x) * 0.5));
    else r = DT_PI_2 - dt_asin_p(x);
    return (float)r;
}
static float det_cosf(float yf) { /* yf in [0, 2 pi] */
    double y = (double)yf;
    if (y > DT_PI) y = 2.0 * DT_PI - y;
    double r;
    if (y <= DT_PI_4) r = dt_cos_p(y);
    else if (y <= 3.0 * DT_PI_4) r = -dt_sin_p(y - DT_PI_2);
    else r = -dt_cos_p(DT_PI - y);
    return (float)r;
}

float orc_det_acosf(float x) { return det_acosf(x); } /* exported for tests/test_oracle_consistency.py */
float orc_det_cosf(float y) { return det_cosf(y); }

/* FastEigen3x3 (:93-154).  evec columns: evec[3*r+c].  NOTE (reference quirk,
 * mirrored): in the general branch the eigenvalues are those of A/max_coeff --
 * they are not scaled back. */
static void fast_eigen3x3(const float *Ain, float *eval, float *evec) {
    float A[9];
    memcpy(A, Ain, sizeof(A));
    float mc = A[0];
    for (int i = 1; i < 9; ++i)
        if (A[i] > mc) mc = A[i];
    if (mc == 0) {
        eval[0] = eval[1] = eval[2] = 0;
        memset(evec, 0, 36);
        evec[0] = evec[4] = evec[8] = 1;
        return;
    }
    for (int i = 0; i < 9; ++i) A[i] /= mc;
    float norm = fmaf(A[5], A[5], fmaf(A[2], A[2], A[1] * A[1]));
    if (norm > 0) {
        float q = (A[0] + A[4] + A[8]) / 3;
        float b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
        float p = sqrtf(fmaf(norm, 2.f, fmaf(b22, b22, fmaf(b11, b11, b00 * b00))) / 6);
        float c00 = det2f(b11, b22, A[5], A[5]);
        float c01 = det2f(A[1], b22, A[5], A[2]);
        float c02 = det2f(A[1], A[5], b11, A[2]);
        float det = fmaf(A[2], c02, fmaf(-A[1], c01, b00 * c00)) / (p * p * p);
        float half_det = det * 0.5f;
        half_det = fminf(fmaxf(half_det, -1.0f), 1.0f);
        float angle = det_acosf(half_det) / (float)3;
        const float two_thirds_pi = 2.09439510239319549f;
        float beta2 = det_cosf(angle) * 2;
        float beta0 = det_cosf(angle + two_thirds_pi) * 2;
        float beta1 = -(beta0 + beta2);
        eval[0] = fmaf(p, beta0, q);
        eval[1] = fmaf(p, beta1, q);
        eval[2] = fmaf(p, beta2, q);
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
        for (int r = 0; r < 3; ++r) {
            evec[3 * r + 0] = c0[r];
            evec[3 * r + 1] = c1[r];
            evec[3 * r + 2] = c2[r];
        }
    } else {
        eval[0] = Ain[0];
        eval[1] = Ain[4];
        eval[2] = Ain[8];
        memset(evec, 0, 36);
        evec[0] = evec[4] = evec[8] = 1;
    }
}
/* SqrtMatrix3x3 (:172-177): V * diag(sqrt(e)) * V^T */
static void sqrt_matrix3x3(const float *A, float *W) {
    float e[3], V[9], VD[9];
    fast_eigen3x3(A, e, V);
    float s[3] = {sqrtf(e[0]), sqrtf(e[1]), sqrtf(e[2])};
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) VD[3 * i + k] = V[3 * i + k] * s[k];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            W[3 * i + j] = dot3f(VD[3 * i], VD[3 * i + 1], VD[3 * i + 2], V[3 * j], V[3 * j + 1], V[3 * j + 2]);
}
/* Eigen Matrix3f::inverse(): cofactors / det (InverseImpl.h size-3 path) */
static void inverse3x3(const float *m, float *inv) {
    float cof[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            cof[3 * i + j] = det2f(m[3 * i1 + j1], m[3 * i2 + j2], m[3 * i1 + j2], m[3 * i2 + j1]);
        }
    float det = dot3f(cof[0], cof[3], cof[6], m[0], m[3], m[6]);
    float invdet = 1.0f / det;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) inv[3 * i + j] = cof[3 * j + i] * invdet;
}

/* ======================================================================== */
/* EstimateNormals  estimate_normals.cu:38-127, geometry_functor.h:35-55      */
/* ======================================================================== */
/* covariance E[xx^T] - E[x]E[x]^T from the float64 cumulants (also ISS's).  Deviation (DESIGN.md section 4, item 22):
 * the mean and the subtraction are float64, fma(-m_a, m_b, cum / cnt), each coefficient rounded to float once; the
 * reference subtracts in float32.  cnt == 0 gives NaN coefficients. */
static void covariance_from_cumulants(const double cum[9], int cnt, float cov[9]) {
    const double c = (double)cnt;
    const double m0 = cum[0] / c, m1 = cum[1] / c, m2 = cum[2] / c;
    cov[0] = (float)fma(-m0, m0, cum[3] / c);
    cov[4] = (float)fma(-m1, m1, cum[6] / c);
    cov[8] = (float)fma(-m2, m2, cum[8] / c);
    cov[1] = cov[3] = (float)fma(-m0, m1, cum[4] / c);
    cov[2] = cov[6] = (float)fma(-m0, m2, cum[5] / c);
    cov[5] = cov[7] = (float)fma(-m1, m2, cum[7] / c);
}
static int usable_vector(const float *v) {
    const float nn = sqrtf(dot3f(v[0], v[1], v[2], v[0], v[1], v[2]));
    return nn > 0.f && nn <= FLT_MAX; /* false for 0, NaN and inf */
}
/* Deviation (item 22): the smallest eigenvalue's eigenvector where FastEigen3x3's is NaN or zero (eigvec1's signf(0) =
 * 0/0).  e: FastEigen3x3's eigenvalues, those of A = cov / max coefficient.  eigvec0 of A with e[mi] when e[mi] is
 * simple: the middle eigenvalue more than 2^-10 of the spread above it; else (a line) eigvec1's U for the largest
 * eigenvalue's eigenvector, a unit vector perpendicular to it. */
static void normal_direct(const float *cov, const float *e, int mi, float *n) {
    float A[9];
    float mc = cov[0];
    for (int i = 1; i < 9; ++i)
        if (cov[i] > mc) mc = cov[i];
    for (int i = 0; i < 9; ++i) A[i] = cov[i] / mc;
    int ma = 0;
    if (e[1] > e[ma]) ma = 1;
    if (e[2] > e[ma]) ma = 2;
    const float mid = ((e[0] + e[1]) + e[2] - e[mi]) - e[ma];
    if (mid - e[mi] > 0x1p-10f * (e[ma] - e[mi])) {
        eigvec0(A, e[mi], n);
        return;
    }
    float v2[3];
    eigvec0(A, e[ma], v2);
    const float mx = fmaxf(fabsf(v2[0]), fabsf(v2[1]));
    const float inv_len = 1 / sqrtf(fmaf(v2[2], v2[2], mx * mx));
    if (fabsf(v2[0]) > fabsf(v2[1])) {
        n[0] = -v2[2]; n[1] = 0; n[2] = v2[0];
    } else {
        n[0] = 0; n[1] = v2[2]; n[2] = -v2[1];
    }
    for (int i = 0; i < 3; ++i) n[i] *= inv_len;
}
void orc_normals_from_neighbors(const float *pts, int n, const int32_t *nbr,
                                int k, float *out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        double cum[9] = {0};
        int cnt = 0;
        for (int j = 0; j < k; ++j) {
            int id = nbr[(size_t)i * k + j];
            if (id < 0) continue;
            const float *p = pts + 3 * (size_t)id;
            cum[0] += p[0]; cum[1] += p[1]; cum[2] += p[2];
            cum[3] += (double)p[0] * p[0]; cum[4] += (double)p[0] * p[1];
            cum[5] += (double)p[0] * p[2]; cum[6] += (double)p[1] * p[1];
            cum[7] += (double)p[1] * p[2]; cum[8] += (double)p[2] * p[2];
            ++cnt;
        }
        float *o = out + 3 * (size_t)i;
        if (cnt < 3) { o[0] = 0; o[1] = 0; o[2] = 1; continue; }
        float cov[9];
        covariance_from_cumulants(cum, cnt, cov);
        float e[3], V[9];
        fast_eigen3x3(cov, e, V);
        int mi = 0; /* Eigen minCoeff: first minimum */
        if (e[1] < e[mi]) mi = 1;
        if (e[2] < e[mi]) mi = 2;
        float v[3] = {V[mi], V[3 + mi], V[6 + mi]};
        if (!usable_vector(v)) normal_direct(cov, e, mi, v);
        if (!usable_vector(v)) { v[0] = 0; v[1] = 0; v[2] = 1; } /* a covariance that is not finite */
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
    }
}
void orc_estimate_normals(const float *pts, int n, int knn, float radius,
                          int max_nn, float *out) {
    int k = (knn > 0) ? knn : max_nn;
    if (k <= 0) {
        for (int i = 0; i < n; ++i) { out[3 * i] = 0; out[3 * i + 1] = 0; out[3 * i + 2] = 1; }
        return;
    }
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * k);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * k);
    orc_kdtree *t = orc_kdtree_build(pts, n);
    orc_kdtree_search(t, pts, n, k, (knn > 0) ? -1.0f : radius, idx, d2);
    orc_normals_from_neighbors(pts, n, idx, k, out);
    orc_kdtree_free(t);
    free(idx);
    free(d2);
}

/* ---- outlier filters (kNN consumers, SURVEY 8f rank 4) -------------------- */
/* down_sample.cu:317-354 RemoveRadiusOutliers: SearchRadius(points, r, nb_points + 1) of the cloud against
 * itself (every point finds itself, d2 = 0); a point is kept when MORE than nb_points of its nb_points + 1
 * slots are valid, i.e. when all of them are.  Output: ascending indices.  The reference only logs
 * nb_points < 1 / radius <= 0 and carries on: the search uses float(radius * radius) (kdtree_flann.inl:118), so a
 * negative radius acts as |radius| and radius == 0 matches nothing (strict d2 < 0), i.e. an empty selection. */
int orc_remove_radius_outliers(const float *pts, int n, int nb_points, float radius, int32_t *out_idx) {
    if (n <= 0 || radius == 0.f || nb_points < 0) return 0;
    radius = fabsf(radius);
    const int k = nb_points + 1;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * k);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * k);
    orc_kdtree *t = orc_kdtree_build(pts, n);
    orc_kdtree_search(t, pts, n, k, radius, idx, d2);
    int m = 0;
    for (int i = 0; i < n; ++i) {
        int cnt = 0;
        for (int j = 0; j < k; ++j) cnt += idx[(size_t)i * k + j] >= 0;
        if (cnt > nb_points) out_idx[m++] = i;
    }
    orc_kdtree_free(t);
    free(idx);
    free(d2);
    return m;
}

/* down_sample.cu:356-438 RemoveStatisticalOutliers.  Per point: mean of the SQUARED distances (the kd-tree
 * returns d2 and the reference averages them as they are) of its nb_neighbors nearest points, itself included;
 * slots with inf / negative d2 do not count; no valid slot -> -1.  Cloud mean and Bessel-corrected standard
 * deviation over the points with avg >= 0 (the deviation sum skips avg <= 0, :423-427); keep
 * 0 < avg < mean + std_ratio * std.  Sums: thrust's float reductions have no specified order -- here (and in
 * the kernels) every sum is accumulated in float64 and rounded to float once. */
int orc_remove_statistical_outliers(const float *pts, int n, int nb_neighbors, float std_ratio, int32_t *out_idx,
                                    float *out_avg /* [n] or NULL */, float out_stats[3] /* mean, std, thr */) {
    if (out_stats) out_stats[0] = out_stats[1] = out_stats[2] = 0.f;
    if (n <= 0 || nb_neighbors < 1) return 0;
    const int k = nb_neighbors;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * k);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * k);
    float *avg = (float *)malloc(sizeof(float) * (size_t)n);
    orc_kdtree *t = orc_kdtree_build(pts, n);
    orc_kdtree_search(t, pts, n, k, -1.0f, idx, d2);
    double msum = 0.0;
    long valid = 0;
    for (int i = 0; i < n; ++i) {
        double s = 0.0;
        int c = 0;
        for (int j = 0; j < k; ++j) {
            const float d = d2[(size_t)i * k + j];
            if (isinf(d) || d < 0.f) continue;
            s += (double)d;
            ++c;
        }
        avg[i] = (c > 0) ? (float)s / (float)c : -1.0f;
        if (avg[i] >= 0.f) { msum += (double)avg[i]; ++valid; }
    }
    int m = 0;
    if (valid > 0) {
        float mean = (float)msum;
        mean /= (float)valid;
        double sq = 0.0;
        for (int i = 0; i < n; ++i)
            if (avg[i] > 0.f) {
                const float e = avg[i] - mean;
                sq += (double)(e * e);
            }
        const float sqf = (float)sq;
        const float std_dev = sqrtf(sqf / (float)(valid - 1)); /* valid == 1: x/0 -> inf or nan, as the reference */
        const float thr = mean + std_ratio * std_dev;
        for (int i = 0; i < n; ++i)
            if (avg[i] > 0.f && avg[i] < thr) out_idx[m++] = i;
        if (out_stats) { out_stats[0] = mean; out_stats[1] = std_dev; out_stats[2] = thr; }
    }
    if (out_avg) memcpy(out_avg, avg, sizeof(float) * (size_t)n);
    orc_kdtree_free(t);
    free(idx);
    free(d2);
    free(avg);
    return m;
}

/* pointcloud.cu:56-106,387-433 PointCloud::GaussianFilter: radius search of the cloud against itself
 * (search_radius, num_max_search_points); every output row is the weighted mean of the found neighbours' rows with
 * weight = exp(-0.5 * d2 / sigma2) -- the product and the exponential are evaluated in double (the literal 0.5
 * promotes them) and rounded to float; sums are sequential float32 in slot order.  Returns 0 (and writes nothing)
 * for illegal parameters, as the reference returns an empty cloud. */
int orc_gaussian_filter(const float *pts, const float *nrm, const float *col, int n, float radius, float sigma2, int max_nn,
                        float *out_pts, float *out_nrm, float *out_col) {
    if (radius <= 0.f || sigma2 <= 0.f || max_nn <= 0 || n <= 0) return 0;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * max_nn);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * max_nn);
    orc_kdtree *t = orc_kdtree_build(pts, n);
    orc_kdtree_search(t, pts, n, max_nn, radius, idx, d2);
    for (int i = 0; i < n; ++i) {
        float tw = 0.f, rp[3] = {0, 0, 0}, rn[3] = {0, 0, 0}, rc[3] = {0, 0, 0};
        for (int s = 0; s < max_nn; ++s) {
            const int j = idx[(size_t)i * max_nn + s];
            if (j < 0) continue;
            const float w = (float)exp(-0.5 * (double)d2[(size_t)i * max_nn + s] / (double)sigma2);
            for (int a = 0; a < 3; ++a) {
                rp[a] += w * pts[3 * j + a];
                if (nrm) rn[a] += w * nrm[3 * j + a];
                if (col) rc[a] += w * col[3 * j + a];
            }
            tw += w;
        }
        for (int a = 0; a < 3; ++a) {
            out_pts[3 * i + a] = rp[a] / tw;
            if (nrm) out_nrm[3 * i + a] = rn[a] / tw;
            if (col) out_col[3 * i + a] = rc[a] / tw;
        }
    }
    orc_kdtree_free(t);
    free(idx);
    free(d2);
    return n;
}

/* generalized_icp.cu:18-61: Rx*diag(eps,1,1)*Rx^T, Rx = rotation e1 -> n */
void orc_covariances_from_normals(const float *nrm, int n, float eps, float *out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        const float *x = nrm + 3 * (size_t)i;
        float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        float c = x[0];
        if (!(c < -0.99f)) {
            float v[3] = {0.f, -x[2], x[1]};
            float sv[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
            float ss[9];
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    ss[3 * a + b] = dot3f(sv[3 * a], sv[3 * a + 1], sv[3 * a + 2], sv[b], sv[3 + b], sv[6 + b]);
            float factor = 1 / (1 + c);
            for (int a = 0; a < 9; ++a) R[a] = fmaf(ss[a], factor, R[a] + sv[a]);
        }
        float cd[3] = {eps, 1.f, 1.f}, tmp[9];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) tmp[3 * a + b] = R[3 * a + b] * cd[b];
        float *C = out + 9 * (size_t)i;
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b)
                C[3 * a + b] = dot3f(tmp[3 * a], tmp[3 * a + 1], tmp[3 * a + 2], R[3 * b], R[3 * b + 1], R[3 * b + 2]);
    }
}

static inline float intensity(const float *c) {
    return (float)((double)(c[0] + c[1] + c[2]) / 3.0);
}
/* colored_icp.cu:73-118 compute_color_gradient_functor (slot 0 skipped) */
void orc_color_gradient(const float *pts, const float *nrm, const float *col,
                        int n, const int32_t *nbr, int k, float *out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        const float *vt = pts + 3 * (size_t)i, *nt = nrm + 3 * (size_t)i;
        float it = intensity(col + 3 * (size_t)i);
        float AtA[9] = {0}, Atb[3] = {0};
        int nn = 0;
        for (int j = 1; j < k; ++j) {
            int a = nbr[(size_t)i * k + j];
            if (a < 0) continue;
            const float *va = pts + 3 * (size_t)a;
            float d[3] = {va[0] - vt[0], va[1] - vt[1], va[2] - vt[2]};
            float s = dot3f(d[0], d[1], d[2], nt[0], nt[1], nt[2]);
            float vtmp[3];
            for (int c = 0; c < 3; ++c) vtmp[c] = fmaf(-s, nt[c], va[c]) - vt[c];
            float ia = intensity(col + 3 * (size_t)a);
            float di = ia - it;
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) AtA[3 * r + c] = fmaf(vtmp[r], vtmp[c], AtA[3 * r + c]);
                Atb[r] = fmaf(di, vtmp[r], Atb[r]);
            }
            ++nn;
        }
        float *o = out + 3 * (size_t)i;
        if (nn < 4) { o[0] = o[1] = o[2] = 0; continue; }
        float w = (float)((nn - 1) * (nn - 1));
        for (int r = 0; r < 3; ++r) {
            float wn = w * nt[r];
            for (int c = 0; c < 3; ++c) AtA[3 * r + c] = fmaf(wn, nt[c], AtA[3 * r + c]);
        }
        AtA[0] += 1.0e-6f; AtA[4] += 1.0e-6f; AtA[8] += 1.0e-6f;
        float inv[9];
        inverse3x3(AtA, inv);
        for (int r = 0; r < 3; ++r) o[r] = dot3f(inv[3 * r], inv[3 * r + 1], inv[3 * r + 2], Atb[0], Atb[1], Atb[2]);
    }
}

/* ======================================================================== */
/* estimator rows -> 27(+1) sums    eigen.inl:33-145                           */
/* ======================================================================== */
static inline void acc_row(double *S, const float J[6], float r) {
    /* deliberate deviation shared with the product (DESIGN.md, parity hazard 8): rows with a non-finite entry
     * are dropped (the reference would let the NaN poison the sum, eigenvalue.inl:28 signf(0) = 0/0) */
    float chk = r;
    for (int a = 0; a < 6; ++a) chk += J[a];
    if (!isfinite(chk)) return;
    int p = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) S[p++] += (double)J[a] * (double)J[b];
    for (int a = 0; a < 6; ++a) S[21 + a] += (double)J[a] * (double)r;
    S[27] += (double)r * (double)r;
}
static void rows_for(int kind, const float *vs, const float *ns, const float *cs,
                     const float *Cs, const float *vt, const float *nt,
                     const float *ct, const float *gt, const float *Ct,
                     float sg, float sp, double *S) {
    float J[6], r;
    if (kind == ORC_P2PLANE) { /* transformation_estimation.cu:34-56 */
        float d[3] = {vs[0] - vt[0], vs[1] - vt[1], vs[2] - vt[2]};
        r = dot3f(d[0], d[1], d[2], nt[0], nt[1], nt[2]);
        cross3(vs, nt, J);
        J[3] = nt[0]; J[4] = nt[1]; J[5] = nt[2];
        acc_row(S, J, r);
    } else if (kind == ORC_SYMMETRIC) { /* :58-90 */
        float nn[3] = {ns[0] + nt[0], ns[1] + nt[1], ns[2] + nt[2]};
        float d[3] = {vs[0] - vt[0], vs[1] - vt[1], vs[2] - vt[2]};
        float sm[3] = {vs[0] + vt[0], vs[1] + vt[1], vs[2] + vt[2]};
        r = dot3f(d[0], d[1], d[2], nn[0], nn[1], nn[2]);
        cross3(sm, nn, J);
        J[3] = nn[0]; J[4] = nn[1]; J[5] = nn[2];
        acc_row(S, J, r);
    } else if (kind == ORC_COLORED) { /* colored_icp.cu:150-216 */
        float d[3] = {vs[0] - vt[0], vs[1] - vt[1], vs[2] - vt[2]};
        float dn = dot3f(d[0], d[1], d[2], nt[0], nt[1], nt[2]);
        float cr[3];
        cross3(vs, nt, cr);
        for (int a = 0; a < 3; ++a) { J[a] = sg * cr[a]; J[3 + a] = sg * nt[a]; }
        r = sg * dn;
        acc_row(S, J, r);
        float vp[3], pd[3];
        for (int a = 0; a < 3; ++a) { vp[a] = fmaf(-dn, nt[a], vs[a]); pd[a] = vp[a] - vt[a]; }
        float is = intensity(cs), it = intensity(ct);
        float is0 = dot3f(gt[0], gt[1], gt[2], pd[0], pd[1], pd[2]) + it;
        float M[9];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b)
                M[3 * a + b] = (a == b) ? (float)(1.0 - (double)(nt[a] * nt[a])) : (-nt[a < b ? a : b]) * nt[a < b ? b : a];
        float gm[3];
        for (int b = 0; b < 3; ++b) gm[b] = dot3f(-gt[0], -gt[1], -gt[2], M[b], M[3 + b], M[6 + b]);
        cross3(vs, gm, cr);
        for (int a = 0; a < 3; ++a) { J[a] = sp * cr[a]; J[3 + a] = sp * gm[a]; }
        r = sp * (is - is0);
        acc_row(S, J, r);
    } else if (kind == ORC_GICP) { /* generalized_icp.cu:63-105 */
        float d[3] = {vs[0] - vt[0], vs[1] - vt[1], vs[2] - vt[2]};
        float M[9], Mi[9], W[9];
        for (int a = 0; a < 9; ++a) M[a] = Ct[a] + Cs[a];
        inverse3x3(M, Mi);
        sqrt_matrix3x3(Mi, W);
        for (int i = 0; i < 3; ++i) {
            const float *w = W + 3 * i;
            J[0] = fmaf(w[2], vs[1], -(w[1] * vs[2]));
            J[1] = fmaf(w[2], -vs[0], w[0] * vs[2]);
            J[2] = fmaf(w[1], vs[0], -(w[0] * vs[1]));
            J[3] = w[0]; J[4] = w[1]; J[5] = w[2];
            r = dot3f(w[0], w[1], w[2], d[0], d[1], d[2]);
            acc_row(S, J, r);
        }
    }
}
void orc_jtj_jtr(int kind, const float *src, const float *src_nrm,
                 const float *src_col, const float *src_cov, const float *tgt,
                 const float *tgt_nrm, const float *tgt_col,
                 const float *tgt_grad, const float *tgt_cov,
                 const int32_t *corr, int n_corr, float lambda_geometric,
                 double sums[32]) {
    /* colored_icp.cu:223-226: host double sqrt assigned to float */
    float sg = (float)sqrt((double)lambda_geometric);
    float lp = (float)(1.0 - (double)lambda_geometric);
    float sp = (float)sqrt((double)lp);
    double S[32];
    memset(S, 0, sizeof(S));
#pragma omp parallel
    {
        double L[32];
        memset(L, 0, sizeof(L));
#pragma omp for schedule(static) nowait
        for (int c = 0; c < n_corr; ++c) {
            size_t i = (size_t)corr[2 * c], j = (size_t)corr[2 * c + 1];
            rows_for(kind, src + 3 * i, src_nrm ? src_nrm + 3 * i : 0,
                     src_col ? src_col + 3 * i : 0, src_cov ? src_cov + 9 * i : 0,
                     tgt + 3 * j, tgt_nrm ? tgt_nrm + 3 * j : 0,
                     tgt_col ? tgt_col + 3 * j : 0, tgt_grad ? tgt_grad + 3 * j : 0,
                     tgt_cov ? tgt_cov + 9 * j : 0, sg, sp, L);
        }
#pragma omp critical
        for (int a = 0; a < 32; ++a) S[a] += L[a];
    }
    memcpy(sums, S, sizeof(S));
}

/* ======================================================================== */
/* 6x6 solve + se(3) exp     eigen.cu:28-50,75-122 (host code: no FMA)        */
/* ======================================================================== */
static float det6_partial_piv(const float A_in[36]) { /* Eigen determinant() n>4 -> PartialPivLU */
    float A[36];
    memcpy(A, A_in, sizeof(A));
    float det = 1.f;
    for (int k = 0; k < 6; ++k) {
        int p = k;
        float best = fabsf(A[6 * k + k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabsf(A[6 * i + k]) > best) { best = fabsf(A[6 * i + k]); p = i; }
        if (best == 0.f) return 0.f;
        if (p != k) {
            for (int j = 0; j < 6; ++j) { float t = A[6 * k + j]; A[6 * k + j] = A[6 * p + j]; A[6 * p + j] = t; }
            det = -det;
        }
        float piv = A[6 * k + k];
        det = det * piv;
        for (int i = k + 1; i < 6; ++i) {
            float f = A[6 * i + k] / piv;
            for (int j = k + 1; j < 6; ++j) A[6 * i + j] = A[6 * i + j] - f * A[6 * k + j];
        }
    }
    return det;
}
/* Eigen LDLT.h ldlt_inplace<Lower>::unblocked + _solve_impl, restated */
static void ldlt6_solve(const float A_in[36], const float b[6], float x[6]) {
    float A[36];
    memcpy(A, A_in, sizeof(A));
    int tr[6];
    for (int k = 0; k < 6; ++k) {
        int ib = k;
        float big = fabsf(A[6 * k + k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabsf(A[6 * i + i]) > big) { big = fabsf(A[6 * i + i]); ib = i; }
        tr[k] = ib;
        if (ib != k) {
            for (int j = 0; j < k; ++j) { float t = A[6 * k + j]; A[6 * k + j] = A[6 * ib + j]; A[6 * ib + j] = t; }
            for (int i = ib + 1; i < 6; ++i) { float t = A[6 * i + k]; A[6 * i + k] = A[6 * i + ib]; A[6 * i + ib] = t; }
            { float t = A[6 * k + k]; A[6 * k + k] = A[6 * ib + ib]; A[6 * ib + ib] = t; }
            for (int i = k + 1; i < ib; ++i) { float t = A[6 * i + k]; A[6 * i + k] = A[6 * ib + i]; A[6 * ib + i] = t; }
        }
        float temp[6];
        if (k > 0) {
            for (int j = 0; j < k; ++j) temp[j] = A[6 * j + j] * A[6 * k + j];
            float s = 0.f;
            for (int j = 0; j < k; ++j) s = s + A[6 * k + j] * temp[j];
            A[6 * k + k] = A[6 * k + k] - s;
            for (int i = k + 1; i < 6; ++i) {
                float s2 = 0.f;
                for (int j = 0; j < k; ++j) s2 = s2 + A[6 * i + j] * temp[j];
                A[6 * i + k] = A[6 * i + k] - s2;
            }
        }
        float akk = A[6 * k + k];
        if (fabsf(akk) > 0.f)
            for (int i = k + 1; i < 6; ++i) A[6 * i + k] = A[6 * i + k] / akk;
    }
    float y[6];
    memcpy(y, b, sizeof(y));
    for (int k = 0; k < 6; ++k)
        if (tr[k] != k) { float t = y[k]; y[k] = y[tr[k]]; y[tr[k]] = t; }
    for (int i = 0; i < 6; ++i) {
        float s = y[i];
        for (int j = 0; j < i; ++j) s = s - A[6 * i + j] * y[j];
        y[i] = s;
    }
    for (int i = 0; i < 6; ++i) y[i] = (fabsf(A[6 * i + i]) > FLT_MIN) ? y[i] / A[6 * i + i] : 0.f;
    for (int i = 5; i >= 0; --i) {
        float s = y[i];
        for (int j = i + 1; j < 6; ++j) s = s - A[6 * j + i] * y[j];
        y[i] = s;
    }
    for (int k = 5; k >= 0; --k)
        if (tr[k] != k) { float t = y[k]; y[k] = y[tr[k]]; y[tr[k]] = t; }
    memcpy(x, y, sizeof(y));
}
static void se3_exp(const float x[6], float T[16]) { /* eigen.cu:28-50 */
    memset(T, 0, 64);
    T[0] = T[5] = T[10] = T[15] = 1.f;
    T[3] = x[3]; T[7] = x[4]; T[11] = x[5];
    float th = sqrtf((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
    if (th == 0) return;
    float w0 = x[0] / th, w1 = x[1] / th, w2 = x[2] / th;
    float c = (float)cos((double)th), s = (float)sin((double)th);
    float oc = 1 - c;
    T[0] = c + w0 * w0 * oc;
    T[1] = w0 * w1 * oc - w2 * s;
    T[2] = w1 * s + w0 * w2 * oc;
    T[4] = w2 * s + w0 * w1 * oc;
    T[5] = c + w1 * w1 * oc;
    T[6] = -w0 * s + w1 * w2 * oc;
    T[8] = -w1 * s + w0 * w2 * oc;
    T[9] = w0 * s + w1 * w2 * oc;
    T[10] = c + w2 * w2 * oc;
}
int orc_solve_jtj(const float u[21], const float jtr[6], float det_thresh, float T[16]) {
    float A[36], b[6], x[6];
    int p = 0;
    for (int a = 0; a < 6; ++a)
        for (int c = a; c < 6; ++c) { A[6 * a + c] = u[p]; A[6 * c + a] = u[p]; ++p; }
    for (int a = 0; a < 6; ++a) b[a] = -jtr[a];
    memset(T, 0, 64);
    T[0] = T[5] = T[10] = T[15] = 1.f;
    if (det_thresh > 0) { /* eigen.cu:88-100 */
        float det = det6_partial_piv(A);
        if (fabsf(det) < det_thresh || isnan(det) || isinf(det)) return 0;
    }
    ldlt6_solve(A, b, x);
    se3_exp(x, T);
    return 1;
}
void orc_matmul4(const float A[16], const float B[16], float C[16]) {
    float R[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            R[4 * i + j] = ((A[4 * i] * B[j] + A[4 * i + 1] * B[4 + j]) + A[4 * i + 2] * B[8 + j]) + A[4 * i + 3] * B[12 + j];
    memcpy(C, R, sizeof(R));
}

/* ======================================================================== */
/* Kabsch  kabsch.cu:42-120 (divide-by-model.size() quirk :76-78,107)         */
/* ======================================================================== */
void orc_kabsch_sums(const float *src, const float *tgt, const int32_t *corr,
                     int n_corr, double sums[17]) {
    double S[17];
    memset(S, 0, sizeof(S));
    for (int c = 0; c < n_corr; ++c) {
        const float *s = src + 3 * (size_t)corr[2 * c], *t = tgt + 3 * (size_t)corr[2 * c + 1];
        for (int a = 0; a < 3; ++a) { S[a] += s[a]; S[3 + a] += t[a]; }
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) S[6 + 3 * a + b] += (double)s[a] * (double)t[b];
    }
    S[15] = (double)n_corr;
    memcpy(sums, S, sizeof(S));
}
/* one-sided Jacobi SVD of a 3x3 (double): A = U diag(s) V^T */
static void svd3(const double A[9], double U[9], double s[3], double V[9]) {
    double B[9];
    memcpy(B, A, sizeof(B));
    for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
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
        s[j] = nn;
        for (int i = 0; i < 3; ++i) U[3 * i + j] = (nn > 0) ? B[3 * i + j] / nn : 0.0;
    }
    /* complete U to an orthonormal basis when singular values vanish */
    for (int j = 0; j < 3; ++j)
        if (s[j] == 0) {
            int a = (j + 1) % 3, b = (j + 2) % 3;
            if (s[a] > 0 && s[b] > 0) {
                U[j] = U[3 + a] * U[6 + b] - U[6 + a] * U[3 + b];
                U[3 + j] = U[6 + a] * U[b] - U[a] * U[6 + b];
                U[6 + j] = U[a] * U[3 + b] - U[3 + a] * U[b];
            }
        }
    /* A = 0: Eigen's JacobiSVD returns U = V = I (kabsch.cu:108-113 then gives the identity rotation, not R = 0) */
    if (s[0] == 0 && s[1] == 0 && s[2] == 0)
        for (int i = 0; i < 9; ++i) U[i] = (i % 4 == 0) ? 1.0 : 0.0;
}
static double det3d(const double M[9]) {
    return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}
void orc_kabsch_from_sums(const double S[17], int n_model, float T[16]) {
    memset(T, 0, 64);
    T[0] = T[5] = T[10] = T[15] = 1.f;
    double C = S[15];
    float div = 1.0f / (float)n_model;
    float mc[3], tc[3];
    for (int a = 0; a < 3; ++a) { mc[a] = (float)S[a] * div; tc[a] = (float)S[3 + a] * div; }
    double H[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            double h = S[6 + 3 * a + b] - (double)mc[a] * S[3 + b] - S[a] * (double)tc[b] + C * (double)mc[a] * (double)tc[b];
            H[3 * a + b] = (double)((float)h / (float)n_model);
        }
    double U[9], sv[3], V[9], UV[9];
    svd3(H, U, sv, V);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) UV[3 * i + j] = U[3 * i] * V[j] + U[3 * i + 1] * V[3 + j] + U[3 * i + 2] * V[6 + j];
    double dd = det3d(UV);
    double ss[3] = {1.0, 1.0, dd};
    float R[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double r = 0;
            for (int k = 0; k < 3; ++k) r += V[3 * i + k] * ss[k] * U[3 * j + k];
            R[3 * i + j] = (float)r;
        }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = R[3 * i + j];
        T[4 * i + 3] = tc[i] - dot3f(R[3 * i], R[3 * i + 1], R[3 * i + 2], mc[0], mc[1], mc[2]);
    }
}

/* ======================================================================== */
/* registration::ComputeFPFHFeature (fpfh.cu:34-229)                          */
/* ======================================================================== */
/* deterministic atan2f (specification shared with cupoch_b200/csrc/fpfh.cu): float64, IEEE add / mul / div / sqrt only.
 * atan(t), t >= 0: half-angle reductions t <- t / (1 + sqrt(1 + t^2)) until t <= 0.2 (at most 3), 13 Taylor terms */
static double dt_atan_pos(double t) {
    int doubled = 0;
    for (int k = 0; k < 3; ++k) {
        if (t > 0.2) {
            t = t / (1.0 + sqrt(1.0 + t * t));
            ++doubled;
        }
    }
    const double t2 = t * t;
    double p = 1.0 / 25.0;
    for (int k = 11; k >= 0; --k) p = 1.0 / (double)(2 * k + 1) - t2 * p;
    double a = t * p;
    for (int k = 0; k < doubled; ++k) a = 2.0 * a;
    return a;
}
static float det_atan2f(float yf, float xf) {
    const double y = (double)yf, x = (double)xf;
    if (x == 0.0 && y == 0.0) return copysignf((signbit(xf) ? (float)DT_PI : 0.f), yf);
    const double ay = fabs(y), ax = fabs(x);
    double a;
    if (ay <= ax) a = dt_atan_pos(ay / ax);
    else a = DT_PI_2 - dt_atan_pos(ax / ay);
    if (x < 0.0) a = DT_PI - a;
    return (float)(signbit(y) ? -a : a); /* atan2(-0, x < 0) = -pi, not +pi */
}
float orc_det_atan2f(float y, float x) { return det_atan2f(y, x); }
/* ComputePairFeatures (fpfh.cu:34-69) */
static void pair_features(const float *p1, const float *n1, const float *p2, const float *n2, float f[4]) {
    float d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
    f[0] = f[1] = f[2] = 0.f;
    f[3] = sqrtf(dot3f(d[0], d[1], d[2], d[0], d[1], d[2]));
    if (f[3] == 0.f) return;
    float a[3] = {n1[0], n1[1], n1[2]}, b[3] = {n2[0], n2[1], n2[2]};
    const float angle1 = dot3f(a[0], a[1], a[2], d[0], d[1], d[2]) / f[3];
    const float angle2 = dot3f(b[0], b[1], b[2], d[0], d[1], d[2]) / f[3];
    const float c1 = fabsf(angle1), c2 = fabsf(angle2);
    /* acos(|x|) is NaN beyond 1 (an un-normalised normal): the reference's comparison is then false */
    const int swap = (c1 <= 1.f && c2 <= 1.f) && (det_acosf(c1) > det_acosf(c2));
    if (swap) {
        for (int k = 0; k < 3; ++k) { const float t = a[k]; a[k] = b[k]; b[k] = t; d[k] = -d[k]; }
        f[2] = -angle2;
    } else {
        f[2] = angle1;
    }
    float v[3], w[3];
    cross3(d, a, v);
    const float vn = sqrtf(dot3f(v[0], v[1], v[2], v[0], v[1], v[2]));
    if (vn == 0.f) { f[0] = f[1] = f[2] = f[3] = 0.f; return; }
    for (int k = 0; k < 3; ++k) v[k] = v[k] / vn;
    cross3(a, v, w);
    f[1] = dot3f(v[0], v[1], v[2], b[0], b[1], b[2]);
    f[0] = det_atan2f(dot3f(w[0], w[1], w[2], b[0], b[1], b[2]), dot3f(a[0], a[1], a[2], b[0], b[1], b[2]));
}
static int hist_bin(double x) {
    int h = (int)floor(x);
    return h < 0 ? 0 : (h >= 11 ? 10 : h);
}
/* knn > 0: KDTreeSearchParamKNN, else Radius(radius, max_nn).  out [n][33].  compute_spfh_functor (:71-112) then
 * compute_fpfh_functor (:147-190), both over the SAME neighbour table (nearest first) */
void orc_compute_fpfh_feature(const float *pts, const float *nrm, int n, int knn, float radius, int max_nn, float *out) {
    const int k = knn > 0 ? knn : max_nn;
    if (n <= 0 || k <= 0) return;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * k);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * k);
    float *spfh = (float *)calloc((size_t)n * 33, sizeof(float));
    orc_kdtree *kd = orc_kdtree_build(pts, n);
    orc_kdtree_search(kd, pts, n, k, knn > 0 ? -1.0f : radius, idx, d2);
    orc_kdtree_free(kd);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        float *ft = spfh + (size_t)i * 33;
        int cnt = 0;
        for (int q = 0; q < k; ++q) cnt += idx[(size_t)i * k + q] >= 0;
        const float hist_incr = (float)(100.0 / (double)(float)(cnt - 1));
        for (int q = 0; q < k; ++q) {
            const int j = idx[(size_t)i * k + q];
            if (j < 0 || j == i) continue;
            float pf[4];
            pair_features(pts + 3 * i, nrm + 3 * i, pts + 3 * j, nrm + 3 * j, pf);
            const double PI = 3.14159265358979323846;
            ft[hist_bin(11.0 * ((double)pf[0] + PI) / (2.0 * PI))] += hist_incr;
            ft[11 + hist_bin(11.0 * ((double)pf[1] + 1.0) * 0.5)] += hist_incr;
            ft[22 + hist_bin(11.0 * ((double)pf[2] + 1.0) * 0.5)] += hist_incr;
        }
    }
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        float ft[33], sum[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < 33; ++j) ft[j] = 0.f;
        for (int q = 0; q < k; ++q) {
            const int nb = idx[(size_t)i * k + q];
            if (nb < 0 || nb == i) continue;
            const float dist = d2[(size_t)i * k + q];
            if (dist == 0.f) continue;
            for (int j = 0; j < 33; ++j) {
                const float val = spfh[(size_t)nb * 33 + j] / dist;
                sum[j / 11] = sum[j / 11] + val;
                ft[j] = ft[j] + val;
            }
        }
        for (int j = 0; j < 3; ++j)
            if (sum[j] != 0.f) sum[j] = (float)(100.0 / (double)sum[j]);
        for (int j = 0; j < 33; ++j) out[(size_t)i * 33 + j] = ft[j] * sum[j / 11] + spfh[(size_t)i * 33 + j];
    }
    free(idx);
    free(d2);
    free(spfh);
}

/* ======================================================================== */
/* PointCloud::ClusterDBSCAN (pointcloud_cluster.cu:30-179)                   */
/* ======================================================================== */
/* Restated as the reference runs it: radius search with max_nn = max_edges + 1; degrees (:34-55: the point itself is
 * dropped, a point with fewer than min_points other neighbours loses all its edges); for i = 0..n-1, if i is unvisited,
 * BFS from i over the edges WITHOUT regard to earlier labels (:57-82), label the reached set with the next cluster id, or
 * -1 when it has fewer than min_points members (:150-176).  Returns the number of cluster ids handed out. */
int orc_cluster_dbscan(const float *pts, int n, float eps, int min_points, int max_edges, int32_t *labels) {
    if (n <= 0) return 0;
    const int K = max_edges + 1;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * K);
    float *d2 = (float *)malloc(sizeof(float) * (size_t)n * K);
    orc_kdtree *kd = orc_kdtree_build(pts, n);
    orc_kdtree_search(kd, pts, n, K, eps, idx, d2);
    orc_kdtree_free(kd);
    int *deg = (int *)malloc(sizeof(int) * n), *xa = (int *)malloc(sizeof(int) * n), *queue = (int *)malloc(sizeof(int) * n);
    char *visited = (char *)calloc(n, 1);
    for (int i = 0; i < n; ++i) {
        int c = 0;
        for (int k = 0; k < K; ++k) {
            const int j = idx[(size_t)i * K + k];
            c += (j >= 0 && j != i);
        }
        deg[i] = (c >= min_points) ? c : 0;
        labels[i] = -1;
        xa[i] = -1;
    }
    int cluster = 0;
    for (int i = 0; i < n; ++i) {
        if (visited[i]) continue;
        int head = 0, tail = 0;
        queue[tail++] = i;
        xa[i] = i; /* stamp = seed */
        while (head < tail) {
            const int u = queue[head++];
            if (deg[u] == 0) continue;
            for (int k = 0; k < K; ++k) {
                const int v = idx[(size_t)u * K + k];
                if (v < 0 || v == u || xa[v] == i) continue;
                xa[v] = i;
                queue[tail++] = v;
            }
        }
        const int noise = tail < min_points;
        for (int q = 0; q < tail; ++q) {
            labels[queue[q]] = noise ? -1 : cluster;
            visited[queue[q]] = 1;
        }
        if (!noise) ++cluster;
    }
    free(idx); free(d2); free(deg); free(xa); free(queue); free(visited);
    return cluster;
}

/* ======================================================================== */
/* The other users of the reducer (SURVEY 8f rank 3), on explicit rows        */
/* ======================================================================== */
/* multiple_jtj_jtr_functor (eigen.inl:48-70): per element, rows in order, float32 */
static void private_sums(const float *J, const float *r, int i, int num_j, float v[28]) {
    for (int k = 0; k < 28; ++k) v[k] = 0.f;
    for (int j = 0; j < num_j; ++j) {
        const float *x = J + ((size_t)i * num_j + j) * 6;
        const float rr = r[(size_t)i * num_j + j];
        int p = 0;
        for (int a = 0; a < 6; ++a)
            for (int b = a; b < 6; ++b) { v[p] = v[p] + x[a] * x[b]; ++p; }
        for (int a = 0; a < 6; ++a) v[21 + a] = v[21 + a] + x[a] * rr;
        v[27] = v[27] + rr * rr;
    }
}
/* utility::ComputeJTJandJTr<Matrix6f, Vector6f, NumJ> (eigen.inl:120-145): sums[0..20] JTJ upper, [21..26] JTr, [27] r^2;
 * float32 per-element values accumulated in float64 (the order-independent limit of thrust's float reduction) */
void orc_jtj_rows(const float *J, const float *r, int n, int num_j, double sums[32]) {
    for (int k = 0; k < 32; ++k) sums[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        float v[28];
        private_sums(J, r, i, num_j, v);
        for (int k = 0; k < 28; ++k) sums[k] += (double)v[k];
    }
}
/* utility::ComputeWeightedJTJandJTr (eigen.inl:147-195) with the RGB-D odometry's Student-t weights
 * (odometry.cu:633-648): w_sum = sum_i r2_i (nu + 1.0) / (nu + r2_i / sigma2)   [double product and quotient: the 1.0
 * literal], w_i = (nu + 1) / (nu + r2_i / w_sum)   [float], sums of w_i * (JTJ_i, JTr_i, r2_i). */
float orc_weighted_jtj_rows(const float *J, const float *r, int n, int num_j, float sigma2, float nu, double sums[32]) {
    double ws = 0.0;
    for (int i = 0; i < n; ++i) {
        float v[28];
        private_sums(J, r, i, num_j, v);
        const float r2 = v[27];
        const float den = nu + r2 / sigma2;
        ws += (double)(float)(((double)r2 * ((double)nu + 1.0)) / (double)den);
    }
    const float w_sum = (float)ws;
    for (int k = 0; k < 32; ++k) sums[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        float v[28];
        private_sums(J, r, i, num_j, v);
        const float w = (nu + 1.f) / (nu + v[27] / w_sum);
        for (int k = 0; k < 28; ++k) sums[k] += (double)(v[k] * w);
    }
    return w_sum;
}
/* registration::KabschWeighted (kabsch.cu:138-201): weighted centres, H = sum w^2 (m - mc)(t - tc)^T / sum w^2,
 * R = V diag(1, 1, det(U V)) U^T, t = tc - R mc */
void orc_kabsch_weighted(const float *model, const float *target, const float *weight, int n, float T[16]) {
    memset(T, 0, 64);
    T[0] = T[5] = T[10] = T[15] = 1.f;
    if (n <= 0) return;
    double sw = 0, sm[3] = {0, 0, 0}, st[3] = {0, 0, 0}, sww = 0;
    for (int i = 0; i < n; ++i) {
        const float w = weight[i];
        sw += (double)w;
        for (int a = 0; a < 3; ++a) {
            sm[a] += (double)(model[3 * i + a] * w);
            st[a] += (double)(target[3 * i + a] * w);
        }
        sww += (double)(w * w);
    }
    const float divided_by = 1.0f / (float)sw;
    float mc[3], tc[3];
    for (int a = 0; a < 3; ++a) { mc[a] = (float)sm[a] * divided_by; tc[a] = (float)st[a] * divided_by; }
    const float h_weight = (float)sww;
    double hs[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n; ++i) {
        const float w = weight[i], ww = w * w;
        float cx[3], cy[3];
        for (int a = 0; a < 3; ++a) { cx[a] = ww * (model[3 * i + a] - mc[a]); cy[a] = target[3 * i + a] - tc[a]; }
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) hs[3 * a + b] += (double)(cx[a] * cy[b]);
    }
    double H[9];
    for (int k = 0; k < 9; ++k) H[k] = (double)((float)hs[k] / h_weight);
    double U[9], sv[3], V[9], UV[9];
    svd3(H, U, sv, V);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) UV[3 * i + j] = U[3 * i] * V[j] + U[3 * i + 1] * V[3 + j] + U[3 * i + 2] * V[6 + j];
    double ss[3] = {1.0, 1.0, det3d(UV)};
    for (int i = 0; i < 3; ++i) {
        float Rf[3];
        for (int j = 0; j < 3; ++j) {
            double rr = 0;
            for (int k = 0; k < 3; ++k) rr += V[3 * i + k] * ss[k] * U[3 * j + k];
            Rf[j] = (float)rr;
            T[4 * i + j] = Rf[j];
        }
        T[4 * i + 3] = tc[i] - ((Rf[0] * mc[0] + Rf[1] * mc[1]) + Rf[2] * mc[2]);
    }
}

/* ======================================================================== */
/* registration.cu:33-80 GetRegistrationResultAndCorrespondences             */
/* ======================================================================== */
void orc_correspondences(const float *src, int n, const float *tgt, int m,
                         const orc_kdtree *kd, float max_distance,
                         int32_t *corr, int *n_corr, float *fitness, float *rmse) {
    *n_corr = 0;
    *fitness = 0.f;
    *rmse = 0.f;
    if (max_distance <= 0.0f || n <= 0) return;
    int32_t *idx = (int32_t *)malloc(sizeof(int32_t) * n);
    float *d2 = (float *)malloc(sizeof(float) * n);
    if (kd)
        orc_kdtree_search(kd, src, n, 1, max_distance, idx, d2);
    else
        orc_search_bruteforce(tgt, m, src, n, 1, max_distance, idx, d2);
    double e2 = 0;
    int c = 0;
    for (int i = 0; i < n; ++i)
        if (idx[i] >= 0) {
            corr[2 * c] = i;
            corr[2 * c + 1] = idx[i];
            e2 += d2[i];
            ++c;
        }
    *n_corr = c;
    if (c > 0) {
        *fitness = (float)c / (float)n;
        *rmse = sqrtf((float)e2 / (float)c);
    }
    free(idx);
    free(d2);
}

static void identity4(float T[16]) {
    memset(T, 0, 64);
    T[0] = T[5] = T[10] = T[15] = 1.f;
}
static int is_identity4(const float T[16]) { /* Eigen isIdentity(prec=1e-5) */
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float v = T[4 * i + j];
            if (i == j) { if (fabsf(v - 1.f) > 1e-5f) return 0; }
            else if (fabsf(v) > 1e-5f) return 0;
        }
    return 1;
}
static float *dupf(const float *p, size_t cnt) {
    if (!p) return 0;
    float *q = (float *)malloc(sizeof(float) * (cnt ? cnt : 1));
    memcpy(q, p, sizeof(float) * cnt);
    return q;
}

/* registration.cu:121-173 RegistrationICP */
int orc_registration_icp(const float *src_in, const float *src_nrm_in,
                         const float *src_col, const float *src_cov_in, int n,
                         const float *tgt, const float *tgt_nrm,
                         const float *tgt_col, const float *tgt_grad,
                         const float *tgt_cov, int m, const float init[16],
                         const orc_icp_params *prm, orc_icp_result *res,
                         int32_t *corr, float *trace_T) {
    float T[16];
    memcpy(T, init, 64);
    orc_kdtree *kd = prm->use_kdtree ? orc_kdtree_build(tgt, m) : 0;
    float *src = dupf(src_in, 3 * (size_t)n);
    float *src_nrm = dupf(src_nrm_in, 3 * (size_t)n);
    float *src_cov = dupf(src_cov_in, 9 * (size_t)n);
    if (!is_identity4(init)) {
        orc_transform_points(src, n, init);
        if (src_nrm) orc_transform_normals(src_nrm, n, init);
        if (src_cov) orc_rotate_covariances(src_cov, n, init);
    }
    int nc;
    float fit, rmse;
    orc_correspondences(src, n, tgt, m, kd, prm->max_distance, corr, &nc, &fit, &rmse);
    if (trace_T) memcpy(trace_T, T, 64);
    int it = 0;
    for (int i = 0; i < prm->max_iteration; ++i) {
        float U[16];
        identity4(U);
        if (prm->kind == ORC_P2P) {
            double S[17];
            orc_kabsch_sums(src, tgt, corr, nc, S);
            orc_kabsch_from_sums(S, n, U);
        } else {
            int ok = nc > 0;
            if ((prm->kind == ORC_P2PLANE || prm->kind == ORC_COLORED) && !tgt_nrm) ok = 0;
            if (prm->kind == ORC_SYMMETRIC && (!tgt_nrm || !src_nrm)) ok = 0;
            if (prm->kind == ORC_COLORED && (!tgt_col || !src_col)) ok = 0;
            if (prm->kind == ORC_GICP && (!tgt_cov || !src_cov)) ok = 0;
            if (ok) {
                double S[32];
                orc_jtj_jtr(prm->kind, src, src_nrm, src_col, src_cov, tgt, tgt_nrm,
                            tgt_col, tgt_grad, tgt_cov, corr, nc, prm->lambda_geometric, S);
                float u[21], b[6];
                for (int a = 0; a < 21; ++a) u[a] = (float)S[a];
                for (int a = 0; a < 6; ++a) b[a] = (float)S[21 + a];
                float det_thresh = (prm->kind == ORC_GICP) ? -1.f : prm->det_thresh;
                int solved = orc_solve_jtj(u, b, det_thresh, U);
                if (solved && prm->kind == ORC_SYMMETRIC) {
                    /* transformation_estimation.cu:319-339: R <- R*R in double */
                    double R[9], R2[9];
                    for (int a = 0; a < 3; ++a)
                        for (int c = 0; c < 3; ++c) R[3 * a + c] = (double)U[4 * a + c];
                    for (int a = 0; a < 3; ++a)
                        for (int c = 0; c < 3; ++c)
                            R2[3 * a + c] = R[3 * a] * R[c] + R[3 * a + 1] * R[3 + c] + R[3 * a + 2] * R[6 + c];
                    for (int a = 0; a < 3; ++a)
                        for (int c = 0; c < 3; ++c) U[4 * a + c] = (float)R2[3 * a + c];
                }
            }
        }
        orc_matmul4(U, T, T);
        orc_transform_points(src, n, U);
        if (src_nrm) orc_transform_normals(src_nrm, n, U);
        if (src_cov) orc_rotate_covariances(src_cov, n, U);
        float bf = fit, br = rmse;
        orc_correspondences(src, n, tgt, m, kd, prm->max_distance, corr, &nc, &fit, &rmse);
        ++it;
        if (trace_T) memcpy(trace_T + 16 * it, T, 64);
        if (fabsf(bf - fit) < prm->relative_fitness && fabsf(br - rmse) < prm->relative_rmse) break;
    }
    memcpy(res->transformation, T, 64);
    res->fitness = fit;
    res->inlier_rmse = rmse;
    res->n_corr = nc;
    res->iterations = it;
    orc_kdtree_free(kd);
    free(src);
    free(src_nrm);
    free(src_cov);
    return 0;
}

/* =====================================================================================================================
 * OccupancyGrid (geometry/occupancygrid.cu): dense log-odds grid, Insert by ray traversal, AddVoxels, SetFreeArea,
 * bound-box extraction.  SURVEY 8f rank 2 (second half).  The grid is an array prob[res^3] (NaN = unknown, the default of
 * OccupancyVoxel::prob_log_, occupancygrid.h) + has_index[res^3] (whether grid_index_ was ever written: SetFreeArea does
 * not write it, occupancygrid.cu:441-446, so extracted voxels of such cells carry (0,0,0)) + the u16 bounds.
 * params = { clamping_thres_min, clamping_thres_max, prob_hit_log, prob_miss_log }.
 * ===================================================================================================================*/
static inline long occ_index_of(int x, int y, int z, int res) { /* utility/helper.h:422-424 (int arithmetic) */
    return (long)(x * res * res + y * res + z);
}
static inline int occ_in_range(const int v[3], int res) { /* occupancygrid.cu:173-178 */
    return !(v[0] < 0 || v[1] < 0 || v[2] < 0 || v[0] >= res || v[1] >= res || v[2] >= res);
}
/* add_occupancy_functor (occupancygrid.cu:246-275) for one voxel */
static void occ_add_one(float *prob, uint8_t *has_index, const int v[3], int res, const float params[4], int occupied) {
    const long idx = occ_index_of(v[0], v[1], v[2], res);
    float p = prob[idx];
    p = (p != p) ? 0.f : p;
    p += occupied ? params[2] : params[3];
    prob[idx] = fminf(fmaxf(p, params[0]), params[1]);
    has_index[idx] = 1;
}
/* VoxelTraversal (occupancygrid.cu:57-132): voxels the segment start -> end passes through, the end voxel excluded
 * (unless it is the start voxel), at most n_buffer of them; returns their number.  Mirrors the reference statement by
 * statement (the int += float steps, the tie order, both stop tests) except for the first boundary: cell k is
 * [k vs, (k + 1) vs), and the ray leaves it through (k + 1) vs going up and k vs going down (DESIGN §4 item 27).
 * ref_rule != 0 puts it at (k + 0.5 step) vs like the reference (:83-85), half a voxel off that cell's faces. */
static int occ_voxel_traversal(int (*voxels)[3], int n_buffer, int half, const float start[3], const float end[3], float vs,
                               int ref_rule) {
    int n = 0;
    float ray[3] = {end[0] - start[0], end[1] - start[1], end[2] - start[2]};
    const float length = sqrtf((ray[0] * ray[0] + ray[1] * ray[1]) + ray[2] * ray[2]);
    if (length == 0) return 0;
    for (int a = 0; a < 3; ++a) ray[a] /= length;
    int cur[3], last[3];
    float step[3], tmax[3], tdelta[3];
    for (int a = 0; a < 3; ++a) {
        cur[a] = (int)floorf(start[a] / vs);
        last[a] = (int)floorf(end[a] / vs);
        step[a] = (ray[a] > 0) ? 1.f : ((ray[a] < 0) ? -1.f : 0.f);
        const double off = ref_rule ? 0.5 * (double)step[a] : ((step[a] > 0) ? 1.0 : 0.0);
        const float boundary = (float)(((double)cur[a] + off) * (double)vs);
        tmax[a] = (step[a] != 0) ? (boundary - start[a]) / ray[a] : INFINITY;
        tdelta[a] = (step[a] != 0) ? vs / fabsf(ray[a]) : INFINITY;
    }
    if (n_buffer <= 0) return 0;
    for (int a = 0; a < 3; ++a) voxels[n][a] = cur[a] + half;
    ++n;
    while (n < n_buffer) {
        int ax;
        if (tmax[0] < tmax[1]) ax = (tmax[0] < tmax[2]) ? 0 : 2;
        else ax = (tmax[1] < tmax[2]) ? 1 : 2;
        cur[ax] = (int)((float)cur[ax] + step[ax]);
        tmax[ax] += tdelta[ax];
        if (last[0] == cur[0] && last[1] == cur[1] && last[2] == cur[2]) break;
        const float d = fminf(fminf(tmax[0], tmax[1]), tmax[2]);
        if (d > length) break;
        for (int a = 0; a < 3; ++a) voxels[n][a] = cur[a] + half;
        ++n;
    }
    return n;
}
static void occ_bounds_merge(uint16_t bounds[6], const int v[3]) { /* AddVoxels :585-592: min / max with the list's extremes */
    for (int a = 0; a < 3; ++a) {
        const uint16_t u = (uint16_t)v[a];
        if (u < bounds[a]) bounds[a] = u;
        if (u > bounds[3 + a]) bounds[3 + a] = u;
    }
}
/* OccupancyGrid::AddVoxels (occupancygrid.cu:579-600); voxels [n][3] grid indices.  Like the reference, indices are NOT
 * range-checked here (the callers filter them) -- out-of-range input is the caller's error. */
void orc_occgrid_add_voxels(float *prob, uint8_t *has_index, uint16_t bounds[6], int res, const float params[4],
                            const int32_t *voxels, int n, int occupied) {
    if (n <= 0) return;
    for (int i = 0; i < n; ++i) {
        const int v[3] = {voxels[3 * i], voxels[3 * i + 1], voxels[3 * i + 2]};
        occ_bounds_merge(bounds, v);
        occ_add_one(prob, has_index, v, res, params, occupied);
    }
}
/* OccupancyGrid::Insert (occupancygrid.cu:462-526).  Every voxel is updated at most once per call (the reference sorts and
 * uniques the voxel lists, :179-183,:239-243); free voxels that are also occupied are dropped (set_difference, :516-520).
 * stamp: scratch [res^3] bytes, all zero on entry and on return.  ref_rule: the traversal's boundary rule (see
 * occ_voxel_traversal); 0 is the library's. */
void orc_occgrid_insert(float *prob, uint8_t *has_index, uint8_t *stamp, uint16_t bounds[6], int res, float voxel_size,
                        const float origin[3], const float params[4], const float *points, int n, const float viewpoint[3],
                        float max_range, int ref_rule) {
    if (n <= 0) return;
    const int half = res / 2;
    float *ranged = (float *)malloc(sizeof(float) * 3 * (size_t)n);
    uint8_t *hit = (uint8_t *)malloc((size_t)n);
    float max_dist = -INFINITY;
    for (int i = 0; i < n; ++i) { /* :471-489 */
        const float *pt = points + 3 * i;
        const float d[3] = {pt[0] - viewpoint[0], pt[1] - viewpoint[1], pt[2] - viewpoint[2]};
        const float dist = sqrtf((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
        const int is_hit = max_range < 0 || dist <= max_range;
        float r[3];
        for (int a = 0; a < 3; ++a)
            r[a] = is_hit ? pt[a] : ((dist == 0) ? viewpoint[a] : viewpoint[a] + d[a] / dist * max_range);
        float m = 0.f;
        for (int a = 0; a < 3; ++a) {
            ranged[3 * i + a] = r[a];
            m = fmaxf(m, fabsf(r[a] - viewpoint[a]));
        }
        hit[i] = (uint8_t)is_hit;
        if (m > max_dist) max_dist = m;
    }
    const int n_div = (int)ceilf(max_dist / voxel_size);
    /* pass 1: occupied voxels (:224-244) -> stamp 2 */
    for (int i = 0; i < n; ++i) {
        if (!hit[i]) continue;
        int v[3];
        for (int a = 0; a < 3; ++a) v[a] = (int)floorf((ranged[3 * i + a] - origin[a]) / voxel_size) + half;
        if (!occ_in_range(v, res)) continue;
        stamp[occ_index_of(v[0], v[1], v[2], res)] = 2;
    }
    /* pass 2: free voxels (:152-184), n_step = (n_div + 1) * 3 entries per ray; those not occupied are updated once */
    long n_free = 0, n_occ = 0;
    int free_min[3] = {65536, 65536, 65536}, free_max[3] = {-1, -1, -1};
    if (n_div > 0) {
        const int n_step = (n_div + 1) * 3;
        int(*buf)[3] = (int(*)[3])malloc(sizeof(int) * 3 * (size_t)n_step);
        const float start[3] = {viewpoint[0] - origin[0], viewpoint[1] - origin[1], viewpoint[2] - origin[2]};
        for (int i = 0; i < n; ++i) {
            const float end[3] = {ranged[3 * i] - origin[0], ranged[3 * i + 1] - origin[1], ranged[3 * i + 2] - origin[2]};
            const int m = occ_voxel_traversal(buf, n_step, half, start, end, voxel_size, ref_rule);
            for (int k = 0; k < m; ++k) {
                if (!occ_in_range(buf[k], res)) continue;
                const long idx = occ_index_of(buf[k][0], buf[k][1], buf[k][2], res);
                if (stamp[idx]) continue; /* occupied, or already counted as free */
                stamp[idx] = 1;
                ++n_free;
                for (int a = 0; a < 3; ++a) {
                    if (buf[k][a] < free_min[a]) free_min[a] = buf[k][a];
                    if (buf[k][a] > free_max[a]) free_max[a] = buf[k][a];
                }
                occ_add_one(prob, has_index, buf[k], res, params, 0);
            }
        }
        /* clear the free stamps again (second traversal: cheaper than an n_free list for the oracle's sizes) */
        for (int i = 0; i < n; ++i) {
            const float end[3] = {ranged[3 * i] - origin[0], ranged[3 * i + 1] - origin[1], ranged[3 * i + 2] - origin[2]};
            const int m = occ_voxel_traversal(buf, n_step, half, start, end, voxel_size, ref_rule);
            for (int k = 0; k < m; ++k)
                if (occ_in_range(buf[k], res)) {
                    const long idx = occ_index_of(buf[k][0], buf[k][1], buf[k][2], res);
                    if (stamp[idx] == 1) stamp[idx] = 0;
                }
        }
        free(buf);
        if (n_free > 0) { occ_bounds_merge(bounds, free_min); occ_bounds_merge(bounds, free_max); }
    }
    /* pass 3: the occupied voxels, once each */
    for (int i = 0; i < n; ++i) {
        if (!hit[i]) continue;
        int v[3];
        for (int a = 0; a < 3; ++a) v[a] = (int)floorf((ranged[3 * i + a] - origin[a]) / voxel_size) + half;
        if (!occ_in_range(v, res)) continue;
        const long idx = occ_index_of(v[0], v[1], v[2], res);
        if (stamp[idx] != 2) continue;
        stamp[idx] = 0;
        ++n_occ;
        occ_bounds_merge(bounds, v);
        occ_add_one(prob, has_index, v, res, params, 1);
    }
    (void)n_occ;
    free(ranged);
    free(hit);
}
/* OccupancyGrid::SetFreeArea (occupancygrid.cu:415-460): REPLACES the bounds by the clipped box and adds prob_miss_log to
 * every cell of it, without clamping and without writing grid_index_. */
void orc_occgrid_set_free_area(float *prob, uint16_t bounds[6], int res, float voxel_size, const float origin[3],
                               float prob_miss_log, const float min_bound[3], const float max_bound[3]) {
    const int half = res / 2;
    int lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        int imin = (int)floorf((min_bound[a] - origin[a]) / voxel_size) + half;
        int imax = (int)floorf((max_bound[a] - origin[a]) / voxel_size) + half;
        lo[a] = imin > 0 ? imin : 0;
        hi[a] = imax < res - 1 ? imax : res - 1;
        bounds[a] = (uint16_t)lo[a];
        bounds[3 + a] = (uint16_t)hi[a];
    }
    /* diff = max - min + 1 in u16 arithmetic (:438-439): an inverted box wraps around; mirrored as 'nothing to do' only
     * when a dimension is empty after the u16 cast */
    for (int x = lo[0]; x <= hi[0]; ++x)
        for (int y = lo[1]; y <= hi[1]; ++y)
            for (int z = lo[2]; z <= hi[2]; ++z) {
                const long idx = occ_index_of(x, y, z, res);
                float p = prob[idx];
                p = (p != p) ? 0.f : p;
                prob[idx] = p + prob_miss_log;
            }
}
/* ExtractBoundVoxels (occupancygrid.cu:358-378) with the three predicates (:380-408): which = 0 known, 1 free (<= thres),
 * 2 occupied (> thres).  Box order (x slowest).  out_index [cap][3] = the voxel's stored grid_index_ ((0,0,0) if never
 * written), out_prob [cap].  Returns the count. */
int orc_occgrid_extract(const float *prob, const uint8_t *has_index, const uint16_t bounds[6], int res, float thres, int which,
                        int32_t *out_index, float *out_prob) {
    int m = 0;
    for (int x = bounds[0]; x <= bounds[3]; ++x)
        for (int y = bounds[1]; y <= bounds[4]; ++y)
            for (int z = bounds[2]; z <= bounds[5]; ++z) {
                const long idx = occ_index_of(x, y, z, res);
                const float p = prob[idx];
                if (p != p) continue;
                if (which == 1 && !(p <= thres)) continue;
                if (which == 2 && !(p > thres)) continue;
                const int w = has_index[idx];
                out_index[3 * m] = w ? x : 0; out_index[3 * m + 1] = w ? y : 0; out_index[3 * m + 2] = w ? z : 0;
                out_prob[m] = p;
                ++m;
            }
    return m;
}
/* DenseGrid::GetVoxelIndex (densegrid.inl:137-146): only the LINEAR index is range-checked */
long orc_occgrid_voxel_index(int res, float voxel_size, const float origin[3], const float point[3]) {
    const int half = res / 2;
    int v[3];
    for (int a = 0; a < 3; ++a) v[a] = (int)floorf((point[a] - origin[a]) / voxel_size) + half;
    const int idx = v[0] * res * res + v[1] * res + v[2];
    if (idx < 0 || idx >= res * res * res) return -1;
    return idx;
}
