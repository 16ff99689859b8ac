/* mesh_clean.c -- plain-C restatement of TriangleMesh cleanup, operator+= and GetSelfIntersectingTriangles
 * (geometry/trianglemesh.cu:411-452, 903-1141; meshbase.cu:124-151) for the tests.  DESIGN section 4 item 26.
 *
 * The self-intersection predicate is intersection_test::TriangleTriangle3d (intersection_test.inl:47-69): the six
 * vertices centred on their mean and divided by their per-axis deviation, then Moller's NoDivTriTriIsect
 * (third_party/tomasakeninemoeller/opttritri.h, June 1999 revision) with USE_EPSILON_TEST, in float32 with the published
 * operand order (built with -ffp-contract=off); FABS(x) < EPSILON compares in double, EPSILON being the double 1e-6.
 *
 * Two pair modes, checked against each other by the tests:
 *   ORC_ALL_PAIRS  the reference's loop over every i < j; `filtered` adds the engine's conditions (all nine vertices
 *                  finite, closed float32 boxes overlapping on every axis)
 *   ORC_SWEEP      sort the finite triangles' boxes by their minimum x, sweep, and test the box-overlapping pairs
 *                  (always filtered)
 * Return codes: 0 ok, 1 a vertex index outside [0, nv), 3 capacity too small (*n_out holds the count). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_ALL_PAIRS 0
#define ORC_SWEEP 1

static int bad_indices(const int32_t *tri, long long nt, long long nv) {
    for (long long k = 0; k < 3 * nt; ++k)
        if (tri[k] < 0 || tri[k] >= nv) return 1;
    return 0;
}

/* ---------------------------------------------------------------------------------------- RemoveDuplicatedVertices */
static const float *g_v;
static int cmp_vertex(const void *pa, const void *pb) {
    const int a = *(const int *)pa, b = *(const int *)pb;
    const float *x = g_v + 3 * (size_t)a, *y = g_v + 3 * (size_t)b;
    const int na = isnan(x[0]) || isnan(x[1]) || isnan(x[2]), nb = isnan(y[0]) || isnan(y[1]) || isnan(y[2]);
    if (na != nb) return na - nb;
    if (!na) {
        for (int k = 0; k < 3; ++k)
            if (x[k] != y[k]) return x[k] < y[k] ? -1 : 1;
    }
    return (a > b) - (a < b);
}

/* outputs sized like the inputs; vn / vc may be NULL; -> *n_out the vertex count */
int orc_remove_duplicated_vertices(const float *v, const float *vn, const float *vc, long long nv, const int32_t *tri, long long nt,
                                   float *ov, float *on, float *oc, int32_t *ot, long long *n_out) {
    *n_out = 0;
    if (bad_indices(tri, nt, nv)) return 1;
    int *perm = (int *)malloc(sizeof(int) * (size_t)(nv + 1));
    int *o2n = (int *)malloc(sizeof(int) * (size_t)(nv + 1));
    for (long long i = 0; i < nv; ++i) perm[i] = (int)i;
    g_v = v;
    qsort(perm, (size_t)nv, sizeof(int), cmp_vertex);
    long long k = -1;
    for (long long p = 0; p < nv; ++p) {
        const float *x = v + 3 * (size_t)perm[p];
        int head = p == 0 || isnan(x[0]) || isnan(x[1]) || isnan(x[2]);
        if (!head) {
            const float *y = v + 3 * (size_t)perm[p - 1];
            head = !(x[0] == y[0] && x[1] == y[1] && x[2] == y[2]);
        }
        if (head) {
            ++k;
            memcpy(ov + 3 * k, x, 12);
            if (vn) memcpy(on + 3 * k, vn + 3 * (size_t)perm[p], 12);
            if (vc) memcpy(oc + 3 * k, vc + 3 * (size_t)perm[p], 12);
        }
        o2n[perm[p]] = (int)k;
    }
    for (long long c = 0; c < 3 * nt; ++c) ot[c] = o2n[tri[c]];
    *n_out = k + 1;
    free(perm);
    free(o2n);
    return 0;
}

/* --------------------------------------------------------------------------------------- RemoveDuplicatedTriangles */
static const int32_t *g_t;
static int cmp_tri(const void *pa, const void *pb) {
    const int a = *(const int *)pa, b = *(const int *)pb;
    for (int k = 0; k < 3; ++k)
        if (g_t[3 * (size_t)a + k] != g_t[3 * (size_t)b + k]) return g_t[3 * (size_t)a + k] < g_t[3 * (size_t)b + k] ? -1 : 1;
    return (a > b) - (a < b);
}

int orc_remove_duplicated_triangles(const int32_t *tri, const float *tn, long long nt, long long nv, int32_t *ot, float *otn, long long *n_out) {
    *n_out = 0;
    if (bad_indices(tri, nt, nv)) return 1;
    int32_t *al = (int32_t *)malloc(sizeof(int32_t) * (size_t)(3 * nt + 3));
    int *perm = (int *)malloc(sizeof(int) * (size_t)(nt + 1));
    for (long long t = 0; t < nt; ++t) {  /* align_triangle_functor (trianglemesh.cu:95-105) */
        const int32_t a = tri[3 * t], b = tri[3 * t + 1], c = tri[3 * t + 2];
        int32_t *r = al + 3 * t;
        if (a <= b) {
            if (a <= c) r[0] = a, r[1] = b, r[2] = c;
            else r[0] = c, r[1] = a, r[2] = b;
        } else {
            if (b <= c) r[0] = b, r[1] = c, r[2] = a;
            else r[0] = c, r[1] = a, r[2] = b;
        }
        perm[t] = (int)t;
    }
    g_t = al;
    qsort(perm, (size_t)nt, sizeof(int), cmp_tri);
    long long k = 0;
    for (long long p = 0; p < nt; ++p) {
        const int32_t *r = al + 3 * (size_t)perm[p];
        if (p > 0) {
            const int32_t *q = al + 3 * (size_t)perm[p - 1];
            if (r[0] == q[0] && r[1] == q[1] && r[2] == q[2]) continue;
        }
        memcpy(ot + 3 * k, r, 12);
        if (tn) memcpy(otn + 3 * k, tn + 3 * (size_t)perm[p], 12);
        ++k;
    }
    *n_out = k;
    free(al);
    free(perm);
    return 0;
}

/* -------------------------------------------------------------------------------------- RemoveUnreferencedVertices */
int orc_remove_unreferenced_vertices(const float *v, const float *vn, const float *vc, long long nv, const int32_t *tri, long long nt,
                                     float *ov, float *on, float *oc, int32_t *ot, long long *n_out) {
    *n_out = 0;
    if (bad_indices(tri, nt, nv)) return 1;
    char *ref = (char *)calloc((size_t)nv + 1, 1);
    int *o2n = (int *)malloc(sizeof(int) * (size_t)(nv + 1));
    for (long long c = 0; c < 3 * nt; ++c) ref[tri[c]] = 1;
    long long k = 0;
    for (long long i = 0; i < nv; ++i) {
        if (!ref[i]) continue;
        memcpy(ov + 3 * k, v + 3 * i, 12);
        if (vn) memcpy(on + 3 * k, vn + 3 * i, 12);
        if (vc) memcpy(oc + 3 * k, vc + 3 * i, 12);
        o2n[i] = (int)k++;
    }
    for (long long c = 0; c < 3 * nt; ++c) ot[c] = o2n[tri[c]];
    *n_out = k;
    free(ref);
    free(o2n);
    return 0;
}

/* --------------------------------------------------------------------------------------- RemoveDegenerateTriangles */
int orc_remove_degenerate_triangles(const int32_t *tri, const float *tn, long long nt, long long nv, int32_t *ot, float *otn, long long *n_out) {
    *n_out = 0;
    if (bad_indices(tri, nt, nv)) return 1;
    long long k = 0;
    for (long long t = 0; t < nt; ++t) {
        const int32_t *r = tri + 3 * t;
        if (r[0] == r[1] || r[1] == r[2] || r[2] == r[0]) continue;
        memcpy(ot + 3 * k, r, 12);
        if (tn) memcpy(otn + 3 * k, tn + 3 * t, 12);
        ++k;
    }
    *n_out = k;
    return 0;
}

/* ------------------------------------------------------------------------------------------------------ operator+= */
int orc_append_triangles(const int32_t *a, long long nta, long long nva, const int32_t *b, long long ntb, long long nvb, int32_t *out) {
    if (bad_indices(a, nta, nva) || bad_indices(b, ntb, nvb)) return 1;
    for (long long c = 0; c < 3 * nta; ++c) out[c] = a[c];
    for (long long c = 0; c < 3 * ntb; ++c) out[3 * nta + c] = (int32_t)(b[c] + nva);
    return 0;
}

/* ------------------------------------------------------------------------------------------------- the predicate */
static int edge_edge(float Ax, float Ay, const float *V0, const float *U0, const float *U1, int i0, int i1) {
    float Bx = U0[i0] - U1[i0];
    float By = U0[i1] - U1[i1];
    float Cx = V0[i0] - U0[i0];
    float Cy = V0[i1] - U0[i1];
    float f = Ay * Bx - Ax * By;
    float d = By * Cx - Bx * Cy;
    if ((f > 0 && d >= 0 && d <= f) || (f < 0 && d <= 0 && d >= f)) {
        float e = Ax * Cy - Ay * Cx;
        if (f > 0) {
            if (e >= 0 && e <= f) return 1;
        } else {
            if (e <= 0 && e >= f) return 1;
        }
    }
    return 0;
}

static int edge_against_tri_edges(const float *V0, const float *V1, const float *U0, const float *U1, const float *U2, int i0, int i1) {
    float Ax = V1[i0] - V0[i0];
    float Ay = V1[i1] - V0[i1];
    if (edge_edge(Ax, Ay, V0, U0, U1, i0, i1)) return 1;
    if (edge_edge(Ax, Ay, V0, U1, U2, i0, i1)) return 1;
    if (edge_edge(Ax, Ay, V0, U2, U0, i0, i1)) return 1;
    return 0;
}

static int point_in_tri(const float *V0, const float *U0, const float *U1, const float *U2, int i0, int i1) {
    float a, b, c, d0, d1, d2;
    a = U1[i1] - U0[i1];
    b = -(U1[i0] - U0[i0]);
    c = -a * U0[i0] - b * U0[i1];
    d0 = a * V0[i0] + b * V0[i1] + c;
    a = U2[i1] - U1[i1];
    b = -(U2[i0] - U1[i0]);
    c = -a * U1[i0] - b * U1[i1];
    d1 = a * V0[i0] + b * V0[i1] + c;
    a = U0[i1] - U2[i1];
    b = -(U0[i0] - U2[i0]);
    c = -a * U2[i0] - b * U2[i1];
    d2 = a * V0[i0] + b * V0[i1] + c;
    if (d0 * d1 > 0.0) {
        if (d0 * d2 > 0.0) return 1;
    }
    return 0;
}

static int coplanar_tri_tri(const float *N, const float *V0, const float *V1, const float *V2, const float *U0, const float *U1,
                            const float *U2) {
    float A[3];
    int i0, i1;
    A[0] = fabsf(N[0]);
    A[1] = fabsf(N[1]);
    A[2] = fabsf(N[2]);
    if (A[0] > A[1]) {
        if (A[0] > A[2]) {
            i0 = 1;
            i1 = 2;
        } else {
            i0 = 0;
            i1 = 1;
        }
    } else {
        if (A[2] > A[1]) {
            i0 = 0;
            i1 = 1;
        } else {
            i0 = 0;
            i1 = 2;
        }
    }
    if (edge_against_tri_edges(V0, V1, U0, U1, U2, i0, i1)) return 1;
    if (edge_against_tri_edges(V1, V2, U0, U1, U2, i0, i1)) return 1;
    if (edge_against_tri_edges(V2, V0, U0, U1, U2, i0, i1)) return 1;
    if (point_in_tri(V0, U0, U1, U2, i0, i1)) return 1;
    if (point_in_tri(U0, V0, V1, V2, i0, i1)) return 1;
    return 0;
}

/* NEWCOMPUTE_INTERVALS -> 0 when the triangles are coplanar */
static int intervals(float VV0, float VV1, float VV2, float D0, float D1, float D2, float D0D1, float D0D2, float *A, float *B, float *C,
                     float *X0, float *X1) {
    if (D0D1 > 0.0f) {
        *A = VV2; *B = (VV0 - VV2) * D2; *C = (VV1 - VV2) * D2; *X0 = D2 - D0; *X1 = D2 - D1;
    } else if (D0D2 > 0.0f) {
        *A = VV1; *B = (VV0 - VV1) * D1; *C = (VV2 - VV1) * D1; *X0 = D1 - D0; *X1 = D1 - D2;
    } else if (D1 * D2 > 0.0f || D0 != 0.0f) {
        *A = VV0; *B = (VV1 - VV0) * D0; *C = (VV2 - VV0) * D0; *X0 = D0 - D1; *X1 = D0 - D2;
    } else if (D1 != 0.0f) {
        *A = VV1; *B = (VV0 - VV1) * D1; *C = (VV2 - VV1) * D1; *X0 = D1 - D0; *X1 = D1 - D2;
    } else if (D2 != 0.0f) {
        *A = VV2; *B = (VV0 - VV2) * D2; *C = (VV1 - VV2) * D2; *X0 = D2 - D0; *X1 = D2 - D1;
    } else {
        return 0;
    }
    return 1;
}

#define ORC_EPSILON 0.000001
static float eps0(float x) { return (double)fabsf(x) < ORC_EPSILON ? 0.0f : x; }
static float dot3f(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static void cross3f(float *d, const float *a, const float *b) {
    d[0] = a[1] * b[2] - a[2] * b[1];
    d[1] = a[2] * b[0] - a[0] * b[2];
    d[2] = a[0] * b[1] - a[1] * b[0];
}

static int no_div_tri_tri_isect(const float *V0, const float *V1, const float *V2, const float *U0, const float *U1, const float *U2) {
    float E1[3], E2[3], N1[3], N2[3], D[3];
    for (int k = 0; k < 3; ++k) E1[k] = V1[k] - V0[k], E2[k] = V2[k] - V0[k];
    cross3f(N1, E1, E2);
    float d1 = -dot3f(N1, V0);
    float du0 = eps0(dot3f(N1, U0) + d1), du1 = eps0(dot3f(N1, U1) + d1), du2 = eps0(dot3f(N1, U2) + d1);
    float du0du1 = du0 * du1, du0du2 = du0 * du2;
    if (du0du1 > 0.0f && du0du2 > 0.0f) return 0;
    for (int k = 0; k < 3; ++k) E1[k] = U1[k] - U0[k], E2[k] = U2[k] - U0[k];
    cross3f(N2, E1, E2);
    float d2 = -dot3f(N2, U0);
    float dv0 = eps0(dot3f(N2, V0) + d2), dv1 = eps0(dot3f(N2, V1) + d2), dv2 = eps0(dot3f(N2, V2) + d2);
    float dv0dv1 = dv0 * dv1, dv0dv2 = dv0 * dv2;
    if (dv0dv1 > 0.0f && dv0dv2 > 0.0f) return 0;
    cross3f(D, N1, N2);
    float max = fabsf(D[0]), bb = fabsf(D[1]), cc = fabsf(D[2]);
    int index = 0;
    if (bb > max) max = bb, index = 1;
    if (cc > max) max = cc, index = 2;
    float a, b, c, x0, x1, d, e, f, y0, y1;
    if (!intervals(V0[index], V1[index], V2[index], dv0, dv1, dv2, dv0dv1, dv0dv2, &a, &b, &c, &x0, &x1))
        return coplanar_tri_tri(N1, V0, V1, V2, U0, U1, U2);
    if (!intervals(U0[index], U1[index], U2[index], du0, du1, du2, du0du1, du0du2, &d, &e, &f, &y0, &y1))
        return coplanar_tri_tri(N1, V0, V1, V2, U0, U1, U2);
    float xx = x0 * x1, yy = y0 * y1, xxyy = xx * yy, tmp, s1[2], s2[2];
    tmp = a * xxyy;
    s1[0] = tmp + b * x1 * yy;
    s1[1] = tmp + c * x0 * yy;
    tmp = d * xxyy;
    s2[0] = tmp + e * xx * y1;
    s2[1] = tmp + f * xx * y0;
    if (s1[0] > s1[1]) tmp = s1[0], s1[0] = s1[1], s1[1] = tmp;
    if (s2[0] > s2[1]) tmp = s2[0], s2[0] = s2[1], s2[1] = tmp;
    if (s1[1] < s2[0] || s2[1] < s1[0]) return 0;
    return 1;
}

/* p, q: 3 vertices of 3 floats each */
int orc_tritri(const float *p, const float *q) {
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
    return no_div_tri_tri_isect(pm, pm + 3, pm + 6, qm, qm + 3, qm + 6);
}

/* ----------------------------------------------------------------------------------- GetSelfIntersectingTriangles */
typedef struct {
    float lo[3], hi[3];
    int finite;
} TBox;

static void tri_box(const float *v, const int32_t *t, TBox *b) {
    b->finite = 1;
    for (int k = 0; k < 3; ++k) {
        const float x = v[3 * (size_t)t[0] + k], y = v[3 * (size_t)t[1] + k], z = v[3 * (size_t)t[2] + k];
        b->finite = b->finite && isfinite(x) && isfinite(y) && isfinite(z);
        b->lo[k] = fminf(fminf(x, y), z);
        b->hi[k] = fmaxf(fmaxf(x, y), z);
    }
}
static int boxes_overlap(const TBox *a, const TBox *b) {
    for (int k = 0; k < 3; ++k)
        if (!(a->lo[k] <= b->hi[k] && b->lo[k] <= a->hi[k])) return 0;
    return 1;
}
static int share_index(const int32_t *a, const int32_t *b) {
    for (int x = 0; x < 3; ++x)
        for (int y = 0; y < 3; ++y)
            if (a[x] == b[y]) return 1;
    return 0;
}
static int pair_hits(const float *v, const int32_t *tri, long long i, long long j) {
    float p[9], q[9];
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) {
            p[3 * c + k] = v[3 * (size_t)tri[3 * i + c] + k];
            q[3 * c + k] = v[3 * (size_t)tri[3 * j + c] + k];
        }
    return orc_tritri(p, q);
}

static TBox *g_boxes;
static int cmp_lox(const void *pa, const void *pb) {
    const int a = *(const int *)pa, b = *(const int *)pb;
    if (g_boxes[a].lo[0] != g_boxes[b].lo[0]) return g_boxes[a].lo[0] < g_boxes[b].lo[0] ? -1 : 1;
    return (a > b) - (a < b);
}
static int cmp_pair(const void *pa, const void *pb) {
    const int32_t *a = (const int32_t *)pa, *b = (const int32_t *)pb;
    if (a[0] != b[0]) return a[0] < b[0] ? -1 : 1;
    return (a[1] > b[1]) - (a[1] < b[1]);
}

/* pairs [cap][2] int32 in ascending (i, j) order */
int orc_self_intersections(const float *v, long long nv, const int32_t *tri, long long nt, int mode, int filtered, int32_t *pairs,
                           long long cap, long long *n_out) {
    *n_out = 0;
    if (bad_indices(tri, nt, nv)) return 1;
    TBox *bx = (TBox *)malloc(sizeof(TBox) * (size_t)(nt + 1));
    for (long long t = 0; t < nt; ++t) tri_box(v, tri + 3 * t, bx + t);
    long long n = 0;
    if (mode == ORC_ALL_PAIRS) {
        for (long long i = 0; i < nt; ++i)
            for (long long j = i + 1; j < nt; ++j) {
                if (share_index(tri + 3 * i, tri + 3 * j)) continue;
                if (filtered && !(bx[i].finite && bx[j].finite && boxes_overlap(bx + i, bx + j))) continue;
                if (!pair_hits(v, tri, i, j)) continue;
                if (n < cap) pairs[2 * n] = (int32_t)i, pairs[2 * n + 1] = (int32_t)j;
                ++n;
            }
    } else {
        int *ord = (int *)malloc(sizeof(int) * (size_t)(nt + 1));
        long long m = 0;
        for (long long t = 0; t < nt; ++t)
            if (bx[t].finite) ord[m++] = (int)t;
        g_boxes = bx;
        qsort(ord, (size_t)m, sizeof(int), cmp_lox);
        for (long long a = 0; a < m; ++a)
            for (long long b = a + 1; b < m && bx[ord[b]].lo[0] <= bx[ord[a]].hi[0]; ++b) {
                const long long i = ord[a] < ord[b] ? ord[a] : ord[b], j = ord[a] < ord[b] ? ord[b] : ord[a];
                if (!boxes_overlap(bx + i, bx + j) || share_index(tri + 3 * i, tri + 3 * j)) continue;
                if (!pair_hits(v, tri, i, j)) continue;
                if (n < cap) pairs[2 * n] = (int32_t)i, pairs[2 * n + 1] = (int32_t)j;
                ++n;
            }
        free(ord);
        if (n <= cap) qsort(pairs, (size_t)n, 2 * sizeof(int32_t), cmp_pair);
    }
    free(bx);
    *n_out = n;
    return n > cap ? 3 : 0;
}
