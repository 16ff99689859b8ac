/* collision.c -- CPU restatement of collision::ComputeIntersection (collision.cu:1137-1231) over grid elements and
 * primitives, by brute force: every (target, query) pair is tested, in ascending target order, and a query element's
 * answer is the first (= smallest) target index that collides.  It shares no lookup structure with the device
 * (cupoch_b200/csrc/collision.cu), which is the point of having it.
 *
 * A grid element is an integer key k with the box [k * vs + o, (k + 1) * vs + o] and an index (a VoxelGrid's position,
 * an OccupancyGrid cell's linear index; the caller lists the target in ascending index order).  The tests restate
 * intersection_test.inl:120-262 and distance_test.inl:47-110 in float, every operation rounded on its own
 * (-ffp-contract=off), in the operand order of DESIGN.md's collision entry. */
#include <float.h>
#include <math.h>
#include <stdint.h>

typedef struct {
    int32_t type; /* 1 Box, 2 Sphere, 3 Capsule, 4 Cylinder */
    float transform[16]; /* row-major */
    float lengths[3];
    float radius;
    float height;
} orc_prim;

static float dot3(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

static float point_aabb2(const float p[3], const float lo[3], const float hi[3]) {
    float d2 = 0.f;
    for (int i = 0; i < 3; ++i) {
        float v = p[i];
        if (v < lo[i]) d2 += (lo[i] - v) * (lo[i] - v);
        if (v > hi[i]) d2 += (v - hi[i]) * (v - hi[i]);
    }
    return d2;
}

static float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

static float seg_seg2(const float p0[3], const float q0[3], const float p1[3], const float q1[3]) {
    float d0[3], d1[3], r[3];
    for (int i = 0; i < 3; ++i) { d0[i] = q0[i] - p0[i]; d1[i] = q1[i] - p1[i]; r[i] = p0[i] - p1[i]; }
    float a = dot3(d0, d0), e = dot3(d1, d1), f = dot3(d1, r);
    float s, t;
    if (a <= FLT_EPSILON && e <= FLT_EPSILON) {
        s = 0.f; t = 0.f;
    } else if (a <= FLT_EPSILON) {
        s = 0.f; t = clamp01(f / e);
    } else {
        float c = dot3(d0, r);
        if (e <= FLT_EPSILON) {
            t = 0.f; s = clamp01(-c / a);
        } else {
            float b = dot3(d0, d1);
            float denom = a * e - b * b;
            s = (denom != 0.f) ? clamp01((b * f - c * e) / denom) : 0.f;
            t = (b * s + f) / e;
            if (t < 0.f) { t = 0.f; s = clamp01(-c / a); }
            else if (t > 1.f) { t = 1.f; s = clamp01((b - c) / a); }
        }
    }
    float w[3];
    for (int i = 0; i < 3; ++i) w[i] = (p0[i] + s * d0[i]) - (p1[i] + t * d1[i]);
    return dot3(w, w);
}

static int capsule_aabb(float radius, const float p[3], const float d[3], const float lo[3], const float hi[3]) {
    float elo[3], ehi[3];
    for (int i = 0; i < 3; ++i) { elo[i] = lo[i] - radius; ehi[i] = hi[i] + radius; }
    float tmin = 0.f, tmax = FLT_MAX;
    for (int i = 0; i < 3; ++i) {
        if (fabsf(d[i]) < FLT_EPSILON) {
            if (p[i] < elo[i] || p[i] > ehi[i]) return 0;
        } else {
            float ood = 1.0f / d[i];
            float t1 = (elo[i] - p[i]) * ood, t2 = (ehi[i] - p[i]) * ood;
            if (t1 > t2) { float x = t1; t1 = t2; t2 = x; }
            if (t1 > tmin) tmin = t1;
            if (t2 < tmax) tmax = t2;
            if (tmin > tmax) return 0;
        }
    }
    if (tmin > 1.0f) return 0;
    int u = 0, v = 0;
    for (int i = 0; i < 3; ++i) {
        float q = p[i] + d[i] * tmin;
        if (q < lo[i]) u |= 1 << i;
        if (q > hi[i]) v |= 1 << i;
    }
    int m = u + v;
    if (m == 7) return 1;
    if ((m & (m - 1)) == 0) return 1;
    float pd[3], c0[3], c1[3];
    for (int i = 0; i < 3; ++i) {
        pd[i] = p[i] + d[i];
        c0[i] = ((u ^ 7) & 1) ? hi[i] : lo[i];
        c1[i] = (v & 1) ? hi[i] : lo[i];
    }
    return seg_seg2(p, pd, c0, c1) <= radius * radius;
}

static int box_box(const float e1[3], const float R[9], const float c1[3], const float e2[3], const float c2[3]) {
    float r[9], ar[9], t[3], dc[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            r[3 * i + j] = (R[3 * i] * (j == 0 ? 1.f : 0.f) + R[3 * i + 1] * (j == 1 ? 1.f : 0.f)) + R[3 * i + 2] * (j == 2 ? 1.f : 0.f);
            ar[3 * i + j] = fabsf(r[3 * i + j]) + FLT_EPSILON;
        }
    for (int i = 0; i < 3; ++i) dc[i] = c2[i] - c1[i];
    for (int i = 0; i < 3; ++i) t[i] = (R[3 * i] * dc[0] + R[3 * i + 1] * dc[1]) + R[3 * i + 2] * dc[2];
#define RR(i, j) r[3 * (i) + (j)]
#define AR(i, j) ar[3 * (i) + (j)]
    for (int i = 0; i < 3; ++i)
        if (fabsf(t[i]) > e1[i] + ((AR(i, 0) * e2[0] + AR(i, 1) * e2[1]) + AR(i, 2) * e2[2])) return 0;
    for (int i = 0; i < 3; ++i)
        if (fabsf((t[0] * RR(0, i) + t[1] * RR(1, i)) + t[2] * RR(2, i)) > ((AR(0, i) * e1[0] + AR(1, i) * e1[1]) + AR(2, i) * e1[2]) + e2[i])
            return 0;
    float ra, rb;
    ra = e1[1] * AR(2, 0) + e1[2] * AR(1, 0); rb = e2[1] * AR(0, 2) + e2[2] * AR(0, 1);
    if (fabsf(t[2] * RR(1, 0) - t[1] * RR(2, 0)) > ra + rb) return 0;
    ra = e1[1] * AR(2, 1) + e1[2] * AR(1, 1); rb = e2[0] * AR(0, 2) + e2[2] * AR(0, 0);
    if (fabsf(t[2] * RR(1, 1) - t[1] * RR(2, 1)) > ra + rb) return 0;
    ra = e1[1] * AR(2, 2) + e1[2] * AR(1, 2); rb = e2[0] * AR(0, 1) + e2[1] * AR(0, 0);
    if (fabsf(t[2] * RR(1, 2) - t[1] * RR(2, 2)) > ra + rb) return 0;
    ra = e1[0] * AR(2, 0) + e1[2] * AR(0, 0); rb = e2[1] * AR(1, 2) + e2[2] * AR(1, 1);
    if (fabsf(t[0] * RR(2, 0) - t[2] * RR(0, 0)) > ra + rb) return 0;
    ra = e1[0] * AR(2, 1) + e1[2] * AR(0, 1); rb = e2[0] * AR(1, 2) + e2[2] * AR(1, 0);
    if (fabsf(t[0] * RR(2, 1) - t[2] * RR(0, 1)) > ra + rb) return 0;
    ra = e1[0] * AR(2, 2) + e1[2] * AR(0, 2); rb = e2[0] * AR(1, 1) + e2[1] * AR(1, 0);
    if (fabsf(t[0] * RR(2, 2) - t[2] * RR(0, 2)) > ra + rb) return 0;
    ra = e1[0] * AR(1, 0) + e1[1] * AR(0, 0); rb = e2[1] * AR(2, 2) + e2[2] * AR(2, 1);
    if (fabsf(t[1] * RR(0, 1) - t[0] * RR(1, 0)) > ra + rb) return 0; /* intersection_test.inl:198 reads r(0, 1) */
    ra = e1[0] * AR(1, 1) + e1[1] * AR(0, 1); rb = e2[0] * AR(2, 2) + e2[2] * AR(2, 0);
    if (fabsf(t[1] * RR(0, 1) - t[0] * RR(1, 1)) > ra + rb) return 0;
    ra = e1[0] * AR(1, 2) + e1[1] * AR(0, 2); rb = e2[0] * AR(2, 1) + e2[1] * AR(2, 0);
    if (fabsf(t[1] * RR(0, 2) - t[0] * RR(1, 2)) > ra + rb) return 0;
#undef RR
#undef AR
    return 1;
}

/* a primitive against the grid element with key k (collision.cu:221-298) */
int orc_coll_prim_elem(const orc_prim *p, const int32_t k[3], float vs, const float o[3], float margin) {
    const float half = vs / 2.f;
    float c[3], lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        c[a] = ((float)k[a] + 0.5f) * vs + o[a];
        lo[a] = c[a] - half;
        hi[a] = c[a] + half;
    }
    const float *T = p->transform;
    if (p->type == 1) {
        const float e1[3] = {p->lengths[0] * 0.5f, p->lengths[1] * 0.5f, p->lengths[2] * 0.5f};
        const float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
        const float t1[3] = {T[3], T[7], T[11]};
        const float e2[3] = {half + margin, half + margin, half + margin};
        return box_box(e1, R, t1, e2, c);
    }
    if (p->type == 2) {
        const float r = p->radius + margin;
        const float ctr[3] = {T[3], T[7], T[11]};
        return point_aabb2(ctr, lo, hi) <= r * r;
    }
    if (p->type == 3) {
        const float r = p->radius + margin;
        const float hh = 0.5f * p->height;
        const float s[3] = {T[3] - hh * T[2], T[7] - hh * T[6], T[11] - hh * T[10]};
        const float d[3] = {p->height * T[2], p->height * T[6], p->height * T[10]};
        return capsule_aabb(r, s, d, lo, hi);
    }
    return 0;
}

/* query grid element box widened by margin against target element box, inclusive (lbvh aabb.cuh:19-25) */
int orc_coll_elem_elem(const int32_t kt[3], float tvs, const float to[3], const int32_t kq[3], float qvs, const float qo[3],
                       float margin) {
    for (int a = 0; a < 3; ++a) {
        float tlo = (float)kt[a] * tvs + to[a], thi = (float)(kt[a] + 1) * tvs + to[a];
        float qlo = (float)kq[a] * qvs + qo[a] - margin, qhi = (float)(kq[a] + 1) * qvs + qo[a] + margin;
        if (!(qlo <= thi && qhi >= tlo)) return 0;
    }
    return 1;
}

/* best[j] = index of the first target element (ascending) that collides with query element j, or -1 */
void orc_coll_grid_grid(const int32_t *tk, const int32_t *tid, int64_t nt, float tvs, const float *to, const int32_t *qk, int64_t nq,
                        float qvs, const float *qo, float margin, int32_t *best) {
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t j = 0; j < nq; ++j) {
        int32_t b = -1;
        for (int64_t i = 0; i < nt; ++i)
            if (orc_coll_elem_elem(tk + 3 * i, tvs, to, qk + 3 * j, qvs, qo, margin)) { b = tid[i]; break; }
        best[j] = b;
    }
}

/* prims_are_target: best[j] for grid query element j = first primitive that collides; else best[j] for primitive j =
 * first grid element (ascending) it collides with */
void orc_coll_prim_grid(const orc_prim *prims, int64_t np, const int32_t *gk, const int32_t *gid, int64_t ng, float vs, const float *o,
                        float margin, int prims_are_target, int32_t *best) {
    if (prims_are_target) {
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t j = 0; j < ng; ++j) {
            int32_t b = -1;
            for (int64_t i = 0; i < np; ++i)
                if (orc_coll_prim_elem(prims + i, gk + 3 * j, vs, o, margin)) { b = (int32_t)i; break; }
            best[j] = b;
        }
    } else {
#pragma omp parallel for schedule(dynamic, 1)
        for (int64_t j = 0; j < np; ++j) {
            int32_t b = -1;
            for (int64_t i = 0; i < ng; ++i)
                if (orc_coll_prim_elem(prims + j, gk + 3 * i, vs, o, margin)) { b = gid[i]; break; }
            best[j] = b;
        }
    }
}
