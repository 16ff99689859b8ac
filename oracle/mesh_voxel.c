/* VoxelGrid::CreateFromTriangleMeshWithinBounds restated in plain C (DESIGN section 4 item 25), for the tests of
 * csrc/voxelgrid.cu's mesh voxelisation.
 *
 * A key k (0 <= k_a < n_a, n_a = (int)roundf((max_a - min_a) / vs)) is a voxel when Akenine-Moeller's triangle/box
 * overlap test says some triangle meets the closed cell of centre ((float)k + 0.5f) * vs + min_a (corner = 0), or,
 * for comparison with the reference, of centre (float)k * vs + min_a (corner = 1).  Half size 0.5f * vs.  A triangle
 * with a non-finite vertex meets no cell.  IEEE float32 throughout, built with -ffp-contract=off.
 *
 * Two enumerations that must agree:
 *   mode 0, cell-major: the reference's loop, every cell against every triangle until one hits (small inputs only);
 *   mode 1, triangle-major: every cell of each triangle's clamped bounding box, widened by two cells, then sort and
 *           unique.
 * Keys come out unique and in lexicographic order.  Return codes: 0 ok, 1 a vertex index outside [0, nv), 2 a bad
 * voxel size, bounds or count, 3 capacity too small (*n_out is still the count). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define AXIS_LIMIT (1 << 21)

static void order2(float a, float b, float *mn, float *mx) {
    if (a < b) {
        *mn = a;
        *mx = b;
    } else {
        *mn = b;
        *mx = a;
    }
}

/* the published triBoxOverlap: 9 edge x axis tests, the 3 box axes, then the plane (planeBoxOverlap) */
int orc_tri_box(const float c[3], float h, const float A[3], const float B[3], const float C[3]) {
    float v0[3], v1[3], v2[3], e0[3], e1[3], e2[3], mn, mx, p0, p1, p2, rad, fx, fy, fz;
    for (int q = 0; q < 3; ++q) {
        v0[q] = A[q] - c[q];
        v1[q] = B[q] - c[q];
        v2[q] = C[q] - c[q];
    }
    for (int q = 0; q < 3; ++q) {
        e0[q] = v1[q] - v0[q];
        e1[q] = v2[q] - v1[q];
        e2[q] = v0[q] - v2[q];
    }
    /* edge 0: AXISTEST_X01, _Y02, _Z12 */
    fx = fabsf(e0[0]), fy = fabsf(e0[1]), fz = fabsf(e0[2]);
    p0 = e0[2] * v0[1] - e0[1] * v0[2], p2 = e0[2] * v2[1] - e0[1] * v2[2];
    order2(p0, p2, &mn, &mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return 0;
    p0 = -e0[2] * v0[0] + e0[0] * v0[2], p2 = -e0[2] * v2[0] + e0[0] * v2[2];
    order2(p0, p2, &mn, &mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    p1 = e0[1] * v1[0] - e0[0] * v1[1], p2 = e0[1] * v2[0] - e0[0] * v2[1];
    order2(p2, p1, &mn, &mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    /* edge 1: AXISTEST_X01, _Y02, _Z0 */
    fx = fabsf(e1[0]), fy = fabsf(e1[1]), fz = fabsf(e1[2]);
    p0 = e1[2] * v0[1] - e1[1] * v0[2], p2 = e1[2] * v2[1] - e1[1] * v2[2];
    order2(p0, p2, &mn, &mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return 0;
    p0 = -e1[2] * v0[0] + e1[0] * v0[2], p2 = -e1[2] * v2[0] + e1[0] * v2[2];
    order2(p0, p2, &mn, &mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    p0 = e1[1] * v0[0] - e1[0] * v0[1], p1 = e1[1] * v1[0] - e1[0] * v1[1];
    order2(p0, p1, &mn, &mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    /* edge 2: AXISTEST_X2, _Y1, _Z12 */
    fx = fabsf(e2[0]), fy = fabsf(e2[1]), fz = fabsf(e2[2]);
    p0 = e2[2] * v0[1] - e2[1] * v0[2], p1 = e2[2] * v1[1] - e2[1] * v1[2];
    order2(p0, p1, &mn, &mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return 0;
    p0 = -e2[2] * v0[0] + e2[0] * v0[2], p1 = -e2[2] * v1[0] + e2[0] * v1[2];
    order2(p0, p1, &mn, &mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    p1 = e2[1] * v1[0] - e2[0] * v1[1], p2 = e2[1] * v2[0] - e2[0] * v2[1];
    order2(p2, p1, &mn, &mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return 0;
    /* the box axes (FINDMINMAX) */
    for (int q = 0; q < 3; ++q) {
        mn = mx = v0[q];
        if (v1[q] < mn) mn = v1[q];
        if (v1[q] > mx) mx = v1[q];
        if (v2[q] < mn) mn = v2[q];
        if (v2[q] > mx) mx = v2[q];
        if (mn > h || mx < -h) return 0;
    }
    /* the plane: normal e0 x e1 */
    const float n[3] = {e0[1] * e1[2] - e0[2] * e1[1], e0[2] * e1[0] - e0[0] * e1[2], e0[0] * e1[1] - e0[1] * e1[0]};
    float vmin[3], vmax[3];
    for (int q = 0; q < 3; ++q) {
        if (n[q] > 0.0f) {
            vmin[q] = -h - v0[q];
            vmax[q] = h - v0[q];
        } else {
            vmin[q] = h - v0[q];
            vmax[q] = -h - v0[q];
        }
    }
    if (n[0] * vmin[0] + n[1] * vmin[1] + n[2] * vmin[2] > 0.0f) return 0;
    return n[0] * vmax[0] + n[1] * vmax[1] + n[2] * vmax[2] >= 0.0f;
}

/* the count rule and the argument checks: 0 ok, 2 rejected */
int orc_mesh_voxel_counts(float vs, const float mnb[3], const float mxb[3], long long cnt[3]) {
    if (!(isfinite(vs) && vs > 0.0f)) return 2;
    for (int a = 0; a < 3; ++a) {
        if (!isfinite(mnb[a]) || !isfinite(mxb[a])) return 2;
        volatile float ext = mxb[a] - mnb[a];
        volatile float q = ext / vs;
        const float c = roundf(q);
        if (!(c >= 0.0f && c < (float)AXIS_LIMIT)) return 2;
        cnt[a] = (long long)c;
    }
    return 0;
}

static float centre(long long k, float vs, float o, int corner) {
    return corner ? (float)k * vs + o : ((float)k + 0.5f) * vs + o;
}

static int finite_tri(const float *v, const int32_t *t, long long i, const float *P[3]) {
    for (int j = 0; j < 3; ++j) {
        P[j] = v + 3 * (long long)t[3 * i + j];
        for (int q = 0; q < 3; ++q)
            if (!isfinite(P[j][q])) return 0;
    }
    return 1;
}

static int cmp_u64(const void *a, const void *b) {
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : x > y;
}

int orc_mesh_voxel(const float *v, long long nv, const int32_t *t, long long nt, float vs, const float mnb[3], const float mxb[3],
                   int mode, int corner, int32_t *out, long long capacity, long long *n_out) {
    *n_out = 0;
    long long n[3];
    if (orc_mesh_voxel_counts(vs, mnb, mxb, n)) return 2;
    for (long long i = 0; i < 3 * nt; ++i)
        if (t[i] < 0 || t[i] >= nv) return 1;
    const float h = vs * 0.5f;
    long long m = 0;
    if (mode == 0) {
        for (long long x = 0; x < n[0]; ++x)
            for (long long y = 0; y < n[1]; ++y)
                for (long long z = 0; z < n[2]; ++z) {
                    const float c[3] = {centre(x, vs, mnb[0], corner), centre(y, vs, mnb[1], corner), centre(z, vs, mnb[2], corner)};
                    for (long long i = 0; i < nt; ++i) {
                        const float *P[3];
                        if (finite_tri(v, t, i, P) && orc_tri_box(c, h, P[0], P[1], P[2])) {
                            if (m < capacity) {
                                out[3 * m] = (int32_t)x;
                                out[3 * m + 1] = (int32_t)y;
                                out[3 * m + 2] = (int32_t)z;
                            }
                            ++m;
                            break;
                        }
                    }
                }
        *n_out = m;
        return m > capacity ? 3 : 0;
    }
    size_t cap = 1024, cnt = 0;
    uint64_t *keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
    for (long long i = 0; i < nt; ++i) {
        const float *P[3];
        if (!finite_tri(v, t, i, P)) continue;
        long long lo[3], hi[3];
        int empty = 0;
        for (int a = 0; a < 3; ++a) {
            const double mn = fmin(fmin(P[0][a], P[1][a]), P[2][a]), mx = fmax(fmax(P[0][a], P[1][a]), P[2][a]);
            const double flo = floor((mn - (double)mnb[a]) / (double)vs) - 2.0, fhi = floor((mx - (double)mnb[a]) / (double)vs) + 2.0;
            lo[a] = flo < 0.0 ? 0 : (long long)flo;
            hi[a] = fhi > (double)(n[a] - 1) ? n[a] - 1 : (long long)fhi;
            if (lo[a] > hi[a]) empty = 1;
        }
        if (empty) continue;
        for (long long x = lo[0]; x <= hi[0]; ++x)
            for (long long y = lo[1]; y <= hi[1]; ++y)
                for (long long z = lo[2]; z <= hi[2]; ++z) {
                    const float c[3] = {centre(x, vs, mnb[0], corner), centre(y, vs, mnb[1], corner), centre(z, vs, mnb[2], corner)};
                    if (!orc_tri_box(c, h, P[0], P[1], P[2])) continue;
                    if (cnt == cap) {
                        cap *= 2;
                        keys = (uint64_t *)realloc(keys, cap * sizeof(uint64_t));
                    }
                    keys[cnt++] = ((uint64_t)x << 42) | ((uint64_t)y << 21) | (uint64_t)z;
                }
    }
    qsort(keys, cnt, sizeof(uint64_t), cmp_u64);
    for (size_t i = 0; i < cnt; ++i) {
        if (i && keys[i] == keys[i - 1]) continue;
        if (m < capacity) {
            out[3 * m] = (int32_t)(keys[i] >> 42);
            out[3 * m + 1] = (int32_t)((keys[i] >> 21) & (AXIS_LIMIT - 1));
            out[3 * m + 2] = (int32_t)(keys[i] & (AXIS_LIMIT - 1));
        }
        ++m;
    }
    free(keys);
    *n_out = m;
    return m > capacity ? 3 : 0;
}
