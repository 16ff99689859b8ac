/* voxelgrid_ops.c -- plain-C restatement of the VoxelGrid operations of cupoch_b200/csrc/voxelgrid.cu (CreateDense,
 * CheckIfIncluded, carving, += / AddVoxels).  Built by oracle.build("voxelgrid_ops"); loader voxelgrid_ops_py.py.
 *
 * Every float operation is rounded on its own (-ffp-contract=off) except the projection's, which states its fused
 * multiply-adds with fmaf() in the order the kernel uses __fmaf_rn. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* CreateDense's counts: int(roundf(extent / voxel_size)) per axis; 0 ok, -1 rejected */
int orc_vg_dense_counts(float vs, float w, float h, float d, long long cnt[3]) {
    const float e[3] = {w, h, d};
    if (!(isfinite(vs) && vs > 0.f)) return -1;
    for (int a = 0; a < 3; ++a) {
        const float c = roundf(e[a] / vs);
        if (!(c >= 0.f && c < 2147483648.f)) return -1;
        cnt[a] = (long long)c;
    }
    return 0;
}

void orc_vg_dense(const long long cnt[3], int32_t *keys, float *colors) {
    size_t i = 0;
    for (long long x = 0; x < cnt[0]; ++x)
        for (long long y = 0; y < cnt[1]; ++y)
            for (long long z = 0; z < cnt[2]; ++z, ++i) {
                keys[3 * i] = (int32_t)x;
                keys[3 * i + 1] = (int32_t)y;
                keys[3 * i + 2] = (int32_t)z;
                colors[3 * i] = colors[3 * i + 1] = colors[3 * i + 2] = 1.f;
            }
}

static int cmp_key(const int32_t *a, const int32_t *b) {
    for (int k = 0; k < 3; ++k)
        if (a[k] != b[k]) return a[k] < b[k] ? -1 : 1;
    return 0;
}
static int cmp_key3(const void *a, const void *b) { return cmp_key((const int32_t *)a, (const int32_t *)b); }

/* CheckIfIncluded: the cell floor((q - o) / vs) of each query, looked up among the keys (sorted copy + bsearch) */
void orc_vg_included(const int32_t *keys, long long n, float vs, const float o[3], const float *q, long long nq, uint8_t *out) {
    int32_t *s = (int32_t *)malloc(sizeof(int32_t) * 3 * (n ? n : 1));
    memcpy(s, keys, sizeof(int32_t) * 3 * n);
    qsort(s, (size_t)n, 12, cmp_key3);
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < nq; ++i) {
        int32_t k[3];
        int ok = 1;
        for (int a = 0; a < 3; ++a) {
            const float f = floorf((q[3 * i + a] - o[a]) / vs);
            if (!(f >= -2147483648.f && f < 2147483648.f)) ok = 0;
            else k[a] = (int32_t)f;
        }
        out[i] = ok && n && bsearch(k, s, (size_t)n, 12, cmp_key3) != NULL;
    }
    free(s);
}

/* FloatValueAt (image.h:240-270) with z == 0 and non-finite u / v outside */
static int sample(const float *img, int w, int h, int sampled, float u, float v, float z, float *d) {
    if (!sampled || z == 0.f || !isfinite(u) || !isfinite(v) || u < 0.f || u > (float)(w - 1) || v < 0.f || v > (float)(h - 1))
        return 0;
    int ui = (int)u, vi = (int)v;
    if (ui > w - 2) ui = w - 2;
    if (ui < 0) ui = 0;
    if (vi > h - 2) vi = h - 2;
    if (vi < 0) vi = 0;
    const float pu = u - (float)ui, pv = v - (float)vi;
    const float v0 = img[(size_t)vi * w + ui], v1 = img[(size_t)(vi + 1) * w + ui];
    const float v2 = img[(size_t)vi * w + ui + 1], v3 = img[(size_t)(vi + 1) * w + ui + 1];
    const float qv = 1.f - pv, qu = 1.f - pu;
    const float a = v0 * qv + v1 * pv, b = v2 * qv + v3 * pv;
    *d = a * qu + b * pu;
    return 1;
}

/* compute_carve_functor: keep[i] = 1 when the voxel survives.  K row-major 3x3, E row-major 4x4. */
void orc_vg_carve(const int32_t *keys, long long n, float vs, const float o[3], const float *img, int w, int h, int sampled,
                  const float K[9], const float E[16], int keep_outside, uint8_t *keep) {
    const float r = vs * 0.5f;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        float c[3];
        for (int a = 0; a < 3; ++a) c[a] = ((float)keys[3 * i + a] + 0.5f) * vs + o[a];
        int kept = 0;
        for (int j = 0; j < 8 && !kept; ++j) {
            const float p[3] = {c[0] + ((j & 2) ? r : -r), c[1] + ((j & 4) ? r : -r), c[2] + ((j & 1) ? r : -r)};
            float x[3], m[3];
            for (int a = 0; a < 3; ++a) x[a] = fmaf(E[4 * a + 2], p[2], fmaf(E[4 * a + 1], p[1], E[4 * a] * p[0])) + E[4 * a + 3];
            for (int a = 0; a < 3; ++a) m[a] = fmaf(K[3 * a + 2], x[2], fmaf(K[3 * a + 1], x[1], K[3 * a] * x[0]));
            const float z = m[2], u = m[0] / z, v = m[1] / z;
            float d = 0.f;
            const int within = sample(img, w, h, sampled, u, v, z, &d);
            kept = (!within && keep_outside) || (within && d > 0.f && z >= d);
        }
        keep[i] = (uint8_t)kept;
    }
}

/* += (average = 1) and AddVoxels (average = 0): a's voxels then b's, sorted by (key, position), one voxel per key */
static const int32_t *g_keys;
static int cmp_pos(const void *a, const void *b) {
    const long long i = *(const long long *)a, j = *(const long long *)b;
    const int c = cmp_key(g_keys + 3 * i, g_keys + 3 * j);
    return c ? c : (i < j ? -1 : i > j);
}
long long orc_vg_merge(const int32_t *keys, const float *colors, long long n, int average, int32_t *out_keys, float *out_colors) {
    long long *ord = (long long *)malloc(sizeof(long long) * (n ? n : 1));
    for (long long i = 0; i < n; ++i) ord[i] = i;
    g_keys = keys;
    qsort(ord, (size_t)n, sizeof(long long), cmp_pos);
    long long m = 0;
    for (long long b = 0; b < n;) {
        long long e = b + 1;
        while (e < n && cmp_key(keys + 3 * ord[e], keys + 3 * ord[b]) == 0) ++e;
        const long long f = ord[b];
        float c[3] = {colors[3 * f], colors[3 * f + 1], colors[3 * f + 2]};
        if (average) {
            for (long long t = b + 1; t < e; ++t)
                for (int a = 0; a < 3; ++a) c[a] = c[a] + colors[3 * ord[t] + a];
            for (int a = 0; a < 3; ++a) c[a] = c[a] / (float)(int)(e - b);
        }
        for (int a = 0; a < 3; ++a) {
            out_keys[3 * m + a] = keys[3 * f + a];
            out_colors[3 * m + a] = c[a];
        }
        ++m;
        b = e;
    }
    free(ord);
    return m;
}
