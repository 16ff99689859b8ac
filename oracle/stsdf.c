/* stsdf.c -- plain-C restatement of integration::ScalableTSDFVolume as cupoch_b200/csrc/stsdf.cu computes it.  Built by
 * oracle.build("stsdf"); loader stsdf_py.py.  It includes depth_cloud.c for the depth projection and the float64 pose,
 * as the kernel shares depth_project.cuh with CreateFromDepthImage.
 *
 * Units live in slots in the order they were first allocated; a plain sorted (key, slot) array finds them.  Packed
 * key: each axis + 2^20 in 21 bits, x highest.  Voxel index in a unit x * 256 + y * 16 + z.  Every float operation is
 * rounded on its own (-ffp-contract=off) except where fmaf() states a fused multiply-add, in the kernel's order.
 * Line numbers cite the reference's integration/scalable_tsdfvolume.cu (ST) and integrate_functor.h (IF). */
#include "depth_cloud.c"

#include <stdlib.h>

#define RES 16
#define VOX 4096
#define BIAS (1 << 20)

typedef struct {
    uint64_t key;
    long long slot;
} Entry;

typedef struct {
    float vl, half, U, trunc, trunc_inv;
    int ct, planes, stride;
    long long count, cap;
    uint64_t *keys;
    float *tw;  /* [cap][4096][2] */
    float *col; /* [cap][planes][4096] */
    Entry *map; /* [count] sorted by key */
} Vol;

static uint64_t pack(long long x, long long y, long long z) {
    return ((uint64_t)(x + BIAS) << 42) | ((uint64_t)(y + BIAS) << 21) | (uint64_t)(z + BIAS);
}
static int axis_of(uint64_t k, int a) { return (int)((k >> (42 - 21 * a)) & 0x1fffff) - BIAS; }
static int cmp_u64(const void *a, const void *b) {
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : x > y;
}
static int cmp_entry(const void *a, const void *b) { return cmp_u64(&((const Entry *)a)->key, &((const Entry *)b)->key); }

static long long find(const Vol *v, long long x, long long y, long long z) {
    if (x < -BIAS || x >= BIAS || y < -BIAS || y >= BIAS || z < -BIAS || z >= BIAS) return -1;
    Entry e = {pack(x, y, z), 0};
    const Entry *r = bsearch(&e, v->map, (size_t)v->count, sizeof(Entry), cmp_entry);
    return r ? r->slot : -1;
}

void *orc_st_create(float vl, float trunc, int ct, int stride) {
    Vol *v = calloc(1, sizeof(Vol));
    v->vl = vl;
    v->half = 0.5f * vl;
    v->U = vl * 16.0f;
    v->trunc = trunc;
    v->trunc_inv = (float)(1.0 / (double)trunc);
    v->ct = ct;
    v->planes = ct == 1 ? 3 : ct == 2 ? 1 : 0;
    v->stride = stride;
    return v;
}

void orc_st_destroy(void *h) {
    Vol *v = h;
    free(v->keys);
    free(v->tw);
    free(v->col);
    free(v->map);
    free(v);
}

void orc_st_reset(void *h) { ((Vol *)h)->count = 0; }
long long orc_st_units(void *h) { return ((Vol *)h)->count; }

void orc_st_data(void *h, uint64_t *keys, float *tw, float *col) {
    const Vol *v = h;
    memcpy(keys, v->keys, (size_t)v->count * 8);
    memcpy(tw, v->tw, (size_t)v->count * VOX * 8);
    if (v->planes) memcpy(col, v->col, (size_t)v->count * v->planes * VOX * 4);
}

/* -> 0, -1 for a singular extrinsic, -2 for a unit key out of range (the volume is then unchanged) */
int orc_st_integrate(void *h, const float *depth, const void *color, int w, int hh, const float K4[4], const float E[16]) {
    Vol *v = h;
    Cam c;
    if (!orc_depth_cloud_pose(E, c.P)) return -1;
    c.fx = K4[0];
    c.fy = K4[1];
    c.cx = K4[2];
    c.cy = K4[3];
    c.cutoff = -1.f;
    c.w = w;
    c.stride = v->stride;
    c.sw = w / v->stride;
    c.sh = hh / v->stride;
    c.bytes = 4;
    c.scale_i = 1;
    c.trunc_i = 0;
    c.depth = depth;
    /* (1) the candidate keys (ST:98-123) */
    size_t n = 0, capk = 1024;
    uint64_t *cand = malloc(capk * 8);
    for (int sr = 0; sr < c.sh; ++sr)
        for (int sc = 0; sc < c.sw; ++sc) {
            float p[3];
            if (!point_at(&c, sr, sc, p)) continue;
            long long lo[3], hi[3];
            for (int a = 0; a < 3; ++a) {
                const float l = floorf((p[a] - v->trunc) / v->U), u = floorf((p[a] + v->trunc) / v->U);
                if (!(l >= (float)-BIAS && u < (float)BIAS)) {
                    free(cand);
                    return -2;
                }
                lo[a] = (long long)l;
                hi[a] = (long long)u;
            }
            for (long long x = lo[0]; x <= hi[0]; ++x)
                for (long long y = lo[1]; y <= hi[1]; ++y)
                    for (long long z = lo[2]; z <= hi[2]; ++z) {
                        if (n == capk) cand = realloc(cand, (capk *= 2) * 8);
                        cand[n++] = pack(x, y, z);
                    }
        }
    /* (2) sorted, unique, the missing ones in ascending order; (4) appended */
    qsort(cand, n, 8, cmp_u64);
    long long m = 0;
    for (size_t i = 0; i < n; ++i)
        if (i == 0 || cand[i] != cand[i - 1]) {
            const uint64_t k = cand[i];
            if (find(v, axis_of(k, 0), axis_of(k, 1), axis_of(k, 2)) < 0) cand[m++] = k;
        }
    if (v->count + m > v->cap) {
        long long cap = v->cap ? v->cap : 1;
        while (cap < v->count + m) cap *= 2;
        v->keys = realloc(v->keys, (size_t)cap * 8);
        v->tw = realloc(v->tw, (size_t)cap * VOX * 8);
        v->col = realloc(v->col, (size_t)cap * (v->planes ? v->planes : 1) * VOX * 4);
        v->map = realloc(v->map, (size_t)cap * sizeof(Entry));
        v->cap = cap;
    }
    for (long long j = 0; j < m; ++j) {
        const long long s = v->count + j;
        v->keys[s] = cand[j];
        for (int t = 0; t < VOX; ++t) v->tw[2 * (s * VOX + t)] = v->tw[2 * (s * VOX + t) + 1] = 0.f;
        for (long long t = 0; t < (long long)v->planes * VOX; ++t) v->col[s * v->planes * VOX + t] = 1.f;
        v->map[s].key = cand[j];
        v->map[s].slot = s;
    }
    v->count += m;
    qsort(v->map, (size_t)v->count, sizeof(Entry), cmp_entry);
    free(cand);
    /* (5) every allocated voxel: ComputeTSDF (IF:84-139) at the column point (fma(vl, x, vl/2) + o0, fma(vl, y, vl/2) + o1,
     * vl/2 + o2), o = key * U, z index z */
    const float fxi = 1.0f / c.fx, fyi = 1.0f / c.fy;
    const float safe_w = (float)w - 0.0001f, safe_h = (float)hh - 0.0001f;
    float S[3];
    for (int r = 0; r < 3; ++r) S[r] = v->vl * E[4 * r + 2];
#pragma omp parallel for schedule(static)
    for (long long s = 0; s < v->count; ++s) {
        const float o[3] = {(float)axis_of(v->keys[s], 0) * v->U, (float)axis_of(v->keys[s], 1) * v->U, (float)axis_of(v->keys[s], 2) * v->U};
        for (int t = 0; t < VOX; ++t) {
            const int x = t >> 8, y = (t >> 4) & 15, z = t & 15;
            const float p0 = fmaf(v->vl, (float)x, v->half) + o[0];
            const float p1 = fmaf(v->vl, (float)y, v->half) + o[1];
            const float p2 = v->half + o[2];
            float cam[3];
            for (int r = 0; r < 3; ++r)
                cam[r] = fmaf((float)z, S[r], fmaf(E[4 * r + 2], p2, fmaf(E[4 * r + 1], p1, E[4 * r] * p0)) + E[4 * r + 3]);
            if (cam[2] <= 0.f) continue;
            const float uf = (cam[0] * c.fx) / cam[2] + c.cx + 0.5f;
            const float vf = (cam[1] * c.fy) / cam[2] + c.cy + 0.5f;
            if (!(uf >= 0.0001f && uf < safe_w && vf >= 0.0001f && vf < safe_h)) continue;
            const int u = (int)floorf(uf), vv = (int)floorf(vf);
            const long long px = (long long)vv * w + u;
            const float d = depth[px];
            if (d <= 0.f) continue;
            const float xx = ((float)u - c.cx) * fxi, yy = ((float)vv - c.cy) * fyi;
            const float sdf = (d - cam[2]) * sqrtf(fmaf(yy, yy, xx * xx) + 1.0f);
            if (!(sdf > -v->trunc)) continue;
            const float tt = fminf(1.0f, sdf * v->trunc_inv);
            float *tw = v->tw + 2 * (s * VOX + t);
            const float w0 = tw[1], w1 = w0 + 1.0f;
            tw[0] = fmaf(tw[0], w0, tt) / w1;
            tw[1] = w1;
            float *cc = v->col + s * v->planes * VOX + t;
            if (v->ct == 1) {
                const uint8_t *rgb = (const uint8_t *)color + 3 * px;
                for (int k = 0; k < 3; ++k) cc[k * VOX] = fmaf(cc[k * VOX], w0, (float)rgb[k]) / w1;
            } else if (v->ct == 2) {
                cc[0] = fmaf(cc[0], w0, ((const float *)color)[px]) / w1;
            }
        }
    }
    return 0;
}

static int band(const float *tw) { return tw[1] != 0.0f && tw[0] < 0.98f && tw[0] >= -0.98f; }

/* voxel k + e_a of unit s: its slot (-1 when missing), k updated */
static long long step(const Vol *v, long long s, int k[3], int a) {
    if (k[a] + 1 < RES) {
        k[a] += 1;
        return s;
    }
    k[a] = 0;
    long long u[3] = {axis_of(v->keys[s], 0), axis_of(v->keys[s], 1), axis_of(v->keys[s], 2)};
    u[a] += 1;
    return find(v, u[0], u[1], u[2]);
}

/* GetTSDFAt (ST:167-213) in the kernel's form */
static float tsdf_at(const Vol *v, const float p[3]) {
    long long u[3];
    int b[3];
    float r[3];
    for (int a = 0; a < 3; ++a) {
        const float pl = p[a] - v->half;
        u[a] = (long long)floorf(pl / v->U);
        const float g = (pl - (float)u[a] * v->U) / v->vl;
        b[a] = (int)floorf(g);
        b[a] = b[a] < 0 ? 0 : b[a] >= RES ? RES - 1 : b[a];
        r[a] = g - (float)b[a];
    }
    const long long s0 = find(v, u[0], u[1], u[2]);
    if (s0 < 0) return 0.f;
    float acc = 0.f;
    for (int k = 0; k < 8; ++k) {
        const int d[3] = {(k >> 2) & 1, (k >> 1) & 1, k & 1};
        int q[3];
        long long uu[3];
        int out = 0;
        for (int a = 0; a < 3; ++a) {
            q[a] = b[a] + d[a];
            uu[a] = u[a];
            if (q[a] >= RES) {
                q[a] -= RES;
                uu[a] += 1;
                out = 1;
            }
        }
        const long long s1 = out ? find(v, uu[0], uu[1], uu[2]) : s0;
        const float f = s1 < 0 ? 0.f : v->tw[2 * (s1 * VOX + q[0] * 256 + q[1] * 16 + q[2])];
        const float wx = d[0] ? r[0] : 1.f - r[0], wy = d[1] ? r[1] : 1.f - r[1], wz = d[2] ? r[2] : 1.f - r[2];
        acc = fmaf((wx * wy) * wz, f, acc);
    }
    return acc;
}

/* ExtractPointCloud (ST:231-289) in slot, voxel, axis order; rows written when pts != NULL -> the row count */
long long orc_st_extract_points(void *h, float *pts, float *nrm, float *cols) {
    const Vol *v = h;
    long long row = 0;
    const float hg = (float)(0.99 * (double)v->vl);
    for (long long s = 0; s < v->count; ++s)
        for (int t = 0; t < VOX; ++t) {
            const float *tw0 = v->tw + 2 * (s * VOX + t);
            if (!band(tw0)) continue;
            const int k0[3] = {t >> 8, (t >> 4) & 15, t & 15};
            for (int a = 0; a < 3; ++a) {
                int k1[3] = {k0[0], k0[1], k0[2]};
                const long long s1 = step(v, s, k1, a);
                if (s1 < 0) continue;
                const int t1 = k1[0] * 256 + k1[1] * 16 + k1[2];
                const float *tw1 = v->tw + 2 * (s1 * VOX + t1);
                if (!(band(tw1) && tw0[0] * tw1[0] < 0.f)) continue;
                if (pts) {
                    const float r0 = fabsf(tw0[0]), r1 = fabsf(tw1[0]), rs = r0 + r1;
                    float p[3];
                    for (int b = 0; b < 3; ++b) p[b] = fmaf(v->vl, (float)k0[b], v->half) + (float)axis_of(v->keys[s], b) * v->U;
                    const float p1a = p[a] + v->vl;
                    p[a] = fmaf(p1a, r0, p[a] * r1) / rs;
                    memcpy(pts + 3 * row, p, 12);
                    float nv[3];
                    for (int b = 0; b < 3; ++b) {
                        float q0[3] = {p[0], p[1], p[2]}, q1[3] = {p[0], p[1], p[2]};
                        q0[b] = p[b] - hg;
                        q1[b] = p[b] + hg;
                        nv[b] = tsdf_at(v, q1) - tsdf_at(v, q0);
                    }
                    const float sq = fmaf(nv[2], nv[2], fmaf(nv[1], nv[1], nv[0] * nv[0]));
                    const float q = sqrtf(sq);
                    for (int b = 0; b < 3; ++b) nrm[3 * row + b] = sq > 0.f ? nv[b] / q : nv[b];
                    if (v->ct == 1) {
                        for (int b = 0; b < 3; ++b) {
                            const float c0 = v->col[(s * 3 + b) * VOX + t], c1 = v->col[(s1 * 3 + b) * VOX + t1];
                            cols[3 * row + b] = (fmaf(c1, r0, c0 * r1) / rs) / 255.0f;
                        }
                    } else if (v->ct == 2) {
                        const float g = fmaf(v->col[s1 * VOX + t1], r0, v->col[s * VOX + t] * r1) / rs;
                        cols[3 * row] = cols[3 * row + 1] = cols[3 * row + 2] = g;
                    }
                }
                ++row;
            }
        }
    return row;
}

/* ExtractVoxelPointCloud: band voxel centres, grey (float)(((double)f + 1) * 0.5) */
long long orc_st_extract_voxels(void *h, float *pts, float *cols) {
    const Vol *v = h;
    long long row = 0;
    for (long long s = 0; s < v->count; ++s)
        for (int t = 0; t < VOX; ++t) {
            const float *tw0 = v->tw + 2 * (s * VOX + t);
            if (!band(tw0)) continue;
            if (pts) {
                const int k[3] = {t >> 8, (t >> 4) & 15, t & 15};
                const float g = (float)(((double)tw0[0] + 1.0) * 0.5);
                for (int a = 0; a < 3; ++a) {
                    pts[3 * row + a] = fmaf(v->vl, (float)k[a], v->half) + (float)axis_of(v->keys[s], a) * v->U;
                    cols[3 * row + a] = g;
                }
            }
            ++row;
        }
    return row;
}
