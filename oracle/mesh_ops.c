/* mesh_ops.c -- plain-C restatement of TriangleMesh's ComputeEdgeList, FilterSharpen / FilterSmoothSimple /
 * FilterSmoothLaplacian / FilterSmoothTaubin, GetSurfaceArea and SamplePointsUniformly (DESIGN section 4 item 24),
 * the bit-for-bit target of the device kernels (cupoch_b200/csrc/mesh.cu).
 *
 * Written from the definitions: float32 throughout, no contraction (-ffp-contract=off), every expression in the
 * reference's order; where the reference's C++ promotes to double (1.0 + N in Simple, the 1e-12 in the Laplacian
 * weights, the per-triangle boundaries) so does this file.  Sums over a vertex's neighbours go left to right in
 * ascending neighbour order from the first term.  The surface area is the float64 sum in the engine's reduction order
 * (sum_values.cuh), the sampling scan the fixed tile order of mesh.cu, and the random draws come from stepping
 * minstd_rand serially from its default seed -- the sequence the device reaches by jump-ahead.
 *
 * Return codes: 0 ok, 1 a vertex index out of range or an edge list out of order, 2 a total area that is not positive
 * and finite, 3 a bad argument. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MINSTD_A 48271u
#define MINSTD_M 2147483647u

static uint32_t minstd_next(uint32_t x) { return (uint32_t)(((uint64_t)x * MINSTD_A) % MINSTD_M); }

/* thrust::uniform_real_distribution<float>(0, 1) of a draw x: (x - min) / (1 + (max - min)), then * (b - a) + a */
static float uniform01(uint32_t x) {
    float r = (float)(x - 1u);
    r /= 1.0f + (float)(2147483646u - 1u);
    return r * (1.0f - 0.0f) + 0.0f;
}

static int cmp_u64(const void *a, const void *b) {
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : x > y;
}

/* ComputeEdgeList -> the number of unique directed edges written to edges [6 nt][2] */
int orc_mesh_edge_list(const int32_t *tri, long long nt, long long nv, int32_t *edges, long long *n_edges) {
    *n_edges = 0;
    uint64_t *k = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(6 * nt + 1));
    for (long long t = 0; t < nt; ++t) {
        for (int j = 0; j < 3; ++j) {
            const int32_t a = tri[3 * t + j], b = tri[3 * t + (j + 1) % 3];
            if (a < 0 || a >= nv || b < 0 || b >= nv) {
                free(k);
                return 1;
            }
            const uint64_t lo = (uint32_t)(a < b ? a : b), hi = (uint32_t)(a < b ? b : a);
            k[6 * t + 2 * j] = lo << 32 | hi;
            k[6 * t + 2 * j + 1] = hi << 32 | lo;
        }
    }
    qsort(k, (size_t)(6 * nt), sizeof(uint64_t), cmp_u64);
    long long n = 0;
    for (long long i = 0; i < 6 * nt; ++i) {
        if (i > 0 && k[i] == k[i - 1]) continue;
        edges[2 * n] = (int32_t)(k[i] >> 32);
        edges[2 * n + 1] = (int32_t)(uint32_t)k[i];
        ++n;
    }
    free(k);
    *n_edges = n;
    return 0;
}

/* one pass of one attribute: in -> out */
static void filter_pass(int kind, float c, const int32_t *e, const long long *rows, const float *w, const float *tw, long long nv,
                        const float *in, float *out) {
    for (long long v = 0; v < nv; ++v) {
        const long long lo = rows[v], hi = rows[v + 1];
        const float *prv = in + 3 * v;
        if (lo == hi) {
            memcpy(out + 3 * v, prv, 12);
            continue;
        }
        float sum[3] = {0.f, 0.f, 0.f};
        for (long long j = lo; j < hi; ++j) {
            const float *x = in + 3 * (long long)e[2 * j + 1];
            for (int k = 0; k < 3; ++k) {
                const float t = kind >= 2 ? w[j] * x[k] : x[k];
                sum[k] = j == lo ? t : sum[k] + t;
            }
        }
        for (int k = 0; k < 3; ++k) {
            if (kind == 0)
                out[3 * v + k] = prv[k] + c * (prv[k] * (float)(uint32_t)(hi - lo) - sum[k]);
            else if (kind == 1)
                out[3 * v + k] = (prv[k] + sum[k]) / (float)(1.0 + (double)(hi - lo));
            else
                out[3 * v + k] = prv[k] + c * (sum[k] / tw[v] - prv[k]);
        }
    }
}

/* kind 0 Sharpen (c0 = strength), 1 Simple, 2 Laplacian (c0 = lambda), 3 Taubin (c0 = lambda, c1 = mu).  in[a] NULL:
 * absent; out[a] receives the filtered attribute when bit a of mask is set and iterations > 0, else a copy. */
int orc_mesh_filter(int kind, int iterations, float c0, float c1, const int32_t *e, long long ne, long long nv, const float *vtx,
                    const float *nrm, const float *col, int mask, float *out_v, float *out_n, float *out_c) {
    if (kind < 0 || kind > 3) return 3;
    for (long long i = 0; i < ne; ++i) {
        const int32_t a = e[2 * i], b = e[2 * i + 1];
        if (a < 0 || a >= nv || b < 0 || b >= nv) return 1;
        if (i > 0 && (e[2 * i - 2] > a || (e[2 * i - 2] == a && e[2 * i - 1] > b))) return 1;
    }
    const float *in[3] = {vtx, nrm, col};
    float *out[3] = {out_v, out_n, out_c};
    const long long passes = iterations > 0 ? (long long)iterations * (kind == 3 ? 2 : 1) : 0;
    long long *rows = (long long *)malloc(sizeof(long long) * (size_t)(nv + 1));
    for (long long v = 0, i = 0; v <= nv; ++v) {
        while (i < ne && e[2 * i] < v) ++i;
        rows[v] = i;
    }
    float *w = (float *)malloc(sizeof(float) * (size_t)(ne + 1)), *tw = (float *)malloc(sizeof(float) * (size_t)(nv + 1));
    if (kind >= 2) {
        for (long long v = 0; v < nv; ++v) {
            float t = 0.f;
            for (long long j = rows[v]; j < rows[v + 1]; ++j) {
                const float *p = vtx + 3 * v, *q = vtx + 3 * (long long)e[2 * j + 1];
                const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
                const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
                w[j] = (float)(1.0 / ((double)dist + 1e-12));
                t = j == rows[v] ? w[j] : t + w[j];
            }
            tw[v] = t;
        }
    }
    float *a_buf = (float *)malloc(12 * (size_t)(nv + 1)), *b_buf = (float *)malloc(12 * (size_t)(nv + 1));
    for (int a = 0; a < 3; ++a) {
        if (!in[a]) continue;
        memcpy(a_buf, in[a], 12 * (size_t)nv);
        if ((mask >> a) & 1) {
            for (long long q = 0; q < passes; ++q) {
                const float c = kind == 3 && q % 2 == 1 ? c1 : c0;
                filter_pass(kind == 3 ? 2 : kind, c, e, rows, w, tw, nv, a_buf, b_buf);
                float *t = a_buf;
                a_buf = b_buf;
                b_buf = t;
            }
        }
        memcpy(out[a], a_buf, 12 * (size_t)nv);
    }
    free(rows);
    free(w);
    free(tw);
    free(a_buf);
    free(b_buf);
    return 0;
}

/* ComputeTriangleArea: 0.5 |(p0 - p1) x (p0 - p2)| in float32; -1 for an index out of range */
static float triangle_area(const float *vtx, long long nv, const int32_t *tri, long long t) {
    for (int j = 0; j < 3; ++j)
        if (tri[3 * t + j] < 0 || tri[3 * t + j] >= nv) return -1.f;
    const float *p0 = vtx + 3 * (long long)tri[3 * t], *p1 = vtx + 3 * (long long)tri[3 * t + 1], *p2 = vtx + 3 * (long long)tri[3 * t + 2];
    const float x0 = p0[0] - p1[0], x1 = p0[1] - p1[1], x2 = p0[2] - p1[2];
    const float y0 = p0[0] - p2[0], y1 = p0[1] - p2[1], y2 = p0[2] - p2[2];
    const float c0 = x1 * y2 - x2 * y1, c1 = x2 * y0 - x0 * y2, c2 = x0 * y1 - x1 * y0;
    return 0.5f * sqrtf(c0 * c0 + c1 * c1 + c2 * c2);
}

/* GetSurfaceArea: areas [nt] (may be NULL), *total = the float64 sum in the engine's reduction order, as float */
int orc_mesh_surface_area(const float *vtx, long long nv, const int32_t *tri, long long nt, float *areas, float *total) {
    *total = 0.f;
    if (nt == 0) return 0;
    float *ar = (float *)malloc(sizeof(float) * (size_t)nt);
    for (long long t = 0; t < nt; ++t) {
        ar[t] = triangle_area(vtx, nv, tri, t);
        if (ar[t] < 0.f) {
            free(ar);
            return 1;
        }
    }
    if (areas) memcpy(areas, ar, sizeof(float) * (size_t)nt);
    const long long block = 256, max_blocks = 592;
    long long grid = (nt + block - 1) / block;
    if (grid > max_blocks) grid = max_blocks;
    double sum = 0.0;
    for (long long b = 0; b < grid; ++b) {
        double part = 0.0;
        for (int warp = 0; warp < 8; ++warp) {
            double lane[32];
            for (int l = 0; l < 32; ++l) {
                double acc = 0.0;
                for (long long i = b * block + warp * 32 + l; i < nt; i += grid * block) acc += (double)ar[i];
                lane[l] = acc;
            }
            for (int o = 16; o > 0; o >>= 1) {
                double nxt[32];
                for (int l = 0; l < 32; ++l) nxt[l] = lane[l] + lane[l ^ o];
                memcpy(lane, nxt, sizeof(lane));
            }
            part += lane[0];
        }
        sum += part;
    }
    *total = (float)sum;
    free(ar);
    return 0;
}

#define TILE_THREAD 8
#define TILE (256 * TILE_THREAD)

/* SamplePointsUniformly: points / normals / colours [n][3]; normals from tn when given, else interpolated vn; NULL
 * outputs are skipped.  Also the boundaries bnd [nt + 1] when bnd is not NULL. */
int orc_mesh_sample(const float *vtx, long long nv, const int32_t *tri, long long nt, const float *vn, const float *tn, const float *vc,
                    long long n, float *pts, float *nrm, float *col, uint32_t *bnd_out) {
    if (n <= 0 || n > 1073741823ll || nt <= 0) return 3;
    double *S = (double *)malloc(sizeof(double) * (size_t)nt);
    const long long nb = (nt + TILE - 1) / TILE;
    double B = 0.0; /* exclusive sum of the block totals */
    for (long long b = 0; b < nb; ++b) {
        double T = 0.0; /* exclusive sum of the thread totals */
        for (int t = 0; t < 256; ++t) {
            double L = 0.0;
            for (int j = 0; j < TILE_THREAD; ++j) {
                const long long i = b * TILE + t * TILE_THREAD + j;
                if (i >= nt) break;
                const float a = triangle_area(vtx, nv, tri, i);
                if (a < 0.f) {
                    free(S);
                    return 1;
                }
                L = L + (double)a;
                S[i] = T + L; /* B added below, once the block is done */
            }
            T = T + L;
        }
        for (long long i = b * TILE; i < nt && i < (b + 1) * TILE; ++i) S[i] = B + S[i];
        B = B + T;
    }
    const double total = B;
    if (!(total > 0.0 && total <= 1.7976931348623157e308)) {
        free(S);
        return 2;
    }
    uint32_t *bnd = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(nt + 1));
    bnd[0] = 0;
    for (long long i = 0; i < nt; ++i) {
        long long x = llrint(S[i] / total * (double)n);
        if (x < (long long)bnd[i]) x = bnd[i];
        if (x > n) x = n;
        bnd[i + 1] = (uint32_t)x;
    }
    bnd[nt] = (uint32_t)n;
    uint32_t x = 1u; /* the default seed */
    for (long long i = 0; i < nt; ++i) {
        const int32_t *f = tri + 3 * i;
        for (long long p = bnd[i]; p < bnd[i + 1]; ++p) {
            x = minstd_next(x);
            const float r1 = uniform01(x);
            x = minstd_next(x);
            const float r2 = uniform01(x);
            const float sr = sqrtf(r1);
            const float a = 1.f - sr, b = sr * (1.f - r2), c = sr * r2;
            for (int k = 0; k < 3; ++k) {
                pts[3 * p + k] = a * vtx[3 * f[0] + k] + b * vtx[3 * f[1] + k] + c * vtx[3 * f[2] + k];
                if (nrm) nrm[3 * p + k] = tn ? tn[3 * i + k] : a * vn[3 * f[0] + k] + b * vn[3 * f[1] + k] + c * vn[3 * f[2] + k];
                if (col) col[3 * p + k] = a * vc[3 * f[0] + k] + b * vc[3 * f[1] + k] + c * vc[3 * f[2] + k];
            }
        }
    }
    if (bnd_out) memcpy(bnd_out, bnd, sizeof(uint32_t) * (size_t)(nt + 1));
    free(bnd);
    free(S);
    return 0;
}
