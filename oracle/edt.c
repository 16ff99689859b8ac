/*
 * edt.c -- CPU restatement of cupoch's geometry::DistanceTransform (geometry/distancetransform.cu) as the product
 * defines it (DESIGN.md section 4, parity hazard 13).  TEST INFRASTRUCTURE ONLY, like oracle.c: loaded by tests/ and
 * tools/bench_ops.py through edt_py.py, never by the product.  Built by edt_py.build() with oracle/Makefile's flags
 * (-ffp-contract=off, no -ffast-math, OpenMP).
 *
 * The transform is separable: along z the nearest site of each row, along y then x the lower envelope of the
 * candidates the previous pass left on each line (Felzenszwalb-Huttenlocher with integer breakpoints).  Every
 * comparison lets the smaller coordinate win a tie, which makes the result the lexicographically smallest of the
 * equidistant sites.  Squared distances are exact integers; distance = sqrtf((float)d2) * voxel_size.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

#define DT_NONE (-1)

int orc_dt_voxel_size_ok(float vs_dt, float vs_vg);
void orc_dt_key_cells(const int32_t *keys, int64_t n, float vs, const float o_vg[3], const float o_dt[3], int res,
                      int32_t *cells, uint8_t *inside);
void orc_dt_compute(int res, const int32_t *cells, int64_t n, int with_distance, float vs, uint16_t *nearest,
                    uint8_t *state, float *dist);
void orc_dt_distance_index(const float *pts, int64_t n, float vs, const float o[3], int res, int64_t *idx);
void orc_dt_voxel_index(const float *pts, int64_t n, float vs, const float o[3], int res, int64_t *idx);

/* distancetransform.cu:331-337 */
int orc_dt_voxel_size_ok(float vs_dt, float vs_vg) { return !(fabsf(vs_dt - vs_vg) > FLT_EPSILON); }

/* compute_obstacle_cells_functor (:254-260): floor(((k * vs + o_vg) - o_dt) / vs) + res / 2, one rounding per operation */
void orc_dt_key_cells(const int32_t *keys, int64_t n, float vs, const float o_vg[3], const float o_dt[3], int res,
                      int32_t *cells, uint8_t *inside) {
    const int half = res / 2;
    for (int64_t i = 0; i < n; ++i) {
        int in = 1;
        for (int a = 0; a < 3; ++a) {
            const float p = (float)keys[3 * i + a] * vs;
            const float q = p + o_vg[a];
            const float d = q - o_dt[a];
            const float f = floorf(d / vs);
            const int ok = f >= (float)-half && f < (float)(res - half);
            in = in && ok;
            cells[3 * i + a] = ok ? (int32_t)f + half : 0;
        }
        inside[i] = (uint8_t)in;
    }
}

/* site packed as x << 20 | y << 10 | z, DT_NONE when the pass found none */
static inline int sx(int32_t p) { return (p >> 20) & 1023; }
static inline int sy(int32_t p) { return (p >> 10) & 1023; }
static inline int sz(int32_t p) { return p & 1023; }

static inline int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

/* one line of pass y (axis 1) or x (axis 0): in[] / out[] at base + t * step; (fa, fz) are the line's fixed
 * coordinates (axis 1: x = fa; axis 0: y = fa).  v / st: scratch of res entries. */
static void envelope_line(const int32_t *in, int32_t *out, int64_t base, int64_t step, int res, int axis, int fa, int fz,
                          int32_t *v, int64_t *st) {
    int k = 0;
    for (int t = 0; t < res; ++t) {
        const int32_t c = in[base + t * step];
        if (c == DT_NONE) continue;
        const int64_t Fc = axis == 1 ? (int64_t)(sz(c) - fz) * (sz(c) - fz)
                                     : (int64_t)(sy(c) - fa) * (sy(c) - fa) + (int64_t)(sz(c) - fz) * (sz(c) - fz);
        int64_t s = 0;
        while (k > 0) {
            const int32_t b = v[k - 1];
            const int qb = axis == 1 ? sy(b) : sx(b);
            const int64_t Fb = axis == 1 ? (int64_t)(sz(b) - fz) * (sz(b) - fz)
                                         : (int64_t)(sy(b) - fa) * (sy(b) - fa) + (int64_t)(sz(b) - fz) * (sz(b) - fz);
            /* first t at which c is strictly nearer than b: (t - t_c)^2 + Fc < (t - qb)^2 + Fb */
            s = floor_div(Fc - Fb + (int64_t)t * t - (int64_t)qb * qb, 2 * (int64_t)(t - qb)) + 1;
            if (s > st[k - 1]) break;
            --k;
            s = 0;
        }
        if (k > 0 && s >= res) continue;
        v[k] = c;
        st[k] = k > 0 ? s : 0;
        ++k;
    }
    int j = 0;
    for (int t = 0; t < res; ++t) {
        while (j + 1 < k && st[j + 1] <= t) ++j;
        out[base + t * step] = k ? v[j] : DT_NONE;
    }
}

void orc_dt_compute(int res, const int32_t *cells, int64_t n, int with_distance, float vs, uint16_t *nearest,
                    uint8_t *state, float *dist) {
    const int64_t r = res, rr = r * r, cn = rr * r;
    uint8_t *site = (uint8_t *)calloc((size_t)cn, 1);
    int32_t *a = (int32_t *)malloc(sizeof(int32_t) * (size_t)cn);
    int32_t *b = (int32_t *)malloc(sizeof(int32_t) * (size_t)cn);
    for (int64_t i = 0; i < n; ++i) {
        const int x = cells[3 * i], y = cells[3 * i + 1], z = cells[3 * i + 2];
        if (x < 0 || y < 0 || z < 0 || x >= res || y >= res || z >= res) continue; /* ignored (hazard 13) */
        site[(x * r + y) * r + z] = 1;
    }
    /* pass z: nearest site of the row, the smaller z on a tie */
#pragma omp parallel for schedule(static)
    for (int64_t line = 0; line < rr; ++line) {
        const int x = (int)(line / r), y = (int)(line % r);
        const int64_t base = line * r;
        int prev = -1;
        for (int z = 0; z < res; ++z) {
            if (site[base + z]) prev = z;
            a[base + z] = prev;
        }
        int next = -1;
        for (int z = res - 1; z >= 0; --z) {
            if (site[base + z]) next = z;
            const int p = a[base + z];
            int best = p;
            if (next >= 0 && (p < 0 || next - z < z - p)) best = next;
            a[base + z] = best < 0 ? DT_NONE : (int32_t)((x << 20) | (y << 10) | best);
        }
    }
    free(site);
    /* pass y: lines (x, ., z) from a into b; pass x: lines (., y, z) from b into a */
#pragma omp parallel
    {
        int32_t *v = (int32_t *)malloc(sizeof(int32_t) * (size_t)res);
        int64_t *st = (int64_t *)malloc(sizeof(int64_t) * (size_t)res);
#pragma omp for schedule(static)
        for (int64_t line = 0; line < rr; ++line)
            envelope_line(a, b, (line / r) * rr + line % r, r, res, 1, (int)(line / r), (int)(line % r), v, st);
#pragma omp for schedule(static)
        for (int64_t line = 0; line < rr; ++line)
            envelope_line(b, a, (line / r) * r + line % r, rr, res, 0, (int)(line / r), (int)(line % r), v, st);
        free(v);
        free(st);
    }
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < cn; ++i) {
        const int x = (int)(i / rr), y = (int)((i / r) % r), z = (int)(i % r);
        const int32_t p = a[i];
        const int nx = p == DT_NONE ? 0 : sx(p), ny = p == DT_NONE ? 0 : sy(p), nz = p == DT_NONE ? 0 : sz(p);
        nearest[3 * i] = (uint16_t)nx;
        nearest[3 * i + 1] = (uint16_t)ny;
        nearest[3 * i + 2] = (uint16_t)nz;
        state[i] = p == DT_NONE ? 2 : 0; /* DistanceVoxel::NotSite */
        const int d2 = (nx - x) * (nx - x) + (ny - y) * (ny - y) + (nz - z) * (nz - z);
        dist[i] = with_distance ? sqrtf((float)d2) * vs : 0.0f;
    }
    free(a);
    free(b);
}

/* get_index_functor / GetDistance (:263-279, :411-419): floor(((q - o) + (0.5 * vs) * res) / vs); -1 outside or NaN */
void orc_dt_distance_index(const float *pts, int64_t n, float vs, const float o[3], int res, int64_t *idx) {
    const float shift = (0.5f * vs) * (float)res;
    for (int64_t i = 0; i < n; ++i) {
        int64_t id = 0;
        int in = 1;
        for (int a = 0; a < 3; ++a) {
            const float d = pts[3 * i + a] - o[a];
            const float f = floorf((d + shift) / vs);
            in = in && f >= 0.0f && f < (float)res;
            id = id * res + (in ? (int64_t)f : 0);
        }
        idx[i] = in ? id : -1;
    }
}

/* DenseGrid::GetVoxelIndex (densegrid.inl:137-146): floor((q - o) / vs) + res / 2; -1 outside (any axis) or NaN */
void orc_dt_voxel_index(const float *pts, int64_t n, float vs, const float o[3], int res, int64_t *idx) {
    const int half = res / 2;
    for (int64_t i = 0; i < n; ++i) {
        int64_t id = 0;
        int in = 1;
        for (int a = 0; a < 3; ++a) {
            const float f = floorf((pts[3 * i + a] - o[a]) / vs);
            in = in && f >= (float)-half && f < (float)(res - half);
            id = id * res + (in ? (int64_t)f + half : 0);
        }
        idx[i] = in ? id : -1;
    }
}
