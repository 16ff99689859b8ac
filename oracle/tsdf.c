/* tsdf.c -- plain-C restatement of integration::UniformTSDFVolume and the RGB-D conversion of cupoch_b200/csrc/tsdf.cu.
 * Built by oracle.build("tsdf"); loader tsdf_py.py.
 *
 * The volume is the kernel's layout: tw[2 * N] = (tsdf, weight) per voxel, voxel idx = x res^2 + y res + z, and the
 * colour planes col[c * N + idx] (3 planes for RGB8, 1 for Gray32, whose three channels are always equal, none for
 * NoColor).  Every float operation is rounded on its own (-ffp-contract=off) except where fmaf() states a fused
 * multiply-add, in the order the kernel uses __fmaf_rn.  Line numbers cite the reference's
 * integration/integrate_functor.h (IF), integration/uniform_tsdfvolume.cu (UT), geometry/image.cu (IM) and
 * geometry/image_factory.cu (IFC). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_COLOR 0
#define RGB8 1
#define GRAY32 2

/* ---------------------------------------------------------------------------------------------- RGB-D conversion */
/* ConvertDepthToFloatImage (IM:339-348, 413-421): CreateFloatImage's value (raw * 1/255 for 8-bit, raw otherwise),
 * then / (float)(int)depth_scale, and 0 where it is >= (float)(int)depth_trunc */
void orc_tsdf_depth_to_float(const void *src, int bytes, long long n, int scale_i, int trunc_i, float *out) {
    const float denom = bytes == 1 ? (float)(1.0 / 255.0) : 1.f;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        float f = bytes == 1 ? (float)((const uint8_t *)src)[i] : bytes == 2 ? (float)((const uint16_t *)src)[i] : ((const float *)src)[i];
        f = f * denom;
        f = f / (float)scale_i;
        if (f >= (float)trunc_i) f = 0.f;
        out[i] = f;
    }
}

/* CreateFloatImage(WEIGHTED) (IFC:54-118, 201-224): 1 channel: v * denom; 3 channels:
 * fma(0.1140, p2, fma(0.5870, p1, 0.2990 * p0)) * denom; denom = 1/255 for 8-bit input, 1 otherwise */
void orc_tsdf_intensity(const void *src, int channels, int bytes, long long n, float *out) {
    const float denom = bytes == 1 ? (float)(1.0 / 255.0) : 1.f;
    const float w0 = 0.2990f, w1 = 0.5870f, w2 = 0.1140f;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        float p[3];
        for (int c = 0; c < channels; ++c) {
            const long long k = i * channels + c;
            p[c] = bytes == 1 ? (float)((const uint8_t *)src)[k] : bytes == 2 ? (float)((const uint16_t *)src)[k] : ((const float *)src)[k];
        }
        const float g = channels == 1 ? p[0] : fmaf(w2, p[2], fmaf(w1, p[1], w0 * p[0]));
        out[i] = g * denom;
    }
}

/* ---------------------------------------------------------------------------------------------- the volume */
typedef struct {
    int res, h, ct;
    float vl, half, trunc, trunc_inv, o[3];
} Vol;

static Vol vol(float length, int res, float trunc, int ct, const float o[3]) {
    Vol v;
    v.res = res;
    v.h = res / 2;
    v.ct = ct;
    v.vl = length / (float)res;     /* TSDFVolume(length / (float)resolution, ...) (UT:650) */
    v.half = 0.5f * v.vl;
    v.trunc = trunc;
    v.trunc_inv = (float)(1.0 / (double)trunc); /* sdf_trunc_inv_(1.0 / sdf_trunc) (IF:52) */
    for (int a = 0; a < 3; ++a) v.o[a] = o[a];
    return v;
}

static long long idx_of(int x, int y, int z, int res) { return ((long long)x * res + y) * res + z; }

/* the initial voxel: tsdf 0, weight 0, colour (1, 1, 1) */
void orc_tsdf_reset(float *tw, float *col, int ncol, long long n) {
    for (long long i = 0; i < n; ++i) tw[2 * i] = tw[2 * i + 1] = 0.f;
    for (long long i = 0; i < n * ncol; ++i) col[i] = 1.f;
}

/* uniform_integrate_functor (IF:84-139, 182-190).  K4 = (fx, fy, cx, cy); E = world-to-camera 4x4, row-major.
 *   column point p = (fma(vl, kx, half) + ox, fma(vl, ky, half) + oy, half + oz), k = index - res / 2;
 *   cam_r = fma(E[r][2], p2, fma(E[r][1], p1, E[r][0] * p0)) + E[r][3], then cam_r = fma(kz, vl * E[r][2], cam_r);
 *   u = (cam0 * fx) / cam2 + cx + 0.5 (left to right), the same for v;
 *   multiplier = sqrt(fma(yy, yy, xx * xx) + 1), xx = ((float)u - cx) * (1 / fx), yy alike (IFC:136-164);
 *   sdf = (d - cam2) * multiplier; tsdf' = fma(tsdf, w, min(1, sdf * trunc_inv)) / (w + 1), colour alike. */
void orc_tsdf_integrate(float *tw, float *col, float length, int res, float trunc, int ct, const float o[3], const float *depth,
                        const void *color, int w, int h, const float K4[4], const float E[16]) {
    const Vol V = vol(length, res, trunc, ct, o);
    const float fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    const float fxi = 1.0f / fx, fyi = 1.0f / fy;
    const float safe_w = (float)w - 0.0001f, safe_h = (float)h - 0.0001f;
    float S[3];
    for (int r = 0; r < 3; ++r) S[r] = V.vl * E[4 * r + 2];
    const long long N = (long long)res * res * res;
#pragma omp parallel for schedule(static) collapse(2)
    for (int x = 0; x < res; ++x)
        for (int y = 0; y < res; ++y) {
            const float p0 = fmaf(V.vl, (float)(x - V.h), V.half) + o[0];
            const float p1 = fmaf(V.vl, (float)(y - V.h), V.half) + o[1];
            const float p2 = V.half + o[2];
            float base[3];
            for (int r = 0; r < 3; ++r) base[r] = fmaf(E[4 * r + 2], p2, fmaf(E[4 * r + 1], p1, E[4 * r] * p0)) + E[4 * r + 3];
            for (int z = 0; z < res; ++z) {
                const float kz = (float)(z - V.h);
                const float c0 = fmaf(kz, S[0], base[0]), c1 = fmaf(kz, S[1], base[1]), c2 = fmaf(kz, S[2], base[2]);
                if (c2 <= 0.f) continue;
                const float uf = (c0 * fx) / c2 + cx + 0.5f;
                const float vf = (c1 * fy) / c2 + cy + 0.5f;
                if (!(uf >= 0.0001f && uf < safe_w && vf >= 0.0001f && vf < safe_h)) continue;
                const int u = (int)floorf(uf), v = (int)floorf(vf);
                const float d = depth[(long long)v * w + u];
                if (d <= 0.f) continue;
                const float xx = ((float)u - cx) * fxi, yy = ((float)v - cy) * fyi;
                const float mult = sqrtf(fmaf(yy, yy, xx * xx) + 1.0f);
                const float sdf = (d - c2) * mult;
                if (!(sdf > -trunc)) continue;
                const float t = fminf(1.0f, sdf * V.trunc_inv);
                const long long i = idx_of(x, y, z, res);
                const float w0 = tw[2 * i + 1], w1 = w0 + 1.0f;
                tw[2 * i] = fmaf(tw[2 * i], w0, t) / w1;
                if (ct == RGB8) {
                    const uint8_t *rgb = (const uint8_t *)color + 3 * ((long long)v * w + u);
                    for (int c = 0; c < 3; ++c) col[c * N + i] = fmaf(col[c * N + i], w0, (float)rgb[c]) / w1;
                } else if (ct == GRAY32) {
                    col[i] = fmaf(col[i], w0, ((const float *)color)[(long long)v * w + u]) / w1;
                }
                tw[2 * i + 1] = w1;
            }
        }
}

static int band(const float *tw, long long i) {
    const float f = tw[2 * i], w = tw[2 * i + 1];
    return w != 0.0f && f < 0.98f && f >= -0.98f;
}

/* GetTSDFAt (UT:36-65): g = p / vl - 0.5, base floor(g), r = g - base; the 8 terms in the source's order, each added as
 * acc = fma((a * b) * c ... , v, acc) with the weight product rounded left to right */
static float tsdf_at(const float *tw, const float p[3], float vl, int res) {
    int b[3];
    float r[3];
    for (int a = 0; a < 3; ++a) {
        const float g = p[a] / vl - 0.5f;
        b[a] = (int)floorf(g);
        r[a] = g - (float)b[a];
    }
    float acc = 0.f;
    for (int k = 0; k < 8; ++k) {
        const int dx = (k >> 2) & 1, dy = (k >> 1) & 1, dz = k & 1;
        const float wx = dx ? r[0] : 1.f - r[0], wy = dy ? r[1] : 1.f - r[1], wz = dz ? r[2] : 1.f - r[2];
        acc = fmaf((wx * wy) * wz, tw[2 * idx_of(b[0] + dx, b[1] + dy, b[2] + dz, res)], acc);
    }
    return acc;
}

/* GetNormalAt (UT:67-83): half_gap is a double, so p(i) -+ half_gap is rounded from double; Eigen's normalized():
 * v / sqrt(fma(z, z, fma(y, y, x * x))) when that sum is > 0, else v unchanged (Eigen >= 3.3) */
static void normal_at(const float *tw, const float p[3], float vl, int res, float n[3]) {
    const double half_gap = 0.99 * (double)vl;
    for (int i = 0; i < 3; ++i) {
        float p0[3] = {p[0], p[1], p[2]}, p1[3] = {p[0], p[1], p[2]};
        p0[i] = (float)((double)p0[i] - half_gap);
        p1[i] = (float)((double)p1[i] + half_gap);
        n[i] = tsdf_at(tw, p1, vl, res) - tsdf_at(tw, p0, vl, res);
    }
    const float s = fmaf(n[2], n[2], fmaf(n[1], n[1], n[0] * n[0]));
    if (s > 0.f) {
        const float q = sqrtf(s);
        for (int i = 0; i < 3; ++i) n[i] = n[i] / q;
    }
}

/* which of the axes of interior voxel (x, y, z) emit a point: bit i (extract_pointcloud_functor, UT:104-140) */
static int emit_mask(const float *tw, int x, int y, int z, int res) {
    if (x < 1 || y < 1 || z < 1 || x > res - 2 || y > res - 2 || z > res - 2) return 0;
    const long long i0 = idx_of(x, y, z, res);
    if (!band(tw, i0)) return 0;
    const float f0 = tw[2 * i0];
    int m = 0;
    const int k[3] = {x, y, z};
    for (int i = 0; i < 3; ++i) {
        if (k[i] + 1 >= res - 1) continue;
        const long long i1 = idx_of(x + (i == 0), y + (i == 1), z + (i == 2), res);
        if (band(tw, i1) && f0 * tw[2 * i1] < 0.f) m |= 1 << i;
    }
    return m;
}

/* ExtractPointCloud (UT:85-156, 703-737), sized by the exact number of crossings (the reference sizes its output by
 * the band voxels and can write past it).  Rows in (x, y, z, axis) order.  Crossing on axis i between voxels 0 and 1:
 *   p0 = fma(vl, k, half) per axis, p1(i) = p0(i) + vl, r0 = |f0|, r1 = |f1|,
 *   p(i) = fma(p1(i), r0, p0(i) * r1) / (r0 + r1); point = (p + origin) - (float)(res / 2) * vl;
 *   colour = fma(c1, r0, c0 * r1) / (r0 + r1) (/ 255 for RGB8); normal = GetNormalAt(p).
 * -> the number of rows; only the first cap rows are written (cap may be 0 to count). */
long long orc_tsdf_extract_points(const float *tw, const float *col, float length, int res, float trunc, int ct, const float o[3],
                                  float *pts, float *nrm, float *cols, long long cap) {
    const Vol V = vol(length, res, trunc, ct, o);
    const long long N = (long long)res * res * res;
    const float hres = (float)(res / 2) * V.vl;
    long long cnt = 0;
    for (int x = 1; x <= res - 2; ++x)
        for (int y = 1; y <= res - 2; ++y)
            for (int z = 1; z <= res - 2; ++z) {
                const int m = emit_mask(tw, x, y, z, res);
                if (!m) continue;
                const long long i0 = idx_of(x, y, z, res);
                const int k[3] = {x, y, z};
                for (int i = 0; i < 3; ++i) {
                    if (!(m >> i & 1)) continue;
                    if (cnt < cap) {
                        const long long i1 = idx_of(x + (i == 0), y + (i == 1), z + (i == 2), res);
                        const float r0 = fabsf(tw[2 * i0]), r1 = fabsf(tw[2 * i1]), rs = r0 + r1;
                        float p[3];
                        for (int a = 0; a < 3; ++a) p[a] = fmaf(V.vl, (float)k[a], V.half);
                        const float p1i = p[i] + V.vl;
                        p[i] = fmaf(p1i, r0, p[i] * r1) / rs;
                        for (int a = 0; a < 3; ++a) pts[3 * cnt + a] = (p[a] + o[a]) - hres;
                        normal_at(tw, p, V.vl, res, nrm + 3 * cnt);
                        for (int a = 0; a < 3; ++a) {
                            float c = 0.f;
                            if (ct == RGB8) c = (fmaf(col[a * N + i1], r0, col[a * N + i0] * r1) / rs) / 255.0f;
                            else if (ct == GRAY32) c = fmaf(col[i1], r0, col[i0] * r1) / rs;
                            if (cols) cols[3 * cnt + a] = c;
                        }
                    }
                    ++cnt;
                }
            }
    return cnt;
}

/* ExtractVoxelPointCloud and ExtractVoxelGrid (UT:352-408, 840-895): every band voxel in index order (lexicographic
 * keys, no sort); key (x, y, z), point fma(vl, k - res / 2, half) + origin, grey (float)(((double)f + 1) * 0.5).
 * -> the number of voxels; the first cap are written (any output may be NULL). */
long long orc_tsdf_extract_voxels(const float *tw, float length, int res, const float o[3], int32_t *keys, float *pts, float *cols,
                                  long long cap) {
    const Vol V = vol(length, res, 1.f, NO_COLOR, o);
    long long cnt = 0;
    for (int x = 0; x < res; ++x)
        for (int y = 0; y < res; ++y)
            for (int z = 0; z < res; ++z) {
                const long long i = idx_of(x, y, z, res);
                if (!band(tw, i)) continue;
                if (cnt < cap) {
                    const int k[3] = {x, y, z};
                    const float g = (float)(((double)tw[2 * i] + 1.0) * 0.5);
                    for (int a = 0; a < 3; ++a) {
                        if (keys) keys[3 * cnt + a] = k[a];
                        if (pts) pts[3 * cnt + a] = fmaf(V.vl, (float)(k[a] - V.h), V.half) + o[a];
                        if (cols) cols[3 * cnt + a] = g;
                    }
                }
                ++cnt;
            }
    return cnt;
}

/* InterpolateTrilinearly (UT:447-484): base = (int)p, minus 1 where p < base + 0.5; a = p - (base + 0.5);
 * terms v_k * A * B * C in the source's order, acc = fma((v_k * A) * B, C, acc) */
static float interp(const float *tw, const float p[3], int res) {
    int b[3];
    float a[3];
    for (int i = 0; i < 3; ++i) {
        b[i] = (int)p[i];
        if (p[i] < (float)b[i] + 0.5f) b[i] -= 1;
        a[i] = p[i] - ((float)b[i] + 0.5f);
    }
    float acc = 0.f;
    for (int k = 0; k < 8; ++k) {
        const int dx = (k >> 2) & 1, dy = (k >> 1) & 1, dz = k & 1;
        const float A = dx ? a[0] : 1.f - a[0], B = dy ? a[1] : 1.f - a[1], C = dz ? a[2] : 1.f - a[2];
        acc = fmaf((tw[2 * idx_of(b[0] + dx, b[1] + dy, b[2] + dz, res)] * A) * B, C, acc);
    }
    return acc;
}

/* the camera pose (InverseTransform, eigen.cu:67-73): R^T and fma(-R[2][r], t2, fma(-R[1][r], t1, -R[0][r] * t0)) */
void orc_tsdf_pose(const float E[16], float P[12]) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) P[4 * r + c] = E[4 * c + r];
        P[4 * r + 3] = fmaf(-E[8 + r], E[11], fmaf(-E[4 + r], E[7], -E[r] * E[3]));
    }
}

/* the ray's entry and exit times on the box of the cells the march may sample, [-(res/2) vl, (res - 1 - res/2) vl]^3
 * (origin-relative; cells [0, res - 1) per axis), or 0 when the ray misses it.  A zero direction component keeps the slab when t lies inside it and misses otherwise.  (The
 * reference's GetMinTime / GetMaxTime use [0, length]^3 and divide 0 / 0.) */
static int ray_box(const float t[3], const float d[3], float lo, float hi, float *t0, float *t1) {
    float a = -INFINITY, b = INFINITY;
    for (int i = 0; i < 3; ++i) {
        if (d[i] == 0.f) {
            if (!(t[i] >= lo && t[i] <= hi)) return 0;
            continue;
        }
        const float e = ((d[i] > 0.f ? lo : hi) - t[i]) / d[i], x = ((d[i] > 0.f ? hi : lo) - t[i]) / d[i];
        a = fmaxf(a, e);
        b = fminf(b, x);
    }
    *t0 = a;
    *t1 = b;
    return 1;
}

static int cell(const float t[3], const float d[3], float len, float vl, int res, int h, int lo, int k[3]) {
    for (int a = 0; a < 3; ++a) {
        const float g = floorf(fmaf(d[a], len, t[a]) / vl);
        if (!(g >= (float)(lo - h) && g < (float)(res - 1 - h))) return 0;
        k[a] = (int)g + h;
    }
    return 1;
}

/* raycast_tsdf_functor (UT:509-639) for pixel (x, y).  dir = R * ((x - cx) / fx, (y - cy) / fy, 1) with
 * fma(R[r][2], 1, fma(R[r][1], q1, R[r][0] * q0)), divided by its norm sqrt(fma(z, z, fma(y, y, x * x))); the march
 * starts one voxel past the entry, steps trunc / 2 up to length sqrt(2) further, skips cells outside [1, res - 1)
 * without touching the previous value, stops at a - to + crossing and interpolates a + to - one:
 * t* = len - ((trunc * 0.5) * f_prev) / (f - f_prev), vertex = fma(dir, t*, t), loc = vertex / vl + res / 2; the
 * normal is the central difference of InterpolateTrilinearly at loc -+ 1 per axis, normalised; the colour is the voxel
 * at (int)loc.  A step that no longer advances the ray length ends the march as a miss.  -> 1 with the row, or 0. */
static int ray(const float *tw, const float *col, const Vol *V, long long N, const float P[12], const float K4[4], float trunc, int x,
               int y, float out[9]) {
    const int res = V->res, h = V->h;
    const float length = (float)res * V->vl;
    const float q0 = ((float)x - K4[2]) / K4[0], q1 = ((float)y - K4[3]) / K4[1];
    float d[3], t[3];
    for (int r = 0; r < 3; ++r) d[r] = fmaf(P[4 * r + 2], 1.0f, fmaf(P[4 * r + 1], q1, P[4 * r] * q0));
    const float dn = sqrtf(fmaf(d[2], d[2], fmaf(d[1], d[1], d[0] * d[0])));
    if (dn == 0.f) return 0;
    for (int r = 0; r < 3; ++r) {
        d[r] = d[r] / dn;
        t[r] = P[4 * r + 3] - V->o[r];
    }
    float len, tmax;
    if (!ray_box(t, d, -(float)h * V->vl, (float)(res - 1 - h) * V->vl, &len, &tmax)) return 0;
    len = fmaxf(len, 0.f);
    if (!(len < tmax)) return 0;
    len = len + V->vl;
    int k[3];
    if (!cell(t, d, len, V->vl, res, h, 0, k)) return 0;
    float f = tw[2 * idx_of(k[0], k[1], k[2], res)];
    const float step = trunc * 0.5f;
    const float lim = len + length * sqrtf(2.0f);
    for (; len < lim; len = len + step) {
        if (!(len + step > len)) return 0;
        if (!cell(t, d, len + step, V->vl, res, h, 1, k)) continue;
        const float fp = f;
        f = tw[2 * idx_of(k[0], k[1], k[2], res)];
        if (fp < 0.f && f > 0.f) return 0;
        if (fp > 0.f && f < 0.f) {
            const float ts = len - (step * fp) / (f - fp);
            float vx[3], loc[3], n[3];
            for (int a = 0; a < 3; ++a) {
                vx[a] = fmaf(d[a], ts, t[a]);
                loc[a] = vx[a] / V->vl + (float)h;
                if (!(loc[a] >= 1.f && loc[a] < (float)(res - 1))) return 0;
            }
            for (int a = 0; a < 3; ++a) {
                float s[3] = {loc[0], loc[1], loc[2]};
                s[a] = loc[a] + 1.f;
                if (s[a] >= (float)(res - 1)) return 0;
                const float f1 = interp(tw, s, res);
                s[a] = loc[a] - 1.f;
                if (s[a] < 1.f) return 0;
                n[a] = f1 - interp(tw, s, res);
            }
            const float nn = sqrtf(fmaf(n[2], n[2], fmaf(n[1], n[1], n[0] * n[0])));
            if (nn == 0.f) return 0;
            const long long ci = idx_of((int)loc[0], (int)loc[1], (int)loc[2], res);
            for (int a = 0; a < 3; ++a) {
                out[a] = vx[a] + V->o[a];
                out[3 + a] = n[a] / nn;
                const float c = V->ct == RGB8 ? col[a * N + ci] / 255.0f : V->ct == GRAY32 ? col[ci] : 0.f;
                out[6 + a] = c;
            }
            return 1;
        }
    }
    return 0;
}

/* Raycast (UT:924-951): one row per pixel (row-major), NaN rows for misses; hit[i] = 1 for a hit.  E is the
 * world-to-camera extrinsic. */
void orc_tsdf_raycast(const float *tw, const float *col, float length, int res, int ct, const float o[3], int w, int h,
                      const float K4[4], const float E[16], float trunc, float *pts, float *nrm, float *cols, uint8_t *hit) {
    const Vol V = vol(length, res, trunc, ct, o);
    const long long N = (long long)res * res * res;
    float P[12];
    orc_tsdf_pose(E, P);
#pragma omp parallel for schedule(dynamic, 64)
    for (long long i = 0; i < (long long)w * h; ++i) {
        float r[9];
        const int ok = ray(tw, col, &V, N, P, K4, trunc, (int)(i % w), (int)(i / w), r);
        if (!ok)
            for (int a = 0; a < 9; ++a) r[a] = NAN;
        for (int a = 0; a < 3; ++a) {
            pts[3 * i + a] = r[a];
            nrm[3 * i + a] = r[3 + a];
            cols[3 * i + a] = r[6 + a];
        }
        hit[i] = (uint8_t)ok;
    }
}
