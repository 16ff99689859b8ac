/* depth_cloud.c -- plain-C restatement of PointCloud::CreateFromDepthImage / CreateFromRGBDImage as
 * cupoch_b200/csrc/depth_cloud.cu computes them.  Built by oracle.build("depth_cloud"); loader depth_cloud_py.py.
 *
 * Every float operation is rounded on its own (-ffp-contract=off) except where fmaf() states a fused multiply-add, in
 * the order the kernel uses __fmaf_rn.  Line numbers cite the reference's geometry/pointcloud_factory.cu (PF) and
 * geometry/image.cu (IM). */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct {
    float P[12]; /* camera pose = extrinsic^-1, rows 0..2 */
    float fx, fy, cx, cy, cutoff;
    int w, sw, sh, stride, bytes, scale_i, trunc_i;
    const void *depth;
} Cam;

/* the inverse of the row-major extrinsic E by Gauss-Jordan elimination with partial pivoting in double, rows 0..2
 * rounded to float.  -> 0 for a singular or non-finite result */
int orc_depth_cloud_pose(const float E[16], float P[12]) {
    double a[4][8];
    for (int r = 0; r < 4; ++r)
        for (int q = 0; q < 4; ++q) {
            a[r][q] = (double)E[4 * r + q];
            a[r][4 + q] = r == q ? 1.0 : 0.0;
        }
    for (int q = 0; q < 4; ++q) {
        int piv = q;
        for (int r = q + 1; r < 4; ++r)
            if (fabs(a[r][q]) > fabs(a[piv][q])) piv = r;
        if (!(fabs(a[piv][q]) > 0.0)) return 0;
        for (int k = 0; k < 8; ++k) {
            const double t = a[q][k];
            a[q][k] = a[piv][k];
            a[piv][k] = t;
        }
        const double d = a[q][q];
        for (int k = 0; k < 8; ++k) a[q][k] = a[q][k] / d;
        for (int r = 0; r < 4; ++r) {
            if (r == q) continue;
            const double f = a[r][q];
            for (int k = 0; k < 8; ++k) a[r][k] = a[r][k] - f * a[q][k];
        }
    }
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 4; ++q) {
            P[4 * r + q] = (float)a[r][4 + q];
            if (!isfinite(P[4 * r + q])) return 0;
        }
    return 1;
}

/* a float32 depth as it is; uint16 by ConvertDepthToFloatImage (IM:339-348): raw / (float)scale_i, 0 where >= (float)trunc_i */
static float depth_at(const Cam *c, int row, int col) {
    const long long k = (long long)row * c->w + col;
    if (c->bytes == 4) return ((const float *)c->depth)[k];
    const float g = (float)((const uint16_t *)c->depth)[k] / (float)c->scale_i;
    return g >= (float)c->trunc_i ? 0.f : g;
}

/* PF:64-80, 132-145: x = ((col - cx) z) / fx, y alike, p_r = fma(P[r][2], z, fma(P[r][1], y, P[r][0] x)) + P[r][3];
 * a point only for d > 0, below a positive cutoff, with a finite result (RemoveNoneFinitePoints) */
static int point_at(const Cam *c, int sr, int sc, float p[3]) {
    const int row = sr * c->stride, col = sc * c->stride;
    const float z = depth_at(c, row, col);
    if (!(z > 0.f)) return 0;
    if (c->cutoff > 0.f && !(c->cutoff > z)) return 0;
    const float x = (((float)col - c->cx) * z) / c->fx;
    const float y = (((float)row - c->cy) * z) / c->fy;
    for (int r = 0; r < 3; ++r) p[r] = fmaf(c->P[4 * r + 2], z, fmaf(c->P[4 * r + 1], y, c->P[4 * r] * x)) + c->P[4 * r + 3];
    return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
}

/* the structured normal (PF:160-200), every border row and column 0: (left - right) x (up - down), a neighbour
 * without a point as 0, component r = fma(h[a], v[b], -(h[b] v[a])), / sqrtf(fma(n2, n2, fma(n1, n1, n0 n0))),
 * negated when z > 0; a zero cross product stays 0 */
static void normal_at(const Cam *c, int sr, int sc, float n[3]) {
    n[0] = n[1] = n[2] = 0.f;
    if (sr < 1 || sc < 1 || sr >= c->sh - 1 || sc >= c->sw - 1) return;
    float q[4][3];
    const int nb[4][2] = {{sr, sc - 1}, {sr, sc + 1}, {sr - 1, sc}, {sr + 1, sc}};
    for (int k = 0; k < 4; ++k)
        if (!point_at(c, nb[k][0], nb[k][1], q[k])) q[k][0] = q[k][1] = q[k][2] = 0.f;
    float h[3], v[3];
    for (int a = 0; a < 3; ++a) {
        h[a] = q[0][a] - q[1][a];
        v[a] = q[2][a] - q[3][a];
    }
    const float m[3] = {fmaf(h[1], v[2], -(h[2] * v[1])), fmaf(h[2], v[0], -(h[0] * v[2])), fmaf(h[0], v[1], -(h[1] * v[0]))};
    const float len = sqrtf(fmaf(m[2], m[2], fmaf(m[1], m[1], m[0] * m[0])));
    if (len == 0.f) return;
    for (int a = 0; a < 3; ++a) n[a] = m[a] / len;
    if (n[2] > 0.f)
        for (int a = 0; a < 3; ++a) n[a] = -n[a];
}

/* depth: [height][width] uint16 (bytes 2) or float32 (bytes 4); color: NULL, uint8 [h][w][3] (ct 1) or float32 [h][w]
 * (ct 2).  Writes the rows (pixel order; with valid_only only the samples with a point, else NaN rows for the others)
 * when out != NULL -> the row count, or -1 for a singular extrinsic */
long long orc_depth_to_points(const void *depth, int width, int height, int bytes, int scale_i, int trunc_i, int stride, const void *color,
                              int ct, const float K4[4], const float E[16], float cutoff, int normals, int valid_only, float *pts,
                              float *nrm, float *cols) {
    Cam c;
    if (!orc_depth_cloud_pose(E, c.P)) return -1;
    c.fx = K4[0];
    c.fy = K4[1];
    c.cx = K4[2];
    c.cy = K4[3];
    c.cutoff = cutoff;
    c.w = width;
    c.stride = stride;
    c.sw = width / stride;
    c.sh = height / stride;
    c.bytes = bytes;
    c.scale_i = scale_i;
    c.trunc_i = trunc_i;
    c.depth = depth;
    const float nan = nanf("");
    long long row = 0;
    for (int sr = 0; sr < c.sh; ++sr)
        for (int sc = 0; sc < c.sw; ++sc) {
            float p[3], n[3] = {nan, nan, nan}, col[3] = {nan, nan, nan};
            const int ok = point_at(&c, sr, sc, p);
            if (!ok && valid_only) continue;
            if (ok) {
                if (normals) normal_at(&c, sr, sc, n);
                const long long px = (long long)(sr * stride) * width + (long long)(sc * stride);
                if (ct == 1)
                    for (int a = 0; a < 3; ++a) col[a] = (float)((const uint8_t *)color)[3 * px + a] / 255.0f;
                else if (ct == 2)
                    col[0] = col[1] = col[2] = ((const float *)color)[px];
            } else {
                p[0] = p[1] = p[2] = nan;
            }
            if (pts) {
                memcpy(pts + 3 * row, p, 12);
                if (normals) memcpy(nrm + 3 * row, n, 12);
                if (ct) memcpy(cols + 3 * row, col, 12);
            }
            ++row;
        }
    return row;
}
