// depth_project.cuh -- the back-projection of a depth image that PointCloud::CreateFromDepthImage / CreateFromRGBDImage
// (depth_cloud.cu) and ScalableTSDFVolume::Integrate's unit discovery (stsdf.cu) share, so that the two cannot drift
// apart.  Reference: geometry/pointcloud_factory.cu (PF), geometry/image.cu (IM).  The expression order is
// oracle/depth_cloud.c's.
#pragma once
#include <math.h>

#include "cphb_internal.cuh"

struct DepthCam {
    float P[12];  // camera pose = extrinsic^-1 (float64, rounded), rows 0..2
    float fx, fy, cx, cy, cutoff;
    int w, sw, sh, stride, bytes, scale_i, trunc_i;
};

// the depth of pixel (row, col) in metres: a float32 image as it is; a uint16 one by ConvertDepthToFloatImage's rule
// (raw / (float)int(depth_scale), 0 where that is >= (float)int(depth_trunc))
__device__ __forceinline__ float dc_depth(const void *depth, const DepthCam &c, int row, int col) {
    const size_t k = (size_t)row * c.w + col;
    if (c.bytes == 4) return __ldg((const float *)depth + k);
    float g = (float)__ldg((const uint16_t *)depth + k) / (float)c.scale_i;
    return g >= (float)c.trunc_i ? 0.f : g;
}

// the point of sampled pixel (sr, sc) (PF:64-80, 132-145): z = d, x = ((col - cx) z) / fx, y alike, then the pose
// p_r = fma(P[r][2], z, fma(P[r][1], y, P[r][0] x)) + P[r][3].  -> whether it has one: d > 0, d below a positive
// cutoff, and a finite result (the reference drops non-finite rows with RemoveNoneFinitePoints)
__device__ __forceinline__ bool dc_point(const void *depth, const DepthCam &c, int sr, int sc, float p[3]) {
    const int row = sr * c.stride, col = sc * c.stride;
    const float z = dc_depth(depth, c, row, col);
    if (!(z > 0.f)) return false;
    if (c.cutoff > 0.f && !(c.cutoff > z)) return false;
    const float x = (((float)col - c.cx) * z) / c.fx;
    const float y = (((float)row - c.cy) * z) / c.fy;
#pragma unroll
    for (int r = 0; r < 3; ++r) p[r] = __fmaf_rn(c.P[4 * r + 2], z, __fmaf_rn(c.P[4 * r + 1], y, c.P[4 * r] * x)) + c.P[4 * r + 3];
    return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
}

// the camera pose: the inverse of the row-major extrinsic by Gauss-Jordan elimination with partial pivoting in
// float64, rounded to float32 (oracle/depth_cloud.c's pose()).  -> false for a singular or non-finite result.
static inline bool dc_pose(const float E[16], float P[12]) {
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
        if (!(fabs(a[piv][q]) > 0.0)) return false;
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
            if (!isfinite(P[4 * r + q])) return false;
        }
    return true;
}
