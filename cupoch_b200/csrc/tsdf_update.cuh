// tsdf_update.cuh -- the per-voxel update of TSDF integration (integrate_functor::ComputeTSDF, IF:84-139), shared by
// UniformTSDFVolume (tsdf.cu) and ScalableTSDFVolume (stsdf.cu).  The expression order is oracle/tsdf.c's Integrate.
#pragma once
#include "cphb_internal.cuh"

#define TSDF_NO_COLOR 0
#define TSDF_RGB8 1
#define TSDF_GRAY32 2

struct TsdfCam {
    float E[12];  // world-to-camera rows 0..2
    float S[3];   // vl * E[r][2]
    float fx, fy, cx, cy, fxi, fyi, safe_w, safe_h;
    int w;
};

// the camera point of the voxel column at p (its z = 0 voxel's centre) and z index kz:
// fma(kz, vl E[r][2], fma(E[r][2], p2, fma(E[r][1], p1, E[r][0] p0)) + E[r][3])
__device__ __forceinline__ void tsdf_camera_point(const TsdfCam &c, float p0, float p1, float p2, float kz, float cam[3]) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float b = __fmaf_rn(c.E[4 * r + 2], p2, __fmaf_rn(c.E[4 * r + 1], p1, c.E[4 * r] * p0)) + c.E[4 * r + 3];
        cam[r] = __fmaf_rn(kz, c.S[r], b);
    }
}

// ComputeTSDF from the camera point on: the pixel test, the depth-to-camera-distance multiplier of pixel (u, v)
// (IFC:136-164, computed here instead of read from an image), the truncation and the weighted running means of tsdf
// and colour.  tw = the voxel's {tsdf, weight}; its colour channel k is col[k * plane].
template <int CT>
__device__ __forceinline__ void tsdf_update_voxel(const TsdfCam &c, const float cam[3], const float *__restrict__ depth,
                                                  const void *__restrict__ color, float trunc, float trunc_inv, float2 *tw, float *col,
                                                  size_t plane) {
    if (cam[2] <= 0.f) return;
    const float uf = (cam[0] * c.fx) / cam[2] + c.cx + 0.5f;
    const float vf = (cam[1] * c.fy) / cam[2] + c.cy + 0.5f;
    if (!(uf >= 0.0001f && uf < c.safe_w && vf >= 0.0001f && vf < c.safe_h)) return;
    const int u = __float2int_rd(uf), v = __float2int_rd(vf);
    const size_t px = (size_t)v * c.w + u;
    const float d = __ldg(depth + px);
    if (d <= 0.f) return;
    const float xx = ((float)u - c.cx) * c.fxi, yy = ((float)v - c.cy) * c.fyi;
    const float sdf = (d - cam[2]) * sqrtf(__fmaf_rn(yy, yy, xx * xx) + 1.0f);
    if (!(sdf > -trunc)) return;
    const float t = fminf(1.0f, sdf * trunc_inv);
    const float2 cur = *tw;
    const float w1 = cur.y + 1.0f;
    *tw = make_float2(__fmaf_rn(cur.x, cur.y, t) / w1, w1);
    if (CT == TSDF_RGB8) {
        const uint8_t *rgb = (const uint8_t *)color + 3 * px;
#pragma unroll
        for (int k = 0; k < 3; ++k) col[k * plane] = __fmaf_rn(col[k * plane], cur.y, (float)__ldg(rgb + k)) / w1;
    } else if (CT == TSDF_GRAY32) {
        col[0] = __fmaf_rn(col[0], cur.y, __ldg((const float *)color + px)) / w1;
    }
}

// the reference's Integrate format checks (UT:677-695) and this project's: the depth image must match the intrinsic
static inline bool tsdf_bad_format(int ct, int depth_width, int depth_height, int depth_channels, int depth_bytes, int color_width,
                                   int color_height, int color_channels, int color_bytes, int width, int height) {
    return depth_channels != 1 || depth_bytes != 4 || depth_width != width || depth_height != height ||
           (ct == TSDF_RGB8 && (color_channels != 3 || color_bytes != 1)) ||
           (ct == TSDF_GRAY32 && (color_channels != 1 || color_bytes != 4)) ||
           (ct != TSDF_NO_COLOR && (color_width != width || color_height != height));
}

// the camera of one Integrate: the extrinsic's rows, vl * its third column (extrinsic_scaled_, IF:53), the intrinsic
// and safe_width / safe_height (UT:906-907)
static inline TsdfCam tsdf_cam(float vl, const float K[9], const float E[16], int width, int height) {
    TsdfCam c;
    for (int r = 0; r < 3; ++r) {
        for (int q = 0; q < 4; ++q) c.E[4 * r + q] = E[4 * r + q];
        c.S[r] = vl * E[4 * r + 2];
    }
    c.fx = K[0];
    c.fy = K[4];
    c.cx = K[2];
    c.cy = K[5];
    c.fxi = 1.0f / c.fx;
    c.fyi = 1.0f / c.fy;
    c.safe_w = (float)width - 0.0001f;
    c.safe_h = (float)height - 0.0001f;
    c.w = width;
    return c;
}
