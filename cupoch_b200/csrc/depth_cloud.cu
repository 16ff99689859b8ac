// depth_cloud.cu -- PointCloud::CreateFromDepthImage and CreateFromRGBDImage (SURVEY 8f row 15; DESIGN section 4 item
// 20).  Reference: geometry/pointcloud_factory.cu (PF).
//
// One thread per sampled pixel.  With project_valid_depth_only the valid rows are compacted in pixel order by the
// engine's block compaction (a count kernel, the shared block-count scan, a writing kernel that recomputes the point);
// otherwise every sampled pixel writes its own row.  A uint16 depth image is converted inside the projection, by the
// rule of cphb_rgbd_convert's to_depth, so no float image is written first.
//
// The projection itself (dc_point) is depth_project.cuh's, shared with ScalableTSDFVolume::Integrate.
//
// Arithmetic: IEEE (build.py compiles with -fmad=false and without fast-math, so every + - * / and sqrtf below is
// rounded on its own); every fused multiply-add is an explicit __fmaf_rn, in the order oracle/depth_cloud.c states with
// fmaf().
#include <math.h>

#include "depth_project.cuh"

#define DC_BLOCK 256
#define DC_NO_COLOR 0
#define DC_RGB8 1
#define DC_GRAY32 2

static int dc_invalid(const char *what) {
    cphb_set_error("cphb_depth_to_points: %s", what);
    return CPHB_ERR_INVALID;
}

// a neighbour's point, zero when it has none
__device__ __forceinline__ void dc_neighbour(const void *depth, const DepthCam &c, int sr, int sc, float q[3]) {
    if (!dc_point(depth, c, sr, sc, q)) q[0] = q[1] = q[2] = 0.f;
}

// the structured normal (PF:160-200) of an interior sample: hor = left - right, ver = up - down, n = hor x ver with
// each component fma(a, b, -(c d)), divided by sqrt(fma(n2, n2, fma(n1, n1, n0 n0))) and negated when n.z > 0.  A
// sample on any border row or column, or a zero cross product, gets (0, 0, 0).
__device__ __forceinline__ void dc_normal(const void *depth, const DepthCam &c, int sr, int sc, float n[3]) {
    n[0] = n[1] = n[2] = 0.f;
    if (sr < 1 || sc < 1 || sr >= c.sh - 1 || sc >= c.sw - 1) return;
    float l[3], r[3], u[3], d[3], hor[3], ver[3];
    dc_neighbour(depth, c, sr, sc - 1, l);
    dc_neighbour(depth, c, sr, sc + 1, r);
    dc_neighbour(depth, c, sr - 1, sc, u);
    dc_neighbour(depth, c, sr + 1, sc, d);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        hor[a] = l[a] - r[a];
        ver[a] = u[a] - d[a];
    }
    const float m[3] = {__fmaf_rn(hor[1], ver[2], -(hor[2] * ver[1])), __fmaf_rn(hor[2], ver[0], -(hor[0] * ver[2])),
                        __fmaf_rn(hor[0], ver[1], -(hor[1] * ver[0]))};
    const float len = sqrtf(__fmaf_rn(m[2], m[2], __fmaf_rn(m[1], m[1], m[0] * m[0])));
    if (len == 0.f) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) n[a] = m[a] / len;
    if (n[2] > 0.f) {
#pragma unroll
        for (int a = 0; a < 3; ++a) n[a] = -n[a];
    }
}

__global__ void __launch_bounds__(DC_BLOCK) dc_count_kernel(const void *__restrict__ depth, const DepthCam c, unsigned *__restrict__ counts) {
    const unsigned i = blockIdx.x * DC_BLOCK + threadIdx.x;
    const unsigned n = (unsigned)c.sw * (unsigned)c.sh;
    float p[3];
    const bool v = i < n && dc_point(depth, c, (int)(i / (unsigned)c.sw), (int)(i % (unsigned)c.sw), p);
    const unsigned k = block_flag_count(v);
    if (threadIdx.x == 0) counts[blockIdx.x] = k;
}

// the rows of a block's samples: at offsets[block] + rank among its valid samples when offsets is given, else at the
// sample's own index (a sample without a point writes NaN in every attribute)
template <int CT>
__global__ void __launch_bounds__(DC_BLOCK) dc_write_kernel(const void *__restrict__ depth, const void *__restrict__ color, const DepthCam c,
                                                            int want_normals, const unsigned *__restrict__ offsets, float *__restrict__ pts,
                                                            float *__restrict__ nrm, float *__restrict__ cols) {
    const unsigned i = blockIdx.x * DC_BLOCK + threadIdx.x;
    const unsigned n = (unsigned)c.sw * (unsigned)c.sh;
    const int sr = (int)(i / (unsigned)c.sw), sc = (int)(i % (unsigned)c.sw);
    float p[3];
    const bool v = i < n && dc_point(depth, c, sr, sc, p);
    size_t row = i;
    if (offsets) {
        const unsigned r = block_flag_rank(v);
        if (!v) return;
        row = (size_t)offsets[blockIdx.x] + r;
    } else if (i >= n) {
        return;
    }
    const float nan = __int_as_float(0x7fc00000);
    float nv[3] = {nan, nan, nan}, cv[3] = {nan, nan, nan};
    if (v) {
        if (want_normals) dc_normal(depth, c, sr, sc, nv);
        const size_t px = (size_t)(sr * c.stride) * c.w + (size_t)(sc * c.stride);
        if (CT == DC_RGB8) {
#pragma unroll
            for (int a = 0; a < 3; ++a) cv[a] = (float)__ldg((const uint8_t *)color + 3 * px + a) / 255.0f;
        } else if (CT == DC_GRAY32) {
            cv[0] = cv[1] = cv[2] = __ldg((const float *)color + px);
        }
    } else {
        p[0] = p[1] = p[2] = nan;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        pts[3 * row + a] = p[a];
        if (want_normals) nrm[3 * row + a] = nv[a];
        if (CT != DC_NO_COLOR) cols[3 * row + a] = cv[a];
    }
}

extern "C" int cphb_depth_to_points(const void *depth, int width, int height, int depth_channels, int depth_bytes_per_channel,
                                    float depth_scale, float depth_trunc, int stride, const void *color, int color_width,
                                    int color_height, int color_channels, int color_bytes_per_channel, const float h_intrinsic[9],
                                    const float h_extrinsic[16], float depth_cutoff, int compute_normals, int project_valid_depth_only,
                                    float *points, float *normals, float *colors, size_t capacity, size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_intrinsic || !h_extrinsic || !h_count) return dc_invalid("null argument");
    *h_count = 0;
    if (depth_channels != 1 || (depth_bytes_per_channel != 2 && depth_bytes_per_channel != 4))
        return dc_invalid("[PointCloud::CreateFromDepthImage] Unsupported image format.");
    int ct = DC_NO_COLOR;
    if (color) {
        if (color_channels == 3 && color_bytes_per_channel == 1)
            ct = DC_RGB8;
        else if (color_channels == 1 && color_bytes_per_channel == 4)
            ct = DC_GRAY32;
        else
            return dc_invalid("[PointCloud::CreateFromRGBDImage] Unsupported image format.");
        if (color_width != width || color_height != height) return dc_invalid("the colour and depth images differ in size");
    }
    if (width < 0 || height < 0) return dc_invalid("negative image size");
    if (stride < 1) return dc_invalid("stride is not positive");
    if (isnan(depth_cutoff)) return dc_invalid("depth_cutoff is NaN");
    DepthCam c;
    c.bytes = depth_bytes_per_channel;
    c.scale_i = 1;
    c.trunc_i = 0;
    if (c.bytes == 2) {  // the depth_to_float functor takes both as int (IM:339-348); a scale that truncates to 0 would divide by zero
        if (!(depth_scale >= 1.f && depth_scale < 2147483648.f)) return dc_invalid("depth_scale is not in [1, 2^31)");
        if (!(depth_trunc > -2147483648.f && depth_trunc < 2147483648.f)) return dc_invalid("depth_trunc is not finite or outside int range");
        c.scale_i = (int)depth_scale;
        c.trunc_i = (int)depth_trunc;
    }
    if (!dc_pose(h_extrinsic, c.P)) return dc_invalid("the extrinsic is not invertible");
    c.fx = h_intrinsic[0];
    c.fy = h_intrinsic[4];
    c.cx = h_intrinsic[2];
    c.cy = h_intrinsic[5];
    c.cutoff = depth_cutoff;
    c.w = width;
    c.stride = stride;
    c.sw = width / stride;
    c.sh = height / stride;
    const size_t n = (size_t)c.sw * (size_t)c.sh;
    if (n > (size_t)INT32_MAX) return dc_invalid("more than 2^31-1 sampled pixels");
    if (n == 0) return CPHB_OK;
    if (!depth) return dc_invalid("null image");
    const unsigned nb = (unsigned)((n + DC_BLOCK - 1) / DC_BLOCK);
    cphb_scratch sc(s);
    unsigned *counts = nullptr, *total = nullptr;
    size_t m = n;
    if (project_valid_depth_only) {
        int rc = sc.alloc(&counts, (size_t)nb);
        if (!rc) rc = sc.alloc(&total, 1);
        if (rc) return rc;
        CPHB_LAUNCH(dc_count_kernel, nb, DC_BLOCK, 0, s, depth, c, counts);
        cphb_scan_block_counts(counts, nb, total, s);
        unsigned h = 0;
        rc = cphb_read_back(&h, total, sizeof(h), s, "cphb_depth_to_points");
        if (rc) return rc;
        m = h;
    }
    if (m && capacity >= m) {
        if (!points || (compute_normals && !normals) || (ct != DC_NO_COLOR && !colors)) return dc_invalid("null output");
        const int wn = compute_normals ? 1 : 0;
#define DC_WRITE(CT) CPHB_LAUNCH(dc_write_kernel<CT>, nb, DC_BLOCK, 0, s, depth, color, c, wn, counts, points, normals, colors)
        if (ct == DC_RGB8)
            DC_WRITE(DC_RGB8);
        else if (ct == DC_GRAY32)
            DC_WRITE(DC_GRAY32);
        else
            DC_WRITE(DC_NO_COLOR);
#undef DC_WRITE
    }
    const int rc = cphb_read_back(nullptr, nullptr, 0, s, "cphb_depth_to_points");
    if (!rc) *h_count = m;
    return rc;
}
