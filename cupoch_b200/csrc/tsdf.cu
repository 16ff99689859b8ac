// tsdf.cu -- integration::UniformTSDFVolume and the RGB-D conversion it reads (SURVEY 8f row 13; DESIGN section 4 item
// 18).  Reference: integration/{integrate_functor.h (IF), uniform_tsdfvolume.cu (UT)}, geometry/image.cu (IM) and
// image_factory.cu (IFC).
//
// Layout: one float2 {tsdf, weight} plane (one 8-byte load and store per voxel) and colour planes only when the volume
// has colour: three float planes for RGB8, one for Gray32 (its three channels are always equal).  Voxel
// idx = x res^2 + y res + z.  Integrate is one thread per voxel with z fastest; a voxel that skips touches no voxel
// memory, and no two threads share a voxel, so there are no atomics.  The extractions are a flag kernel (one byte per
// voxel), the stable compaction cphb_compact_flags and a writing kernel; ExtractPointCloud adds one exclusive CUB scan
// of the flag popcounts over the compacted voxels.  Raycast is one thread per pixel on 8x4-pixel warp tiles.
//
// Arithmetic: IEEE (build.py compiles with -fmad=false and without fast-math, so every + - * / and sqrtf below is
// rounded on its own); every fused multiply-add is an explicit __fmaf_rn, in the order oracle/tsdf.c states with fmaf().
#include <math.h>

#include <cub/device/device_scan.cuh>
#include <memory>

#include "tsdf_update.cuh"

#define TSDF_MAX_RES 1290  // res^3 <= 2^31 - 1: cphb_compact_flags writes int32 positions

struct cphb_tsdf {
    float length, vl, half, trunc, trunc_inv, o[3];
    int res, h, ct, planes;
    size_t n;
    float2 *tw = nullptr;  // {tsdf, weight}[n]
    float *col = nullptr;  // [planes][n]
    cphb_arena arena;
};

static int tsdf_invalid(const char *who, const char *what) {
    cphb_set_error("%s: %s", who, what);
    return CPHB_ERR_INVALID;
}
static unsigned tsdf_blocks(size_t n, unsigned b) { return n ? (unsigned)((n + b - 1) / b) : 1u; }

__device__ __forceinline__ size_t tsdf_idx(int x, int y, int z, int res) { return ((size_t)x * res + y) * res + z; }

// 32 z x 8 y voxels per block: each warp covers 32 consecutive voxels of one column
static dim3 tsdf_vox_grid(int res) { return dim3((unsigned)((res + 31) / 32), (unsigned)((res + 7) / 8), (unsigned)res); }
static const dim3 TSDF_VOX_BLOCK(32, 8);

// ------------------------------------------------------------------------------------------------ RGB-D conversion
__device__ __forceinline__ float tsdf_raw(const void *src, int bytes, size_t k) {
    return bytes == 1 ? (float)__ldg((const uint8_t *)src + k)
                      : bytes == 2 ? (float)__ldg((const uint16_t *)src + k) : __ldg((const float *)src + k);
}

// to_depth: ConvertDepthToFloatImage (IM:339-348, 413-421) -- CreateFloatImage's value, / (float)scale_i, 0 where it is
// >= (float)trunc_i.  Otherwise CreateFloatImage(WEIGHTED) (IFC:54-118, 201-224): 1 channel v * denom, 3 channels
// fma(0.1140, p2, fma(0.5870, p1, 0.2990 * p0)) * denom; denom = 1/255 for 8-bit input, 1 otherwise.
__global__ void __launch_bounds__(256) rgbd_convert_kernel(const void *__restrict__ src, size_t n, int channels, int bytes, int to_depth,
                                                           int scale_i, int trunc_i, float *__restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float denom = bytes == 1 ? (float)(1.0 / 255.0) : 1.f;
    float g;
    if (channels == 1) {
        g = tsdf_raw(src, bytes, i);
    } else {
        const float p0 = tsdf_raw(src, bytes, 3 * i), p1 = tsdf_raw(src, bytes, 3 * i + 1), p2 = tsdf_raw(src, bytes, 3 * i + 2);
        g = __fmaf_rn(0.1140f, p2, __fmaf_rn(0.5870f, p1, 0.2990f * p0));
    }
    g = g * denom;
    if (to_depth) {
        g = g / (float)scale_i;
        if (g >= (float)trunc_i) g = 0.f;
    }
    out[i] = g;
}

extern "C" int cphb_rgbd_convert(const void *src, int width, int height, int channels, int bytes_per_channel, int to_depth,
                                 float depth_scale, float depth_trunc, float *out, void *stream) {
    const char *who = "cphb_rgbd_convert";
    if (width < 0 || height < 0) return tsdf_invalid(who, "negative image size");
    const size_t n = (size_t)width * height;
    if (n && (!src || !out)) return tsdf_invalid(who, "null argument");
    if (bytes_per_channel != 1 && bytes_per_channel != 2 && bytes_per_channel != 4)
        return tsdf_invalid(who, "bytes_per_channel is not 1, 2 or 4");
    if (channels != 1 && (to_depth || channels != 3)) return tsdf_invalid(who, to_depth ? "a depth image has one channel" : "an image to convert to intensity has 1 or 3 channels");
    int scale_i = 1, trunc_i = 0;
    if (to_depth) {
        // depth_to_float_functor takes both as int (IM:339-348); a scale that truncates to 0 would divide by zero
        if (!(depth_scale >= 1.f && depth_scale < 2147483648.f)) return tsdf_invalid(who, "depth_scale is not in [1, 2^31)");
        if (!(depth_trunc > -2147483648.f && depth_trunc < 2147483648.f)) return tsdf_invalid(who, "depth_trunc is not finite or outside int range");
        scale_i = (int)depth_scale;
        trunc_i = (int)depth_trunc;
    }
    if (n == 0) return CPHB_OK;
    CPHB_LAUNCH(rgbd_convert_kernel, tsdf_blocks(n, 256), 256, 0, stream, src, n, channels, bytes_per_channel, to_depth ? 1 : 0, scale_i,
                trunc_i, out);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// ------------------------------------------------------------------------------------------------ the handle
__global__ void __launch_bounds__(256) tsdf_reset_kernel(float2 *__restrict__ tw, float *__restrict__ col, size_t n, int planes) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        tw[i] = make_float2(0.f, 0.f);
        for (int c = 0; c < planes; ++c) col[c * n + i] = 1.f;
    }
}

static int tsdf_reset(cphb_tsdf *v, cudaStream_t s) {
    CPHB_LAUNCH(tsdf_reset_kernel, (unsigned)min((size_t)CPHB_SMS * 8, (v->n + 255) / 256), 256, 0, s, v->tw, v->col, v->n, v->planes);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

extern "C" int cphb_tsdf_create(float length, int resolution, float sdf_trunc, int color_type, const float origin[3], void *stream,
                                cphb_tsdf **out) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_create";
    if (!out) return tsdf_invalid(who, "null argument");
    *out = nullptr;
    if (resolution < 2 || resolution > TSDF_MAX_RES) {
        cphb_set_error("%s: resolution %d outside [2, %d] (the voxel count must fit int32)", who, resolution, TSDF_MAX_RES);
        return CPHB_ERR_INVALID;
    }
    if (!(isfinite(length) && length > 0.f)) return tsdf_invalid(who, "length is not positive and finite");
    if (!(isfinite(sdf_trunc) && sdf_trunc > 0.f)) return tsdf_invalid(who, "sdf_trunc is not positive and finite");
    if (color_type < TSDF_NO_COLOR || color_type > TSDF_GRAY32) return tsdf_invalid(who, "unknown color_type");
    std::unique_ptr<cphb_tsdf> v(new cphb_tsdf());
    v->length = length;
    v->res = resolution;
    v->h = resolution / 2;
    v->vl = length / (float)resolution;  // TSDFVolume(length / (float)resolution, ...) (UT:650)
    if (!(v->vl > 0.f)) return tsdf_invalid(who, "length / resolution underflows to 0");
    v->half = 0.5f * v->vl;
    v->trunc = sdf_trunc;
    v->trunc_inv = (float)(1.0 / (double)sdf_trunc);  // sdf_trunc_inv_(1.0 / sdf_trunc) (IF:52)
    v->ct = color_type;
    v->planes = color_type == TSDF_RGB8 ? 3 : color_type == TSDF_GRAY32 ? 1 : 0;
    for (int a = 0; a < 3; ++a) v->o[a] = origin ? origin[a] : 0.f;
    v->n = (size_t)resolution * resolution * resolution;
    v->arena.slice(&v->tw, v->n);
    v->arena.slice(&v->col, v->n * v->planes, v->planes > 0);
    int rc = v->arena.alloc(s);
    if (!rc) rc = tsdf_reset(v.get(), s);
    if (rc) return rc;
    *out = v.release();
    return CPHB_OK;
}

extern "C" void cphb_tsdf_destroy(cphb_tsdf *v) { delete v; }

// Reset: every voxel back to its initial state (the reference clears the vector, after which every Extract* reads an
// empty buffer, UT:668)
extern "C" int cphb_tsdf_reset(cphb_tsdf *v, void *stream) {
    if (!v) return tsdf_invalid("cphb_tsdf_reset", "null volume");
    return tsdf_reset(v, (cudaStream_t)stream);
}

extern "C" int cphb_tsdf_data(const cphb_tsdf *v, float **tw, float **col) {
    if (!v || !tw || !col) return tsdf_invalid("cphb_tsdf_data", "null argument");
    *tw = (float *)v->tw;
    *col = v->col;
    return CPHB_OK;
}

// ------------------------------------------------------------------------------------------------ Integrate
// uniform_integrate_functor (IF:84-139, 182-190); the expression order is oracle/tsdf.c's Integrate
template <int CT>
__global__ void __launch_bounds__(256) tsdf_integrate_kernel(float2 *__restrict__ tw, float *__restrict__ col, size_t n, int res, int h,
                                                             float vl, float half, float ox, float oy, float oz, float trunc,
                                                             float trunc_inv, const TsdfCam c, const float *__restrict__ depth,
                                                             const void *__restrict__ color) {
    const int z = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, x = blockIdx.z;
    if (z >= res || y >= res) return;
    const float p0 = __fmaf_rn(vl, (float)(x - h), half) + ox;
    const float p1 = __fmaf_rn(vl, (float)(y - h), half) + oy;
    const float p2 = half + oz;
    const float kz = (float)(z - h);
    float cam[3];
    tsdf_camera_point(c, p0, p1, p2, kz, cam);
    const size_t i = tsdf_idx(x, y, z, res);
    tsdf_update_voxel<CT>(c, cam, depth, color, trunc, trunc_inv, tw + i, col + i, n);
}

// the reference's format checks (UT:677-695) and this project's: the depth image must match the intrinsic too
extern "C" int cphb_tsdf_integrate(cphb_tsdf *v, const float *depth, int depth_width, int depth_height, int depth_channels,
                                   int depth_bytes_per_channel, const void *color, int color_width, int color_height,
                                   int color_channels, int color_bytes_per_channel, int width, int height, const float h_intrinsic[9],
                                   const float h_extrinsic[16], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_integrate";
    if (!v || !h_intrinsic || !h_extrinsic) return tsdf_invalid(who, "null argument");
    const bool bad = tsdf_bad_format(v->ct, depth_width, depth_height, depth_channels, depth_bytes_per_channel, color_width, color_height,
                                     color_channels, color_bytes_per_channel, width, height);
    if (bad) return tsdf_invalid(who, "[UniformTSDFVolume::Integrate] Unsupported image format.");
    if (width <= 0 || height <= 0) return tsdf_invalid(who, "the intrinsic's image size is not positive");
    if (!depth || (v->ct != TSDF_NO_COLOR && !color)) return tsdf_invalid(who, "null image");
    const TsdfCam c = tsdf_cam(v->vl, h_intrinsic, h_extrinsic, width, height);
    const dim3 g = tsdf_vox_grid(v->res);
#define TSDF_INTEGRATE(CT)                                                                                                        \
    CPHB_LAUNCH(tsdf_integrate_kernel<CT>, g, TSDF_VOX_BLOCK, 0, s, v->tw, v->col, v->n, v->res, v->h, v->vl, v->half, v->o[0], v->o[1], \
                v->o[2], v->trunc, v->trunc_inv, c, depth, color)
    if (v->ct == TSDF_RGB8)
        TSDF_INTEGRATE(TSDF_RGB8);
    else if (v->ct == TSDF_GRAY32)
        TSDF_INTEGRATE(TSDF_GRAY32);
    else
        TSDF_INTEGRATE(TSDF_NO_COLOR);
#undef TSDF_INTEGRATE
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// ------------------------------------------------------------------------------------------------ extraction
__device__ __forceinline__ bool tsdf_band(float2 v) { return v.y != 0.0f && v.x < 0.98f && v.x >= -0.98f; }

// mode 0: bit i set when interior voxel (x, y, z) emits ExtractPointCloud's point on axis i (UT:104-140);
// mode 1: 1 for a band voxel (the voxel extractions, UT:352-408)
__global__ void __launch_bounds__(256) tsdf_flag_kernel(const float2 *__restrict__ tw, int res, int mode, uint8_t *__restrict__ flags) {
    const int z = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, x = blockIdx.z;
    if (z >= res || y >= res) return;
    const size_t i0 = tsdf_idx(x, y, z, res);
    const float2 v0 = tw[i0];
    uint8_t m = 0;
    if (mode == 1) {
        m = tsdf_band(v0) ? 1 : 0;
    } else if (x >= 1 && y >= 1 && z >= 1 && x <= res - 2 && y <= res - 2 && z <= res - 2 && tsdf_band(v0)) {
        const int k[3] = {x, y, z};
        const size_t stride[3] = {(size_t)res * res, (size_t)res, 1};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (k[a] + 1 >= res - 1) continue;
            const float2 v1 = tw[i0 + stride[a]];
            if (tsdf_band(v1) && v0.x * v1.x < 0.f) m |= (uint8_t)(1 << a);
        }
    }
    flags[i0] = m;
}

__global__ void __launch_bounds__(256) tsdf_popc_kernel(const int32_t *__restrict__ pos, size_t m, const uint8_t *__restrict__ flags,
                                                        unsigned long long *__restrict__ cnt) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j < m) cnt[j] = (unsigned long long)__popc(flags[pos[j]]);
    if (j == m) cnt[j] = 0ull;  // the scan runs over m + 1 entries: its last output is the total
}

// GetTSDFAt (UT:36-65): g = p / vl - 0.5, base floor(g), r = g - base; acc = fma((wx * wy) * wz, tsdf, acc) over the
// 8 corners in the source's order
__device__ float tsdf_at(const float2 *__restrict__ tw, const float p[3], float vl, int res) {
    int b[3];
    float r[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float g = p[a] / vl - 0.5f;
        b[a] = (int)floorf(g);
        r[a] = g - (float)b[a];
    }
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int dx = (k >> 2) & 1, dy = (k >> 1) & 1, dz = k & 1;
        const float wx = dx ? r[0] : 1.f - r[0], wy = dy ? r[1] : 1.f - r[1], wz = dz ? r[2] : 1.f - r[2];
        acc = __fmaf_rn((wx * wy) * wz, tw[tsdf_idx(b[0] + dx, b[1] + dy, b[2] + dz, res)].x, acc);
    }
    return acc;
}

// ExtractPointCloud's rows of compacted voxel j (UT:85-156), at out rows off[j] ...; the expression order is
// oracle/tsdf.c's ExtractPointCloud
template <int CT>
__global__ void __launch_bounds__(128) tsdf_points_kernel(const float2 *__restrict__ tw, const float *__restrict__ col, size_t n, int res,
                                                          float vl, float half, float hres, float ox, float oy, float oz,
                                                          const int32_t *__restrict__ pos, size_t m, const uint8_t *__restrict__ flags,
                                                          const unsigned long long *__restrict__ off, float *__restrict__ pts,
                                                          float *__restrict__ nrm, float *__restrict__ cols) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const size_t i0 = (size_t)pos[j];
    const int mask = flags[i0];
    const size_t rr = (size_t)res * res;
    const int k[3] = {(int)(i0 / rr), (int)((i0 / res) % res), (int)(i0 % res)};
    const size_t stride[3] = {rr, (size_t)res, 1};
    const float o[3] = {ox, oy, oz};
    size_t row = off[j];
    const float f0 = tw[i0].x;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (!(mask >> i & 1)) continue;
        const size_t i1 = i0 + stride[i];
        const float r0 = fabsf(f0), r1 = fabsf(tw[i1].x), rs = r0 + r1;
        float p[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) p[a] = __fmaf_rn(vl, (float)k[a], half);
        const float p1i = p[i] + vl;
        p[i] = __fmaf_rn(p1i, r0, p[i] * r1) / rs;
#pragma unroll
        for (int a = 0; a < 3; ++a) pts[3 * row + a] = (p[a] + o[a]) - hres;
        // GetNormalAt (UT:67-83): half_gap is a double; Eigen's normalized() leaves a zero vector unchanged
        const double half_gap = 0.99 * (double)vl;
        float nv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float q0[3] = {p[0], p[1], p[2]}, q1[3] = {p[0], p[1], p[2]};
            q0[a] = (float)((double)p[a] - half_gap);
            q1[a] = (float)((double)p[a] + half_gap);
            nv[a] = tsdf_at(tw, q1, vl, res) - tsdf_at(tw, q0, vl, res);
        }
        const float sq = __fmaf_rn(nv[2], nv[2], __fmaf_rn(nv[1], nv[1], nv[0] * nv[0]));
        const float q = sqrtf(sq);
#pragma unroll
        for (int a = 0; a < 3; ++a) nrm[3 * row + a] = sq > 0.f ? nv[a] / q : nv[a];
        if (CT == TSDF_RGB8) {
#pragma unroll
            for (int a = 0; a < 3; ++a) cols[3 * row + a] = (__fmaf_rn(col[a * n + i1], r0, col[a * n + i0] * r1) / rs) / 255.0f;
        } else if (CT == TSDF_GRAY32) {
            const float g = __fmaf_rn(col[i1], r0, col[i0] * r1) / rs;
            cols[3 * row] = cols[3 * row + 1] = cols[3 * row + 2] = g;
        }
        ++row;
    }
}

// ExtractVoxelPointCloud / ExtractVoxelGrid (UT:352-408): key (x, y, z), point fma(vl, k - res / 2, half) + origin, grey
// (float)(((double)f + 1) * 0.5)
__global__ void __launch_bounds__(256) tsdf_voxels_kernel(const float2 *__restrict__ tw, int res, int h, float vl, float half, float ox,
                                                          float oy, float oz, const int32_t *__restrict__ pos, size_t m,
                                                          int32_t *__restrict__ keys, float *__restrict__ pts, float *__restrict__ cols) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const size_t i = (size_t)pos[j];
    const size_t rr = (size_t)res * res;
    const int k[3] = {(int)(i / rr), (int)((i / res) % res), (int)(i % res)};
    const float o[3] = {ox, oy, oz};
    const float g = (float)(((double)tw[i].x + 1.0) * 0.5);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (keys) keys[3 * j + a] = k[a];
        if (pts) pts[3 * j + a] = __fmaf_rn(vl, (float)(k[a] - h), half) + o[a];
        cols[3 * j + a] = g;
    }
}

// flags of every voxel, then the ascending positions of the flagged ones; *m = their number (synchronises)
static int tsdf_flag_compact(const cphb_tsdf *v, int mode, cphb_scratch &sc, uint8_t **flags, int32_t **pos, size_t *m, cudaStream_t s) {
    int rc = sc.alloc(flags, v->n);
    if (!rc) rc = sc.alloc(pos, v->n);
    if (rc) return rc;
    CPHB_LAUNCH(tsdf_flag_kernel, tsdf_vox_grid(v->res), TSDF_VOX_BLOCK, 0, s, v->tw, v->res, mode, *flags);
    return cphb_compact_flags(*flags, v->n, *pos, m, s);
}

static int tsdf_scan(const unsigned long long *cnt, unsigned long long *off, size_t n, cphb_scratch &sc, cudaStream_t s) {
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, cnt, off, (int64_t)n, s));
    char *tmp = nullptr;
    const int rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, cnt, off, (int64_t)n, s));
    g_cphb_launches += 2;  // CUB's init and scan kernels
    return CPHB_OK;
}

extern "C" int cphb_tsdf_extract_points(const cphb_tsdf *v, float *points, float *normals, float *colors, size_t capacity, size_t *h_count,
                                        void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_extract_points";
    if (!v || !h_count) return tsdf_invalid(who, "null argument");
    *h_count = 0;
    if (capacity && (!points || !normals || (v->ct != TSDF_NO_COLOR && !colors))) return tsdf_invalid(who, "null output");
    cphb_scratch sc(s);
    uint8_t *flags = nullptr;
    int32_t *pos = nullptr;
    size_t m = 0;
    int rc = tsdf_flag_compact(v, 0, sc, &flags, &pos, &m, s);
    if (rc) return rc;
    // output offsets: exclusive scan of the popcounts of the m surface voxels' masks and one trailing 0, so off[m] is the
    // total.  The scan runs also when m == 0, so the call's launches do not depend on the data.
    unsigned long long *cnt = nullptr, *off = nullptr;
    rc = sc.alloc(&cnt, m + 1);
    if (!rc) rc = sc.alloc(&off, m + 1);
    if (rc) return rc;
    CPHB_LAUNCH(tsdf_popc_kernel, tsdf_blocks(m + 1, 256), 256, 0, s, pos, m, flags, cnt);
    rc = tsdf_scan(cnt, off, m + 1, sc, s);
    if (rc) return rc;
    unsigned long long total = 0;
    rc = cphb_read_back(&total, off + m, sizeof(unsigned long long), s, who);
    if (rc) return rc;
    const size_t mw = total && capacity >= total ? m : 0;  // the writing launch always happens: a fixed launch count
#define TSDF_POINTS(CT)                                                                                                               \
    CPHB_LAUNCH(tsdf_points_kernel<CT>, tsdf_blocks(mw, 128), 128, 0, s, v->tw, v->col, v->n, v->res, v->vl, v->half, (float)v->h * v->vl, \
                v->o[0], v->o[1], v->o[2], pos, mw, flags, off, points, normals, colors)
    if (v->ct == TSDF_RGB8)
        TSDF_POINTS(TSDF_RGB8);
    else if (v->ct == TSDF_GRAY32)
        TSDF_POINTS(TSDF_GRAY32);
    else
        TSDF_POINTS(TSDF_NO_COLOR);
#undef TSDF_POINTS
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_count = (size_t)total;
    return rc;
}

extern "C" int cphb_tsdf_extract_voxels(const cphb_tsdf *v, int32_t *keys, float *points, float *colors, size_t capacity, size_t *h_count,
                                        void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_extract_voxels";
    if (!v || !h_count) return tsdf_invalid(who, "null argument");
    *h_count = 0;
    if (capacity && !colors) return tsdf_invalid(who, "null output");
    cphb_scratch sc(s);
    uint8_t *flags = nullptr;
    int32_t *pos = nullptr;
    size_t m = 0;
    int rc = tsdf_flag_compact(v, 1, sc, &flags, &pos, &m, s);
    if (rc) return rc;
    const size_t mw = capacity >= m ? m : 0;
    CPHB_LAUNCH(tsdf_voxels_kernel, tsdf_blocks(mw, 256), 256, 0, s, v->tw, v->res, v->h, v->vl, v->half, v->o[0], v->o[1], v->o[2], pos,
                mw, keys, points, colors);
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_count = m;
    return rc;
}

// ------------------------------------------------------------------------------------------------ ExtractTriangleMesh
// Welded marching cubes (DESIGN section 4 item 19).  The tables are printed by tools/gen_mc_tables.py, whose docstring
// states the rule; oracle/tsdf_mesh.c carries the same text.
#define MC_TABLE static __device__ const
/* BEGIN tables printed by tools/gen_mc_tables.py */
#define MC_MAX_TRIS 5 /* the most triangles any configuration produces */
/* corner i of a cube: its voxel offset */
MC_TABLE int8_t mc_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
/* edge e: origin corner offset and axis */
MC_TABLE int8_t mc_edge[12][4] = {{0, 0, 0, 0}, {1, 0, 0, 1}, {0, 1, 0, 0}, {0, 0, 0, 1}, {0, 0, 1, 0}, {1, 0, 1, 1}, {0, 1, 1, 0}, {0, 0, 1, 1}, {0, 0, 0, 2}, {1, 0, 0, 2}, {1, 1, 0, 2}, {0, 1, 0, 2}};
/* bit e: edge e is crossed */
MC_TABLE uint16_t mc_edge_table[256] = {
    0x000, 0x109, 0x203, 0x30a, 0x406, 0x50f, 0x605, 0x70c, 0x80c, 0x905, 0xa0f, 0xb06, 0xc0a, 0xd03, 0xe09, 0xf00,
    0x190, 0x099, 0x393, 0x29a, 0x596, 0x49f, 0x795, 0x69c, 0x99c, 0x895, 0xb9f, 0xa96, 0xd9a, 0xc93, 0xf99, 0xe90,
    0x230, 0x339, 0x033, 0x13a, 0x636, 0x73f, 0x435, 0x53c, 0xa3c, 0xb35, 0x83f, 0x936, 0xe3a, 0xf33, 0xc39, 0xd30,
    0x3a0, 0x2a9, 0x1a3, 0x0aa, 0x7a6, 0x6af, 0x5a5, 0x4ac, 0xbac, 0xaa5, 0x9af, 0x8a6, 0xfaa, 0xea3, 0xda9, 0xca0,
    0x460, 0x569, 0x663, 0x76a, 0x066, 0x16f, 0x265, 0x36c, 0xc6c, 0xd65, 0xe6f, 0xf66, 0x86a, 0x963, 0xa69, 0xb60,
    0x5f0, 0x4f9, 0x7f3, 0x6fa, 0x1f6, 0x0ff, 0x3f5, 0x2fc, 0xdfc, 0xcf5, 0xfff, 0xef6, 0x9fa, 0x8f3, 0xbf9, 0xaf0,
    0x650, 0x759, 0x453, 0x55a, 0x256, 0x35f, 0x055, 0x15c, 0xe5c, 0xf55, 0xc5f, 0xd56, 0xa5a, 0xb53, 0x859, 0x950,
    0x7c0, 0x6c9, 0x5c3, 0x4ca, 0x3c6, 0x2cf, 0x1c5, 0x0cc, 0xfcc, 0xec5, 0xdcf, 0xcc6, 0xbca, 0xac3, 0x9c9, 0x8c0,
    0x8c0, 0x9c9, 0xac3, 0xbca, 0xcc6, 0xdcf, 0xec5, 0xfcc, 0x0cc, 0x1c5, 0x2cf, 0x3c6, 0x4ca, 0x5c3, 0x6c9, 0x7c0,
    0x950, 0x859, 0xb53, 0xa5a, 0xd56, 0xc5f, 0xf55, 0xe5c, 0x15c, 0x055, 0x35f, 0x256, 0x55a, 0x453, 0x759, 0x650,
    0xaf0, 0xbf9, 0x8f3, 0x9fa, 0xef6, 0xfff, 0xcf5, 0xdfc, 0x2fc, 0x3f5, 0x0ff, 0x1f6, 0x6fa, 0x7f3, 0x4f9, 0x5f0,
    0xb60, 0xa69, 0x963, 0x86a, 0xf66, 0xe6f, 0xd65, 0xc6c, 0x36c, 0x265, 0x16f, 0x066, 0x76a, 0x663, 0x569, 0x460,
    0xca0, 0xda9, 0xea3, 0xfaa, 0x8a6, 0x9af, 0xaa5, 0xbac, 0x4ac, 0x5a5, 0x6af, 0x7a6, 0x0aa, 0x1a3, 0x2a9, 0x3a0,
    0xd30, 0xc39, 0xf33, 0xe3a, 0x936, 0x83f, 0xb35, 0xa3c, 0x53c, 0x435, 0x73f, 0x636, 0x13a, 0x033, 0x339, 0x230,
    0xe90, 0xf99, 0xc93, 0xd9a, 0xa96, 0xb9f, 0x895, 0x99c, 0x69c, 0x795, 0x49f, 0x596, 0x29a, 0x393, 0x099, 0x190,
    0xf00, 0xe09, 0xd03, 0xc0a, 0xb06, 0xa0f, 0x905, 0x80c, 0x70c, 0x605, 0x50f, 0x406, 0x30a, 0x203, 0x109, 0x000,
};
MC_TABLE uint8_t mc_tri_count[256] = {
    0, 1, 1, 2, 1, 2, 2, 3, 1, 2, 2, 3, 2, 3, 3, 2, 1, 2, 2, 3, 2, 3, 3, 4, 2, 3, 3, 4, 3, 4, 4, 3,
    1, 2, 2, 3, 2, 3, 3, 4, 2, 3, 3, 4, 3, 4, 4, 3, 2, 3, 3, 2, 3, 4, 4, 3, 3, 4, 4, 3, 4, 5, 5, 2,
    1, 2, 2, 3, 2, 3, 3, 4, 2, 3, 3, 4, 3, 4, 4, 3, 2, 3, 3, 4, 3, 4, 4, 5, 3, 4, 4, 5, 4, 5, 5, 4,
    2, 3, 3, 4, 3, 4, 2, 3, 3, 4, 4, 5, 4, 5, 3, 2, 3, 4, 4, 3, 4, 5, 3, 2, 4, 5, 5, 4, 5, 2, 4, 1,
    1, 2, 2, 3, 2, 3, 3, 4, 2, 3, 3, 4, 3, 4, 4, 3, 2, 3, 3, 4, 3, 4, 4, 5, 3, 2, 4, 3, 4, 3, 5, 2,
    2, 3, 3, 4, 3, 4, 4, 5, 3, 4, 4, 5, 4, 5, 5, 4, 3, 4, 4, 3, 4, 5, 5, 4, 4, 3, 5, 2, 5, 4, 2, 1,
    2, 3, 3, 4, 3, 4, 4, 5, 3, 4, 4, 5, 2, 3, 3, 2, 3, 4, 4, 5, 4, 5, 5, 2, 4, 3, 5, 4, 3, 2, 4, 1,
    3, 4, 4, 5, 4, 5, 3, 4, 4, 5, 5, 2, 3, 4, 2, 1, 2, 3, 3, 2, 3, 4, 2, 1, 3, 2, 4, 1, 2, 1, 1, 0,
};
/* the edges of each triangle, -1 past mc_tri_count */
MC_TABLE int8_t mc_tri_table[256][3 * MC_MAX_TRIS] = {
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 10, 0, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 9, 2, 9, 10, -1, -1, -1, -1, -1, -1},
    {2, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 8, 1, 8, 9, -1, -1, -1, -1, -1, -1},
    {1, 10, 11, 1, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 11, 0, 11, 8, -1, -1, -1, -1, -1, -1},
    {0, 9, 10, 0, 10, 11, 0, 11, 3, -1, -1, -1, -1, -1, -1},
    {8, 9, 10, 8, 10, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 7, 1, 7, 4, 1, 4, 9, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, 4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 4, 1, 10, 2, -1, -1, -1, -1, -1, -1},
    {0, 9, 10, 0, 10, 2, 4, 8, 7, -1, -1, -1, -1, -1, -1},
    {2, 3, 7, 2, 7, 4, 2, 4, 9, 2, 9, 10, -1, -1, -1},
    {2, 11, 3, 4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 7, 0, 7, 4, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 11, 3, 4, 8, 7, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 7, 1, 7, 4, 1, 4, 9, -1, -1, -1},
    {1, 10, 11, 1, 11, 3, 4, 8, 7, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 11, 0, 11, 7, 0, 7, 4, -1, -1, -1},
    {0, 9, 10, 0, 10, 11, 0, 11, 3, 4, 8, 7, -1, -1, -1},
    {4, 9, 10, 4, 10, 11, 4, 11, 7, -1, -1, -1, -1, -1, -1},
    {4, 5, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 4, 5, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 0, 5, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 4, 1, 4, 5, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, 4, 5, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 10, 2, 4, 5, 9, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 0, 5, 10, 0, 10, 2, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 4, 2, 4, 5, 2, 5, 10, -1, -1, -1},
    {2, 11, 3, 4, 5, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 8, 4, 5, 9, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 0, 5, 1, 2, 11, 3, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 8, 1, 8, 4, 1, 4, 5, -1, -1, -1},
    {1, 10, 11, 1, 11, 3, 4, 5, 9, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 11, 0, 11, 8, 4, 5, 9, -1, -1, -1},
    {0, 4, 5, 0, 5, 10, 0, 10, 11, 0, 11, 3, -1, -1, -1},
    {4, 5, 10, 4, 10, 11, 4, 11, 8, -1, -1, -1, -1, -1, -1},
    {5, 9, 8, 5, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 5, 0, 5, 9, -1, -1, -1, -1, -1, -1},
    {0, 8, 7, 0, 7, 5, 0, 5, 1, -1, -1, -1, -1, -1, -1},
    {1, 3, 7, 1, 7, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, 5, 9, 8, 5, 8, 7, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 5, 0, 5, 9, 1, 10, 2, -1, -1, -1},
    {0, 8, 7, 0, 7, 5, 0, 5, 10, 0, 10, 2, -1, -1, -1},
    {2, 3, 7, 2, 7, 5, 2, 5, 10, -1, -1, -1, -1, -1, -1},
    {2, 11, 3, 5, 9, 8, 5, 8, 7, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 7, 0, 7, 5, 0, 5, 9, -1, -1, -1},
    {0, 8, 7, 0, 7, 5, 0, 5, 1, 2, 11, 3, -1, -1, -1},
    {1, 2, 11, 1, 11, 7, 1, 7, 5, -1, -1, -1, -1, -1, -1},
    {1, 10, 11, 1, 11, 3, 5, 9, 8, 5, 8, 7, -1, -1, -1},
    {0, 1, 10, 0, 10, 11, 0, 11, 7, 0, 7, 5, 0, 5, 9},
    {0, 8, 7, 0, 7, 5, 0, 5, 10, 0, 10, 11, 0, 11, 3},
    {5, 10, 11, 5, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 9, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {1, 5, 6, 1, 6, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 5, 6, 1, 6, 2, -1, -1, -1, -1, -1, -1},
    {0, 9, 5, 0, 5, 6, 0, 6, 2, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 9, 2, 9, 5, 2, 5, 6, -1, -1, -1},
    {2, 11, 3, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 8, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 11, 3, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 8, 1, 8, 9, 5, 6, 10, -1, -1, -1},
    {1, 5, 6, 1, 6, 11, 1, 11, 3, -1, -1, -1, -1, -1, -1},
    {0, 1, 5, 0, 5, 6, 0, 6, 11, 0, 11, 8, -1, -1, -1},
    {0, 9, 5, 0, 5, 6, 0, 6, 11, 0, 11, 3, -1, -1, -1},
    {5, 6, 11, 5, 11, 8, 5, 8, 9, -1, -1, -1, -1, -1, -1},
    {4, 8, 7, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 4, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 4, 8, 7, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {1, 3, 7, 1, 7, 4, 1, 4, 9, 5, 6, 10, -1, -1, -1},
    {1, 5, 6, 1, 6, 2, 4, 8, 7, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 4, 1, 5, 6, 1, 6, 2, -1, -1, -1},
    {0, 9, 5, 0, 5, 6, 0, 6, 2, 4, 8, 7, -1, -1, -1},
    {2, 3, 7, 2, 7, 4, 2, 4, 9, 2, 9, 5, 2, 5, 6},
    {2, 11, 3, 4, 8, 7, 5, 6, 10, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 7, 0, 7, 4, 5, 6, 10, -1, -1, -1},
    {0, 9, 1, 2, 11, 3, 4, 8, 7, 5, 6, 10, -1, -1, -1},
    {1, 2, 11, 1, 11, 7, 1, 7, 4, 1, 4, 9, 5, 6, 10},
    {1, 5, 6, 1, 6, 11, 1, 11, 3, 4, 8, 7, -1, -1, -1},
    {0, 1, 5, 0, 5, 6, 0, 6, 11, 0, 11, 7, 0, 7, 4},
    {0, 9, 5, 0, 5, 6, 0, 6, 11, 0, 11, 3, 4, 8, 7},
    {9, 5, 6, 9, 6, 11, 9, 11, 7, 9, 7, 4, -1, -1, -1},
    {4, 6, 10, 4, 10, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 4, 6, 10, 4, 10, 9, -1, -1, -1, -1, -1, -1},
    {0, 4, 6, 0, 6, 10, 0, 10, 1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 4, 1, 4, 6, 1, 6, 10, -1, -1, -1},
    {1, 9, 4, 1, 4, 6, 1, 6, 2, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 9, 4, 1, 4, 6, 1, 6, 2, -1, -1, -1},
    {0, 4, 6, 0, 6, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 4, 2, 4, 6, -1, -1, -1, -1, -1, -1},
    {2, 11, 3, 4, 6, 10, 4, 10, 9, -1, -1, -1, -1, -1, -1},
    {0, 2, 11, 0, 11, 8, 4, 6, 10, 4, 10, 9, -1, -1, -1},
    {0, 4, 6, 0, 6, 10, 0, 10, 1, 2, 11, 3, -1, -1, -1},
    {1, 2, 11, 1, 11, 8, 1, 8, 4, 1, 4, 6, 1, 6, 10},
    {1, 9, 4, 1, 4, 6, 1, 6, 11, 1, 11, 3, -1, -1, -1},
    {1, 9, 4, 1, 4, 6, 1, 6, 11, 1, 11, 8, 1, 8, 0},
    {0, 4, 6, 0, 6, 11, 0, 11, 3, -1, -1, -1, -1, -1, -1},
    {4, 6, 11, 4, 11, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {6, 10, 9, 6, 9, 8, 6, 8, 7, -1, -1, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 6, 0, 6, 10, 0, 10, 9, -1, -1, -1},
    {0, 8, 7, 0, 7, 6, 0, 6, 10, 0, 10, 1, -1, -1, -1},
    {1, 3, 7, 1, 7, 6, 1, 6, 10, -1, -1, -1, -1, -1, -1},
    {1, 9, 8, 1, 8, 7, 1, 7, 6, 1, 6, 2, -1, -1, -1},
    {7, 6, 2, 7, 2, 1, 7, 1, 9, 7, 9, 0, 7, 0, 3},
    {0, 8, 7, 0, 7, 6, 0, 6, 2, -1, -1, -1, -1, -1, -1},
    {2, 3, 7, 2, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 11, 3, 6, 10, 9, 6, 9, 8, 6, 8, 7, -1, -1, -1},
    {0, 2, 11, 0, 11, 7, 0, 7, 6, 0, 6, 10, 0, 10, 9},
    {0, 8, 7, 0, 7, 6, 0, 6, 10, 0, 10, 1, 2, 11, 3},
    {1, 2, 11, 1, 11, 7, 1, 7, 6, 1, 6, 10, -1, -1, -1},
    {1, 9, 8, 1, 8, 7, 1, 7, 6, 1, 6, 11, 1, 11, 3},
    {0, 1, 9, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 7, 0, 7, 6, 0, 6, 11, 0, 11, 3, -1, -1, -1},
    {6, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {6, 7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 6, 7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 6, 7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 9, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, 6, 7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 10, 2, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {0, 9, 10, 0, 10, 2, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 9, 2, 9, 10, 6, 7, 11, -1, -1, -1},
    {2, 6, 7, 2, 7, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 2, 6, 0, 6, 7, 0, 7, 8, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 6, 7, 2, 7, 3, -1, -1, -1, -1, -1, -1},
    {1, 2, 6, 1, 6, 7, 1, 7, 8, 1, 8, 9, -1, -1, -1},
    {1, 10, 6, 1, 6, 7, 1, 7, 3, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 6, 0, 6, 7, 0, 7, 8, -1, -1, -1},
    {0, 9, 10, 0, 10, 6, 0, 6, 7, 0, 7, 3, -1, -1, -1},
    {6, 7, 8, 6, 8, 9, 6, 9, 10, -1, -1, -1, -1, -1, -1},
    {4, 8, 11, 4, 11, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 11, 0, 11, 6, 0, 6, 4, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 4, 8, 11, 4, 11, 6, -1, -1, -1, -1, -1, -1},
    {1, 3, 11, 1, 11, 6, 1, 6, 4, 1, 4, 9, -1, -1, -1},
    {1, 10, 2, 4, 8, 11, 4, 11, 6, -1, -1, -1, -1, -1, -1},
    {0, 3, 11, 0, 11, 6, 0, 6, 4, 1, 10, 2, -1, -1, -1},
    {0, 9, 10, 0, 10, 2, 4, 8, 11, 4, 11, 6, -1, -1, -1},
    {3, 11, 6, 3, 6, 4, 3, 4, 9, 3, 9, 10, 3, 10, 2},
    {2, 6, 4, 2, 4, 8, 2, 8, 3, -1, -1, -1, -1, -1, -1},
    {0, 2, 6, 0, 6, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 6, 4, 2, 4, 8, 2, 8, 3, -1, -1, -1},
    {1, 2, 6, 1, 6, 4, 1, 4, 9, -1, -1, -1, -1, -1, -1},
    {1, 10, 6, 1, 6, 4, 1, 4, 8, 1, 8, 3, -1, -1, -1},
    {0, 1, 10, 0, 10, 6, 0, 6, 4, -1, -1, -1, -1, -1, -1},
    {10, 6, 4, 10, 4, 8, 10, 8, 3, 10, 3, 0, 10, 0, 9},
    {4, 9, 10, 4, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 5, 9, 6, 7, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 4, 5, 9, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 0, 5, 1, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 4, 1, 4, 5, 6, 7, 11, -1, -1, -1},
    {1, 10, 2, 4, 5, 9, 6, 7, 11, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 10, 2, 4, 5, 9, 6, 7, 11, -1, -1, -1},
    {0, 4, 5, 0, 5, 10, 0, 10, 2, 6, 7, 11, -1, -1, -1},
    {2, 3, 8, 2, 8, 4, 2, 4, 5, 2, 5, 10, 6, 7, 11},
    {2, 6, 7, 2, 7, 3, 4, 5, 9, -1, -1, -1, -1, -1, -1},
    {0, 2, 6, 0, 6, 7, 0, 7, 8, 4, 5, 9, -1, -1, -1},
    {0, 4, 5, 0, 5, 1, 2, 6, 7, 2, 7, 3, -1, -1, -1},
    {1, 2, 6, 1, 6, 7, 1, 7, 8, 1, 8, 4, 1, 4, 5},
    {1, 10, 6, 1, 6, 7, 1, 7, 3, 4, 5, 9, -1, -1, -1},
    {0, 1, 10, 0, 10, 6, 0, 6, 7, 0, 7, 8, 4, 5, 9},
    {0, 4, 5, 0, 5, 10, 0, 10, 6, 0, 6, 7, 0, 7, 3},
    {10, 6, 7, 10, 7, 8, 10, 8, 4, 10, 4, 5, -1, -1, -1},
    {5, 9, 8, 5, 8, 11, 5, 11, 6, -1, -1, -1, -1, -1, -1},
    {0, 3, 11, 0, 11, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1},
    {0, 8, 11, 0, 11, 6, 0, 6, 5, 0, 5, 1, -1, -1, -1},
    {1, 3, 11, 1, 11, 6, 1, 6, 5, -1, -1, -1, -1, -1, -1},
    {1, 10, 2, 5, 9, 8, 5, 8, 11, 5, 11, 6, -1, -1, -1},
    {0, 3, 11, 0, 11, 6, 0, 6, 5, 0, 5, 9, 1, 10, 2},
    {0, 8, 11, 0, 11, 6, 0, 6, 5, 0, 5, 10, 0, 10, 2},
    {3, 11, 6, 3, 6, 5, 3, 5, 10, 3, 10, 2, -1, -1, -1},
    {2, 6, 5, 2, 5, 9, 2, 9, 8, 2, 8, 3, -1, -1, -1},
    {0, 2, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1, -1, -1, -1},
    {8, 3, 2, 8, 2, 6, 8, 6, 5, 8, 5, 1, 8, 1, 0},
    {1, 2, 6, 1, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {6, 5, 9, 6, 9, 8, 6, 8, 3, 6, 3, 1, 6, 1, 10},
    {0, 1, 10, 0, 10, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1},
    {0, 8, 3, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 7, 11, 5, 11, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 5, 7, 11, 5, 11, 10, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 5, 7, 11, 5, 11, 10, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 1, 8, 9, 5, 7, 11, 5, 11, 10, -1, -1, -1},
    {1, 5, 7, 1, 7, 11, 1, 11, 2, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 1, 5, 7, 1, 7, 11, 1, 11, 2, -1, -1, -1},
    {0, 9, 5, 0, 5, 7, 0, 7, 11, 0, 11, 2, -1, -1, -1},
    {2, 3, 8, 2, 8, 9, 2, 9, 5, 2, 5, 7, 2, 7, 11},
    {2, 10, 5, 2, 5, 7, 2, 7, 3, -1, -1, -1, -1, -1, -1},
    {0, 2, 10, 0, 10, 5, 0, 5, 7, 0, 7, 8, -1, -1, -1},
    {0, 9, 1, 2, 10, 5, 2, 5, 7, 2, 7, 3, -1, -1, -1},
    {2, 10, 5, 2, 5, 7, 2, 7, 8, 2, 8, 9, 2, 9, 1},
    {1, 5, 7, 1, 7, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 5, 0, 5, 7, 0, 7, 8, -1, -1, -1, -1, -1, -1},
    {0, 9, 5, 0, 5, 7, 0, 7, 3, -1, -1, -1, -1, -1, -1},
    {5, 7, 8, 5, 8, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 8, 11, 4, 11, 10, 4, 10, 5, -1, -1, -1, -1, -1, -1},
    {0, 3, 11, 0, 11, 10, 0, 10, 5, 0, 5, 4, -1, -1, -1},
    {0, 9, 1, 4, 8, 11, 4, 11, 10, 4, 10, 5, -1, -1, -1},
    {3, 11, 10, 3, 10, 5, 3, 5, 4, 3, 4, 9, 3, 9, 1},
    {1, 5, 4, 1, 4, 8, 1, 8, 11, 1, 11, 2, -1, -1, -1},
    {11, 2, 1, 11, 1, 5, 11, 5, 4, 11, 4, 0, 11, 0, 3},
    {5, 4, 8, 5, 8, 11, 5, 11, 2, 5, 2, 0, 5, 0, 9},
    {2, 3, 11, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 5, 2, 5, 4, 2, 4, 8, 2, 8, 3, -1, -1, -1},
    {0, 2, 10, 0, 10, 5, 0, 5, 4, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, 2, 10, 5, 2, 5, 4, 2, 4, 8, 2, 8, 3},
    {2, 10, 5, 2, 5, 4, 2, 4, 9, 2, 9, 1, -1, -1, -1},
    {1, 5, 4, 1, 4, 8, 1, 8, 3, -1, -1, -1, -1, -1, -1},
    {0, 1, 5, 0, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 4, 8, 5, 8, 3, 5, 3, 0, 5, 0, 9, -1, -1, -1},
    {4, 9, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 11, 4, 11, 10, 4, 10, 9, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, 4, 7, 11, 4, 11, 10, 4, 10, 9, -1, -1, -1},
    {0, 4, 7, 0, 7, 11, 0, 11, 10, 0, 10, 1, -1, -1, -1},
    {1, 3, 8, 1, 8, 4, 1, 4, 7, 1, 7, 11, 1, 11, 10},
    {1, 9, 4, 1, 4, 7, 1, 7, 11, 1, 11, 2, -1, -1, -1},
    {0, 3, 8, 1, 9, 4, 1, 4, 7, 1, 7, 11, 1, 11, 2},
    {0, 4, 7, 0, 7, 11, 0, 11, 2, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 4, 2, 4, 7, 2, 7, 11, -1, -1, -1},
    {2, 10, 9, 2, 9, 4, 2, 4, 7, 2, 7, 3, -1, -1, -1},
    {2, 10, 9, 2, 9, 4, 2, 4, 7, 2, 7, 8, 2, 8, 0},
    {4, 7, 3, 4, 3, 2, 4, 2, 10, 4, 10, 1, 4, 1, 0},
    {1, 2, 10, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 4, 1, 4, 7, 1, 7, 3, -1, -1, -1, -1, -1, -1},
    {1, 9, 4, 1, 4, 7, 1, 7, 8, 1, 8, 0, -1, -1, -1},
    {0, 4, 7, 0, 7, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 11, 10, 8, 10, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 11, 0, 11, 10, 0, 10, 9, -1, -1, -1, -1, -1, -1},
    {0, 8, 11, 0, 11, 10, 0, 10, 1, -1, -1, -1, -1, -1, -1},
    {1, 3, 11, 1, 11, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 8, 1, 8, 11, 1, 11, 2, -1, -1, -1, -1, -1, -1},
    {11, 2, 1, 11, 1, 9, 11, 9, 0, 11, 0, 3, -1, -1, -1},
    {0, 8, 11, 0, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 9, 2, 9, 8, 2, 8, 3, -1, -1, -1, -1, -1, -1},
    {0, 2, 10, 0, 10, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 3, 2, 8, 2, 10, 8, 10, 1, 8, 1, 0, -1, -1, -1},
    {1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 8, 1, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
};
/* END tables printed by tools/gen_mc_tables.py */
#undef MC_TABLE

// cube byte at the cube's origin voxel (x, y, z), x, y, z <= res - 2: the cube index (bit i: corner i's tsdf < 0) when
// all 8 corner weights are nonzero and the index is neither 0 nor 255, else 0 (UT:184-210 and its 0 / 255 filter)
__global__ void __launch_bounds__(256) tsdf_mc_cube_kernel(const float2 *__restrict__ tw, int res, uint8_t *__restrict__ cb) {
    const int z = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, x = blockIdx.z;
    if (z >= res || y >= res) return;
    int ci = 0;
    bool ok = x < res - 1 && y < res - 1 && z < res - 1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (!ok) break;
        const float2 c = tw[tsdf_idx(x + mc_corner[i][0], y + mc_corner[i][1], z + mc_corner[i][2], res)];
        ok = c.y != 0.0f;
        ci |= (c.x < 0.0f ? 1 : 0) << i;
    }
    cb[tsdf_idx(x, y, z, res)] = ok && ci != 255 ? (uint8_t)ci : 0;
}

// bit a of voxel v's mask: edge (v, a) is a vertex, i.e. it is crossed in a cube that emits.  The cube at v - d holds
// the edge as its edge e with origin corner d and axis a, so the bit is the OR of mc_edge_table[cb[v - d]] >> e.
__global__ void __launch_bounds__(256) tsdf_mc_edge_kernel(const uint8_t *__restrict__ cb, int res, uint8_t *__restrict__ em) {
    const int z = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, x = blockIdx.z;
    if (z >= res || y >= res) return;
    uint8_t m = 0;
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        const int cx = x - mc_edge[e][0], cy = y - mc_edge[e][1], cz = z - mc_edge[e][2];
        if (cx < 0 || cy < 0 || cz < 0) continue;
        if (mc_edge_table[__ldg(cb + tsdf_idx(cx, cy, cz, res))] >> e & 1) m |= (uint8_t)(1 << mc_edge[e][3]);
    }
    em[tsdf_idx(x, y, z, res)] = m;
}

// vcnt[j] = popcount of compacted voxel j's edge mask, tcnt[j] = triangle count of compacted cube j; each array ends
// with one 0, so the exclusive scans' last outputs are the totals
__global__ void __launch_bounds__(256) tsdf_mc_count_kernel(const int32_t *__restrict__ vpos, size_t mv, const uint8_t *__restrict__ em,
                                                            const int32_t *__restrict__ cpos, size_t mc, const uint8_t *__restrict__ cb,
                                                            unsigned long long *__restrict__ vcnt, unsigned long long *__restrict__ tcnt) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j < mv) vcnt[j] = (unsigned long long)__popc(em[vpos[j]]);
    if (j == mv) vcnt[j] = 0ull;
    if (j < mc) tcnt[j] = (unsigned long long)mc_tri_count[cb[cpos[j]]];
    if (j == mc) tcnt[j] = 0ull;
}

// the vertices of compacted voxel j, at rows voff[j] ...; vbase[v] = voff[j] for the triangle kernel.  The expression
// order is oracle/tsdf_mesh.c's ExtractTriangleMesh.
template <int CT>
__global__ void __launch_bounds__(128) tsdf_mc_vertex_kernel(const float2 *__restrict__ tw, const float *__restrict__ col, size_t n, int res,
                                                             float vl, float half, float hres, float ox, float oy, float oz,
                                                             const int32_t *__restrict__ vpos, size_t mv, const uint8_t *__restrict__ em,
                                                             const unsigned long long *__restrict__ voff, int32_t *__restrict__ vbase,
                                                             float *__restrict__ verts, float *__restrict__ vcols) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= mv) return;
    const size_t i0 = (size_t)vpos[j];
    const int mask = em[i0];
    const size_t rr = (size_t)res * res;
    const int k[3] = {(int)(i0 / rr), (int)((i0 / res) % res), (int)(i0 % res)};
    const size_t stride[3] = {rr, (size_t)res, 1};
    const float o[3] = {ox, oy, oz};
    size_t row = voff[j];
    vbase[i0] = (int32_t)row;
    const float f0 = fabsf(tw[i0].x);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!(mask >> a & 1)) continue;
        const size_t i1 = i0 + stride[a];
        const float f1 = fabsf(tw[i1].x), fs = f0 + f1;
        float p[3];
#pragma unroll
        for (int b = 0; b < 3; ++b) p[b] = __fmaf_rn(vl, (float)k[b], half);
        p[a] = p[a] + (f0 * vl) / fs;
#pragma unroll
        for (int b = 0; b < 3; ++b) verts[3 * row + b] = (p[b] + o[b]) - hres;
        if (CT == TSDF_RGB8) {
#pragma unroll
            for (int b = 0; b < 3; ++b) vcols[3 * row + b] = __fmaf_rn(f0, col[b * n + i1] / 255.0f, f1 * (col[b * n + i0] / 255.0f)) / fs;
        } else if (CT == TSDF_GRAY32) {
            const float g = __fmaf_rn(f0, col[i1], f1 * col[i0]) / fs;
            vcols[3 * row] = vcols[3 * row + 1] = vcols[3 * row + 2] = g;
        }
        ++row;
    }
}

// the triangles of compacted cube j, at rows toff[j] ...: edge e of the cube at c is vertex vbase[v] + popc(em[v] &
// ((1 << a) - 1)), v = c + its origin corner, a = its axis
__global__ void __launch_bounds__(128) tsdf_mc_triangle_kernel(const int32_t *__restrict__ cpos, size_t mc, const uint8_t *__restrict__ cb,
                                                               const uint8_t *__restrict__ em, const int32_t *__restrict__ vbase, int res,
                                                               const unsigned long long *__restrict__ toff, int32_t *__restrict__ tris) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= mc) return;
    const size_t c = (size_t)cpos[j];
    const int ci = cb[c];
    const int nt = mc_tri_count[ci];
    int32_t *out = tris + 3 * toff[j];
    for (int t = 0; t < 3 * nt; ++t) {
        const int e = mc_tri_table[ci][t];
        const size_t v = c + ((size_t)mc_edge[e][0] * res + mc_edge[e][1]) * res + mc_edge[e][2];
        out[t] = __ldg(vbase + v) + __popc(__ldg(em + v) & ((1 << mc_edge[e][3]) - 1));
    }
}

extern "C" int cphb_tsdf_extract_mesh(const cphb_tsdf *v, float *vertices, float *colors, int32_t *triangles, size_t vertex_capacity,
                                      size_t triangle_capacity, size_t *h_n_vertices, size_t *h_n_triangles, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_extract_mesh";
    if (!v || !h_n_vertices || !h_n_triangles) return tsdf_invalid(who, "null argument");
    *h_n_vertices = *h_n_triangles = 0;
    if ((vertex_capacity || triangle_capacity) && (!vertices || !triangles || (v->ct != TSDF_NO_COLOR && !colors)))
        return tsdf_invalid(who, "null output");
    cphb_scratch sc(s);
    uint8_t *cb = nullptr, *em = nullptr;
    int32_t *vpos = nullptr, *cpos = nullptr, *vbase = nullptr;
    int rc = sc.alloc(&cb, v->n);
    if (!rc) rc = sc.alloc(&em, v->n);
    if (!rc) rc = sc.alloc(&vpos, v->n);
    if (!rc) rc = sc.alloc(&cpos, v->n);
    if (!rc) rc = sc.alloc(&vbase, v->n);
    if (rc) return rc;
    const dim3 g = tsdf_vox_grid(v->res);
    CPHB_LAUNCH(tsdf_mc_cube_kernel, g, TSDF_VOX_BLOCK, 0, s, v->tw, v->res, cb);
    CPHB_LAUNCH(tsdf_mc_edge_kernel, g, TSDF_VOX_BLOCK, 0, s, cb, v->res, em);
    size_t mv = 0, mc = 0;
    rc = cphb_compact_flags(em, v->n, vpos, &mv, s);
    if (!rc) rc = cphb_compact_flags(cb, v->n, cpos, &mc, s);
    if (rc) return rc;
    // output offsets: exclusive scans of the vertex counts of the mv edge voxels and of the triangle counts of the mc
    // emitting cubes, each with one trailing 0.  They run also when a count is 0, so the launches do not depend on
    // the data.
    unsigned long long *vcnt = nullptr, *voff = nullptr, *tcnt = nullptr, *toff = nullptr;
    rc = sc.alloc(&vcnt, mv + 1);
    if (!rc) rc = sc.alloc(&voff, mv + 1);
    if (!rc) rc = sc.alloc(&tcnt, mc + 1);
    if (!rc) rc = sc.alloc(&toff, mc + 1);
    if (rc) return rc;
    CPHB_LAUNCH(tsdf_mc_count_kernel, tsdf_blocks(max(mv, mc) + 1, 256), 256, 0, s, vpos, mv, em, cpos, mc, cb, vcnt, tcnt);
    rc = tsdf_scan(vcnt, voff, mv + 1, sc, s);
    if (!rc) rc = tsdf_scan(tcnt, toff, mc + 1, sc, s);
    unsigned long long nv = 0, nt = 0;
    if (!rc) rc = cphb_read_back(&nv, voff + mv, sizeof(nv), s, who);
    if (!rc) rc = cphb_read_back(&nt, toff + mc, sizeof(nt), s, who);
    if (rc) return rc;
    if (nv > (unsigned long long)INT32_MAX) {  // vertex indices are int32: refuse rather than truncate
        cphb_set_error("%s: the mesh has %llu vertices, more than int32 vertex indices can name", who, nv);
        return CPHB_ERR_INVALID;
    }
    // the writing launches always happen: a fixed launch count
    const bool write = nv && vertex_capacity >= nv && triangle_capacity >= nt;
    const size_t mvw = write ? mv : 0, mcw = write ? mc : 0;
#define TSDF_MC_VERTS(CT)                                                                                                    \
    CPHB_LAUNCH(tsdf_mc_vertex_kernel<CT>, tsdf_blocks(mvw, 128), 128, 0, s, v->tw, v->col, v->n, v->res, v->vl, v->half,  \
                (float)v->h * v->vl, v->o[0], v->o[1], v->o[2], vpos, mvw, em, voff, vbase, vertices, colors)
    if (v->ct == TSDF_RGB8)
        TSDF_MC_VERTS(TSDF_RGB8);
    else if (v->ct == TSDF_GRAY32)
        TSDF_MC_VERTS(TSDF_GRAY32);
    else
        TSDF_MC_VERTS(TSDF_NO_COLOR);
#undef TSDF_MC_VERTS
    CPHB_LAUNCH(tsdf_mc_triangle_kernel, tsdf_blocks(mcw, 128), 128, 0, s, cpos, mcw, cb, em, vbase, v->res, toff, triangles);
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) {
        *h_n_vertices = (size_t)nv;
        *h_n_triangles = (size_t)nt;
    }
    return rc;
}

// ------------------------------------------------------------------------------------------------ Raycast
struct TsdfRay {
    float P[12];  // camera pose (InverseTransform of the extrinsic), rows 0..2
    float fx, fy, cx, cy, trunc, lo, hi;
    int w, h_img;
};

// InterpolateTrilinearly (UT:447-484): base (int)p, minus 1 where p < base + 0.5; acc = fma((tsdf * A) * B, C, acc)
__device__ float tsdf_interp(const float2 *__restrict__ tw, const float p[3], int res) {
    int b[3];
    float a[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        b[i] = (int)p[i];
        if (p[i] < (float)b[i] + 0.5f) b[i] -= 1;
        a[i] = p[i] - ((float)b[i] + 0.5f);
    }
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int dx = (k >> 2) & 1, dy = (k >> 1) & 1, dz = k & 1;
        const float A = dx ? a[0] : 1.f - a[0], B = dy ? a[1] : 1.f - a[1], C = dz ? a[2] : 1.f - a[2];
        acc = __fmaf_rn((__ldg(&tw[tsdf_idx(b[0] + dx, b[1] + dy, b[2] + dz, res)].x) * A) * B, C, acc);
    }
    return acc;
}

// the grid cell of t + dir * len, or false when it lies outside [lo, res - 1) on an axis (range-checked before the cast)
__device__ __forceinline__ bool tsdf_cell(const float t[3], const float d[3], float len, float vl, int res, int h, int lo, int k[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float g = floorf(__fmaf_rn(d[a], len, t[a]) / vl);
        if (!(g >= (float)(lo - h) && g < (float)(res - 1 - h))) return false;
        k[a] = (int)g + h;
    }
    return true;
}

// raycast_tsdf_functor (UT:509-639); the expression order and the entry / exit times on the grid's real box are
// oracle/tsdf.c's ray()
__device__ bool tsdf_ray(const float2 *__restrict__ tw, int res, int h, float vl, const float o[3], const TsdfRay &c, int x, int y,
                         float out[9], size_t *ci) {
    const float length = (float)res * vl;
    const float q0 = ((float)x - c.cx) / c.fx, q1 = ((float)y - c.cy) / c.fy;
    float d[3], t[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) d[r] = __fmaf_rn(c.P[4 * r + 2], 1.0f, __fmaf_rn(c.P[4 * r + 1], q1, c.P[4 * r] * q0));
    const float dn = sqrtf(__fmaf_rn(d[2], d[2], __fmaf_rn(d[1], d[1], d[0] * d[0])));
    if (dn == 0.f) return false;
    float len = -INFINITY, tmax = INFINITY;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        d[r] = d[r] / dn;
        t[r] = c.P[4 * r + 3] - o[r];
        if (d[r] == 0.f) {  // parallel to the slab: inside it for every time, or never
            if (!(t[r] >= c.lo && t[r] <= c.hi)) return false;
            continue;
        }
        len = fmaxf(len, ((d[r] > 0.f ? c.lo : c.hi) - t[r]) / d[r]);
        tmax = fminf(tmax, ((d[r] > 0.f ? c.hi : c.lo) - t[r]) / d[r]);
    }
    len = fmaxf(len, 0.f);
    if (!(len < tmax)) return false;
    len = len + vl;
    int k[3];
    if (!tsdf_cell(t, d, len, vl, res, h, 0, k)) return false;
    float f = __ldg(&tw[tsdf_idx(k[0], k[1], k[2], res)].x);
    const float step = c.trunc * 0.5f;
    const float lim = len + length * sqrtf(2.0f);
    for (; len < lim; len = len + step) {
        if (!(len + step > len)) return false;  // the step no longer advances the ray: the reference would loop for ever
        if (!tsdf_cell(t, d, len + step, vl, res, h, 1, k)) continue;
        const float fp = f;
        f = __ldg(&tw[tsdf_idx(k[0], k[1], k[2], res)].x);
        if (fp < 0.f && f > 0.f) return false;
        if (fp > 0.f && f < 0.f) {
            const float ts = len - (step * fp) / (f - fp);
            float loc[3], n[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                out[a] = __fmaf_rn(d[a], ts, t[a]);
                loc[a] = out[a] / vl + (float)h;
                if (!(loc[a] >= 1.f && loc[a] < (float)(res - 1))) return false;
            }
            for (int a = 0; a < 3; ++a) {
                float s[3] = {loc[0], loc[1], loc[2]};
                s[a] = loc[a] + 1.f;
                if (s[a] >= (float)(res - 1)) return false;
                const float f1 = tsdf_interp(tw, s, res);
                s[a] = loc[a] - 1.f;
                if (s[a] < 1.f) return false;
                n[a] = f1 - tsdf_interp(tw, s, res);
            }
            const float nn = sqrtf(__fmaf_rn(n[2], n[2], __fmaf_rn(n[1], n[1], n[0] * n[0])));
            if (nn == 0.f) return false;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                out[a] = out[a] + o[a];
                out[3 + a] = n[a] / nn;
            }
            *ci = tsdf_idx((int)loc[0], (int)loc[1], (int)loc[2], res);
            return true;
        }
    }
    return false;
}

// one thread per pixel; a block is 8 x 16 pixels, so each warp marches an 8 x 4 tile of neighbouring rays.  Rows go to
// pts / nrm / cols (NaN for a miss) and, when hit is given, the hit flag.
template <int CT>
__global__ void __launch_bounds__(128) tsdf_raycast_kernel(const float2 *__restrict__ tw, const float *__restrict__ col, size_t n, int res,
                                                           int h, float vl, float ox, float oy, float oz, const TsdfRay c,
                                                           float *__restrict__ pts, float *__restrict__ nrm, float *__restrict__ cols,
                                                           uint8_t *__restrict__ hit) {
    const int x = blockIdx.x * 8 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y;
    if (x >= c.w || y >= c.h_img) return;
    const float o[3] = {ox, oy, oz};
    float r[9];
    size_t ci = 0;
    const bool ok = tsdf_ray(tw, res, h, vl, o, c, x, y, r, &ci);
    if (ok) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
            r[6 + a] = CT == TSDF_RGB8 ? __ldg(col + a * n + ci) / 255.0f : CT == TSDF_GRAY32 ? __ldg(col + ci) : 0.f;
    } else {
#pragma unroll
        for (int a = 0; a < 9; ++a) r[a] = __int_as_float(0x7fc00000);
    }
    const size_t i = (size_t)y * c.w + x;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        pts[3 * i + a] = r[a];
        nrm[3 * i + a] = r[3 + a];
        cols[3 * i + a] = r[6 + a];
    }
    if (hit) hit[i] = ok ? 1 : 0;
}

extern "C" int cphb_tsdf_raycast(const cphb_tsdf *v, int width, int height, const float h_intrinsic[9], const float h_extrinsic[16],
                                 float sdf_trunc, int project_valid_depth_only, float *points, float *normals, float *colors,
                                 size_t capacity, size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_tsdf_raycast";
    if (!v || !h_intrinsic || !h_extrinsic || !h_count) return tsdf_invalid(who, "null argument");
    *h_count = 0;
    if (width <= 0 || height <= 0) return tsdf_invalid(who, "the intrinsic's image size is not positive");
    // a step of sdf_trunc / 2 that is not positive would march for ever
    if (!(isfinite(sdf_trunc) && sdf_trunc > 0.f)) return tsdf_invalid(who, "sdf_trunc is not positive and finite");
    const size_t npx = (size_t)width * height;
    if (npx > (size_t)INT32_MAX) return tsdf_invalid(who, "more than 2^31-1 pixels");
    if (capacity < npx || !points || !normals || !colors) return tsdf_invalid(who, "the outputs need width * height rows");
    TsdfRay c;
    const float *E = h_extrinsic;
    for (int r = 0; r < 3; ++r) {  // InverseTransform (eigen.cu:67-73): R^T, -R^T t
        for (int q = 0; q < 3; ++q) c.P[4 * r + q] = E[4 * q + r];
        c.P[4 * r + 3] = fmaf(-E[8 + r], E[11], fmaf(-E[4 + r], E[7], -E[r] * E[3]));
    }
    c.fx = h_intrinsic[0];
    c.fy = h_intrinsic[4];
    c.cx = h_intrinsic[2];
    c.cy = h_intrinsic[5];
    c.trunc = sdf_trunc;
    // the box of the cells the march may sample, origin-relative: cells [0, res - 1) per axis.  (The first sample is one
    // voxel past the entry and must lie in a cell below res - 1, so a ray entering through a high face of the whole
    // grid's box would always miss.)
    c.lo = -(float)v->h * v->vl;
    c.hi = (float)(v->res - 1 - v->h) * v->vl;
    c.w = width;
    c.h_img = height;
    cphb_scratch sc(s);
    float *rp = points, *rn = normals, *rc_ = colors;
    uint8_t *hit = nullptr;
    int32_t *sel = nullptr;
    if (project_valid_depth_only) {
        int rc = sc.alloc(&rp, 3 * npx);
        if (!rc) rc = sc.alloc(&rn, 3 * npx);
        if (!rc) rc = sc.alloc(&rc_, 3 * npx);
        if (!rc) rc = sc.alloc(&hit, npx);
        if (!rc) rc = sc.alloc(&sel, npx);
        if (rc) return rc;
    }
    const dim3 g((unsigned)((width + 7) / 8), (unsigned)((height + 15) / 16)), b(8, 16);
#define TSDF_RAYCAST(CT) \
    CPHB_LAUNCH(tsdf_raycast_kernel<CT>, g, b, 0, s, v->tw, v->col, v->n, v->res, v->h, v->vl, v->o[0], v->o[1], v->o[2], c, rp, rn, rc_, hit)
    if (v->ct == TSDF_RGB8)
        TSDF_RAYCAST(TSDF_RGB8);
    else if (v->ct == TSDF_GRAY32)
        TSDF_RAYCAST(TSDF_GRAY32);
    else
        TSDF_RAYCAST(TSDF_NO_COLOR);
#undef TSDF_RAYCAST
    size_t m = npx;
    if (project_valid_depth_only) {  // RemoveNoneFinitePoints(true, true) (UT:948-949): the hit rows, in pixel order
        int rc = cphb_compact_flags(hit, npx, sel, &m, s);
        if (!rc) rc = cphb_select_by_index(rp, rn, rc_, npx, sel, m, points, normals, colors, s);
        if (rc) return rc;
    }
    const int rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_count = m;
    return rc;
}
