// stsdf.cu -- integration::ScalableTSDFVolume (SURVEY 8f row 16; DESIGN section 4 item 21).  Reference:
// integration/scalable_tsdfvolume.cu (ST) and integrate_functor.h (IF).
//
// Storage: 16^3-voxel units in a pool of slots.  Slot s holds one float2 {tsdf, weight} block of 4096 voxels at
// tw[s * 4096] and, with colour, its colour planes at col[(s * planes + k) * 4096] (the layout decision of tsdf.cu).
// Voxel index in a unit: x * 256 + y * 16 + z.  keys[s] is the unit's packed key: each axis of floor(p / U) biased by
// 2^20 into 21 bits, x highest, so ascending packed keys are ascending (x, y, z).  An open-addressing table (linear
// probing, capacity a power of two at least twice the pool's) maps a packed key to its slot.
//
// Integrate: (1) the strided depth points (depth_project.cuh, the projection PointCloud::CreateFromDepthImage uses) and
// per point every unit key in [floor((P - trunc) / U), floor((P + trunc) / U)] per axis, by count, CUB scan and write;
// (2) CUB radix sort and unique of the candidates, a table lookup each, the missing ones compacted in ascending key
// order; (3) the pool grows by doubling when they do not fit (a new arena first, so a failed allocation
// changes nothing); (4) the new units are appended and initialised; (5) one thread per voxel of every allocated unit
// runs tsdf_update.cuh's update, a block per 256 consecutive voxels of one unit (block b: slot b / 16).  Nothing changes before step (3)
// succeeds, and every rejection (format, key range, unit count, allocation) happens before it.
//
// Unit order is the frame that first touched the unit, then ascending key; it does not depend on map_size or growth.
// The extractions go in slot order, then voxel index, then axis.
//
// Arithmetic: IEEE, no contraction; every fused multiply-add is an explicit __fmaf_rn, in the order oracle/stsdf.c
// states with fmaf().
#include <math.h>

#include <memory>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "depth_project.cuh"
#include "tsdf_update.cuh"

#define ST_RES 16
#define ST_VOX 4096
#define ST_BIAS (1 << 20)
#define ST_EMPTY 0xffffffffffffffffull
#define ST_MAX_UNITS (INT32_MAX / ST_VOX)  // the extractions' compaction writes int32 voxel positions

struct cphb_stsdf {
    float vl, half, U, trunc, trunc_inv;
    int ct, planes, stride;
    size_t cap = 0, count = 0, hcap = 0;
    float2 *tw = nullptr;
    float *col = nullptr;
    uint64_t *keys = nullptr;   // [cap] slot -> packed key
    uint64_t *hkeys = nullptr;  // [hcap] table keys (ST_EMPTY: free)
    int32_t *hvals = nullptr;   // [hcap] table slots
    std::unique_ptr<cphb_arena> arena;  // all of the above: one block, replaced whole when the pool grows
};

static int st_invalid(const char *who, const char *what) {
    cphb_set_error("%s: %s", who, what);
    return CPHB_ERR_INVALID;
}
static unsigned st_blocks(size_t n, unsigned b) { return n ? (unsigned)((n + b - 1) / b) : 1u; }

__host__ __device__ __forceinline__ uint64_t st_pack(int x, int y, int z) {
    return ((uint64_t)(x + ST_BIAS) << 42) | ((uint64_t)(y + ST_BIAS) << 21) | (uint64_t)(z + ST_BIAS);
}
__device__ __forceinline__ int st_axis(uint64_t k, int a) { return (int)((k >> (42 - 21 * a)) & 0x1fffff) - ST_BIAS; }
__device__ __forceinline__ bool st_in_range(int k) { return k >= -ST_BIAS && k < ST_BIAS; }

__device__ __forceinline__ uint64_t st_hash(uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    return k ^ (k >> 33);
}
// slot of a packed key, or -1
__device__ __forceinline__ int st_find(const uint64_t *__restrict__ hk, const int32_t *__restrict__ hv, size_t hcap, uint64_t k) {
    if (!hcap) return -1;
    for (size_t h = st_hash(k) & (hcap - 1);; h = (h + 1) & (hcap - 1)) {
        const uint64_t q = hk[h];
        if (q == k) return hv[h];
        if (q == ST_EMPTY) return -1;
    }
}
// slot of unit key (x, y, z), -1 when it is outside the key range or not allocated
__device__ __forceinline__ int st_find3(const uint64_t *hk, const int32_t *hv, size_t hcap, int x, int y, int z) {
    if (!st_in_range(x) || !st_in_range(y) || !st_in_range(z)) return -1;
    return st_find(hk, hv, hcap, st_pack(x, y, z));
}

__global__ void __launch_bounds__(256) st_insert_kernel(const uint64_t *__restrict__ keys, size_t first, size_t n, uint64_t *hk,
                                                        int32_t *hv, size_t hcap) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint64_t k = keys[first + j];
    for (size_t h = st_hash(k) & (hcap - 1);; h = (h + 1) & (hcap - 1)) {
        const unsigned long long prev = atomicCAS((unsigned long long *)&hk[h], ST_EMPTY, (unsigned long long)k);
        if (prev == ST_EMPTY || prev == k) {
            hv[h] = (int32_t)(first + j);
            return;
        }
    }
}

// ------------------------------------------------------------------------------------------------ the handle
extern "C" int cphb_stsdf_create(float voxel_length, float sdf_trunc, int color_type, int depth_sampling_stride, int map_size, void *stream,
                                 cphb_stsdf **out) {
    const char *who = "cphb_stsdf_create";
    if (!out) return st_invalid(who, "null argument");
    *out = nullptr;
    if (!(isfinite(voxel_length) && voxel_length > 0.f)) return st_invalid(who, "voxel_length is not positive and finite");
    if (!(isfinite(sdf_trunc) && sdf_trunc > 0.f)) return st_invalid(who, "sdf_trunc is not positive and finite");
    if (color_type < TSDF_NO_COLOR || color_type > TSDF_GRAY32) return st_invalid(who, "unknown color_type");
    if (depth_sampling_stride < 1) return st_invalid(who, "depth_sampling_stride is not positive");
    if (map_size < 1) return st_invalid(who, "map_size is not positive");
    std::unique_ptr<cphb_stsdf> v(new cphb_stsdf());
    v->vl = voxel_length;
    v->half = 0.5f * voxel_length;
    v->U = voxel_length * (float)ST_RES;  // volume_unit_length_ = voxel_length * 16 (ST:300)
    if (!(isfinite(v->U) && v->U > 0.f)) return st_invalid(who, "voxel_length * 16 is not finite");
    // a point touches at most (2 trunc / U + 2)^3 units; keep that count small enough for the 32-bit per-point counts
    if (!(sdf_trunc / v->U < 64.f)) return st_invalid(who, "sdf_trunc is more than 64 units (1024 voxels)");
    v->trunc = sdf_trunc;
    v->trunc_inv = (float)(1.0 / (double)sdf_trunc);
    v->ct = color_type;
    v->planes = color_type == TSDF_RGB8 ? 3 : color_type == TSDF_GRAY32 ? 1 : 0;
    v->stride = depth_sampling_stride;
    v->cap = (size_t)std::min(map_size, ST_MAX_UNITS);
    // storage is allocated by the first Integrate that needs it (map_size is the pool's first capacity, not a limit)
    *out = v.release();
    return CPHB_OK;
}

extern "C" void cphb_stsdf_destroy(cphb_stsdf *v) { delete v; }

// Reset: no unit is allocated (the pool and the table keep their capacity)
extern "C" int cphb_stsdf_reset(cphb_stsdf *v, void *stream) {
    if (!v) return st_invalid("cphb_stsdf_reset", "null volume");
    v->count = 0;
    if (v->hcap) CPHB_CUDA(cudaMemsetAsync(v->hkeys, 0xff, v->hcap * sizeof(uint64_t), (cudaStream_t)stream));
    return CPHB_OK;
}

extern "C" int cphb_stsdf_data(const cphb_stsdf *v, size_t *h_units, uint64_t **keys, float **tw, float **col) {
    if (!v || !h_units || !keys || !tw || !col) return st_invalid("cphb_stsdf_data", "null argument");
    *h_units = v->count;
    *keys = v->keys;
    *tw = (float *)v->tw;
    *col = v->col;
    return CPHB_OK;
}

extern "C" int cphb_stsdf_info(const cphb_stsdf *v, size_t *h_units, size_t *h_capacity, size_t *h_device_bytes) {
    if (!v || !h_units || !h_capacity || !h_device_bytes) return st_invalid("cphb_stsdf_info", "null argument");
    *h_units = v->count;
    *h_capacity = v->hkeys ? v->cap : 0;
    *h_device_bytes = v->hkeys ? v->cap * (ST_VOX * (8 + 4 * (size_t)v->planes) + 8) + v->hcap * 12 : 0;
    return CPHB_OK;
}

// ------------------------------------------------------------------------------------------------ Integrate
// OpenVolumeUnitKernel's ranges (ST:98-123), bounds-checked: lo = floor((P - trunc) / U), hi = floor((P + trunc) / U)
// per axis.  -> the number of keys of sample i (0 without a point); *bad set when a key leaves the 21-bit range
__device__ __forceinline__ unsigned st_range(const void *depth, const DepthCam &c, float trunc, float U, unsigned i, int lo[3], int hi[3],
                                             unsigned *bad) {
    float p[3];
    if (!dc_point(depth, c, (int)(i / (unsigned)c.sw), (int)(i % (unsigned)c.sw), p)) return 0;
    unsigned n = 1;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float l = floorf((p[a] - trunc) / U), h = floorf((p[a] + trunc) / U);
        if (!(l >= (float)-ST_BIAS && h < (float)ST_BIAS)) {
            atomicOr(bad, 1u);
            return 0;
        }
        lo[a] = (int)l;
        hi[a] = (int)h;
        n *= (unsigned)(hi[a] - lo[a] + 1);
    }
    return n;
}

__global__ void __launch_bounds__(256) st_count_kernel(const float *__restrict__ depth, const DepthCam c, float trunc, float U,
                                                       unsigned long long *__restrict__ cnt, unsigned *bad) {
    const unsigned i = blockIdx.x * 256 + threadIdx.x;
    const unsigned n = (unsigned)c.sw * (unsigned)c.sh;
    if (i > n) return;
    int lo[3], hi[3];
    cnt[i] = i < n ? st_range(depth, c, trunc, U, i, lo, hi, bad) : 0ull;  // the scan's last output is the total
}

__global__ void __launch_bounds__(256) st_keys_kernel(const float *__restrict__ depth, const DepthCam c, float trunc, float U,
                                                      const unsigned long long *__restrict__ off, uint64_t *__restrict__ out, unsigned *bad) {
    const unsigned i = blockIdx.x * 256 + threadIdx.x;
    if (i >= (unsigned)c.sw * (unsigned)c.sh) return;
    int lo[3], hi[3];
    if (!st_range(depth, c, trunc, U, i, lo, hi, bad)) return;
    size_t o = off[i];
    for (int x = lo[0]; x <= hi[0]; ++x)
        for (int y = lo[1]; y <= hi[1]; ++y)
            for (int z = lo[2]; z <= hi[2]; ++z) out[o++] = st_pack(x, y, z);
}

__global__ void __launch_bounds__(256) st_missing_kernel(const uint64_t *__restrict__ uniq, const unsigned *__restrict__ n_uniq,
                                                         const uint64_t *__restrict__ hk, const int32_t *__restrict__ hv, size_t hcap,
                                                         size_t n, uint8_t *__restrict__ flags) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j < n) flags[j] = j < *n_uniq && st_find(hk, hv, hcap, uniq[j]) < 0 ? 1 : 0;
}

// the new units: slot count + j gets key uniq[pos[j]], tsdf 0, weight 0, colour 1 (uniform_tsdfvolume.h:38-40)
__global__ void __launch_bounds__(256) st_append_kernel(const uint64_t *__restrict__ uniq, const int32_t *__restrict__ pos, size_t count,
                                                        uint64_t *__restrict__ keys, float2 *__restrict__ tw, float *__restrict__ col,
                                                        int planes) {
    const size_t slot = count + (blockIdx.x >> 4);
    const unsigned t = (blockIdx.x & 15) * 256 + threadIdx.x;
    if (t == 0) keys[slot] = uniq[pos[blockIdx.x >> 4]];
    tw[slot * ST_VOX + t] = make_float2(0.f, 0.f);
    for (int k = 0; k < planes; ++k) col[(slot * planes + k) * ST_VOX + t] = 1.f;
}

// scalable_integrate_functor (ST:80-95, IF:84-139): voxel (x, y, z) of the unit with origin key * U has the column point
// (fma(vl, x, vl / 2) + o0, fma(vl, y, vl / 2) + o1, vl / 2 + o2) and z index z
template <int CT>
__global__ void __launch_bounds__(256) st_integrate_kernel(const uint64_t *__restrict__ keys, float2 *__restrict__ tw, float *__restrict__ col,
                                                           int planes, float vl, float half, float U, float trunc, float trunc_inv,
                                                           const TsdfCam c, const float *__restrict__ depth, const void *__restrict__ color) {
    const size_t slot = blockIdx.x >> 4;
    const int t = (blockIdx.x & 15) * 256 + threadIdx.x;
    const int x = t >> 8, y = (t >> 4) & 15, z = t & 15;
    const uint64_t k = keys[slot];
    const float o0 = (float)st_axis(k, 0) * U, o1 = (float)st_axis(k, 1) * U, o2 = (float)st_axis(k, 2) * U;
    const float p0 = __fmaf_rn(vl, (float)x, half) + o0;
    const float p1 = __fmaf_rn(vl, (float)y, half) + o1;
    const float p2 = half + o2;
    float cam[3];
    tsdf_camera_point(c, p0, p1, p2, (float)z, cam);
    tsdf_update_voxel<CT>(c, cam, depth, color, trunc, trunc_inv, tw + slot * ST_VOX + t, col + slot * planes * ST_VOX + t, ST_VOX);
}

// a larger pool and table, the old slots copied and the table rebuilt; on failure nothing is changed
static int st_grow(cphb_stsdf *v, size_t need, cudaStream_t s) {
    size_t cap = v->cap;
    while (cap < need) cap *= 2;
    if (cap > (size_t)ST_MAX_UNITS) cap = ST_MAX_UNITS;
    size_t hcap = 1;
    while (hcap < 2 * cap) hcap *= 2;
    float2 *tw = nullptr;
    float *col = nullptr;
    uint64_t *keys = nullptr, *hk = nullptr;
    int32_t *hv = nullptr;
    std::unique_ptr<cphb_arena> a(new cphb_arena());
    a->slice(&tw, cap * ST_VOX);
    a->slice(&col, cap * v->planes * ST_VOX, v->planes > 0);
    a->slice(&keys, cap);
    a->slice(&hk, hcap);
    a->slice(&hv, hcap);
    int rc = a->alloc(s);
    if (rc) return rc;  // nothing allocated, the volume unchanged
    if (v->count) {
        CPHB_CUDA(cudaMemcpyAsync(tw, v->tw, v->count * ST_VOX * sizeof(float2), cudaMemcpyDeviceToDevice, s));
        if (v->planes) CPHB_CUDA(cudaMemcpyAsync(col, v->col, v->count * v->planes * ST_VOX * sizeof(float), cudaMemcpyDeviceToDevice, s));
        CPHB_CUDA(cudaMemcpyAsync(keys, v->keys, v->count * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    }
    CPHB_CUDA(cudaMemsetAsync(hk, 0xff, hcap * sizeof(uint64_t), s));
    if (v->count) CPHB_LAUNCH(st_insert_kernel, st_blocks(v->count, 256), 256, 0, s, keys, (size_t)0, v->count, hk, hv, hcap);
    CPHB_CHECK_LAUNCH();
    v->arena = std::move(a);  // the old block goes back to the pool on its stream
    v->tw = tw;
    v->col = col;
    v->keys = keys;
    v->hkeys = hk;
    v->hvals = hv;
    v->cap = cap;
    v->hcap = hcap;
    return CPHB_OK;
}

extern "C" int cphb_stsdf_integrate(cphb_stsdf *v, const float *depth, int depth_width, int depth_height, int depth_channels,
                                    int depth_bytes_per_channel, const void *color, int color_width, int color_height, int color_channels,
                                    int color_bytes_per_channel, int width, int height, const float h_intrinsic[9],
                                    const float h_extrinsic[16], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_stsdf_integrate";
    if (!v || !h_intrinsic || !h_extrinsic) return st_invalid(who, "null argument");
    if (tsdf_bad_format(v->ct, depth_width, depth_height, depth_channels, depth_bytes_per_channel, color_width, color_height, color_channels,
                        color_bytes_per_channel, width, height))
        return st_invalid(who, "[ScalableTSDFVolume::Integrate] Unsupported image format.");
    if (width <= 0 || height <= 0) return st_invalid(who, "the intrinsic's image size is not positive");
    if (!depth || (v->ct != TSDF_NO_COLOR && !color)) return st_invalid(who, "null image");
    // (1) CreateFromDepthImage(depth, intrinsic, extrinsic, 1000, 1000, stride) (ST:333-335): float depth as it is
    DepthCam dc;
    if (!dc_pose(h_extrinsic, dc.P)) return st_invalid(who, "the extrinsic is not invertible");
    dc.fx = h_intrinsic[0];
    dc.fy = h_intrinsic[4];
    dc.cx = h_intrinsic[2];
    dc.cy = h_intrinsic[5];
    dc.cutoff = -1.f;
    dc.w = width;
    dc.stride = v->stride;
    dc.sw = width / v->stride;
    dc.sh = height / v->stride;
    dc.bytes = 4;
    dc.scale_i = 1;
    dc.trunc_i = 0;
    const size_t n = (size_t)dc.sw * dc.sh;
    if (n >= (size_t)UINT32_MAX) return st_invalid(who, "too many sampled pixels");
    cphb_scratch sc(s);
    unsigned long long *cnt = nullptr, *off = nullptr;
    unsigned *bad = nullptr;
    int rc = sc.alloc(&cnt, n + 1);
    if (!rc) rc = sc.alloc(&off, n + 1);
    if (!rc) rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(unsigned), s));
    CPHB_LAUNCH(st_count_kernel, st_blocks(n + 1, 256), 256, 0, s, depth, dc, v->trunc, v->U, cnt, bad);
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, cnt, off, (int64_t)(n + 1), s));
    char *tmp = nullptr;
    rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, cnt, off, (int64_t)(n + 1), s));
    g_cphb_launches += 2;
    unsigned long long head[2] = {0, 0};
    rc = cphb_read_back(&head[0], off + n, sizeof(unsigned long long), s, who);
    if (!rc) rc = cphb_read_back(&head[1], bad, sizeof(unsigned), s, who);
    if (rc) return rc;
    if (head[1]) return st_invalid(who, "a unit key is outside [-2^20, 2^20) (the frame is rejected)");
    const size_t total = head[0];
    // (2) sort, unique, look up; the missing keys in ascending order
    size_t m = 0;
    uint64_t *uniq = nullptr;
    int32_t *pos = nullptr;
    if (total) {
        uint64_t *cand = nullptr, *sorted = nullptr;
        unsigned *n_uniq = nullptr;
        uint8_t *flags = nullptr;
        rc = sc.alloc(&cand, total);
        if (!rc) rc = sc.alloc(&sorted, total);
        if (!rc) rc = sc.alloc(&uniq, total);
        if (!rc) rc = sc.alloc(&n_uniq, 1);
        if (!rc) rc = sc.alloc(&flags, total);
        if (!rc) rc = sc.alloc(&pos, total);
        if (rc) return rc;
        CPHB_LAUNCH(st_keys_kernel, st_blocks(n, 256), 256, 0, s, depth, dc, v->trunc, v->U, off, cand, bad);
        size_t sb = 0, ub = 0;
        CPHB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sb, cand, sorted, (int64_t)total, 0, 63, s));
        CPHB_CUDA(cub::DeviceSelect::Unique(nullptr, ub, sorted, uniq, n_uniq, (int64_t)total, s));
        char *t2 = nullptr;
        rc = sc.alloc(&t2, std::max(std::max(sb, ub), (size_t)16));
        if (rc) return rc;
        CPHB_CUDA(cub::DeviceRadixSort::SortKeys(t2, sb, cand, sorted, (int64_t)total, 0, 63, s));
        CPHB_CUDA(cub::DeviceSelect::Unique(t2, ub, sorted, uniq, n_uniq, (int64_t)total, s));
        CPHB_LAUNCH(st_missing_kernel, st_blocks(total, 256), 256, 0, s, uniq, n_uniq, v->hkeys, v->hvals, v->hcap, total, flags);
        rc = cphb_compact_flags(flags, total, pos, &m, s);
        if (rc) return rc;
    }
    if (v->count + m > (size_t)ST_MAX_UNITS) return st_invalid(who, "more than 524287 units (the voxel count must fit int32)");
    // (3) room for the new units
    if (!v->hkeys || v->count + m > v->cap) {
        rc = st_grow(v, v->count + m, s);
        if (rc) return rc;
    }
    // (4) append and initialise, then enter them into the table
    if (m) {
        CPHB_LAUNCH(st_append_kernel, (unsigned)(m * 16), 256, 0, s, uniq, pos, v->count, v->keys, v->tw, v->col, v->planes);
        CPHB_LAUNCH(st_insert_kernel, st_blocks(m, 256), 256, 0, s, v->keys, v->count, m, v->hkeys, v->hvals, v->hcap);
        v->count += m;
    }
    // (5) every allocated unit
    if (v->count) {
        const TsdfCam c = tsdf_cam(v->vl, h_intrinsic, h_extrinsic, width, height);
        const unsigned g = (unsigned)(v->count * 16);
#define ST_INTEGRATE(CT)                                                                                                                    \
    CPHB_LAUNCH(st_integrate_kernel<CT>, g, 256, 0, s, v->keys, v->tw, v->col, v->planes, v->vl, v->half, v->U, v->trunc, v->trunc_inv, c, \
                depth, color)
        if (v->ct == TSDF_RGB8)
            ST_INTEGRATE(TSDF_RGB8);
        else if (v->ct == TSDF_GRAY32)
            ST_INTEGRATE(TSDF_GRAY32);
        else
            ST_INTEGRATE(TSDF_NO_COLOR);
#undef ST_INTEGRATE
    }
    return cphb_read_back(nullptr, nullptr, 0, s, who);
}

// ------------------------------------------------------------------------------------------------ extraction
__device__ __forceinline__ bool st_band(float2 v) { return v.y != 0.0f && v.x < 0.98f && v.x >= -0.98f; }

struct StView {
    const uint64_t *keys, *hk;
    const int32_t *hv;
    const float2 *tw;
    const float *col;
    size_t hcap;
    int planes;
    float vl, half, U;
};

// voxel (x, y, z) + e_a of unit `slot`: the slot holding it (-1 when that unit is missing) and its index there
__device__ __forceinline__ int st_step(const StView &V, int slot, uint64_t key, int xyz[3], int a) {
    if (xyz[a] + 1 < ST_RES) {
        xyz[a] += 1;
        return slot;
    }
    xyz[a] = 0;
    int k[3] = {st_axis(key, 0), st_axis(key, 1), st_axis(key, 2)};
    k[a] += 1;
    return st_find3(V.hk, V.hv, V.hcap, k[0], k[1], k[2]);
}

// mode 0: bit a set when voxel i emits ExtractPointCloud's point on axis a (ST:231-289); mode 1: 1 for a band voxel
__global__ void __launch_bounds__(256) st_flag_kernel(const StView V, int mode, uint8_t *__restrict__ flags) {
    const size_t slot = blockIdx.x >> 4;
    const int t = (blockIdx.x & 15) * 256 + threadIdx.x;
    const size_t i = slot * ST_VOX + t;
    const float2 v0 = V.tw[i];
    uint8_t m = 0;
    if (st_band(v0)) {
        if (mode == 1) {
            m = 1;
        } else {
            const uint64_t key = V.keys[slot];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                int xyz[3] = {t >> 8, (t >> 4) & 15, t & 15};
                const int s1 = st_step(V, (int)slot, key, xyz, a);
                if (s1 < 0) continue;  // a missing unit counts as weight 0
                const float2 v1 = V.tw[(size_t)s1 * ST_VOX + xyz[0] * 256 + xyz[1] * 16 + xyz[2]];
                if (st_band(v1) && v0.x * v1.x < 0.f) m |= (uint8_t)(1 << a);
            }
        }
    }
    flags[i] = m;
}

__global__ void __launch_bounds__(256) st_popc_kernel(const int32_t *__restrict__ pos, size_t m, const uint8_t *__restrict__ flags,
                                                      unsigned long long *__restrict__ cnt) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j < m) cnt[j] = (unsigned long long)__popc(flags[pos[j]]);
    if (j == m) cnt[j] = 0ull;
}

// GetTSDFAt (ST:167-213): p_locate = p - vl / 2, unit floor(p_locate / U), g = (p_locate - unit * U) / vl, idx0 =
// floor(g) clamped to [0, 15], r = g - idx0; a corner past the unit comes from the next unit (0 when it is missing);
// acc = fma((wx * wy) * wz, f, acc) over the 8 corners in tsdf.cu's order; 0 when the unit is missing
__device__ float st_tsdf_at(const StView &V, const float p[3]) {
    int u[3], b[3];
    float r[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float pl = p[a] - V.half;
        u[a] = (int)floorf(pl / V.U);
        const float g = (pl - (float)u[a] * V.U) / V.vl;
        b[a] = (int)floorf(g);
        b[a] = b[a] < 0 ? 0 : b[a] >= ST_RES ? ST_RES - 1 : b[a];
        r[a] = g - (float)b[a];
    }
    const int s0 = st_find3(V.hk, V.hv, V.hcap, u[0], u[1], u[2]);
    if (s0 < 0) return 0.f;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int d[3] = {(k >> 2) & 1, (k >> 1) & 1, k & 1};
        int q[3], uu[3];
        bool out = false;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            q[a] = b[a] + d[a];
            uu[a] = u[a];
            if (q[a] >= ST_RES) {
                q[a] -= ST_RES;
                uu[a] += 1;
                out = true;
            }
        }
        const int s1 = out ? st_find3(V.hk, V.hv, V.hcap, uu[0], uu[1], uu[2]) : s0;
        const float f = s1 < 0 ? 0.f : V.tw[(size_t)s1 * ST_VOX + q[0] * 256 + q[1] * 16 + q[2]].x;
        const float wx = d[0] ? r[0] : 1.f - r[0], wy = d[1] ? r[1] : 1.f - r[1], wz = d[2] ? r[2] : 1.f - r[2];
        acc = __fmaf_rn((wx * wy) * wz, f, acc);
    }
    return acc;
}

// the rows of compacted voxel j (ST:231-289) at out rows off[j] ...: p0 = fma(vl, k, vl / 2) + unit * U per axis, the
// crossing fma(p0_a + vl, r0, p0_a r1) / (r0 + r1), GetNormalAt's central differences with half_gap (float)(0.99 vl),
// colour fma(c1, r0, c0 r1) / (r0 + r1) (/ 255 for RGB8)
template <int CT>
__global__ void __launch_bounds__(128) st_points_kernel(const StView V, const int32_t *__restrict__ pos, size_t m,
                                                        const uint8_t *__restrict__ flags, const unsigned long long *__restrict__ off,
                                                        float *__restrict__ pts, float *__restrict__ nrm, float *__restrict__ cols) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const size_t i0 = (size_t)pos[j];
    const int slot = (int)(i0 / ST_VOX), t = (int)(i0 % ST_VOX);
    const uint64_t key = V.keys[slot];
    const int mask = flags[i0];
    const float f0 = V.tw[i0].x;
    size_t row = off[j];
    const int k0[3] = {t >> 8, (t >> 4) & 15, t & 15};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!(mask >> a & 1)) continue;
        int xyz[3] = {k0[0], k0[1], k0[2]};
        const int s1 = st_step(V, slot, key, xyz, a);
        const size_t i1 = (size_t)s1 * ST_VOX + xyz[0] * 256 + xyz[1] * 16 + xyz[2];
        const float r0 = fabsf(f0), r1 = fabsf(V.tw[i1].x), rs = r0 + r1;
        float p[3];
#pragma unroll
        for (int b = 0; b < 3; ++b) p[b] = __fmaf_rn(V.vl, (float)k0[b], V.half) + (float)st_axis(key, b) * V.U;
        const float p1a = p[a] + V.vl;
        p[a] = __fmaf_rn(p1a, r0, p[a] * r1) / rs;
#pragma unroll
        for (int b = 0; b < 3; ++b) pts[3 * row + b] = p[b];
        const float hg = (float)(0.99 * (double)V.vl);
        float nv[3];
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            float q0[3] = {p[0], p[1], p[2]}, q1[3] = {p[0], p[1], p[2]};
            q0[b] = p[b] - hg;
            q1[b] = p[b] + hg;
            nv[b] = st_tsdf_at(V, q1) - st_tsdf_at(V, q0);
        }
        const float sq = __fmaf_rn(nv[2], nv[2], __fmaf_rn(nv[1], nv[1], nv[0] * nv[0]));
        const float q = sqrtf(sq);
#pragma unroll
        for (int b = 0; b < 3; ++b) nrm[3 * row + b] = sq > 0.f ? nv[b] / q : nv[b];
        if (CT == TSDF_RGB8) {
#pragma unroll
            for (int b = 0; b < 3; ++b) {
                const float c0 = V.col[((size_t)slot * 3 + b) * ST_VOX + t], c1 = V.col[((size_t)s1 * 3 + b) * ST_VOX + (i1 % ST_VOX)];
                cols[3 * row + b] = (__fmaf_rn(c1, r0, c0 * r1) / rs) / 255.0f;
            }
        } else if (CT == TSDF_GRAY32) {
            const float c0 = V.col[(size_t)slot * ST_VOX + t], c1 = V.col[(size_t)s1 * ST_VOX + (i1 % ST_VOX)];
            const float g = __fmaf_rn(c1, r0, c0 * r1) / rs;
            cols[3 * row] = cols[3 * row + 1] = cols[3 * row + 2] = g;
        }
        ++row;
    }
}

// ExtractVoxelPointCloud: the centre fma(vl, k, vl / 2) + unit * U of every band voxel, grey (float)(((double)f + 1) * 0.5)
__global__ void __launch_bounds__(256) st_voxels_kernel(const StView V, const int32_t *__restrict__ pos, size_t m, float *__restrict__ pts,
                                                        float *__restrict__ cols) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= m) return;
    const size_t i = (size_t)pos[j];
    const int slot = (int)(i / ST_VOX), t = (int)(i % ST_VOX);
    const uint64_t key = V.keys[slot];
    const int k[3] = {t >> 8, (t >> 4) & 15, t & 15};
    const float g = (float)(((double)V.tw[i].x + 1.0) * 0.5);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        pts[3 * j + a] = __fmaf_rn(V.vl, (float)k[a], V.half) + (float)st_axis(key, a) * V.U;
        cols[3 * j + a] = g;
    }
}

static StView st_view(const cphb_stsdf *v) {
    StView V;
    V.keys = v->keys;
    V.hk = v->hkeys;
    V.hv = v->hvals;
    V.tw = v->tw;
    V.col = v->col;
    V.hcap = v->hcap;
    V.planes = v->planes;
    V.vl = v->vl;
    V.half = v->half;
    V.U = v->U;
    return V;
}

static int st_flag_compact(const cphb_stsdf *v, int mode, cphb_scratch &sc, uint8_t **flags, int32_t **pos, size_t *m, cudaStream_t s) {
    const size_t n = v->count * ST_VOX;
    int rc = sc.alloc(flags, n);
    if (!rc) rc = sc.alloc(pos, n);
    if (rc) return rc;
    CPHB_LAUNCH(st_flag_kernel, (unsigned)(v->count * 16), 256, 0, s, st_view(v), mode, *flags);
    return cphb_compact_flags(*flags, n, *pos, m, s);
}

extern "C" int cphb_stsdf_extract_points(const cphb_stsdf *v, float *points, float *normals, float *colors, size_t capacity,
                                         size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_stsdf_extract_points";
    if (!v || !h_count) return st_invalid(who, "null argument");
    *h_count = 0;
    if (capacity && (!points || !normals || (v->ct != TSDF_NO_COLOR && !colors))) return st_invalid(who, "null output");
    if (!v->count) return CPHB_OK;
    cphb_scratch sc(s);
    uint8_t *flags = nullptr;
    int32_t *pos = nullptr;
    size_t m = 0;
    int rc = st_flag_compact(v, 0, sc, &flags, &pos, &m, s);
    if (rc) return rc;
    unsigned long long *cnt = nullptr, *off = nullptr;
    rc = sc.alloc(&cnt, m + 1);
    if (!rc) rc = sc.alloc(&off, m + 1);
    if (rc) return rc;
    CPHB_LAUNCH(st_popc_kernel, st_blocks(m + 1, 256), 256, 0, s, pos, m, flags, cnt);
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, cnt, off, (int64_t)(m + 1), s));
    char *tmp = nullptr;
    rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, cnt, off, (int64_t)(m + 1), s));
    g_cphb_launches += 2;
    unsigned long long total = 0;
    rc = cphb_read_back(&total, off + m, sizeof(total), s, who);
    if (rc) return rc;
    const size_t mw = total && capacity >= total ? m : 0;
    if (mw) {
#define ST_POINTS(CT) CPHB_LAUNCH(st_points_kernel<CT>, st_blocks(mw, 128), 128, 0, s, st_view(v), pos, mw, flags, off, points, normals, colors)
        if (v->ct == TSDF_RGB8)
            ST_POINTS(TSDF_RGB8);
        else if (v->ct == TSDF_GRAY32)
            ST_POINTS(TSDF_GRAY32);
        else
            ST_POINTS(TSDF_NO_COLOR);
#undef ST_POINTS
    }
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_count = (size_t)total;
    return rc;
}

extern "C" int cphb_stsdf_extract_voxels(const cphb_stsdf *v, float *points, float *colors, size_t capacity, size_t *h_count,
                                         void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_stsdf_extract_voxels";
    if (!v || !h_count) return st_invalid(who, "null argument");
    *h_count = 0;
    if (capacity && (!points || !colors)) return st_invalid(who, "null output");
    if (!v->count) return CPHB_OK;
    cphb_scratch sc(s);
    uint8_t *flags = nullptr;
    int32_t *pos = nullptr;
    size_t m = 0;
    int rc = st_flag_compact(v, 1, sc, &flags, &pos, &m, s);
    if (rc) return rc;
    if (m && capacity >= m) CPHB_LAUNCH(st_voxels_kernel, st_blocks(m, 256), 256, 0, s, st_view(v), pos, m, points, colors);
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_count = m;
    return rc;
}
