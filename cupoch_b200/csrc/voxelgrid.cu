// voxelgrid.cu -- VoxelGrid::CreateFromPointCloudWithinBounds (voxelgrid_factory.cu:164-219; SURVEY 8f rank 2).
//
// The reference computes an int3 key per point, sorts the (key, Voxel) pairs with a comparison sort,
// reduce_by_key's the colours and divides by the counts.  Here: the key is packed into 64 bits relative to the
// smallest grid index that occurs (so points below min_bound, whose indices are negative, pack as well), one
// stable radix sort over exactly the bits that can differ, head flags + stable compaction for the segment
// starts, and one thread per voxel adds its points' colours in float64 in original index order (the stable sort
// keeps it) -- the same order and arithmetic as the CPU restatement the tests compare with, so the parity is
// bit-exact.
#include <math.h>

#include <cub/device/device_scan.cuh>

#include "voxelkey.cuh"

struct VgParams {
    float org[3];
    float voxel;
    int kmin[3];
    int sz, sy;  // shifts of the y and x fields
};

// voxelgrid_factory.cu:73-76: floor((p - min_bound) / voxel_size), IEEE subtraction and division
__device__ __forceinline__ int vg_index(float p, float org, float voxel) {
    return (int)floorf(__fdiv_rn(__fsub_rn(p, org), voxel));
}

__global__ void __launch_bounds__(256) vg_key_kernel(const float *__restrict__ pts, size_t n, VgParams P,
                                                     unsigned long long *__restrict__ keys, uint32_t *__restrict__ vals) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long kx = (unsigned long long)(long long)(vg_index(pts[3 * i], P.org[0], P.voxel) - P.kmin[0]);
    const unsigned long long ky = (unsigned long long)(long long)(vg_index(pts[3 * i + 1], P.org[1], P.voxel) - P.kmin[1]);
    const unsigned long long kz = (unsigned long long)(long long)(vg_index(pts[3 * i + 2], P.org[2], P.voxel) - P.kmin[2]);
    keys[i] = (kx << P.sy) | (ky << P.sz) | kz;
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) vg_head_kernel(const unsigned long long *__restrict__ sorted, size_t n,
                                                      uint8_t *__restrict__ head) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    head[i] = (i == 0 || sorted[i] != sorted[i - 1]) ? 1 : 0;
}

__global__ void __launch_bounds__(256) vg_reduce_kernel(const unsigned long long *__restrict__ sorted,
                                                        const uint32_t *__restrict__ order, const int32_t *__restrict__ starts,
                                                        size_t n_out, size_t n, const float *__restrict__ colors, VgParams P,
                                                        int32_t *__restrict__ out_keys, float *__restrict__ out_colors) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v >= n_out) return;
    const size_t b = (size_t)starts[v], e = (v + 1 < n_out) ? (size_t)starts[v + 1] : n;
    const unsigned long long key = sorted[b];
    const unsigned long long mz = (P.sz >= 64) ? ~0ull : ((1ull << P.sz) - 1ull);
    const unsigned long long my = (P.sy - P.sz >= 64) ? ~0ull : ((1ull << (P.sy - P.sz)) - 1ull);
    out_keys[3 * v] = (int32_t)((long long)(key >> P.sy) + P.kmin[0]);
    out_keys[3 * v + 1] = (int32_t)((long long)((key >> P.sz) & my) + P.kmin[1]);
    out_keys[3 * v + 2] = (int32_t)((long long)(key & mz) + P.kmin[2]);
    if (colors) {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (size_t t = b; t < e; ++t) {
            const size_t i = order[t];
            s0 += (double)colors[3 * i];
            s1 += (double)colors[3 * i + 1];
            s2 += (double)colors[3 * i + 2];
        }
        const float cnt = (float)(e - b);
        out_colors[3 * v] = __fdiv_rn((float)s0, cnt);      // divide_voxel_color_functor (voxelgrid.h:75-82)
        out_colors[3 * v + 1] = __fdiv_rn((float)s1, cnt);
        out_colors[3 * v + 2] = __fdiv_rn((float)s2, cnt);
    } else {  // Voxel's default colour (voxelgrid.h:61)
        out_colors[3 * v] = 1.f;
        out_colors[3 * v + 1] = 1.f;
        out_colors[3 * v + 2] = 1.f;
    }
}

static int bits_for_span(long long cells) {  // bits needed for values 0 .. cells-1
    int b = 1;
    while (b < 63 && (1ll << b) < cells) ++b;
    return b;
}

extern "C" int cphb_voxel_grid_from_point_cloud(const float *points, const float *colors, size_t n, float voxel_size,
                                                const float h_min_bound[3], const float h_max_bound[3], int32_t *out_keys,
                                                float *out_colors, size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out || !h_min_bound || !h_max_bound) {
        cphb_set_error("cphb_voxel_grid_from_point_cloud: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    // the reference only logs these two (voxelgrid_factory.cu:170-177) and goes on to divide by the bad size;
    // an empty grid is the defined behaviour here
    if (voxel_size <= 0.0f || n == 0) return CPHB_OK;
    float ext = 0.f;
    for (int a = 0; a < 3; ++a)
        if (h_max_bound[a] - h_min_bound[a] > ext) ext = h_max_bound[a] - h_min_bound[a];
    if (voxel_size * (float)2147483647 < ext) return CPHB_OK;
    if (!points || !out_keys || !out_colors) {
        cphb_set_error("cphb_voxel_grid_from_point_cloud: null argument");
        return CPHB_ERR_INVALID;
    }
    if (n > 0x7fffffffull) {
        cphb_set_error("cphb_voxel_grid_from_point_cloud: n exceeds int32");
        return CPHB_ERR_INVALID;
    }
    float mn[3], mx[3];
    int rc = cphb_min_max_bound(points, n, mn, mx, stream);
    if (rc) return rc;
    VgParams P;
    P.voxel = voxel_size;
    long long span[3];
    for (int a = 0; a < 3; ++a) {
        P.org[a] = h_min_bound[a];
        // floor((x - org) / voxel) is monotone in x: every point's index lies between those of the bounds
        const volatile float dlo = mn[a] - h_min_bound[a], dhi = mx[a] - h_min_bound[a];
        const volatile float qlo = dlo / voxel_size, qhi = dhi / voxel_size;
        const double klo = floor((double)qlo), khi = floor((double)qhi);
        if (!(klo >= -2147483648.0 && khi <= 2147483647.0)) {
            cphb_set_error("cphb_voxel_grid_from_point_cloud: grid index outside int32 (voxel_size too small for the bounds)");
            return CPHB_ERR_UNSUPPORTED;
        }
        P.kmin[a] = (int)klo;
        span[a] = (long long)khi - (long long)klo + 1;
    }
    const int bx = bits_for_span(span[0]), by = bits_for_span(span[1]), bz = bits_for_span(span[2]);
    if (bx + by + bz > 64) {
        cphb_set_error("cphb_voxel_grid_from_point_cloud: grid needs %d key bits (> 64)", bx + by + bz);
        return CPHB_ERR_UNSUPPORTED;
    }
    P.sz = bz;
    P.sy = by + bz;

    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = cphb_align(off + bytes, 256); return o; };
    const size_t o_k = take(n * 8), o_k2 = take(n * 8), o_v = take(n * 4), o_ord = take(n * 4), o_head = take(n), o_st = take(n * 4);
    cphb_scratch sc(s);
    char *base = nullptr;
    rc = sc.alloc(&base, off);
    if (rc) return rc;
    unsigned long long *keys = (unsigned long long *)(base + o_k), *keys2 = (unsigned long long *)(base + o_k2);
    uint32_t *vals = (uint32_t *)(base + o_v), *order = (uint32_t *)(base + o_ord);
    uint8_t *head = (uint8_t *)(base + o_head);
    int32_t *starts = (int32_t *)(base + o_st);
    const unsigned grid = (unsigned)((n + 255) / 256);
    CPHB_LAUNCH(vg_key_kernel, grid, 256, 0, s, points, n, P, keys, vals);
    rc = cphb_sort_pairs_u64((const uint64_t *)keys, (uint64_t *)keys2, vals, order, n, bx + by + bz, s);
    size_t n_out = 0;
    if (!rc) {
        CPHB_LAUNCH(vg_head_kernel, grid, 256, 0, s, keys2, n, head);
        rc = cphb_compact_flags(head, n, starts, &n_out, s);
    }
    if (!rc && n_out) {
        CPHB_LAUNCH(vg_reduce_kernel, (unsigned)((n_out + 255) / 256), 256, 0, s, keys2, order, starts, n_out, n, colors, P, out_keys,
                    out_colors);
        rc = cphb_read_back(nullptr, nullptr, 0, s, "cphb_voxel_grid_from_point_cloud");
    }
    sc.release();
    cudaStreamSynchronize(s);
    if (!rc) *h_n_out = n_out;
    return rc;
}

// Batched VoxelGrid::GetVoxel (voxelgrid.cu:338-341): out[i] = floor((p_i - origin) / voxel_size) per axis, the
// arithmetic every voxel kernel of this library uses for its keys -- callers that must agree with those keys (the
// slab partition of the sharded VoxelDownSample) take the indices from here instead of recomputing them.
__global__ void __launch_bounds__(256) vg_indices_kernel(const float *__restrict__ pts, size_t n, float ox, float oy, float oz,
                                                         float voxel, int32_t *__restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[3 * i] = vg_index(pts[3 * i], ox, voxel);
    out[3 * i + 1] = vg_index(pts[3 * i + 1], oy, voxel);
    out[3 * i + 2] = vg_index(pts[3 * i + 2], oz, voxel);
}

extern "C" int cphb_voxel_indices(const float *points, size_t n, float voxel_size, const float h_origin[3], int32_t *out_indices,
                                  void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return CPHB_OK;
    if (!points || !h_origin || !out_indices || !(voxel_size > 0.f)) {
        cphb_set_error("cphb_voxel_indices: invalid argument");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(vg_indices_kernel, (unsigned)((n + 255) / 256), 256, 0, s, points, n, h_origin[0], h_origin[1], h_origin[2], voxel_size,
                out_indices);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// The rest of VoxelGrid (voxelgrid.cu:235-475, voxelgrid_factory.cu:134-162,283-305; SURVEY 8f rank 12).  Every
// operation is a fixed number of coalesced passes: CreateDense writes keys already in lexicographic order (no sort, no
// unique); lookups and merges go through the packed-key sort of voxelkey.cuh (one sort per call, then a binary
// search per query or a head-flag compaction); carving and the inverted selection are a flag kernel, the stable
// compaction and a gather, so survivors keep their order.
// ---------------------------------------------------------------------------------------------------------------------
#define VGO_BLOCK 256
static unsigned vgo_grid(size_t n) { return (unsigned)((n + VGO_BLOCK - 1) / VGO_BLOCK); }
// at least one block: a launch whose work can be empty (no survivors) still happens, so the launch count of a call does
// not depend on its data
static unsigned vgo_grid1(size_t n) { return n ? vgo_grid(n) : 1u; }
static unsigned vgo_capped(size_t n) {
    const unsigned g = vgo_grid(n);
    return g < CPHB_SMS * 32 ? g : CPHB_SMS * 32;
}
static int vgo_invalid(const char *who, const char *what) {
    cphb_set_error("%s: %s", who, what);
    return CPHB_ERR_INVALID;
}

// create_dense_functor (voxelgrid_factory.cu:42-55): voxel i is (i / (nh nd), (i / nd) % nh, i % nd)
template <class I>
__global__ void __launch_bounds__(VGO_BLOCK) vgo_dense_kernel(I total, I nh, I nd, int32_t *__restrict__ keys, float *__restrict__ colors) {
    for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
        const I hd = nh * nd;
        const I w = i / hd, r = i - w * hd, h = r / nd;
        keys[3 * (size_t)i] = (int32_t)w;
        keys[3 * (size_t)i + 1] = (int32_t)h;
        keys[3 * (size_t)i + 2] = (int32_t)(r - h * nd);
        colors[3 * (size_t)i] = 1.f;
        colors[3 * (size_t)i + 1] = 1.f;
        colors[3 * (size_t)i + 2] = 1.f;
    }
}

extern "C" int cphb_voxel_grid_create_dense(float voxel_size, float width, float height, float depth, int32_t *out_keys,
                                            float *out_colors, size_t capacity, size_t *h_n, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_create_dense";
    if (!h_n) return vgo_invalid(who, "null argument");
    *h_n = 0;
    if (!(isfinite(voxel_size) && voxel_size > 0.f)) return vgo_invalid(who, "voxel_size is not positive and finite");
    const float ext[3] = {width, height, depth};
    unsigned long long cnt[3];
    for (int a = 0; a < 3; ++a) {
        const volatile float q = ext[a] / voxel_size;  // int(std::round(w / voxel_size)) in float
        const float c = roundf(q);
        if (!(c >= 0.f && c < 2147483648.f)) {
            cphb_set_error("%s: axis %d count round(%g / %g) is negative, not finite or >= 2^31", who, a, (double)ext[a],
                           (double)voxel_size);
            return CPHB_ERR_INVALID;
        }
        cnt[a] = (unsigned long long)c;
    }
    // the total in 64 bits, with its keys and colours (24 bytes a voxel) addressable by size_t
    const unsigned long long lim = (unsigned long long)(SIZE_MAX / 24);
    unsigned long long total = cnt[0];
    if (cnt[1] && total > lim / cnt[1]) return vgo_invalid(who, "voxel count overflows");
    total *= cnt[1];
    if (cnt[2] && total > lim / cnt[2]) return vgo_invalid(who, "voxel count overflows");
    total *= cnt[2];
    *h_n = (size_t)total;
    if (total == 0 || capacity < total) return CPHB_OK;
    if (!out_keys || !out_colors) return vgo_invalid(who, "null output");
    // the 32-bit index path only when the grid-stride step cannot wrap past 2^32
    if (total <= 0xffffffffull - (unsigned long long)vgo_capped(total) * VGO_BLOCK)
        CPHB_LAUNCH(vgo_dense_kernel<uint32_t>, vgo_capped(total), VGO_BLOCK, 0, s, (uint32_t)total, (uint32_t)cnt[1], (uint32_t)cnt[2],
                    out_keys, out_colors);
    else
        CPHB_LAUNCH(vgo_dense_kernel<unsigned long long>, vgo_capped(total), VGO_BLOCK, 0, s, total, cnt[1], cnt[2], out_keys, out_colors);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// CheckIfIncluded: the GetVoxel cell of each query, looked up among the sorted packed keys
__global__ void __launch_bounds__(VGO_BLOCK) vgo_included_kernel(const uint64_t *__restrict__ skeys, size_t n, int3 lo3, int3 hi3,
                                                                 float voxel, float ox, float oy, float oz,
                                                                 const float *__restrict__ q, size_t nq, uint8_t *__restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const int lo[3] = {lo3.x, lo3.y, lo3.z}, hi[3] = {hi3.x, hi3.y, hi3.z};
    const float o[3] = {ox, oy, oz};
    int k[3];
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        // vg_index's expression; a NaN or out-of-range floor fails the test before the cast
        const float f = floorf(__fdiv_rn(__fsub_rn(q[3 * i + a], o[a]), voxel));
        in = in && (double)f >= (double)lo[a] && (double)f <= (double)hi[a];
        k[a] = in ? (int)f : lo[a];
    }
    if (in) {
        const uint64_t key = cphb_key_pack(lo, k[0], k[1], k[2]);
        const size_t p = cphb_key_lower_bound(skeys, n, key);
        in = p < n && skeys[p] == key;
    }
    out[i] = in ? 1 : 0;
}

extern "C" int cphb_voxel_grid_check_if_included(const int32_t *keys, size_t n, float voxel_size, const float h_origin[3],
                                                 const float *queries, size_t nq, uint8_t *out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_check_if_included";
    if (!h_origin || (n && !keys) || (nq && (!queries || !out))) return vgo_invalid(who, "null argument");
    if (n && !(isfinite(voxel_size) && voxel_size > 0.f)) return vgo_invalid(who, "voxel_size is not positive and finite");
    if (n > (size_t)INT32_MAX) return vgo_invalid(who, "more than 2^31-1 voxels");
    if (nq == 0) return CPHB_OK;
    if (n == 0) {
        CPHB_CUDA(cudaMemsetAsync(out, 0, nq, s));
        return cphb_read_back(nullptr, nullptr, 0, s, who);
    }
    cphb_scratch sc(s);
    cphb_sorted_keys sk;
    int rc = cphb_sort_voxel_keys(keys, n, sc, &sk, s, who);
    if (rc) return rc;
    CPHB_LAUNCH(vgo_included_kernel, vgo_grid(nq), VGO_BLOCK, 0, s, sk.skeys, n, make_int3(sk.lo[0], sk.lo[1], sk.lo[2]),
                make_int3(sk.hi[0], sk.hi[1], sk.hi[2]), voxel_size, h_origin[0], h_origin[1], h_origin[2], queries, nq, out);
    return cphb_read_back(nullptr, nullptr, 0, s, who);
}

__global__ void __launch_bounds__(VGO_BLOCK) vgo_has_key_kernel(const int32_t *__restrict__ keys, size_t n, int x, int y, int z,
                                                                int *found) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (keys[3 * i] == x && keys[3 * i + 1] == y && keys[3 * i + 2] == z) *found = 1;
}

extern "C" int cphb_voxel_grid_has_key(const int32_t *keys, size_t n, const int32_t h_key[3], int *h_found, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_has_key";
    if (!h_key || !h_found || (n && !keys)) return vgo_invalid(who, "null argument");
    *h_found = 0;
    if (n == 0) return CPHB_OK;
    cphb_scratch sc(s);
    int *d_found = nullptr;
    int rc = sc.alloc(&d_found, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(d_found, 0, sizeof(int), s));
    CPHB_LAUNCH(vgo_has_key_kernel, vgo_capped(n), VGO_BLOCK, 0, s, keys, n, h_key[0], h_key[1], h_key[2], d_found);
    return cphb_read_back(h_found, d_found, sizeof(int), s, who);
}

// ------------------------------------------------------------------------------------------------ carving
struct VgoCamera {
    float K[9], R[9], t[3];
    float o[3], voxel;
    int width, height;
    int sampled;  // the image is 1-channel float32 (FloatValueAt's only readable kind)
    int keep_outside;
};

// FloatValueAt (image.h:240-270) with the defined outside cases: z == 0 or a non-finite u / v is outside
__device__ __forceinline__ bool vgo_sample(const float *__restrict__ img, const VgoCamera &c, float u, float v, float z, float &d) {
    if (!c.sampled || z == 0.f || !isfinite(u) || !isfinite(v) || u < 0.f || u > (float)(c.width - 1) || v < 0.f ||
        v > (float)(c.height - 1))
        return false;
    const int ui = max(min((int)u, c.width - 2), 0), vi = max(min((int)v, c.height - 2), 0);
    const float pu = __fsub_rn(u, (float)ui), pv = __fsub_rn(v, (float)vi);
    const float v0 = __ldg(img + (size_t)vi * c.width + ui), v1 = __ldg(img + (size_t)(vi + 1) * c.width + ui);
    const float v2 = __ldg(img + (size_t)vi * c.width + ui + 1), v3 = __ldg(img + (size_t)(vi + 1) * c.width + ui + 1);
    const float qv = __fsub_rn(1.f, pv), qu = __fsub_rn(1.f, pu);
    const float a = __fadd_rn(__fmul_rn(v0, qv), __fmul_rn(v1, pv)), b = __fadd_rn(__fmul_rn(v2, qv), __fmul_rn(v3, pv));
    d = __fadd_rn(__fmul_rn(a, qu), __fmul_rn(b, pu));
    return true;
}

// compute_carve_functor (voxelgrid.cu:58-123), keep[i] = !carve.  The projection's expression order (oracle/voxelgrid_ops.c
// restates it): centre c = ((float)k + 0.5f) * vs + o; corner p = c +- vs / 2 in GetVoxelBoundingPoints' order;
// x = fma(R2, p2, fma(R1, p1, R0 * p0)) + t per row; (u', v', z) = fma(K2, x2, fma(K1, x1, K0 * x0)) per row;
// u = u' / z, v = v' / z.
__global__ void __launch_bounds__(VGO_BLOCK) vgo_carve_kernel(const int32_t *__restrict__ keys, size_t n, const float *__restrict__ img,
                                                              const VgoCamera c, uint8_t *__restrict__ keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float r = __fmul_rn(c.voxel, 0.5f);
    float ctr[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) ctr[a] = __fadd_rn(__fmul_rn(__fadd_rn((float)keys[3 * i + a], 0.5f), c.voxel), c.o[a]);
    bool kept = false;
#pragma unroll 1
    for (int j = 0; j < 8 && !kept; ++j) {
        const float p[3] = {__fadd_rn(ctr[0], (j & 2) ? r : -r), __fadd_rn(ctr[1], (j & 4) ? r : -r), __fadd_rn(ctr[2], (j & 1) ? r : -r)};
        float x[3], w[3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            x[a] = __fadd_rn(__fmaf_rn(c.R[3 * a + 2], p[2], __fmaf_rn(c.R[3 * a + 1], p[1], __fmul_rn(c.R[3 * a], p[0]))), c.t[a]);
#pragma unroll
        for (int a = 0; a < 3; ++a) w[a] = __fmaf_rn(c.K[3 * a + 2], x[2], __fmaf_rn(c.K[3 * a + 1], x[1], __fmul_rn(c.K[3 * a], x[0])));
        const float z = w[2], u = __fdiv_rn(w[0], z), v = __fdiv_rn(w[1], z);
        float d = 0.f;
        const bool within = vgo_sample(img, c, u, v, z, d);
        kept = (!within && c.keep_outside) || (within && d > 0.f && z >= d);
    }
    keep[i] = kept ? 1 : 0;
}

template <class I>
__global__ void __launch_bounds__(VGO_BLOCK) vgo_gather_kernel(const I *__restrict__ sel, size_t m, const int32_t *__restrict__ keys,
                                                               const float *__restrict__ colors, int32_t *__restrict__ out_keys,
                                                               float *__restrict__ out_colors) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    const size_t i = (size_t)sel[t];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        out_keys[3 * t + a] = keys[3 * i + a];
        out_colors[3 * t + a] = colors[3 * i + a];
    }
}

extern "C" int cphb_voxel_grid_carve(const int32_t *keys, const float *colors, size_t n, float voxel_size, const float h_origin[3],
                                     const void *image, int width, int height, int num_of_channels, int bytes_per_channel,
                                     const float h_intrinsic[9], const float h_extrinsic[16], int keep_outside, int32_t *out_keys,
                                     float *out_colors, size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_carve";
    if (!h_n_out || !h_origin || !h_intrinsic || !h_extrinsic) return vgo_invalid(who, "null argument");
    *h_n_out = 0;
    if (width < 2 || height < 2) return vgo_invalid(who, "the image is narrower or lower than 2 pixels");
    VgoCamera c;
    c.sampled = num_of_channels == 1 && bytes_per_channel == 4;
    if (c.sampled && !image) return vgo_invalid(who, "null image");
    if (n == 0) return CPHB_OK;
    if (!keys || !colors || !out_keys || !out_colors) return vgo_invalid(who, "null argument");
    if (n > (size_t)INT32_MAX) return vgo_invalid(who, "more than 2^31-1 voxels");
    for (int a = 0; a < 9; ++a) c.K[a] = h_intrinsic[a];
    for (int r = 0; r < 3; ++r) {
        for (int q = 0; q < 3; ++q) c.R[3 * r + q] = h_extrinsic[4 * r + q];
        c.t[r] = h_extrinsic[4 * r + 3];
        c.o[r] = h_origin[r];
    }
    c.voxel = voxel_size;
    c.width = width;
    c.height = height;
    c.keep_outside = keep_outside ? 1 : 0;
    cphb_scratch sc(s);
    uint8_t *keep = nullptr;
    int32_t *sel = nullptr;
    int rc = sc.alloc(&keep, n);
    if (!rc) rc = sc.alloc(&sel, n);
    if (rc) return rc;
    CPHB_LAUNCH(vgo_carve_kernel, vgo_grid(n), VGO_BLOCK, 0, s, keys, n, c.sampled ? (const float *)image : nullptr, c, keep);
    size_t m = 0;
    rc = cphb_compact_flags(keep, n, sel, &m, s);
    if (rc) return rc;
    CPHB_LAUNCH(vgo_gather_kernel<int32_t>, vgo_grid1(m), VGO_BLOCK, 0, s, sel, m, keys, colors, out_keys, out_colors);
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_n_out = m;
    return rc;
}

// ------------------------------------------------------------------------------------------------ += and AddVoxels
// one thread per run of equal keys: a's voxels precede b's in the concatenation and the stable sort keeps that order
__global__ void __launch_bounds__(VGO_BLOCK) vgo_merge_kernel(const uint32_t *__restrict__ sidx, const int32_t *__restrict__ starts,
                                                              size_t n_out, size_t n, const int32_t *__restrict__ keys,
                                                              const float *__restrict__ colors, int average,
                                                              int32_t *__restrict__ out_keys, float *__restrict__ out_colors) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v >= n_out) return;
    const size_t b = (size_t)starts[v], e = (v + 1 < n_out) ? (size_t)starts[v + 1] : n;
    const size_t f = sidx[b];
    float c[3] = {colors[3 * f], colors[3 * f + 1], colors[3 * f + 2]};
    if (average) {
        for (size_t t = b + 1; t < e; ++t) {  // add_voxel_color_functor, left to right
            const size_t i = sidx[t];
#pragma unroll
            for (int a = 0; a < 3; ++a) c[a] = __fadd_rn(c[a], colors[3 * i + a]);
        }
        const float cnt = (float)(int)(e - b);  // divide_voxel_color_functor (voxelgrid.h:75-82)
#pragma unroll
        for (int a = 0; a < 3; ++a) c[a] = __fdiv_rn(c[a], cnt);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        out_keys[3 * v + a] = keys[3 * f + a];
        out_colors[3 * v + a] = c[a];
    }
}

extern "C" int cphb_voxel_grid_merge(const int32_t *keys_a, const float *colors_a, size_t na, const int32_t *keys_b,
                                     const float *colors_b, size_t nb, int average, int32_t *out_keys, float *out_colors,
                                     size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_merge";
    if (!h_n_out || (na && (!keys_a || !colors_a)) || (nb && (!keys_b || !colors_b))) return vgo_invalid(who, "null argument");
    *h_n_out = 0;
    const size_t n = na + nb;
    if (n == 0) return CPHB_OK;
    if (!out_keys || !out_colors) return vgo_invalid(who, "null output");
    if (na > (size_t)INT32_MAX || nb > (size_t)INT32_MAX || n > (size_t)INT32_MAX) return vgo_invalid(who, "more than 2^31-1 voxels");
    cphb_scratch sc(s);
    int32_t *keys = nullptr, *starts = nullptr;
    float *colors = nullptr;
    uint8_t *head = nullptr;
    int rc = sc.alloc(&keys, 3 * n);
    if (!rc) rc = sc.alloc(&colors, 3 * n);
    if (!rc) rc = sc.alloc(&head, n);
    if (!rc) rc = sc.alloc(&starts, n);
    if (rc) return rc;
    if (na) {
        CPHB_CUDA(cudaMemcpyAsync(keys, keys_a, 12 * na, cudaMemcpyDeviceToDevice, s));
        CPHB_CUDA(cudaMemcpyAsync(colors, colors_a, 12 * na, cudaMemcpyDeviceToDevice, s));
    }
    if (nb) {
        CPHB_CUDA(cudaMemcpyAsync(keys + 3 * na, keys_b, 12 * nb, cudaMemcpyDeviceToDevice, s));
        CPHB_CUDA(cudaMemcpyAsync(colors + 3 * na, colors_b, 12 * nb, cudaMemcpyDeviceToDevice, s));
    }
    cphb_sorted_keys sk;
    rc = cphb_sort_voxel_keys(keys, n, sc, &sk, s, who);
    if (rc) return rc;
    CPHB_LAUNCH(vg_head_kernel, vgo_grid(n), VGO_BLOCK, 0, s, (const unsigned long long *)sk.skeys, n, head);
    size_t n_out = 0;
    rc = cphb_compact_flags(head, n, starts, &n_out, s);
    if (rc) return rc;
    CPHB_LAUNCH(vgo_merge_kernel, vgo_grid(n_out), VGO_BLOCK, 0, s, sk.sidx, starts, n_out, n, keys, colors, average ? 1 : 0, out_keys,
                out_colors);
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_n_out = n_out;
    return rc;
}

// ------------------------------------------------------------------------------------------------ paint and select
__global__ void __launch_bounds__(VGO_BLOCK) vgo_bad_index_kernel(const int64_t *__restrict__ idx, size_t m, long long n, int *bad) {
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < m; t += (size_t)gridDim.x * blockDim.x)
        if (idx[t] < 0 || idx[t] >= n) *bad = 1;
}
__global__ void __launch_bounds__(VGO_BLOCK) vgo_paint_kernel(float *__restrict__ colors, const int64_t *__restrict__ idx, size_t m,
                                                              float c0, float c1, float c2) {
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < m; t += (size_t)gridDim.x * blockDim.x) {
        const size_t i = idx ? (size_t)idx[t] : t;
        colors[3 * i] = c0;
        colors[3 * i + 1] = c1;
        colors[3 * i + 2] = c2;
    }
}
__global__ void __launch_bounds__(VGO_BLOCK) vgo_unmark_kernel(const int64_t *__restrict__ idx, size_t m, uint8_t *keep) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t < m) keep[idx[t]] = 0;
}

// CPHB_ERR_INVALID when an index is outside [0, n); synchronises
static int vgo_check_indices(const int64_t *idx, size_t m, size_t n, cphb_scratch &sc, cudaStream_t s, const char *who) {
    int *d_bad = nullptr;
    int rc = sc.alloc(&d_bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), s));
    CPHB_LAUNCH(vgo_bad_index_kernel, m ? vgo_capped(m) : 1u, VGO_BLOCK, 0, s, idx, m, (long long)n, d_bad);
    int bad = 0;
    rc = cphb_read_back(&bad, d_bad, sizeof(int), s, who);
    if (rc) return rc;
    if (bad) {
        cphb_set_error("%s: an index is outside [0, %zu)", who, n);
        return CPHB_ERR_INVALID;
    }
    return CPHB_OK;
}

extern "C" int cphb_voxel_grid_paint(float *colors, size_t n, const int64_t *indices, size_t m, const float h_color[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_paint";
    if (!h_color || (n && !colors) || (indices == nullptr && m != 0) || (m && !indices)) return vgo_invalid(who, "null argument");
    const size_t cnt = indices ? m : n;
    if (cnt == 0) return CPHB_OK;
    cphb_scratch sc(s);
    if (indices) {
        const int rc = vgo_check_indices(indices, m, n, sc, s, who);
        if (rc) return rc;
    }
    CPHB_LAUNCH(vgo_paint_kernel, vgo_capped(cnt), VGO_BLOCK, 0, s, colors, indices, cnt, h_color[0], h_color[1], h_color[2]);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

extern "C" int cphb_voxel_grid_select_by_index(const int32_t *keys, const float *colors, size_t n, const int64_t *indices, size_t m,
                                               int invert, int32_t *out_keys, float *out_colors, size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_select_by_index";
    if (!h_n_out || (n && (!keys || !colors)) || (m && !indices)) return vgo_invalid(who, "null argument");
    *h_n_out = 0;
    if (n > (size_t)INT32_MAX) return vgo_invalid(who, "more than 2^31-1 voxels");
    const size_t rows = invert ? n : m;
    if (rows && (!out_keys || !out_colors)) return vgo_invalid(who, "null output");
    cphb_scratch sc(s);
    if (rows == 0) return CPHB_OK;
    int rc = vgo_check_indices(indices, m, n, sc, s, who);
    if (rc) return rc;
    size_t w = m;
    if (!invert) {
        CPHB_LAUNCH(vgo_gather_kernel<int64_t>, vgo_grid(m), VGO_BLOCK, 0, s, indices, m, keys, colors, out_keys, out_colors);
    } else {
        uint8_t *keep = nullptr;
        int32_t *sel = nullptr;
        rc = sc.alloc(&keep, n);
        if (!rc) rc = sc.alloc(&sel, n);
        if (rc) return rc;
        CPHB_CUDA(cudaMemsetAsync(keep, 1, n, s));
        CPHB_LAUNCH(vgo_unmark_kernel, vgo_grid1(m), VGO_BLOCK, 0, s, indices, m, keep);
        rc = cphb_compact_flags(keep, n, sel, &w, s);
        if (rc) return rc;
        CPHB_LAUNCH(vgo_gather_kernel<int32_t>, vgo_grid1(w), VGO_BLOCK, 0, s, sel, w, keys, colors, out_keys, out_colors);
    }
    rc = cphb_read_back(nullptr, nullptr, 0, s, who);
    if (!rc) *h_n_out = w;
    return rc;
}

// ------------------------------------------------------------------------------------------------ from an OccupancyGrid
// compute_points_from_occvoxels_functor (pointcloud_factory.cu:239-256): (cell + c) * vs + o, c = (float)(-res / 2 + 0.5)
__global__ void __launch_bounds__(VGO_BLOCK) vgo_occ_points_kernel(const int32_t *__restrict__ cells, size_t m, float c, float voxel,
                                                                   float ox, float oy, float oz, float *__restrict__ pts,
                                                                   float *__restrict__ colors) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    const float o[3] = {ox, oy, oz};
#pragma unroll
    for (int a = 0; a < 3; ++a) pts[3 * t + a] = __fadd_rn(__fmul_rn(__fadd_rn((float)cells[3 * t + a], c), voxel), o[a]);
    colors[3 * t] = 0.f;  // OccupancyVoxel's colour (occupancygrid.h:33-72)
    colors[3 * t + 1] = 0.f;
    colors[3 * t + 2] = 1.f;
}

static int vgo_occ_check(const cphb_occgrid *grid, float *vs, float o[3], int *res, const char *who) {
    if (!grid) return vgo_invalid(who, "null OccupancyGrid");
    cphb_occgrid_geometry(grid, vs, o);
    cphb_occgrid_view v;
    cphb_occgrid_view_of(grid, &v);
    *res = v.res;
    if (!(*vs > 0.f)) return vgo_invalid(who, "occupancy grid voxel_size <= 0");  // voxelgrid_factory.cu:287-290
    return CPHB_OK;
}

extern "C" int cphb_voxel_grid_from_occgrid(const cphb_occgrid *grid, int32_t *out_keys, float *out_colors, size_t capacity,
                                            size_t *h_count, float h_origin[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_from_occgrid";
    if (!h_count || !h_origin) return vgo_invalid(who, "null argument");
    *h_count = 0;
    float vs, o[3];
    int res;
    int rc = vgo_occ_check(grid, &vs, o, &res, who);
    if (rc) return rc;
    const float half = (float)(res / 2);
    for (int a = 0; a < 3; ++a) h_origin[a] = o[a] - half * vs;
    if (capacity && (!out_keys || !out_colors)) return vgo_invalid(who, "null output");
    size_t cnt = 0;
    rc = cphb_occgrid_extract(grid, 2, capacity ? out_keys : nullptr, nullptr, capacity, &cnt, stream);
    if (rc) return rc;
    *h_count = cnt;
    if (cnt == 0 || capacity < cnt) return cphb_read_back(nullptr, nullptr, 0, s, who);
    CPHB_LAUNCH(vgo_paint_kernel, vgo_capped(cnt), VGO_BLOCK, 0, s, out_colors, nullptr, cnt, 0.f, 0.f, 1.f);
    return cphb_read_back(nullptr, nullptr, 0, s, who);
}

extern "C" int cphb_point_cloud_from_occgrid(const cphb_occgrid *grid, float *out_points, float *out_colors, size_t capacity,
                                             size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_point_cloud_from_occgrid";
    if (!h_count) return vgo_invalid(who, "null argument");
    *h_count = 0;
    float vs, o[3];
    int res;
    int rc = vgo_occ_check(grid, &vs, o, &res, who);
    if (rc) return rc;
    if (capacity && (!out_points || !out_colors)) return vgo_invalid(who, "null output");
    cphb_scratch sc(s);
    int32_t *cells = nullptr;
    if (capacity) {
        rc = sc.alloc(&cells, 3 * capacity);
        if (rc) return rc;
    }
    size_t cnt = 0;
    rc = cphb_occgrid_extract(grid, 2, cells, nullptr, capacity, &cnt, stream);
    if (rc) return rc;
    *h_count = cnt;
    if (cnt == 0 || capacity < cnt) return cphb_read_back(nullptr, nullptr, 0, s, who);
    const float c = (float)(-(res / 2) + 0.5);
    CPHB_LAUNCH(vgo_occ_points_kernel, vgo_grid(cnt), VGO_BLOCK, 0, s, cells, cnt, c, vs, o[0], o[1], o[2], out_points, out_colors);
    return cphb_read_back(nullptr, nullptr, 0, s, who);
}

// ------------------------------------------------------------------------------------------------ from a TriangleMesh
// CreateFromTriangleMeshWithinBounds (voxelgrid_factory.cu:229-272; DESIGN section 4 item 25).  The reference runs
// one thread per cell of the dense box and tests every triangle against it; here the work follows the surface:
//   1. one thread per triangle checks its indices and finds, per axis, the exact range of cells whose centre passes
//      the test's own box-axis comparison (a binary search on the float predicate, which is monotone in k), and its
//      dominant normal axis d.  Its work items are the columns of that box along d (the cells in the other two axes);
//   2. a 64-bit CUB exclusive scan of the column counts, then one thread per (triangle, column) finds its triangle by
//      binary search and walks the cells of the column whose centre lies within the triangle plane's reach (the
//      plane's slab in float64, widened by a bound on the float test's own rounding), testing each exactly;
//   3. the hits go through the block compaction as packed keys, the radix sort and a head-flag unique, then are
//      unpacked to [m][3].
// A degenerate triangle (zero float64 normal) walks its whole box.  The walk only has to be a superset of the cells
// that pass: the exact test decides every key, so the result does not depend on how the work is split.
#define MV_BLOCK 256

// component a of (x, y, z) for a run-time a, by selects (an indexed local array would live in local memory)
template <class T>
__host__ __device__ __forceinline__ T mv_pick(int a, T x, T y, T z) { return a == 0 ? x : (a == 1 ? y : z); }

struct MvTri {
    int lo[3], hi[3];  // per axis, the cells that pass the box-axis comparison
    int d;             // column axis; + 4 when degenerate (the whole range is walked)
};

// cell centre on one axis: ((float)k + 0.5f) * vs + o, each step rounded (carving's rule, DESIGN item 17)
// (plain operators: -fmad=false keeps every one rounded, and the host build of the tests' harness does the same)
__host__ __device__ __forceinline__ float mv_centre(int k, float vs, float o) { return ((float)k + 0.5f) * vs + o; }

__host__ __device__ __forceinline__ void mv_order(float a, float b, float &mn, float &mx) {
    if (a < b) {
        mn = a;
        mx = b;
    } else {
        mn = b;
        mx = a;
    }
}

// Akenine-Moeller's triangle/box overlap test (the separating axes: 9 edge x box-axis cross products, then the 3 box
// axes, then the triangle's plane), with the operand order and comparisons of the published triBoxOverlap.  c: box
// centre, h: half size, A, B, C: the triangle.  IEEE float32, no contraction (-fmad=false); oracle/mesh_voxel.c
// restates it.
__host__ __device__ __forceinline__ bool mv_tri_box(const float c[3], float h, const float A[3], const float B[3], const float C[3]) {
    float v0[3], v1[3], v2[3], e0[3], e1[3], e2[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        v0[q] = A[q] - c[q];
        v1[q] = B[q] - c[q];
        v2[q] = C[q] - c[q];
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        e0[q] = v1[q] - v0[q];
        e1[q] = v2[q] - v1[q];
        e2[q] = v0[q] - v2[q];
    }
    float mn, mx, p0, p1, p2, rad, fx, fy, fz;
    fx = fabsf(e0[0]), fy = fabsf(e0[1]), fz = fabsf(e0[2]);
    p0 = e0[2] * v0[1] - e0[1] * v0[2], p2 = e0[2] * v2[1] - e0[1] * v2[2];  // x * e0
    mv_order(p0, p2, mn, mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return false;
    p0 = -e0[2] * v0[0] + e0[0] * v0[2], p2 = -e0[2] * v2[0] + e0[0] * v2[2];  // y * e0
    mv_order(p0, p2, mn, mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return false;
    p1 = e0[1] * v1[0] - e0[0] * v1[1], p2 = e0[1] * v2[0] - e0[0] * v2[1];  // z * e0
    mv_order(p2, p1, mn, mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return false;
    fx = fabsf(e1[0]), fy = fabsf(e1[1]), fz = fabsf(e1[2]);
    p0 = e1[2] * v0[1] - e1[1] * v0[2], p2 = e1[2] * v2[1] - e1[1] * v2[2];  // x * e1
    mv_order(p0, p2, mn, mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return false;
    p0 = -e1[2] * v0[0] + e1[0] * v0[2], p2 = -e1[2] * v2[0] + e1[0] * v2[2];  // y * e1
    mv_order(p0, p2, mn, mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return false;
    p0 = e1[1] * v0[0] - e1[0] * v0[1], p1 = e1[1] * v1[0] - e1[0] * v1[1];  // z * e1
    mv_order(p0, p1, mn, mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return false;
    fx = fabsf(e2[0]), fy = fabsf(e2[1]), fz = fabsf(e2[2]);
    p0 = e2[2] * v0[1] - e2[1] * v0[2], p1 = e2[2] * v1[1] - e2[1] * v1[2];  // x * e2
    mv_order(p0, p1, mn, mx), rad = fz * h + fy * h;
    if (mn > rad || mx < -rad) return false;
    p0 = -e2[2] * v0[0] + e2[0] * v0[2], p1 = -e2[2] * v1[0] + e2[0] * v1[2];  // y * e2
    mv_order(p0, p1, mn, mx), rad = fz * h + fx * h;
    if (mn > rad || mx < -rad) return false;
    p1 = e2[1] * v1[0] - e2[0] * v1[1], p2 = e2[1] * v2[0] - e2[0] * v2[1];  // z * e2
    mv_order(p2, p1, mn, mx), rad = fy * h + fx * h;
    if (mn > rad || mx < -rad) return false;
#pragma unroll
    for (int q = 0; q < 3; ++q) {  // the box axes
        mn = mx = v0[q];
        if (v1[q] < mn) mn = v1[q];
        if (v1[q] > mx) mx = v1[q];
        if (v2[q] < mn) mn = v2[q];
        if (v2[q] > mx) mx = v2[q];
        if (mn > h || mx < -h) return false;
    }
    const float n[3] = {e0[1] * e1[2] - e0[2] * e1[1], e0[2] * e1[0] - e0[0] * e1[2], e0[0] * e1[1] - e0[1] * e1[0]};
    float vmin[3], vmax[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        if (n[q] > 0.f) {
            vmin[q] = -h - v0[q];
            vmax[q] = h - v0[q];
        } else {
            vmin[q] = h - v0[q];
            vmax[q] = -h - v0[q];
        }
    }
    if (n[0] * vmin[0] + n[1] * vmin[1] + n[2] * vmin[2] > 0.f) return false;
    return n[0] * vmax[0] + n[1] * vmax[1] + n[2] * vmax[2] >= 0.f;
}

// the first k in [lo, hi] at which a predicate that is false, then true, turns true; hi + 1 when it never does
template <class P>
__host__ __device__ __forceinline__ int mv_first(int lo, int hi, P p) {
    int a = lo, b = hi + 1;
    while (a < b) {
        const int m = a + ((b - a) >> 1);
        if (p(m)) b = m;
        else a = m + 1;
    }
    return a;
}

struct MvGrid {
    float o[3], vs, h;
    int n[3];
};

__host__ __device__ __forceinline__ bool mv_load(const float *__restrict__ vtx, const int32_t *__restrict__ tri, size_t t, float P[3][3]) {
    bool finite = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const size_t v = (size_t)tri[3 * t + j];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            P[j][q] = vtx[3 * v + q];
            finite = finite && isfinite(P[j][q]);
        }
    }
    return finite;
}

// the triangle's normal (v1 - v0) x (v2 - v1) in float64, the orientation of the float test's normal
__host__ __device__ __forceinline__ void mv_normal64(const float P[3][3], double nD[3]) {
    double e0[3], e1[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        e0[q] = (double)P[1][q] - (double)P[0][q];
        e1[q] = (double)P[2][q] - (double)P[1][q];
    }
    nD[0] = e0[1] * e1[2] - e0[2] * e1[1];
    nD[1] = e0[2] * e1[0] - e0[0] * e1[2];
    nD[2] = e0[0] * e1[1] - e0[1] * e1[0];
}

// a finite triangle's record and its column count (0 when its box misses the grid)
__host__ __device__ __forceinline__ unsigned long long mv_setup(const float P[3][3], const MvGrid &g, MvTri &r) {
    long long span[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float mn = fminf(fminf(P[0][a], P[1][a]), P[2][a]), mx = fmaxf(fmaxf(P[0][a], P[1][a]), P[2][a]);
        const float o = g.o[a], vs = g.vs, h = g.h;
        // the test's box-axis comparison: min_j (v_j - c) > h or max_j (v_j - c) < -h rejects, and v - c is monotone in c
        r.lo[a] = mv_first(0, g.n[a] - 1, [&](int k) { return mn - mv_centre(k, vs, o) <= h; });
        r.hi[a] = mv_first(0, g.n[a] - 1, [&](int k) { return !(mx - mv_centre(k, vs, o) >= -h); }) - 1;
        span[a] = (long long)r.hi[a] - r.lo[a] + 1;
        if (span[a] <= 0) return 0ull;
    }
    double nD[3];
    mv_normal64(P, nD);
    const double m0 = fabs(nD[0]), m1 = fabs(nD[1]), m2 = fabs(nD[2]);
    if (m0 + m1 + m2 > 0.0) {
        r.d = (m0 >= m1 && m0 >= m2) ? 0 : (m1 >= m2 ? 1 : 2);
    } else {  // degenerate: walk the longest axis of the box
        r.d = (span[0] >= span[1] && span[0] >= span[2]) ? 0 : (span[1] >= span[2] ? 1 : 2);
        r.d += 4;
    }
    const int d = r.d & 3;
    return (unsigned long long)mv_pick((d + 1) % 3, span[0], span[1], span[2]) * (unsigned long long)mv_pick((d + 2) % 3, span[0], span[1], span[2]);
}

__global__ void __launch_bounds__(MV_BLOCK) mv_setup_kernel(const float *__restrict__ vtx, size_t nv, const int32_t *__restrict__ tri, size_t nt,
                                                            MvGrid g, MvTri *__restrict__ info, unsigned long long *__restrict__ cols,
                                                            unsigned long long *__restrict__ bad) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t > nt) return;
    if (t == nt) {  // the scan's extra entry: its exclusive sum is the total
        cols[nt] = 0ull;
        return;
    }
    cols[t] = 0ull;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const int32_t v = tri[3 * t + j];
        ok = ok && v >= 0 && (size_t)v < nv;
    }
    if (!ok) {
        *bad = 1ull;
        return;
    }
    float P[3][3];
    if (!mv_load(vtx, tri, t, P)) return;  // a non-finite vertex meets no cell
    MvTri r;
    const unsigned long long c = mv_setup(P, g, r);
    if (c) {
        info[t] = r;
        cols[t] = c;
    }
}

// one work item: a column of one triangle along axis d, at cells ki, kj on axes i = (d + 1) % 3, j = (d + 2) % 3
// (centres ci, cj); the walk tests cells k0 .. k0 + len - 1 along d
struct MvColumn {
    float P[3][3];
    float ci, cj;
    int ki, kj, k0, d;
};

__host__ __device__ __forceinline__ int mv_column(const float *__restrict__ vtx, const int32_t *__restrict__ tri, size_t nt, const MvTri *__restrict__ info,
                                         const unsigned long long *__restrict__ off, unsigned long long w, unsigned long long W, const MvGrid &g,
                                         MvColumn &col) {
    col.d = 0;
    col.ci = col.cj = 0.f;
    col.ki = col.kj = col.k0 = 0;
    if (w >= W) return 0;
    size_t a = 0, b = nt;  // the last triangle whose first item is <= w
    while (b - a > 1) {
        const size_t m = (a + b) >> 1;
        if (off[m] <= w) a = m;
        else b = m;
    }
    const size_t t = a;
    const MvTri r = info[t];
    const int d = r.d & 3, i = (d + 1) % 3, j = (d + 2) % 3;
    col.d = d;
    const int loi = mv_pick(i, r.lo[0], r.lo[1], r.lo[2]), loj = mv_pick(j, r.lo[0], r.lo[1], r.lo[2]);
    const int hij = mv_pick(j, r.hi[0], r.hi[1], r.hi[2]);
    const unsigned long long local = w - off[t], nj = (unsigned long long)(hij - loj + 1);
    col.ki = loi + (int)(local / nj);
    col.kj = loj + (int)(local % nj);
    col.ci = mv_centre(col.ki, g.vs, mv_pick(i, g.o[0], g.o[1], g.o[2]));
    col.cj = mv_centre(col.kj, g.vs, mv_pick(j, g.o[0], g.o[1], g.o[2]));
    mv_load(vtx, tri, t, col.P);
    int k0 = mv_pick(d, r.lo[0], r.lo[1], r.lo[2]), k1 = mv_pick(d, r.hi[0], r.hi[1], r.hi[2]);
    if (!(r.d & 4)) {
        // The plane meets the closed cell of centre c when |n . (P0 - c)| <= h (|n0| + |n1| + |n2|), i.e. c_d within
        // rr of tc.  The float test computes its normal per cell from centre-relative vertices (|v| <= V = E + vs for
        // every cell that passes the box axes, E the triangle's extent), so its normal is off by about u E V and its
        // dot by about u |n| V (u = 2^-24): the slab is widened by 2^-16 (E V^2 / |n_d| + 4 V), far above those, plus
        // 2^-140 / |n_d| for underflow in the float products.
        double nD[3];
        mv_normal64(col.P, nD);
        const double nd = mv_pick(d, nD[0], nD[1], nD[2]), ni = mv_pick(i, nD[0], nD[1], nD[2]), nj2 = mv_pick(j, nD[0], nD[1], nD[2]);
        double E = 0.0;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const double lo = fmin(fmin((double)col.P[0][q], (double)col.P[1][q]), (double)col.P[2][q]);
            const double hi = fmax(fmax((double)col.P[0][q], (double)col.P[1][q]), (double)col.P[2][q]);
            E = fmax(E, hi - lo);
        }
        const double V = E + (double)g.vs, ad = fabs(nd);
        const double slack = 0x1p-16 * (E * V * V / ad + 4.0 * V) + 0x1p-140 / ad;
        const double p0i = mv_pick(i, col.P[0][0], col.P[0][1], col.P[0][2]), p0j = mv_pick(j, col.P[0][0], col.P[0][1], col.P[0][2]);
        const double p0d = mv_pick(d, col.P[0][0], col.P[0][1], col.P[0][2]);
        const double tc = p0d + (ni * (p0i - (double)col.ci) + nj2 * (p0j - (double)col.cj)) / nd;
        const double rr = (double)g.h * (fabs(nD[0]) + fabs(nD[1]) + fabs(nD[2])) / ad;
        const double clo = tc - rr - slack, chi = tc + rr + slack;
        const float o = mv_pick(d, g.o[0], g.o[1], g.o[2]), vs = g.vs;
        const int lo = k0, hi = k1;
        k0 = mv_first(lo, hi, [&](int k) { return (double)mv_centre(k, vs, o) >= clo; });
        k1 = mv_first(lo, hi, [&](int k) { return (double)mv_centre(k, vs, o) > chi; }) - 1;
    }
    col.k0 = k0;
    return k1 >= k0 ? k1 - k0 + 1 : 0;
}

// step s of the walk: whether cell k0 + s of the column passes the test; its key to key[]
__host__ __device__ __forceinline__ bool mv_step_hit(int s, int len, const MvColumn &col, const MvGrid &g, int key[3]) {
    if (s >= len) return false;
    const int kd = col.k0 + s, d = col.d;
    const float cd = mv_centre(kd, g.vs, mv_pick(d, g.o[0], g.o[1], g.o[2]));
    float c[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        c[q] = q == d ? cd : (q == (d + 1) % 3 ? col.ci : col.cj);
        key[q] = q == d ? kd : (q == (d + 1) % 3 ? col.ki : col.kj);
    }
    return mv_tri_box(c, g.h, col.P[0], col.P[1], col.P[2]);
}

// per block: the number of hits (block_flag_count per step of the walk); their total to *hits
__global__ void __launch_bounds__(MV_BLOCK) mv_count_kernel(const float *__restrict__ vtx, const int32_t *__restrict__ tri, size_t nt,
                                                            const MvTri *__restrict__ info, const unsigned long long *__restrict__ off,
                                                            unsigned long long W, MvGrid g, unsigned *__restrict__ counts,
                                                            unsigned long long *__restrict__ hits) {
    MvColumn col;
    int key[3];
    const int len = mv_column(vtx, tri, nt, info, off, blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x, W, g, col);
    unsigned total = 0;
    for (int s = 0; __syncthreads_or(s < len); ++s) total += block_flag_count(mv_step_hit(s, len, col, g, key));
    if (threadIdx.x == 0) {
        counts[blockIdx.x] = total;
        atomicAdd(hits, (unsigned long long)total);
    }
}

// the same walk; hit r of the block goes to keys[offsets[block] + r], packed x | y | z with z lowest.  keys[n_hits]
// gets the sentinel (every sorted bit set), which sorts last, so the sort and the unique run on every non-empty input.
__global__ void __launch_bounds__(MV_BLOCK) mv_write_kernel(const float *__restrict__ vtx, const int32_t *__restrict__ tri, size_t nt,
                                                            const MvTri *__restrict__ info, const unsigned long long *__restrict__ off,
                                                            unsigned long long W, MvGrid g, const unsigned *__restrict__ offsets, int sy,
                                                            int sz, uint64_t sentinel, size_t n_hits, uint64_t *__restrict__ keys) {
    MvColumn col;
    int key[3];
    const int len = mv_column(vtx, tri, nt, info, off, blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x, W, g, col);
    if (blockIdx.x == 0 && threadIdx.x == 0) keys[n_hits] = sentinel;
    size_t base = offsets[blockIdx.x];
    for (int s = 0; __syncthreads_or(s < len); ++s) {
        const bool hit = mv_step_hit(s, len, col, g, key);
        const unsigned r = block_flag_rank(hit);
        if (hit) keys[base + r] = ((uint64_t)key[0] << sy) | ((uint64_t)key[1] << sz) | (uint64_t)key[2];
        base += __syncthreads_count(hit);
    }
}

// thrust::unique of the sorted keys [0, n) as a block compaction (the sentinel at n is never kept)
__device__ __forceinline__ bool mv_first_of_run(const uint64_t *k, size_t i, size_t n) { return i < n && (i == 0 || k[i] != k[i - 1]); }
__global__ void __launch_bounds__(MV_BLOCK) mv_unique_count_kernel(const uint64_t *__restrict__ k, size_t n, unsigned *__restrict__ counts) {
    const unsigned c = block_flag_count(mv_first_of_run(k, blockIdx.x * (size_t)blockDim.x + threadIdx.x, n));
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}
// rows are written only when the total fits the capacity
__global__ void __launch_bounds__(MV_BLOCK) mv_unique_write_kernel(const uint64_t *__restrict__ k, size_t n, const unsigned *__restrict__ offsets,
                                                                   const unsigned *__restrict__ total, size_t capacity, int sy, int sz,
                                                                   int32_t *__restrict__ out_keys, float *__restrict__ out_colors) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool v = mv_first_of_run(k, i, n);
    const unsigned r = block_flag_rank(v);
    if (v && out_keys && *total <= capacity) {
        const size_t o = offsets[blockIdx.x] + (size_t)r;
        const uint64_t key = k[i];
        out_keys[3 * o] = (int32_t)(key >> sy);
        out_keys[3 * o + 1] = (int32_t)((key >> sz) & ((1ull << (sy - sz)) - 1ull));
        out_keys[3 * o + 2] = (int32_t)(key & ((1ull << sz) - 1ull));
        out_colors[3 * o] = 1.f;  // Voxel's default colour (voxelgrid.h:61)
        out_colors[3 * o + 1] = 1.f;
        out_colors[3 * o + 2] = 1.f;
    }
}

extern "C" int cphb_voxel_grid_from_triangle_mesh(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                                  float voxel_size, const float h_min_bound[3], const float h_max_bound[3], int32_t *out_keys,
                                                  float *out_colors, size_t capacity, size_t *h_n, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_voxel_grid_from_triangle_mesh";
    if (!h_n || !h_min_bound || !h_max_bound) return vgo_invalid(who, "null argument");
    *h_n = 0;
    if (!(isfinite(voxel_size) && voxel_size > 0.f)) return vgo_invalid(who, "voxel_size is not positive and finite");
    MvGrid g;
    g.vs = voxel_size;
    g.h = voxel_size * 0.5f;
    for (int a = 0; a < 3; ++a) {
        if (!isfinite(h_min_bound[a]) || !isfinite(h_max_bound[a])) return vgo_invalid(who, "the bounds are not finite");
        const volatile float ext = h_max_bound[a] - h_min_bound[a];
        const volatile float q = ext / voxel_size;  // int(std::round(extent / voxel_size)) in float, as CreateDense
        const float c = roundf(q);
        if (!(c >= 0.f && c < (float)(1 << CPHB_KEY_AXIS_BITS))) {
            cphb_set_error("%s: axis %d count round(%g / %g) is negative or >= 2^%d", who, a, (double)ext, (double)voxel_size,
                           CPHB_KEY_AXIS_BITS);
            return CPHB_ERR_INVALID;
        }
        g.n[a] = (int)c;
        g.o[a] = h_min_bound[a];
    }
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || (n_vertices && !vertices) || (capacity && (!out_keys || !out_colors))) return vgo_invalid(who, "null argument");
    if (n_triangles > (size_t)INT32_MAX) return vgo_invalid(who, "more than 2^31-1 triangles");
    const int bx = bits_for_span(g.n[0]), by = bits_for_span(g.n[1]), bz = bits_for_span(g.n[2]);
    const int sz = bz, sy = by + bz, bits = bx + by + bz;
    const uint64_t sentinel = ~0ull >> (64 - bits);

    cphb_scratch sc(s);
    unsigned long long *meta = nullptr, *cols = nullptr, *off = nullptr;  // meta: index error, columns, hits
    MvTri *info = nullptr;
    int rc = sc.alloc(&meta, 4);
    if (!rc) rc = sc.alloc(&cols, n_triangles + 1);
    if (!rc) rc = sc.alloc(&off, n_triangles + 1);
    if (!rc) rc = sc.alloc(&info, n_triangles);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(meta, 0, 4 * sizeof(unsigned long long), s));
    CPHB_LAUNCH(mv_setup_kernel, vgo_grid(n_triangles + 1), MV_BLOCK, 0, s, vertices, n_vertices, triangles, n_triangles, g, info, cols, meta);
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, cols, off, (int64_t)(n_triangles + 1), s));
    char *tmp = nullptr;
    rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, cols, off, (int64_t)(n_triangles + 1), s));
    g_cphb_launches += 2;  // CUB's init and scan kernels
    CPHB_CUDA(cudaMemcpyAsync(meta + 1, off + n_triangles, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
    unsigned long long h_meta[2] = {0ull, 0ull};
    rc = cphb_read_back(h_meta, meta, 2 * sizeof(unsigned long long), s, who);
    if (rc) return rc;
    if (h_meta[0]) return vgo_invalid(who, "a triangle's vertex index is outside [0, n_vertices)");
    const unsigned long long W = h_meta[1];
    if (W > (unsigned long long)INT32_MAX * MV_BLOCK) return vgo_invalid(who, "more than 2^39 triangle columns");
    const unsigned nb = W ? (unsigned)((W + MV_BLOCK - 1) / MV_BLOCK) : 1u;

    unsigned *counts = nullptr, *total = nullptr;
    rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (rc) return rc;
    CPHB_LAUNCH(mv_count_kernel, nb, MV_BLOCK, 0, s, vertices, triangles, n_triangles, info, off, W, g, counts, meta + 2);
    cphb_scan_block_counts(counts, nb, total, s);
    unsigned long long H = 0;
    rc = cphb_read_back(&H, meta + 2, sizeof(H), s, who);
    if (rc) return rc;
    if (H >= (unsigned long long)INT32_MAX) return vgo_invalid(who, "2^31-1 or more triangle/cell hits");

    uint64_t *keys = nullptr, *skeys = nullptr;
    unsigned *ucounts = nullptr, *utotal = nullptr;
    const size_t nk = (size_t)H + 1;
    const unsigned nbu = (unsigned)((nk + MV_BLOCK - 1) / MV_BLOCK);
    rc = sc.alloc(&keys, nk);
    if (!rc) rc = sc.alloc(&skeys, nk);
    if (!rc) rc = sc.alloc(&ucounts, (size_t)nbu + 4);
    if (!rc) rc = sc.alloc(&utotal, 1);
    if (rc) return rc;
    CPHB_LAUNCH(mv_write_kernel, nb, MV_BLOCK, 0, s, vertices, triangles, n_triangles, info, off, W, g, counts, sy, sz, sentinel, (size_t)H,
                keys);
    rc = cphb_sort_keys_u64(keys, skeys, nk, bits, s);
    if (rc) return rc;
    CPHB_LAUNCH(mv_unique_count_kernel, nbu, MV_BLOCK, 0, s, skeys, (size_t)H, ucounts);
    cphb_scan_block_counts(ucounts, nbu, utotal, s);
    CPHB_LAUNCH(mv_unique_write_kernel, nbu, MV_BLOCK, 0, s, skeys, (size_t)H, ucounts, utotal, capacity, sy, sz, out_keys, out_colors);
    unsigned m = 0;
    rc = cphb_read_back(&m, utotal, sizeof(m), s, who);
    if (rc) return rc;
    *h_n = m;
    return CPHB_OK;
}
