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

#include "cphb_internal.cuh"

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
