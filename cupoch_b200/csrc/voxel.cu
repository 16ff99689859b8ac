// voxel.cu -- PointCloud::VoxelDownSample (down_sample.cu:170-273) as a voxel
// hash build instead of the reference's comparison merge-sort of int3 keys
// with zipped payloads (thrust::sort_by_key + reduce_by_key, :194-222).
//
//   bounds -> key = floor((p - origin)/voxel) (down_sample.cu:64-75)
//   insert : open-addressing table of packed 64-bit keys (atomicCAS, linear
//            probing); lanes of a warp that hold the same key elect one
//            inserter (__match_any_sync), so coherent (scan-ordered) inputs
//            issue one CAS per voxel per warp
//   assign : occupied slots get dense ids
//   accum  : per point, probe (read-only) -> id -> float64 atomic adds of
//            xyz / normal / colour + count (order-independent to 1e-16, so the
//            float32 result is reproducible and equals the oracle's)
//   order  : radix sort of the (few) voxel keys restores the reference's
//            lexicographic (x,y,z) output order (helper.h:113-121)
//   final  : mean; normals mean-then-normalise (down_sample.cu:78-90)
// The table is sized by min(n, #grid cells), so for grids of few cells it stays small enough for L2.
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "cphb_internal.cuh"

#define VX_EMPTY 0xffffffffffffffffull

struct VoxelGrid {
    float org[3];
    float voxel;
    int sy, sz;  // shifts: key = x << (sy) | y << sz | z  (sy = by + bz, sz = bz)
};

__device__ __forceinline__ unsigned long long voxel_key(const float *p, const VoxelGrid &g) {
    // compute_key_functor (down_sample.cu:70-73): floor((pt - min_bound) / voxel_size) cast to int
    long long kx = (long long)(int)floorf(__fdiv_rn(p[0] - g.org[0], g.voxel));
    long long ky = (long long)(int)floorf(__fdiv_rn(p[1] - g.org[1], g.voxel));
    long long kz = (long long)(int)floorf(__fdiv_rn(p[2] - g.org[2], g.voxel));
    return ((unsigned long long)kx << g.sy) | ((unsigned long long)ky << g.sz) | (unsigned long long)kz;
}
__device__ __forceinline__ unsigned hash64(unsigned long long k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (unsigned)k;
}

__global__ void __launch_bounds__(256) voxel_table_init_kernel(unsigned long long *keys, size_t T, unsigned *counter) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < T) keys[i] = VX_EMPTY;
    if (i == 0) *counter = 0;
}

__global__ void __launch_bounds__(256) voxel_insert_kernel(const float *__restrict__ pts, size_t n, VoxelGrid g,
                                                           unsigned long long *keys, unsigned mask) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    bool valid = i < n;
    unsigned long long key = valid ? voxel_key(pts + 3 * i, g) : VX_EMPTY;
    // warp-cooperative dedup of runs: scan-ordered inputs put consecutive points into the same voxel, so a
    // lane whose left neighbour holds the same key leaves the insert to it (one CAS per run per warp).
    // (A full __match_any_sync costs more than the CAS it saves on unordered inputs.)
    const unsigned long long left = __shfl_up_sync(CPHB_FULL, key, 1);
    if (!valid || (lane_id() > 0 && left == key)) return;
    unsigned h = hash64(key) & mask;
    while (true) {
        unsigned long long prev = atomicCAS(&keys[h], VX_EMPTY, key);
        if (prev == VX_EMPTY || prev == key) break;
        h = (h + 1) & mask;
    }
}

__global__ void __launch_bounds__(256) voxel_assign_kernel(const unsigned long long *__restrict__ keys, size_t T,
                                                           unsigned *ids, unsigned long long *dense_keys,
                                                           unsigned *dense_ids, unsigned *counter) {
    __shared__ unsigned s_warp[8];
    __shared__ unsigned s_base;
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    bool occ = i < T && keys[i] != VX_EMPTY;
    unsigned m = __ballot_sync(CPHB_FULL, occ);
    const int warp = threadIdx.x >> 5;
    if (lane_id() == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {  // one global atomic per block (not per warp: 131k same-address atomics serialise)
        unsigned tot = 0;
        for (int w2 = 0; w2 < 8; ++w2) { unsigned c = s_warp[w2]; s_warp[w2] = tot; tot += c; }
        s_base = tot ? atomicAdd(counter, tot) : 0u;
    }
    __syncthreads();
    if (occ) {
        unsigned id = s_base + s_warp[warp] + __popc(m & ((1u << lane_id()) - 1u));
        ids[i] = id;
        dense_keys[id] = keys[i];
        dense_ids[id] = id;
    }
}

__global__ void __launch_bounds__(256) voxel_zero_kernel(double *sums, unsigned *counts, size_t n_sums, size_t n_counts) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n_sums) sums[i] = 0.0;
    if (i < n_counts) counts[i] = 0u;
}

template <int A>  // A attribute vectors per point: 1 points, 2 (+normals or colours), 3 both
__global__ void __launch_bounds__(256) voxel_accum_kernel(const float *__restrict__ pts, const float *__restrict__ a1,
                                                          const float *__restrict__ a2, size_t n, VoxelGrid g,
                                                          const unsigned long long *__restrict__ keys,
                                                          const unsigned *__restrict__ ids, unsigned mask, double *sums,
                                                          unsigned *counts) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    unsigned long long key = voxel_key(p, g);
    unsigned h = hash64(key) & mask;
    while (keys[h] != key) h = (h + 1) & mask;
    const unsigned id = ids[h];
    double *s = sums + (size_t)id * 3 * A;
    atomicAdd(s + 0, (double)p[0]);
    atomicAdd(s + 1, (double)p[1]);
    atomicAdd(s + 2, (double)p[2]);
    if (A >= 2) {
        atomicAdd(s + 3, (double)a1[3 * i]);
        atomicAdd(s + 4, (double)a1[3 * i + 1]);
        atomicAdd(s + 5, (double)a1[3 * i + 2]);
    }
    if (A >= 3) {
        atomicAdd(s + 6, (double)a2[3 * i]);
        atomicAdd(s + 7, (double)a2[3 * i + 1]);
        atomicAdd(s + 8, (double)a2[3 * i + 2]);
    }
    atomicAdd(counts + id, 1u);
}

template <int A>
__global__ void __launch_bounds__(256) voxel_final_kernel(const unsigned *__restrict__ order, unsigned n_out,
                                                          const double *__restrict__ sums,
                                                          const unsigned *__restrict__ counts, int a1_is_normal,
                                                          float *out_p, float *out_a1, float *out_a2) {
    unsigned pos = blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= n_out) return;
    unsigned id = order[pos];
    const double *s = sums + (size_t)id * 3 * A;
    float cnt = (float)counts[id];
    // divide_tuple_functor: x / (float)count
    out_p[3 * pos] = __fdiv_rn((float)s[0], cnt);
    out_p[3 * pos + 1] = __fdiv_rn((float)s[1], cnt);
    out_p[3 * pos + 2] = __fdiv_rn((float)s[2], cnt);
    if (A >= 2) {
        float v[3] = {__fdiv_rn((float)s[3], cnt), __fdiv_rn((float)s[4], cnt), __fdiv_rn((float)s[5], cnt)};
        if (a1_is_normal) {  // normalize_and_divide_tuple_functor (down_sample.cu:78-90)
            float nn = sqrtf(dot3(v[0], v[1], v[2], v[0], v[1], v[2]));
            if (nn > 0.f) { v[0] = __fdiv_rn(v[0], nn); v[1] = __fdiv_rn(v[1], nn); v[2] = __fdiv_rn(v[2], nn); }
        }
        out_a1[3 * pos] = v[0]; out_a1[3 * pos + 1] = v[1]; out_a1[3 * pos + 2] = v[2];
    }
    if (A >= 3) {
        out_a2[3 * pos] = __fdiv_rn((float)s[6], cnt);
        out_a2[3 * pos + 1] = __fdiv_rn((float)s[7], cnt);
        out_a2[3 * pos + 2] = __fdiv_rn((float)s[8], cnt);
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// Dense-grid path.  When the grid has no more cells than about twice the points (config 3 of BASELINE.json: 10 M points
// in 2.0 M cells), hashing buys nothing: every cell gets one 32-byte-aligned accumulator row [sum x, sum y, sum z, count]
// (+ the attribute sums) addressed directly by its lexicographic cell number, so
//   * there is no insert pass, no probe and no dense-id table.  The accumulators of the whole grid (64 MB at config 3)
//     exceed the H100's 50 MB L2, yet the dense path stays the faster one: 10 M points, VoxelDownSample on the H100
//     (profiles/h100_tuning_sweep.txt) at 0.61 / 2.0 / 3.9 M cells (20 / 64 / 126 MB of accumulators): dense 0.68 / 1.08 / 1.26 ms, hash
//     1.26 / 2.36 / 3.02 ms; 2 M points in 2.0 M cells: 0.35 vs 0.63 ms.  So the threshold (cells <= 2 n) stands;
//   * a cell's atomics fall into one sector;
//   * the cells are already in the reference's output order (helper.h:113-121): an ordered compaction replaces the
//     radix sort of the voxel keys.
// Sums are float64 atomics of float32 values exactly as in the hash path (the same, order-independent-to-1e-16 result).
// ---------------------------------------------------------------------------------------------------------------------
struct DenseGrid {
    float org[3];
    float voxel;
    unsigned dy, dz;  // cells along y and z: cell = (kx * dy + ky) * dz + kz
};
template <int A>
__host__ __device__ constexpr int dense_stride() { return A == 1 ? 4 : A == 2 ? 8 : 12; }  // doubles per cell (32-B multiples)

template <int A>
__global__ void __launch_bounds__(256) voxel_dense_accum_kernel(const float *__restrict__ pts, const float *__restrict__ a1,
                                                                const float *__restrict__ a2, size_t n, DenseGrid g,
                                                                double *acc) {
    constexpr int S = dense_stride<A>();
    // 4 consecutive points per thread: 48 B = three 16-byte loads per array when the base is 16-byte aligned
    const size_t i0 = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) * 4;
    if (i0 >= n) return;
    float p[12], q1[12], q2[12];
    const bool vec = (i0 + 4 <= n) && ((reinterpret_cast<uintptr_t>(pts) & 15) == 0) &&
                     (A < 2 || (reinterpret_cast<uintptr_t>(a1) & 15) == 0) && (A < 3 || (reinterpret_cast<uintptr_t>(a2) & 15) == 0);
    const int cnt = (i0 + 4 <= n) ? 4 : (int)(n - i0);
    if (vec) {
#pragma unroll
        for (int v = 0; v < 3; ++v) {
            const float4 x = reinterpret_cast<const float4 *>(pts + 3 * i0)[v];
            p[4 * v] = x.x; p[4 * v + 1] = x.y; p[4 * v + 2] = x.z; p[4 * v + 3] = x.w;
            if (A >= 2) {
                const float4 y = reinterpret_cast<const float4 *>(a1 + 3 * i0)[v];
                q1[4 * v] = y.x; q1[4 * v + 1] = y.y; q1[4 * v + 2] = y.z; q1[4 * v + 3] = y.w;
            }
            if (A >= 3) {
                const float4 z = reinterpret_cast<const float4 *>(a2 + 3 * i0)[v];
                q2[4 * v] = z.x; q2[4 * v + 1] = z.y; q2[4 * v + 2] = z.z; q2[4 * v + 3] = z.w;
            }
        }
    } else {
        for (int k = 0; k < 3 * cnt; ++k) {
            p[k] = pts[3 * i0 + k];
            if (A >= 2) q1[k] = a1[3 * i0 + k];
            if (A >= 3) q2[k] = a2[3 * i0 + k];
        }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        if (t >= cnt) break;
        // compute_key_functor (down_sample.cu:70-73): floor((pt - min_bound) / voxel_size) cast to int
        const unsigned kx = (unsigned)(int)floorf(__fdiv_rn(p[3 * t] - g.org[0], g.voxel));
        const unsigned ky = (unsigned)(int)floorf(__fdiv_rn(p[3 * t + 1] - g.org[1], g.voxel));
        const unsigned kz = (unsigned)(int)floorf(__fdiv_rn(p[3 * t + 2] - g.org[2], g.voxel));
        double *c = acc + ((size_t)(kx * g.dy + ky) * g.dz + kz) * S;
        atomicAdd(c + 0, (double)p[3 * t]);
        atomicAdd(c + 1, (double)p[3 * t + 1]);
        atomicAdd(c + 2, (double)p[3 * t + 2]);
        if (A >= 2) {
            atomicAdd(c + 3, (double)q1[3 * t]);
            atomicAdd(c + 4, (double)q1[3 * t + 1]);
            atomicAdd(c + 5, (double)q1[3 * t + 2]);
        }
        if (A >= 3) {
            atomicAdd(c + 6, (double)q2[3 * t]);
            atomicAdd(c + 7, (double)q2[3 * t + 1]);
            atomicAdd(c + 8, (double)q2[3 * t + 2]);
        }
        atomicAdd(c + (A == 1 ? 3 : A == 2 ? 6 : 9), 1.0);  // the count, exact in float64
    }
}

#define VD_BLOCK 1024
template <int A>
__global__ void __launch_bounds__(VD_BLOCK) voxel_dense_count_kernel(const double *__restrict__ acc, size_t cells, unsigned *block_counts) {
    constexpr int S = dense_stride<A>();
    __shared__ unsigned s_w[32];
    const size_t c = blockIdx.x * (size_t)VD_BLOCK + threadIdx.x;
    const bool occ = c < cells && acc[c * S + (A == 1 ? 3 : A == 2 ? 6 : 9)] > 0.0;
    const unsigned m = __ballot_sync(CPHB_FULL, occ);
    if (lane_id() == 0) s_w[threadIdx.x >> 5] = __popc(m);
    __syncthreads();
    if (threadIdx.x < 32) {
        unsigned v = s_w[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(CPHB_FULL, v, o);
        if (threadIdx.x == 0) block_counts[blockIdx.x] = v;
    }
}
// exclusive scan of the block counts (one block; the grid has cells / 1024 entries), total to *total
__global__ void __launch_bounds__(1024) voxel_dense_scan_kernel(unsigned *block_counts, unsigned nb, unsigned *total) {
    __shared__ unsigned s_w[32];
    __shared__ unsigned s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (unsigned base = 0; base < nb; base += 1024) {
        const unsigned i = base + threadIdx.x;
        const unsigned v = i < nb ? block_counts[i] : 0u;
        unsigned x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(CPHB_FULL, x, o);
            if (lane_id() >= o) x += y;
        }
        if (lane_id() == 31) s_w[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            const unsigned ws = s_w[threadIdx.x];
            unsigned z = ws;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned y = __shfl_up_sync(CPHB_FULL, z, o);
                if (lane_id() >= o) z += y;
            }
            s_w[threadIdx.x] = z - ws;
        }
        __syncthreads();
        const unsigned excl = x - v + s_w[threadIdx.x >> 5] + s_carry;
        if (i < nb) block_counts[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_carry;
}
template <int A>
__global__ void __launch_bounds__(VD_BLOCK) voxel_dense_write_kernel(const double *__restrict__ acc, size_t cells,
                                                                     const unsigned *__restrict__ block_offsets, int a1_is_normal,
                                                                     float *out_p, float *out_a1, float *out_a2) {
    constexpr int S = dense_stride<A>();
    __shared__ unsigned s_w[32];
    const size_t c = blockIdx.x * (size_t)VD_BLOCK + threadIdx.x;
    double cntd = 0.0;
    if (c < cells) cntd = acc[c * S + (A == 1 ? 3 : A == 2 ? 6 : 9)];
    const bool occ = cntd > 0.0;
    const unsigned m = __ballot_sync(CPHB_FULL, occ);
    if (lane_id() == 0) s_w[threadIdx.x >> 5] = __popc(m);
    __syncthreads();
    if (threadIdx.x < 32) {
        const unsigned ws = s_w[threadIdx.x];
        unsigned z = ws;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(CPHB_FULL, z, o);
            if (lane_id() >= o) z += y;
        }
        s_w[threadIdx.x] = z - ws;
    }
    __syncthreads();
    if (!occ) return;
    const size_t pos = (size_t)block_offsets[blockIdx.x] + s_w[threadIdx.x >> 5] + __popc(m & ((1u << lane_id()) - 1u));
    const double *s = acc + c * S;
    const float cnt = (float)cntd;
    // divide_tuple_functor: x / (float)count
    out_p[3 * pos] = __fdiv_rn((float)s[0], cnt);
    out_p[3 * pos + 1] = __fdiv_rn((float)s[1], cnt);
    out_p[3 * pos + 2] = __fdiv_rn((float)s[2], cnt);
    if (A >= 2) {
        float v[3] = {__fdiv_rn((float)s[3], cnt), __fdiv_rn((float)s[4], cnt), __fdiv_rn((float)s[5], cnt)};
        if (a1_is_normal) {  // normalize_and_divide_tuple_functor (down_sample.cu:78-90)
            const float nn = sqrtf(dot3(v[0], v[1], v[2], v[0], v[1], v[2]));
            if (nn > 0.f) { v[0] = __fdiv_rn(v[0], nn); v[1] = __fdiv_rn(v[1], nn); v[2] = __fdiv_rn(v[2], nn); }
        }
        out_a1[3 * pos] = v[0]; out_a1[3 * pos + 1] = v[1]; out_a1[3 * pos + 2] = v[2];
    }
    if (A >= 3) {
        out_a2[3 * pos] = __fdiv_rn((float)s[6], cnt);
        out_a2[3 * pos + 1] = __fdiv_rn((float)s[7], cnt);
        out_a2[3 * pos + 2] = __fdiv_rn((float)s[8], cnt);
    }
}

template <int A>
static int voxel_dense(const float *points, const float *a1, const float *a2, size_t n, const DenseGrid &g, size_t cells,
                       int a1_is_normal, float *out_p, float *out_a1, float *out_a2, size_t *h_n_out, cudaStream_t s) {
    constexpr int S = dense_stride<A>();
    const unsigned nb = (unsigned)((cells + VD_BLOCK - 1) / VD_BLOCK);
    char *base = nullptr;
    const size_t acc_bytes = cphb_align(sizeof(double) * S * cells, 256);
    int rc = cphb_alloc_async((void **)&base, acc_bytes + sizeof(unsigned) * ((size_t)nb + 8), s);
    if (rc) return rc;
    double *acc = (double *)base;
    unsigned *bc = (unsigned *)(base + acc_bytes), *total = bc + nb;
    CPHB_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * S * cells, s));
    CPHB_LAUNCH(voxel_dense_accum_kernel<A>, (unsigned)((n + 1023) / 1024), 256, 0, s, points, a1, a2, n, g, acc);
    CPHB_LAUNCH(voxel_dense_count_kernel<A>, nb, VD_BLOCK, 0, s, acc, cells, bc);
    CPHB_LAUNCH(voxel_dense_scan_kernel, 1, 1024, 0, s, bc, nb, total);
    CPHB_LAUNCH(voxel_dense_write_kernel<A>, nb, VD_BLOCK, 0, s, acc, cells, bc, a1_is_normal, out_p, out_a1, out_a2);
    CPHB_CHECK_LAUNCH();
    unsigned h = 0;
    CPHB_CUDA(cudaMemcpyAsync(&h, total, 4, cudaMemcpyDeviceToHost, s));
    cphb_free_async(base, s);
    CPHB_CUDA(cudaStreamSynchronize(s));
    *h_n_out = h;
    return CPHB_OK;
}

static int bits_for(double cells) {
    int b = 1;
    while (b < 63 && (double)(1ull << b) < cells) ++b;
    return b;
}

// h_origin == nullptr: the reference's origin, min_bound - voxel/2 (down_sample.cu:180).  A caller-supplied origin
// (<= every point, component-wise) lets several ranks down-sample disjoint parts of one cloud on ONE common grid
// (cupoch_b200.distributed.voxel_down_sample).
static int voxel_down_sample_impl(const float *points, const float *normals, const float *colors, size_t n,
                                  float voxel_size, const float *h_origin, float *out_points, float *out_normals,
                                  float *out_colors, size_t *h_n_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_n_out) {
        cphb_set_error("cphb_voxel_down_sample: h_n_out is null");
        return CPHB_ERR_INVALID;
    }
    *h_n_out = 0;
    if (voxel_size <= 0.0f || n == 0) return CPHB_OK;  // down_sample.cu:173-176 (warn + empty cloud)
    if (!points || !out_points || (normals && !out_normals) || (colors && !out_colors)) {
        cphb_set_error("cphb_voxel_down_sample: null argument");
        return CPHB_ERR_INVALID;
    }
    if (n > 0x7fffffffull) {
        cphb_set_error("cphb_voxel_down_sample: n exceeds int32");
        return CPHB_ERR_INVALID;
    }
    float mn[3], mx[3];
    int rc = cphb_min_max_bound(points, n, mn, mx, stream);
    if (rc) return rc;
    VoxelGrid g;
    g.voxel = voxel_size;
    float ext = 0.f;
    double cells = 1.0, dims[3];
    for (int a = 0; a < 3; ++a) {
        g.org[a] = h_origin ? h_origin[a] : mn[a] - voxel_size * 0.5f;       // :180
        if (h_origin && !(h_origin[a] <= mn[a])) {
            cphb_set_error("cphb_voxel_down_sample_origin: origin[%d] = %g lies above the cloud's minimum %g", a, h_origin[a], mn[a]);
            return CPHB_ERR_INVALID;
        }
        float hi = mx[a] + voxel_size * 0.5f;       // :181
        if (hi - g.org[a] > ext) ext = hi - g.org[a];
        dims[a] = (double)floorf((mx[a] - g.org[a]) / voxel_size) + 1.0;
        cells *= dims[a];
    }
    if (voxel_size * (float)2147483647 < ext) return CPHB_OK;  // :183-187 "voxel_size is too small"
    const int A0 = 1 + (normals ? 1 : 0) + (colors ? 1 : 0);
    const bool no_dense = getenv("CPHB_VOXEL_NO_DENSE") != nullptr;  // A/B and test hook: force the hash path
    if (!no_dense && cells <= 2.0 * (double)n + 4096.0 && cells < 2.0e9 && dims[1] * dims[2] < 4.0e9) {
        DenseGrid dg;
        for (int a = 0; a < 3; ++a) dg.org[a] = g.org[a];
        dg.voxel = voxel_size;
        dg.dy = (unsigned)dims[1];
        dg.dz = (unsigned)dims[2];
        const float *d1 = normals ? normals : colors, *d2 = colors;
        float *o1 = normals ? out_normals : out_colors;
        if (A0 == 1) return voxel_dense<1>(points, nullptr, nullptr, n, dg, (size_t)cells, 0, out_points, nullptr, nullptr, h_n_out, s);
        if (A0 == 2) return voxel_dense<2>(points, d1, nullptr, n, dg, (size_t)cells, normals ? 1 : 0, out_points, o1, nullptr, h_n_out, s);
        return voxel_dense<3>(points, normals, colors, n, dg, (size_t)cells, 1, out_points, out_normals, out_colors, h_n_out, s);
    }
    int bx = bits_for(dims[0]), by = bits_for(dims[1]), bz = bits_for(dims[2]);
    if (bx + by + bz > 63) {
        cphb_set_error("cphb_voxel_down_sample: grid %gx%gx%g needs %d key bits (> 63)", dims[0], dims[1], dims[2],
                       bx + by + bz);
        return CPHB_ERR_UNSUPPORTED;
    }
    g.sz = bz;
    g.sy = by + bz;
    const size_t cap = (cells < (double)n) ? (size_t)cells : n;  // max possible voxel count
    size_t T = 1024;
    while (T < 2 * cap) T <<= 1;
    const unsigned mask = (unsigned)(T - 1);
    const int A = 1 + (normals ? 1 : 0) + (colors ? 1 : 0);

    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = cphb_align(off + bytes, 256); return o; };
    size_t o_keys = take(T * 8), o_ids = take(T * 4), o_dk = take(cap * 8), o_dk2 = take(cap * 8);
    size_t o_di = take(cap * 4), o_ord = take(cap * 4), o_sums = take(cap * 3 * A * 8), o_cnt = take(cap * 4), o_ctr = take(16);
    char *base = nullptr;
    rc = cphb_alloc_async((void **)&base, off, s);
    if (rc) return rc;
    unsigned long long *keys = (unsigned long long *)(base + o_keys);
    unsigned *ids = (unsigned *)(base + o_ids);
    unsigned long long *dk = (unsigned long long *)(base + o_dk), *dk2 = (unsigned long long *)(base + o_dk2);
    unsigned *di = (unsigned *)(base + o_di), *order = (unsigned *)(base + o_ord);
    double *sums = (double *)(base + o_sums);
    unsigned *counts = (unsigned *)(base + o_cnt), *counter = (unsigned *)(base + o_ctr);

    CPHB_LAUNCH(voxel_table_init_kernel, (unsigned)((T + 255) / 256), 256, 0, s, keys, T, counter);
    CPHB_LAUNCH(voxel_insert_kernel, (unsigned)((n + 255) / 256), 256, 0, s, points, n, g, keys, mask);
    CPHB_LAUNCH(voxel_assign_kernel, (unsigned)((T + 255) / 256), 256, 0, s, keys, T, ids, dk, di, counter);
    size_t nz = cap * 3 * A;
    CPHB_LAUNCH(voxel_zero_kernel, (unsigned)((nz + 255) / 256), 256, 0, s, sums, counts, nz, cap);
    const float *a1 = normals ? normals : colors, *a2 = colors;
    unsigned gridn = (unsigned)((n + 255) / 256);
    if (A == 1) CPHB_LAUNCH(voxel_accum_kernel<1>, gridn, 256, 0, s, points, a1, a2, n, g, keys, ids, mask, sums, counts);
    else if (A == 2) CPHB_LAUNCH(voxel_accum_kernel<2>, gridn, 256, 0, s, points, a1, a2, n, g, keys, ids, mask, sums, counts);
    else CPHB_LAUNCH(voxel_accum_kernel<3>, gridn, 256, 0, s, points, a1, a2, n, g, keys, ids, mask, sums, counts);
    CPHB_CHECK_LAUNCH();
    unsigned h_cnt = 0;
    CPHB_CUDA(cudaMemcpyAsync(&h_cnt, counter, 4, cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    const unsigned n_out = h_cnt;
    rc = cphb_sort_pairs_u64((const uint64_t *)dk, (uint64_t *)dk2, di, order, n_out, bx + by + bz, s);
    if (rc) { cphb_free_async(base, s); return rc; }
    unsigned gridv = (n_out + 255) / 256;
    if (n_out) {
        if (A == 1) CPHB_LAUNCH(voxel_final_kernel<1>, gridv, 256, 0, s, order, n_out, sums, counts, 0, out_points, nullptr, nullptr);
        else if (A == 2)
            CPHB_LAUNCH(voxel_final_kernel<2>, gridv, 256, 0, s, order, n_out, sums, counts, normals ? 1 : 0, out_points,
                        normals ? out_normals : out_colors, nullptr);
        else CPHB_LAUNCH(voxel_final_kernel<3>, gridv, 256, 0, s, order, n_out, sums, counts, 1, out_points, out_normals, out_colors);
        CPHB_CHECK_LAUNCH();
    }
    cphb_free_async(base, s);
    CPHB_CUDA(cudaStreamSynchronize(s));
    *h_n_out = n_out;
    return CPHB_OK;
}

extern "C" int cphb_voxel_down_sample(const float *points, const float *normals, const float *colors, size_t n,
                                      float voxel_size, float *out_points, float *out_normals, float *out_colors,
                                      size_t *h_n_out, void *stream) {
    return voxel_down_sample_impl(points, normals, colors, n, voxel_size, nullptr, out_points, out_normals, out_colors, h_n_out,
                                  stream);
}

extern "C" int cphb_voxel_down_sample_origin(const float *points, const float *normals, const float *colors, size_t n,
                                             float voxel_size, const float h_origin[3], float *out_points, float *out_normals,
                                             float *out_colors, size_t *h_n_out, void *stream) {
    if (!h_origin) {
        cphb_set_error("cphb_voxel_down_sample_origin: origin is null");
        return CPHB_ERR_INVALID;
    }
    return voxel_down_sample_impl(points, normals, colors, n, voxel_size, h_origin, out_points, out_normals, out_colors, h_n_out,
                                  stream);
}
