// fused_neighbourhood.cuh -- the "k-best search, then a per-point epilogue over the list" form shared by every k-list
// kernel: search.cu (searchk_kernel, whose epilogue writes the [n][k] table), features.cu (EstimateNormals), iss.cu
// (ComputeISSKeypoints) and shot.cu (ComputeSHOTFeature, with shared memory of its own per warp: launch_fused_extra).  The warp's k-best search with its lists in shared memory, its one launch rule
// (launch_fused), the 9 cumulants over a lane's list in list order (geometry_functor.h:35-55) and the covariance
// E[xx^T] - E[x]E[x]^T formed from them; the fused epilogues write no [n][k] table.
// Translation units including this must be compiled with -fmad=false.
#pragma once
#include "cphb_internal.cuh"
#include "cphb_searchk.cuh"

// compute_cumulant_functor (geometry_functor.h:35-55): one neighbour into the 9 cumulants (float64 sums of exact products)
__device__ __forceinline__ void cumulant_add(double (&cum)[9], float x, float y, float z) {
    cum[0] += x; cum[1] += y; cum[2] += z;
    cum[3] = fma((double)x, (double)x, cum[3]); cum[4] = fma((double)x, (double)y, cum[4]);
    cum[5] = fma((double)x, (double)z, cum[5]); cum[6] = fma((double)y, (double)y, cum[6]);
    cum[7] = fma((double)y, (double)z, cum[7]); cum[8] = fma((double)z, (double)z, cum[8]);
}

// covariance E[xx^T] - E[x]E[x]^T in float32 from the cumulants divided by (float)cnt, row-major (estimate_normals.cu:38-54,
// iss_keypoints.cu:51-63).  cnt == 0 gives NaN coefficients.
__device__ __forceinline__ void covariance_from_cumulants(const double (&cum)[9], int cnt, float (&cov)[9]) {
    float c[9];
#pragma unroll
    for (int a = 0; a < 9; ++a) c[a] = (float)cum[a] / (float)cnt;
    cov[0] = __fmaf_rn(-c[0], c[0], c[3]);
    cov[4] = __fmaf_rn(-c[1], c[1], c[6]);
    cov[8] = __fmaf_rn(-c[2], c[2], c[8]);
    cov[1] = cov[3] = __fmaf_rn(-c[0], c[1], c[4]);
    cov[2] = cov[6] = __fmaf_rn(-c[0], c[2], c[5]);
    cov[5] = cov[7] = __fmaf_rn(-c[1], c[2], c[7]);
}

// Per-lane query and empty k-best list of a fused kernel.  Dynamic shared memory per warp: 2 leaf tiles, 2 mbarriers,
// k * 32 list keys (fused_smem_per_warp).  Returns the list's initial key: a slot holds a neighbour iff its key < init.
//   self_order: the queries are the indexed cloud itself, taken in INDEX order (lane = one point of a leaf, so a warp's
//               queries are exactly one leaf and need no ordering pass); original position = ix.pts[i].w
//   otherwise : query i is pts[first + perm[i]] (perm = Hilbert order of the block, or NULL), output row perm[i]
// Every lane of the warp must then call fused_query_search, valid or not (it is warp-collective).
__device__ __forceinline__ unsigned long long fused_query_setup(WarpSearchK &w, unsigned char *smem, const IndexView &ix,
                                                                const float *__restrict__ pts, size_t first, size_t count,
                                                                const uint32_t *__restrict__ perm, int self_order, float r2,
                                                                int k, size_t &pos) {
    const int nwarp = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5;
    float4 *tiles = (float4 *)smem;
    uint64_t *bars = (uint64_t *)(tiles + (size_t)nwarp * 2 * CPHB_LEAF);
    unsigned long long *lists = (unsigned long long *)(bars + 2 * nwarp);
    warp_search_setup(w, tiles + (size_t)warp * 2 * CPHB_LEAF, bars + 2 * warp);
    w.k = k;
    w.list = lists + (size_t)warp * k * 32 + lane_id();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    pos = 0;
    w.qx = w.qy = w.qz = 0.f;
    if (self_order) {
        w.valid = i < (size_t)ix.n_leaves * CPHB_LEAF;
        if (w.valid) {
            const float4 q = ix.pts[i];
            w.valid = __float_as_uint(q.w) != 0xffffffffu;  // padded tail of the index
            pos = __float_as_uint(q.w);
            w.qx = q.x; w.qy = q.y; w.qz = q.z;
        }
    } else {
        w.valid = i < count;
        if (w.valid) {
            pos = perm ? perm[i] : i;
            const float *q = pts + 3 * (first + pos);
            w.qx = q[0]; w.qy = q[1]; w.qz = q[2];
        }
    }
    const unsigned long long init = (r2 > 0.f) ? init_key(r2) : 0ull;
    for (int j = 0; j < k; ++j) w.list[j * 32] = init;
    w.worst = init;
    w.bound = (unsigned)(init >> 32);
    return init;
}

// the k-best search of the warp's valid lanes (a lane may be switched off between setup and search)
template <int TOP>
__device__ __forceinline__ void fused_query_search(const IndexView &ix, WarpSearchK &w) {
    warp_query_box(w);
    if (__any_sync(CPHB_FULL, w.valid)) warp_nn_search<TOP>(ix, w);
}

// the 9 cumulants and the count over this lane's filled slots, in list order (ascending (d2, index))
__device__ __forceinline__ void list_cumulants(const WarpSearchK &w, int k, unsigned long long init,
                                               const float *__restrict__ pts, double (&cum)[9], int &cnt) {
#pragma unroll
    for (int a = 0; a < 9; ++a) cum[a] = 0;
    cnt = 0;
    for (int j = 0; j < k; ++j) {
        const unsigned long long key = w.list[j * 32];
        if (!(key < init)) break;  // ascending: the unfilled slots are at the end
        const size_t id = (unsigned)(key & 0xffffffffull);
        cumulant_add(cum, pts[3 * id], pts[3 * id + 1], pts[3 * id + 2]);
        ++cnt;
    }
}

// dynamic shared memory of one warp of a fused kernel with k-slot lists, plus `extra` bytes of the kernel's own per warp
// (placed after every warp's lists: fused_warp_extra)
static inline size_t fused_smem_per_warp(int k, size_t extra = 0) {
    return 2 * CPHB_LEAF * sizeof(float4) + 2 * sizeof(uint64_t) + (size_t)k * 32 * sizeof(unsigned long long) + extra;
}

// this warp's `extra` bytes of a kernel launched with launch_fused_extra (16-byte aligned when `extra` is a multiple of 16)
__device__ __forceinline__ unsigned char *fused_warp_extra(unsigned char *smem, int k, size_t extra) {
    const size_t nwarp = blockDim.x >> 5;
    unsigned char *lists_end =
        smem + nwarp * (2 * CPHB_LEAF * sizeof(float4) + 2 * sizeof(uint64_t) + (size_t)k * 32 * sizeof(unsigned long long));
    return lists_end + (size_t)(threadIdx.x >> 5) * extra;
}

// launch of one k-list kernel over `lanes` query lanes (one thread each): as many warps per block as fit in 96 KB of
// lists, tiles and `extra` bytes per warp, 1 to 8; the <3> or <5> instance by the index's depth.  The kernel's first
// argument is the index view.
template <class K3, class K5, class... Args>
static int launch_fused_extra(const cphb_index *ix, K3 k3, K5 k5, size_t lanes, int k, size_t extra, cudaStream_t s,
                              Args... args) {
    int warps = (int)((96 * 1024) / fused_smem_per_warp(k, extra));
    if (warps > 8) warps = 8;
    if (warps < 1) warps = 1;
    const size_t smem = fused_smem_per_warp(k, extra) * warps;
    const unsigned block = warps * 32;
    const unsigned grid = (unsigned)((lanes + block - 1) / block);
    if (ix->v.top <= 3) {
        CPHB_CUDA(cudaFuncSetAttribute(k3, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CPHB_LAUNCH(k3, grid, block, smem, s, ix->v, args...);
    } else {
        CPHB_CUDA(cudaFuncSetAttribute(k5, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CPHB_LAUNCH(k5, grid, block, smem, s, ix->v, args...);
    }
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}
template <class K3, class K5, class... Args>
static int launch_fused(const cphb_index *ix, K3 k3, K5 k5, size_t lanes, int k, cudaStream_t s, Args... args) {
    return launch_fused_extra(ix, k3, k5, lanes, k, 0, s, args...);
}
