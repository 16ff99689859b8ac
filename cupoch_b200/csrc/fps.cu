// fps.cu -- PointCloud::FarthestPointDownSample (pointcloud.cu:122-139,301-338): farthest-point sampling.
//
// The reference runs one thrust::transform_reduce per sample (update every point's distance to the selected set, take
// the argmax) and reads the winner back to the host before the next step: one launch and one host round trip per
// sample.  The steps are sequential but each is a tiny amount of work, so here the whole loop is ONE cooperative
// launch of a persistent grid (co-residency guaranteed by cudaLaunchCooperativeKernel):
//   per step  every thread updates its points' running distances and keeps its best key; warps reduce with REDUX
//             (max of the distance bits, then min of the index among the lanes holding that maximum); one atomicMax
//             per block on a 64-bit slot; one grid barrier; every thread reads the winner from the slot and its
//             coordinates from global memory.
//   slots     three, rotated: block 0 clears slot (t+1) % 3 before it arrives at barrier t.  Slot (t+1) % 3 was last
//             read after barrier t-2, and every block has passed those reads once barrier t-1 is complete, so one
//             barrier per step suffices.
//   residency while n <= SMs * FPS_SMEM_POINTS (about 1.9 M points on 132 SMs) each block keeps its contiguous chunk
//             of points as float4 (xyz, running distance) in shared memory for the whole call; above that the points
//             are re-read from the caller's packed xyz and the distances from a global array every step.  Both paths
//             are the same kernel body (fps_kernel<RES>).
//
// Arithmetic (DESIGN.md arithmetic contract; the CPU oracle restates it):
//   d2 = dist2 (the search's operation order), dist = fminf(dist, d2) (a NaN d2 never replaces dist), so every dist
//   lies in [+0, +inf] and its bits order like its value; key = (dist bits << 32) | (0xFFFFFFFF - index), the argmax
//   is the largest key: the farthest point, the smallest index among equal distances.
#include <cooperative_groups.h>

#include "cphb_internal.cuh"

namespace cg = cooperative_groups;

#define FPS_THREADS 1024
#define FPS_SMEM_POINTS 14336  // resident points per block: 224 KB of float4, one block per SM

struct FpsArgs {
    const float *pts;  // packed xyz
    size_t n, num_samples, chunk;  // chunk: points per block
    int32_t *indices_out;
    float *dist;        // streamed path: running distances [n] (d2_out when given)
    float *d2_out;      // resident path: final distances, or NULL
    unsigned long long *slots;  // [3], zero on entry
};

template <bool RES>
__global__ void __launch_bounds__(FPS_THREADS, 1) fps_kernel(FpsArgs a) {
    extern __shared__ float4 s_pt[];  // RES: this block's points, w = running distance
    __shared__ unsigned s_d[FPS_THREADS / 32], s_i[FPS_THREADS / 32];
    cg::grid_group grid = cg::this_grid();
    const size_t lo = (size_t)blockIdx.x * a.chunk;
    const int len = lo < a.n ? (int)min(a.chunk, a.n - lo) : 0;
    const float inf = __int_as_float(0x7f800000);
    if (RES) {  // each thread only ever touches its own positions k: no block barrier needed
#pragma unroll 1  // unrolled, the loads of the copy alone fill the register budget and spill
        for (int k = threadIdx.x; k < len; k += FPS_THREADS) {
            const float *p = a.pts + 3 * (lo + k);
            s_pt[k] = make_float4(p[0], p[1], p[2], inf);
        }
    }
    const int warp = threadIdx.x >> 5, lane = lane_id();
    unsigned far = 0;
    for (size_t t = 0;; ++t) {
        if (blockIdx.x == 0 && threadIdx.x == 0) a.indices_out[t] = (int32_t)far;
        const float fx = __ldg(a.pts + 3 * (size_t)far), fy = __ldg(a.pts + 3 * (size_t)far + 1),
                    fz = __ldg(a.pts + 3 * (size_t)far + 2);
        unsigned long long best = 0ull;  // below every real key (0xFFFFFFFF - index > 0 for n <= 2^31-1)
#pragma unroll 4
        for (int k = threadIdx.x; k < len; k += FPS_THREADS) {
            float x, y, z, d;
            if (RES) {
                const float4 q = s_pt[k];
                x = q.x; y = q.y; z = q.z; d = q.w;
            } else {
                const float *p = a.pts + 3 * (lo + k);
                x = __ldg(p); y = __ldg(p + 1); z = __ldg(p + 2);
                d = t ? a.dist[lo + k] : inf;
            }
            const float nd = fminf(d, dist2(x, y, z, fx, fy, fz));
            if (RES) {
                if (nd < d) s_pt[k].w = nd;
            } else if (nd < d || t == 0) {
                a.dist[lo + k] = nd;
            }
            const unsigned long long key =
                ((unsigned long long)__float_as_uint(nd) << 32) | (0xffffffffu - (unsigned)(lo + k));
            best = key > best ? key : best;
        }
        if (t + 1 == a.num_samples) break;  // the last argmax is never observed
        unsigned hi = (unsigned)(best >> 32), idx = 0xffffffffu - (unsigned)best;
        unsigned m = __reduce_max_sync(CPHB_FULL, hi);
        idx = __reduce_min_sync(CPHB_FULL, hi == m ? idx : 0xffffffffu);
        if (lane == 0) {
            s_d[warp] = m;
            s_i[warp] = idx;
        }
        __syncthreads();
        if (warp == 0) {
            hi = s_d[lane];
            m = __reduce_max_sync(CPHB_FULL, hi);
            idx = __reduce_min_sync(CPHB_FULL, hi == m ? s_i[lane] : 0xffffffffu);
            if (lane == 0) {
                atomicMax(a.slots + t % 3, ((unsigned long long)m << 32) | (0xffffffffu - idx));
                if (blockIdx.x == 0) a.slots[(t + 1) % 3] = 0ull;
            }
        }
        grid.sync();
        far = 0xffffffffu - (unsigned)__ldcg(a.slots + t % 3);  // L2: the slot is rewritten every third step
    }
    if (RES && a.d2_out)
        for (int k = threadIdx.x; k < len; k += FPS_THREADS) a.d2_out[lo + k] = s_pt[k].w;
}

extern "C" int cphb_farthest_point_down_sample(const float *points, size_t n, size_t num_samples, int32_t *indices_out,
                                               float *d2_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n > (size_t)INT32_MAX) {
        cphb_set_error("cphb_farthest_point_down_sample: n = %zu (need n <= 2^31-1)", n);
        return CPHB_ERR_INVALID;
    }
    if (num_samples == 0) return CPHB_OK;
    if (n == 0 || !points || !indices_out) {
        cphb_set_error("cphb_farthest_point_down_sample: %s", n == 0 ? "no points to sample from" : "null argument");
        return CPHB_ERR_INVALID;
    }
    int dev = 0, sms = 0;
    CPHB_CUDA(cudaGetDevice(&dev));
    CPHB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const bool res = n <= (size_t)sms * FPS_SMEM_POINTS;
    const void *fn = res ? (const void *)fps_kernel<true> : (const void *)fps_kernel<false>;
    size_t smem = 0;
    if (res) {
        smem = (n + sms - 1) / sms * sizeof(float4);
        CPHB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, FPS_SMEM_POINTS * (int)sizeof(float4)));
    }
    int per_sm = 0;
    CPHB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, FPS_THREADS, smem));
    if (per_sm < 1) {
        cphb_set_error("cphb_farthest_point_down_sample: the kernel does not fit on an SM");
        return CPHB_ERR_CUDA;
    }
    // every block gets points: blocks without any would only add arrivals to the barrier
    size_t grid = (size_t)sms * per_sm;
    if (grid > (n + FPS_THREADS - 1) / FPS_THREADS) grid = (n + FPS_THREADS - 1) / FPS_THREADS;
    FpsArgs a;
    a.pts = points;
    a.n = n;
    a.num_samples = num_samples;
    a.chunk = (n + grid - 1) / grid;
    a.indices_out = indices_out;
    a.d2_out = d2_out;
    a.dist = nullptr;
    a.slots = nullptr;
    if (res) smem = a.chunk * sizeof(float4);
    cphb_scratch sc(s);
    int rc = sc.alloc(&a.slots, 3);
    if (!rc && !res) {
        if (d2_out) a.dist = d2_out;
        else rc = sc.alloc(&a.dist, n);
    }
    if (!rc) {
        cudaError_t e = cudaMemsetAsync(a.slots, 0, 3 * sizeof(unsigned long long), s);
        void *args[] = {&a};
        if (e == cudaSuccess) e = cudaLaunchCooperativeKernel(fn, dim3((unsigned)grid), dim3(FPS_THREADS), args, smem, s);
        ++g_cphb_launches;
        if (e != cudaSuccess) {
            cphb_set_error("cphb_farthest_point_down_sample: %s", cudaGetErrorString(e));
            rc = CPHB_ERR_CUDA;
        }
    }
    return rc;
}
