// sum_values.cuh -- the engine's fixed-order float64 sum of per-element float32 values (reduce.cu's normal-equation
// sums, mesh.cu's surface area).  Thread t of block b adds its elements b * RED_BLOCK + t + k * grid * RED_BLOCK in
// order from 0.0, the warp adds its lanes by an xor butterfly (offsets 16, 8, 4, 2, 1; every lane ends with the same
// bits), the block adds its warps in order from 0.0, and one thread adds the blocks in order from 0.0.  grid =
// min(ceil(n / RED_BLOCK), RED_MAX_BLOCKS).  The order is part of the answer; oracle/mesh_ops.c restates it.
#pragma once
#include "cphb_internal.cuh"

#define RED_BLOCK 256
#define RED_MAX_BLOCKS 592

// ---------------------------------------------------------------------------------------------------------------------
// fixed-order sum of NV values per element
// ---------------------------------------------------------------------------------------------------------------------
template <int NV, class F>
__global__ void __launch_bounds__(RED_BLOCK) sum_values_kernel(F f, size_t n, double *partials) {
    __shared__ double s_part[RED_BLOCK / 32][NV];
    double acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = 0.0;
    // thread t of block b owns elements b*RED_BLOCK + t + k*gridDim.x*RED_BLOCK: a fixed assignment
    for (size_t i = blockIdx.x * (size_t)RED_BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * RED_BLOCK) {
        float v[NV];
        f(i, v);
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] += (double)v[k];
    }
    // warp: xor butterfly (same bits on every lane); block: warps in order
#pragma unroll
    for (int k = 0; k < NV; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(CPHB_FULL, acc[k], o);
    }
    const int warp = threadIdx.x >> 5;
    if (lane_id() == 0)
#pragma unroll
        for (int k = 0; k < NV; ++k) s_part[warp][k] = acc[k];
    __syncthreads();
    if (threadIdx.x < NV) {
        double t = 0.0;
        for (int w2 = 0; w2 < RED_BLOCK / 32; ++w2) t += s_part[w2][threadIdx.x];
        partials[(size_t)blockIdx.x * NV + threadIdx.x] = t;
    }
}
template <int NV>
__global__ void sum_partials_kernel(const double *partials, unsigned n_blocks, double *total) {
    if (threadIdx.x >= NV) return;
    double t = 0.0;
    for (unsigned b = 0; b < n_blocks; ++b) t += partials[(size_t)b * NV + threadIdx.x];
    total[threadIdx.x] = t;
}

template <int NV, class F>
static int sum_values(const F &f, size_t n, double *h_out, cudaStream_t s) {
    for (int k = 0; k < NV; ++k) h_out[k] = 0.0;
    if (n == 0) return CPHB_OK;
    unsigned grid = (unsigned)((n + RED_BLOCK - 1) / RED_BLOCK);
    if (grid > RED_MAX_BLOCKS) grid = RED_MAX_BLOCKS;
    cphb_scratch sc(s);
    double *buf = nullptr;
    int rc = sc.alloc(&buf, NV * ((size_t)grid + 1));
    if (rc) return rc;
    CPHB_LAUNCH((sum_values_kernel<NV, F>), grid, RED_BLOCK, 0, s, f, n, buf);
    CPHB_LAUNCH(sum_partials_kernel<NV>, 1, 32, 0, s, buf, grid, buf + (size_t)grid * NV);
    return cphb_read_back(h_out, buf + (size_t)grid * NV, sizeof(double) * NV, s, "sum_values");
}
