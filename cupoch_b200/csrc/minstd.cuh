// minstd.cuh -- thrust::default_random_engine (minstd_rand: x_{k+1} = 48271 x_k mod 2^31 - 1) reached by
// jump-ahead: the k-th draw after a seed x0 is a^k x0 mod m, and a^k is the product of the table entries a^(2^j) for
// the set bits j of k.  Shared by SegmentPlane's sampler (segment.cu) and SamplePointsUniformly (mesh.cu);
// oracle/segment_plane.c and oracle/mesh_ops.c restate it.
#pragma once
#include <stdint.h>

#define CPHB_MINSTD_A 48271u
#define CPHB_MINSTD_M 2147483647u

struct cphb_minstd_pow {
    uint32_t p[32];  // a^(2^j) mod m
};

__host__ __device__ __forceinline__ uint32_t cphb_minstd_mulmod(uint32_t x, uint32_t y) {  // x * y mod 2^31 - 1
    const uint64_t p = (uint64_t)x * y;
    uint64_t r = (p & CPHB_MINSTD_M) + (p >> 31);
    r = (r & CPHB_MINSTD_M) + (r >> 31);
    return (uint32_t)(r >= CPHB_MINSTD_M ? r - CPHB_MINSTD_M : r);
}

static inline void cphb_minstd_table(cphb_minstd_pow *pw) {
    pw->p[0] = CPHB_MINSTD_A;
    for (int j = 1; j < 32; ++j) pw->p[j] = cphb_minstd_mulmod(pw->p[j - 1], pw->p[j - 1]);
}

// x a^e mod m, e < 2^32
__host__ __device__ __forceinline__ uint32_t cphb_minstd_jump(uint32_t x, uint64_t e, const cphb_minstd_pow &pw) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
        if ((e >> j) & 1u) x = cphb_minstd_mulmod(x, pw.p[j]);
    return x;
}
