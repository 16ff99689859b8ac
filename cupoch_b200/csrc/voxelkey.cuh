// voxelkey.cuh -- the packed-key lookup of VoxelGrid keys, shared by collision.cu (VoxelGrid targets) and
// voxelgrid_ops.cu (CheckIfIncluded, +=, AddVoxels).
//
// A key (x, y, z) is packed relative to the smallest key on each axis, 21 bits per axis, x highest, so ascending packed
// keys are the keys in lexicographic order.  cphb_sort_voxel_keys sorts the packed keys of any [n][3] int32 key array
// (unsorted and repeated keys included) with their original indices; the CUB radix sort is stable, so equal keys keep
// their original order.
#pragma once

#include "cphb_internal.cuh"

#define CPHB_KEY_AXIS_BITS 21

__device__ __forceinline__ uint64_t cphb_key_pack(const int lo[3], int x, int y, int z) {
    return ((uint64_t)(uint32_t)(x - lo[0]) << (2 * CPHB_KEY_AXIS_BITS)) | ((uint64_t)(uint32_t)(y - lo[1]) << CPHB_KEY_AXIS_BITS) |
           (uint64_t)(uint32_t)(z - lo[2]);
}

// first position of sorted[0, n) whose packed key is >= k
__device__ __forceinline__ size_t cphb_key_lower_bound(const uint64_t *sorted, size_t n, uint64_t k) {
    size_t a = 0, b = n;
    while (a < b) {
        const size_t m = (a + b) >> 1;
        if (sorted[m] < k) a = m + 1;
        else b = m;
    }
    return a;
}

// keys [n][3] (device, n >= 1) -> the key bounds lo / hi (host) and, in buffers taken from sc, the packed keys in
// ascending order with their original indices.  A key span of 2^21 or more on an axis is CPHB_ERR_INVALID, reported
// as "<who>: ...".  collision.cu
struct cphb_sorted_keys {
    const uint64_t *skeys;
    const uint32_t *sidx;
    int lo[3], hi[3];
};
int cphb_sort_voxel_keys(const int32_t *keys, size_t n, cphb_scratch &sc, cphb_sorted_keys *out, cudaStream_t s, const char *who);
