// sort.cu -- radix sort of (key, value) pairs (CUB DeviceRadixSort).
// Used once per index build / per source ordering / per voxel pass; never in
// the per-iteration ICP loop.  Kept in its own translation unit so the
// hand-written kernels compile in seconds.
#include <cub/device/device_radix_sort.cuh>

#include "cphb_internal.cuh"

template <typename K>
static int sort_pairs(const K *keys_in, K *keys_out, const uint32_t *vals_in, uint32_t *vals_out,
                      size_t n, int bits, cudaStream_t s) {
    if (n == 0) return CPHB_OK;
    if (n > (size_t)INT32_MAX) {
        cphb_set_error("sort: n=%zu exceeds 2^31-1", n);
        return CPHB_ERR_INVALID;
    }
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in, keys_out, vals_in, vals_out,
                                              (int)n, 0, bits, s));
    cphb_scratch sc(s);
    char *tmp = nullptr;
    int rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys_in, keys_out, vals_in, vals_out,
                                                    (int)n, 0, bits, s);
    g_cphb_launches += (bits + 7) / 8 + 1;  // histogram + one onesweep pass per 8 bits
    if (e != cudaSuccess) {
        cphb_set_error("cub::DeviceRadixSort::SortPairs: %s", cudaGetErrorString(e));
        return CPHB_ERR_CUDA;
    }
    return CPHB_OK;
}

int cphb_sort_pairs_u32(const uint32_t *keys_in, uint32_t *keys_out, const uint32_t *vals_in,
                        uint32_t *vals_out, size_t n, int bits, cudaStream_t s) {
    return sort_pairs<uint32_t>(keys_in, keys_out, vals_in, vals_out, n, bits, s);
}
int cphb_sort_pairs_u64(const uint64_t *keys_in, uint64_t *keys_out, const uint32_t *vals_in,
                        uint32_t *vals_out, size_t n, int bits, cudaStream_t s) {
    return sort_pairs<uint64_t>(keys_in, keys_out, vals_in, vals_out, n, bits, s);
}

int cphb_sort_keys_u64(const uint64_t *keys_in, uint64_t *keys_out, size_t n, int bits, cudaStream_t s) {
    if (n == 0) return CPHB_OK;
    if (n > (size_t)INT32_MAX) {
        cphb_set_error("sort: n=%zu exceeds 2^31-1", n);
        return CPHB_ERR_INVALID;
    }
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, keys_in, keys_out, (int)n, 0, bits, s));
    cphb_scratch sc(s);
    char *tmp = nullptr;
    int rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    cudaError_t e = cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, keys_in, keys_out, (int)n, 0, bits, s);
    g_cphb_launches += (bits + 7) / 8 + 1;  // as sort_pairs
    if (e != cudaSuccess) {
        cphb_set_error("cub::DeviceRadixSort::SortKeys: %s", cudaGetErrorString(e));
        return CPHB_ERR_CUDA;
    }
    return CPHB_OK;
}
