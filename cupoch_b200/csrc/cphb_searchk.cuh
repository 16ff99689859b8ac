// cphb_searchk.cuh -- the k-best result set of the warp-cooperative traversal (k > 1), used by every k-list kernel
// through fused_neighbourhood.cuh: search.cu (SearchKNN / SearchRadius), features.cu (the fused EstimateNormals kernel)
// and iss.cu (ComputeISSKeypoints).
#pragma once
#include "cphb_internal.cuh"

// ---------------------------------------------------------------------------
// k-best result set per lane, kept in shared memory as list[k][32] (column =
// lane, so any mix of insert positions is bank-conflict free).  Ascending by
// key = (d2 bits, index).  Mirrors KnnRadiusResultSet (result_set.h:372-474):
// strict d2 < r2, unfilled slots idx=-1 / d2=+inf.
// ---------------------------------------------------------------------------
struct WarpSearchK : WarpSearchBase {
    unsigned long long *list;  // this lane's column
    int k;
    unsigned long long worst;  // == list[(k-1)*32]
    __device__ __forceinline__ unsigned lane_bound() const { return (unsigned)(worst >> 32); }
};

__device__ __forceinline__ void scan_tile(const float4 *tile, WarpSearchK &w, unsigned /*need*/) {
    const int k = w.k;
#pragma unroll 4
    for (int j = 0; j < CPHB_LEAF; ++j) {
        float4 p = tile[j];
        float d2 = dist2(w.qx, w.qy, w.qz, p.x, p.y, p.z);
        unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | __float_as_uint(p.w);
        if (key < w.worst) {
            int pos = k - 1;
            while (pos > 0) {
                unsigned long long prev = w.list[(pos - 1) * 32];
                if (prev <= key) break;
                w.list[pos * 32] = prev;
                --pos;
            }
            w.list[pos * 32] = key;
            w.worst = w.list[(k - 1) * 32];
        }
    }
}

