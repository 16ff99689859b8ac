// cphb_internal.cuh -- shared host/device definitions of the H100 engine.
// sm_90a only.  Not part of the public interface (see include/cupoch_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "cupoch_b200.h"

// ---------------------------------------------------------------------------
// Spatial index layout (DESIGN.md "Data layout in HBM")
//   pts   : float4[n_leaves*LEAF]  points in 3-D Hilbert order, w = original
//           index bits; tail padded with (FLT_MAX,FLT_MAX,FLT_MAX, -1)
//   boxes : per level, Box[ceil32(count)]; level 0 = leaves (LEAF consecutive
//           points), level l node j = union of level l-1 nodes [32j, 32j+32).
//           Padding boxes are empty (lo=+inf, hi=-inf) so their distance is
//           +inf and no traversal ever enters them.
// A warp owns 32 queries; it tests the 32 children of a node with one lane per
// child and walks children nearest-first, so the only divergence is the loop
// trip count.  Leaves are fetched by one TMA bulk copy (cp.async.bulk) into a
// per-warp shared-memory tile and scanned with broadcast LDS.128.
// ---------------------------------------------------------------------------
#define CPHB_LEAF 32
#define CPHB_LEVELS 6 /* box levels always built: 32^5 * LEAF points max */
#define CPHB_FULL 0xffffffffu
#define CPHB_SMS 132 /* H100 SXM; grid caps of grid-stride kernels are CPHB_SMS * 8 blocks of 256 */

struct Box {
    float4 lo;
    float4 hi;
};

struct IndexView {
    const float4 *pts;
    const uint32_t *inv;  // inv[original index] = position in Hilbert order
    const Box *boxes[CPHB_LEVELS];
    unsigned long long n;
    unsigned n_leaves;
    int top; /* smallest level with <= 32 nodes */
};

struct cphb_index {
    IndexView v;
    void *arena;
    size_t arena_bytes;
    float *bounds; /* device: 6 ordered-uint encoded floats (min xyz, max xyz) */
    int device;
    cudaStream_t stream; /* stream the arena was allocated on */
};

// ---------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------
void cphb_set_error(const char *fmt, ...);
extern unsigned long long g_cphb_launches;

#define CPHB_CUDA(call)                                                                   \
    do {                                                                                  \
        cudaError_t e__ = (call);                                                         \
        if (e__ != cudaSuccess) {                                                         \
            cphb_set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return CPHB_ERR_CUDA;                                                         \
        }                                                                                 \
    } while (0)

#define CPHB_LAUNCH(kernel, grid, block, smem, stream, ...)                 \
    do {                                                                    \
        kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__); \
        ++g_cphb_launches;                                                  \
    } while (0)

#define CPHB_CHECK_LAUNCH()                                                               \
    do {                                                                                  \
        cudaError_t e__ = cudaGetLastError();                                             \
        if (e__ != cudaSuccess) {                                                         \
            cphb_set_error("%s:%d kernel launch: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return CPHB_ERR_CUDA;                                                         \
        }                                                                                 \
    } while (0)

static inline size_t cphb_align(size_t x, size_t a) { return (x + a - 1) / a * a; }

// stream-ordered allocation (pool retained across calls; no cudaMalloc in loops)
int cphb_alloc_async(void **p, size_t bytes, cudaStream_t s);
void cphb_free_async(void *p, cudaStream_t s);

// radix sort of (key,value) u32 pairs by the low `bits` bits (CUB, stable; index
// build, source ordering and SegmentPlane's sampler -- never inside the ICP
// per-iteration loop). sort.cu
int cphb_sort_pairs_u32(const uint32_t *keys_in, uint32_t *keys_out, const uint32_t *vals_in,
                        uint32_t *vals_out, size_t n, int bits, cudaStream_t s);
int cphb_sort_pairs_u64(const uint64_t *keys_in, uint64_t *keys_out, const uint32_t *vals_in,
                        uint32_t *vals_out, size_t n, int bits, cudaStream_t s);

// stable compaction (filters.cu): ascending positions i < n with keep[i] != 0 -> indices_out, their number to
// *h_n_out (synchronises the stream)
int cphb_compact_flags(const uint8_t *keep, size_t n, int32_t *indices_out, size_t *h_n_out, cudaStream_t s);

// index.cu internals reused by icp.cu (Hilbert-ordering of the source)
// perm_out[pos] = original index of the pos-th point along the Hilbert curve.
// bounds_dev6: device buffer of 6 ordered-uint floats; computed here unless
// bounds_given (then the existing bounds, e.g. the target index's, are used so
// queries and targets share one curve).
int cphb_hilbert_order(const float *xyz, size_t n, uint32_t *perm_out /*device n*/,
                       float *bounds_dev6 /*or NULL*/, int bounds_given, cudaStream_t s);
// same, with the curve resolution chosen for n_ref points (query ordering: n_ref = size of the indexed cloud)
int cphb_hilbert_order_n(const float *xyz, size_t n, uint32_t *perm_out, float *bounds_dev6, int bounds_given,
                         size_t n_ref, cudaStream_t s);

// ---------------------------------------------------------------------------
// communicator for the sharded ICP (comm.cu)
// ---------------------------------------------------------------------------
#define CPHB_COMM_NCCL 1
#define CPHB_COMM_P2P 2
#define CPHB_P2P_MAX_WORLD 16
// mailbox layout per rank: data[2][MAX_WORLD][32] doubles, then flags[2][MAX_WORLD] u64
#define CPHB_P2P_DATA_BYTES (2 * CPHB_P2P_MAX_WORLD * 32 * 8)
#define CPHB_P2P_BOX_BYTES (CPHB_P2P_DATA_BYTES + 2 * CPHB_P2P_MAX_WORLD * 8)
#define CPHB_P2P_ALLOC_BYTES (CPHB_P2P_BOX_BYTES + 64) /* + this rank's private exchange counter */
struct P2pView {
    char *box[CPHB_P2P_MAX_WORLD];  // box[q] = rank q's mailbox as mapped into THIS process
    int rank, world;
};
struct cphb_comm {
    int kind, rank, world, connected;
    void *nccl;
    void *box_local;
    P2pView view;
};
int cphb_nccl_allreduce_f64(void *nccl_comm, const double *send, double *recv, size_t count, cudaStream_t s);

#ifdef __CUDACC__
// One warp (lanes = columns) of every rank calls this the same number of times: returns the sum over
// ranks of `mine`, added in rank order (bit-identical on every rank).  Data and flag stores go straight
// to the peers' HBM over NVLink; the wait spins on this rank's own memory.  The exchange number lives in
// this rank's device memory (every rank executes the same sequence of exchanges, so the counters agree);
// its parity selects one of two slot sets, which is what makes back-to-back exchanges safe: a peer can be
// at most one exchange ahead.
// The wait is bounded (~60 s of SM clock -- far beyond any start-up skew between ranks, which wait for each other here
// in their very first exchange): if a peer never arrives -- its process died, or a one-sided host error kept
// it from launching -- the warp stops waiting, raises *timed_out (when given) and returns what it has, so the GPU is
// released instead of spinning for ever; the host turns the flag into an error (cphb_icp_run).
__device__ __forceinline__ double p2p_exchange_sum(const P2pView &v, double mine, unsigned *timed_out = nullptr) {
    const int c = threadIdx.x & 31;
    unsigned long long *ctr = (unsigned long long *)(v.box[v.rank] + CPHB_P2P_BOX_BYTES);
    const unsigned long long epoch = *(volatile unsigned long long *)ctr + 1ull;
    __syncwarp();
    if (c == 0) *(volatile unsigned long long *)ctr = epoch;
    const int par = (int)(epoch & 1ull);
    for (int q = 0; q < v.world; ++q) {
        double *slot = (double *)v.box[q] + ((size_t)par * CPHB_P2P_MAX_WORLD + v.rank) * 32;
        *((volatile double *)slot + c) = mine;
    }
    __threadfence_system();
    __syncwarp();
    if (c < v.world) {
        volatile unsigned long long *f =
            (volatile unsigned long long *)(v.box[c] + CPHB_P2P_DATA_BYTES) + (size_t)par * CPHB_P2P_MAX_WORLD + v.rank;
        *f = epoch;  // lane c raises this rank's flag in peer c's mailbox
        volatile unsigned long long *mine_f =
            (volatile unsigned long long *)(v.box[v.rank] + CPHB_P2P_DATA_BYTES) + (size_t)par * CPHB_P2P_MAX_WORLD + c;
        const long long t0 = clock64();
        while (*mine_f < epoch) {
            if (clock64() - t0 > 120000000000ll) {
                if (timed_out) atomicExch(timed_out, 1u);
                break;
            }
        }
    }
    __syncwarp();
    __threadfence_system();
    double tot = 0.0;
    for (int q = 0; q < v.world; ++q) {
        const double *slot = (const double *)v.box[v.rank] + ((size_t)par * CPHB_P2P_MAX_WORLD + q) * 32;
        tot += *((const volatile double *)slot + c);
    }
    return tot;
}

// ---------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// order-preserving float <-> uint (for atomicMin/Max and REDUX on signed floats)
__host__ __device__ __forceinline__ unsigned f2ord(float f) {
#ifdef __CUDA_ARCH__
    unsigned u = __float_as_uint(f);
#else
    union { float f; unsigned u; } c; c.f = f; unsigned u = c.u;
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(unsigned o) {
    unsigned u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    union { float f; unsigned u; } c; c.u = u; return c.f;
#endif
}

// squared distance, fixed operation order (DESIGN.md "arithmetic contract"):
// d = q - p per axis; d2 = fma(dz,dz, fma(dx,dx, dy*dy)) -- the order nvcc 12.9 gives the reference's own kernel for
// sm_90a under its --use_fast_math flags (FLANN CudaL2::dist, kdtree_cuda_3d_index.cu:221-227: SASS of
// oracle/_ref shows FMUL dy,dy; FFMA dx,dx; FFMA dz,dz; FFMA dw,dw with dw = 0), so squared distances are bit-identical
// to the reference binary's (tests/test_gpu_flann_ref.py)
__device__ __forceinline__ float dist2(float qx, float qy, float qz, float px, float py, float pz) {
    float dx = qx - px, dy = qy - py, dz = qz - pz;
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}
__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __fmaf_rn(a2, b2, __fmaf_rn(a1, b1, __fmul_rn(a0, b0)));
}
__device__ __forceinline__ float det2(float a, float b, float c, float d) {
    return __fmaf_rn(a, b, -__fmul_rn(c, d));
}

// lower bound of dist2 between any point of box [lo,hi] and any point of the
// query box [qlo,qhi]; same op order as dist2 so it never exceeds a real d2.
__device__ __forceinline__ float box_dist2(const float4 &lo, const float4 &hi, const float (&qlo)[3],
                                           const float (&qhi)[3]) {
    float dx = fmaxf(0.f, fmaxf(lo.x - qhi[0], qlo[0] - hi.x));
    float dy = fmaxf(0.f, fmaxf(lo.y - qhi[1], qlo[1] - hi.y));
    float dz = fmaxf(0.f, fmaxf(lo.z - qhi[2], qlo[2] - hi.z));
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// ---- 3-D Hilbert index, 10 bits per axis (Skilling's transpose form) --------
__device__ __forceinline__ uint32_t hilbert30(uint32_t x, uint32_t y, uint32_t z) {
    uint32_t X[3] = {x, y, z};
    const uint32_t M = 1u << 9;
#pragma unroll
    for (uint32_t Q = M; Q > 1; Q >>= 1) {
        uint32_t P = Q - 1;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            if (X[i] & Q) {
                X[0] ^= P;
            } else {
                uint32_t t = (X[0] ^ X[i]) & P;
                X[0] ^= t;
                X[i] ^= t;
            }
        }
    }
    X[1] ^= X[0];
    X[2] ^= X[1];
    uint32_t t = 0;
#pragma unroll
    for (uint32_t Q = M; Q > 1; Q >>= 1)
        if (X[2] & Q) t ^= Q - 1;
    X[0] ^= t; X[1] ^= t; X[2] ^= t;
    uint32_t key = 0;
#pragma unroll
    for (int b = 9; b >= 0; --b) {
        key = (key << 3) | (((X[0] >> b) & 1u) << 2) | (((X[1] >> b) & 1u) << 1) | ((X[2] >> b) & 1u);
    }
    return key;
}

// ---- TMA bulk copy + mbarrier (raw PTX; SASS: UBLKCP / SYNCS) ----------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes,
                                             uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// sqrt.approx.f32: one MUFU, max relative error 2^-23 (callers pad the result in the safe direction)
__device__ __forceinline__ float sqrt_approx(float x) {
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// ---------------------------------------------------------------------------
// Warp-cooperative exact nearest-neighbour traversal.
//
// A warp owns 32 queries (a compact cluster: queries are processed in Hilbert
// order).  At every node one lane tests one child box:
//   stage 1  box-vs-warp-AABB distance against the warp bound (max over lanes
//            of their current worst accepted d2) -- one instruction stream for
//            32 children;
//   order    children are visited by increasing distance to the warp AABB's
//            centre, so the bound tightens after the first leaves;
//   stage 2  before a child is entered its box is broadcast and every lane
//            tests its OWN query against it with its OWN bound; the child is
//            skipped unless some lane can still improve.
// Leaves are fetched by TMA bulk copies into a double-buffered shared-memory
// tile: the copy of the next candidate leaf is in flight while the current one
// is scanned.  Ties: key = (d2 bits << 32) | original index, so one u64 min
// implements "smaller d2, then smaller index" (the oracle's rule); culling
// uses <= so equal-distance candidates are never skipped.
// ---------------------------------------------------------------------------
struct WarpSearchBase {
    float qx, qy, qz;      // this lane's query
    float wlo[3], whi[3];  // warp-uniform AABB of the valid queries
    float wc[3];           // its centre
    unsigned bound;        // warp-uniform cull bound (d2 bits)
    unsigned phase;        // bit b = parity of mbarrier b
    bool valid;            // lane holds a real query
    bool warm;             // bounds are already tight (ICP warm start): skip the ordering refinements
    int tmax;              // transposed scan when at most this many lanes need the leaf
    float4 *tile;          // per-warp smem: 2 leaf tiles [2][CPHB_LEAF]
    uint64_t *bar;         // per-warp smem: 2 mbarriers
};
struct WarpSearch : WarpSearchBase {
    unsigned long long best;  // this lane's best key
    __device__ __forceinline__ unsigned lane_bound() const { return (unsigned)(best >> 32); }
};

// Certifying variant used by the ICP loop.  Besides the best key it keeps a LOWER BOUND on the squared distance
// from the query to every target point other than the best one:
//   * nodes are culled against the relaxed bound (sqrt(best_d2) + margin)^2 instead of best_d2, so every point
//     that was never evaluated is farther than that (the bound only shrinks during a search, so a node culled
//     against an earlier, larger bound is outside the final one too).  For a lane with no candidate yet best_d2
//     is r^2, so the bound also covers points just outside the radius;
//   * m1 <= m2 are the two smallest d2 among the candidates this lane evaluated in leaf scans.  A leaf is scanned
//     at most once per search and the best point's own leaf always is (its box is inside every bound), so m1 is
//     the best point's d2 and m2 bounds every other evaluated point from below.
// L2 = min(m2, final relaxed bound) lets later ICP iterations prove, from the query's displacement alone, that
// the match cannot have changed (icp.cu) -- the search is then skipped for that lane.  The best key itself is
// found exactly as by WarpSearch: a larger cull bound never hides a candidate.
struct WarpSearchC : WarpSearchBase {
    unsigned long long best;
    unsigned m1, m2;  // d2 bits (0x7f800000 = none yet)
    unsigned rb;      // cached relaxed bound (d2 bits), >= best_d2
    float margin;     // distance units, >= 0
    bool track;       // warp-uniform: some searching lane has margin > 0.  Without a margin the relaxed bound IS
                      // best_d2 and min(m2, bound) = best_d2 whatever m2 is: nothing to track, plain scan
    __device__ __forceinline__ unsigned lane_bound() const { return rb; }
    __device__ __forceinline__ void refresh() {
        const unsigned hi = (unsigned)(best >> 32);
        if (margin > 0.f && hi != 0u) {
            // approximate sqrt (rel. error 2^-23) padded upwards: only has to be >= the exact value
            const float e = __fadd_ru(__fmul_ru(sqrt_approx(__uint_as_float(hi)), 1.000001f), margin);
            rb = max(__float_as_uint(__fmul_ru(e, e)), hi);
        } else {
            rb = hi;
        }
    }
};

// key strictly below (r2, idx 0): accepts exactly d2 < r2
__device__ __forceinline__ unsigned long long init_key(float r2) {
    return ((unsigned long long)__float_as_uint(r2) << 32) - 1ull;
}

template <class W>
__device__ __forceinline__ void warp_query_box(W &w) {
    unsigned lo[3], hi[3];
    lo[0] = w.valid ? f2ord(w.qx) : 0xffffffffu; hi[0] = w.valid ? f2ord(w.qx) : 0u;
    lo[1] = w.valid ? f2ord(w.qy) : 0xffffffffu; hi[1] = w.valid ? f2ord(w.qy) : 0u;
    lo[2] = w.valid ? f2ord(w.qz) : 0xffffffffu; hi[2] = w.valid ? f2ord(w.qz) : 0u;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        w.wlo[a] = ord2f(__reduce_min_sync(CPHB_FULL, lo[a]));
        w.whi[a] = ord2f(__reduce_max_sync(CPHB_FULL, hi[a]));
        w.wc[a] = 0.5f * w.wlo[a] + 0.5f * w.whi[a];
    }
}
template <class W>
__device__ __forceinline__ void warp_update_bound(W &w) {
    w.bound = __reduce_max_sync(CPHB_FULL, w.valid ? w.lane_bound() : 0u);
}

__device__ __forceinline__ void issue_leaf(const IndexView &ix, unsigned leaf, float4 *tile, uint64_t *bar) {
    if (lane_id() == 0) {
        mbar_expect_tx(bar, CPHB_LEAF * 16);
        tma_bulk_g2s(tile, ix.pts + (size_t)leaf * CPHB_LEAF, CPHB_LEAF * 16, bar);
    }
}
template <class W>
__device__ __forceinline__ void wait_leaf(W &w, int b) {
    while (!mbar_try_wait(w.bar + b, (w.phase >> b) & 1u)) {
    }
    w.phase ^= (1u << b);
}

// k = 1 leaf scan.  `need` = lanes whose own bound still reaches this leaf's box.
//   many lanes  : every lane scans the 32 candidates against its own query (broadcast LDS.128);
//   few lanes   : transposed -- lane L holds candidate L, the needing queries are broadcast one at a
//                 time and the 32 distances are min-reduced with REDUX (d2 bits, then index among
//                 equal d2: the same (d2, index) order as the sequential scan).
#define CPHB_TRANSPOSE_MAX 14
__device__ __forceinline__ void scan_tile(const float4 *tile, WarpSearch &w, unsigned need) {
    if (__popc(need) > w.tmax) {
        unsigned long long best = w.best;
#pragma unroll
        for (int j = 0; j < CPHB_LEAF; ++j) {
            float4 p = tile[j];
            float d2 = dist2(w.qx, w.qy, w.qz, p.x, p.y, p.z);
            unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | __float_as_uint(p.w);
            best = (key < best) ? key : best;
        }
        w.best = best;
        return;
    }
    const float4 p = tile[lane_id()];
    const unsigned pidx = __float_as_uint(p.w);
    while (need) {
        const int t = __ffs(need) - 1;
        need &= need - 1;
        const float qx = __shfl_sync(CPHB_FULL, w.qx, t), qy = __shfl_sync(CPHB_FULL, w.qy, t),
                    qz = __shfl_sync(CPHB_FULL, w.qz, t);
        const unsigned db = __float_as_uint(dist2(qx, qy, qz, p.x, p.y, p.z));
        const unsigned m1 = __reduce_min_sync(CPHB_FULL, db);
        const unsigned m2 = __reduce_min_sync(CPHB_FULL, db == m1 ? pidx : 0xffffffffu);
        const unsigned long long key = ((unsigned long long)m1 << 32) | m2;
        if (lane_id() == t && key < w.best) w.best = key;
    }
}

__device__ __forceinline__ void scan_tile(const float4 *tile, WarpSearchC &w, unsigned need) {
    if (!w.track) {  // exactly the WarpSearch scan; rb follows best_d2 (every margin in the warp is 0)
        if (__popc(need) > w.tmax) {
            unsigned long long best = w.best;
#pragma unroll
            for (int j = 0; j < CPHB_LEAF; ++j) {
                const float4 p = tile[j];
                const float d2 = dist2(w.qx, w.qy, w.qz, p.x, p.y, p.z);
                const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | __float_as_uint(p.w);
                best = (key < best) ? key : best;
            }
            w.best = best;
            w.rb = (unsigned)(best >> 32);
            return;
        }
        const float4 p = tile[lane_id()];
        const unsigned pidx = __float_as_uint(p.w);
        while (need) {
            const int t = __ffs(need) - 1;
            need &= need - 1;
            const float qx = __shfl_sync(CPHB_FULL, w.qx, t), qy = __shfl_sync(CPHB_FULL, w.qy, t),
                        qz = __shfl_sync(CPHB_FULL, w.qz, t);
            const unsigned db = __float_as_uint(dist2(qx, qy, qz, p.x, p.y, p.z));
            const unsigned l1 = __reduce_min_sync(CPHB_FULL, db);
            const unsigned li = __reduce_min_sync(CPHB_FULL, db == l1 ? pidx : 0xffffffffu);
            const unsigned long long key = ((unsigned long long)l1 << 32) | li;
            if (lane_id() == t && key < w.best) {
                w.best = key;
                w.rb = l1;
            }
        }
        return;
    }
    if (__popc(need) > w.tmax) {
        unsigned long long best = w.best;
        unsigned m1 = w.m1, m2 = w.m2;
#pragma unroll
        for (int j = 0; j < CPHB_LEAF; ++j) {
            const float4 p = tile[j];
            const unsigned db = __float_as_uint(dist2(w.qx, w.qy, w.qz, p.x, p.y, p.z));
            const unsigned long long key = ((unsigned long long)db << 32) | __float_as_uint(p.w);
            best = (key < best) ? key : best;
            m2 = min(m2, max(db, m1));
            m1 = min(m1, db);
        }
        w.best = best;
        w.m1 = m1;
        w.m2 = m2;
        w.refresh();
        return;
    }
    const float4 p = tile[lane_id()];
    const unsigned pidx = __float_as_uint(p.w);
    while (need) {
        const int t = __ffs(need) - 1;
        need &= need - 1;
        const float qx = __shfl_sync(CPHB_FULL, w.qx, t), qy = __shfl_sync(CPHB_FULL, w.qy, t),
                    qz = __shfl_sync(CPHB_FULL, w.qz, t);
        const unsigned db = __float_as_uint(dist2(qx, qy, qz, p.x, p.y, p.z));
        const unsigned l1 = __reduce_min_sync(CPHB_FULL, db);
        const unsigned li = __reduce_min_sync(CPHB_FULL, db == l1 ? pidx : 0xffffffffu);
        const unsigned l2 = __reduce_min_sync(CPHB_FULL, pidx == li ? 0x7f800000u : db);  // leaf's second smallest
        if (lane_id() == t) {
            const unsigned long long key = ((unsigned long long)l1 << 32) | li;
            if (key < w.best) w.best = key;
            w.m2 = min(max(w.m1, l1), min(w.m2, l2));  // two smallest of {m1, m2, l1, l2}
            w.m1 = min(w.m1, l1);
            w.refresh();
        }
    }
}

// lane index of the active child with the smallest order key, or -1
__device__ __forceinline__ int pick_child(unsigned active, unsigned keybits) {
    unsigned cand = ((active >> lane_id()) & 1u) ? keybits : 0xffffffffu;
    unsigned m = __reduce_min_sync(CPHB_FULL, cand);
    if (m == 0xffffffffu) return -1;
    return __ffs(__ballot_sync(CPHB_FULL, cand == m)) - 1;
}
// stage 2: which lanes can still improve inside box `bx`?  (uniform address: one broadcast load)
template <class W>
__device__ __forceinline__ unsigned lanes_needing(const W &w, const Box *bx) {
    const float4 lo = __ldg(&bx->lo), hi = __ldg(&bx->hi);
    float dx = fmaxf(0.f, fmaxf(lo.x - w.qx, w.qx - hi.x));
    float dy = fmaxf(0.f, fmaxf(lo.y - w.qy, w.qy - hi.y));
    float dz = fmaxf(0.f, fmaxf(lo.z - w.qz, w.qz - hi.z));
    float d = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    return __ballot_sync(CPHB_FULL, w.valid && __float_as_uint(d) <= w.lane_bound());
}

template <int LV, class W>
struct Visit {
    static __device__ __forceinline__ void run(const IndexView &ix, unsigned group, W &w) {
        const Box *gbox = ix.boxes[LV] + (size_t)group * 32;
        unsigned dcull, dkey;
        {
            const float4 lo = __ldg(&gbox[lane_id()].lo), hi = __ldg(&gbox[lane_id()].hi);
            dcull = __float_as_uint(box_dist2(lo, hi, w.wlo, w.whi));
            // order key: distance of the box to the warp centre (+inf for empty boxes stays +inf)
            const float c3[3] = {w.wc[0], w.wc[1], w.wc[2]};
            dkey = __float_as_uint(box_dist2(lo, hi, c3, c3));
            // boxes containing the centre all have key 0: break those ties by the distance of the box
            // centre so the box "around" the warp comes first
            if (!w.warm && dkey == 0u) {
                const float mx = 0.5f * lo.x + 0.5f * hi.x - c3[0], my = 0.5f * lo.y + 0.5f * hi.y - c3[1],
                            mz = 0.5f * lo.z + 0.5f * hi.z - c3[2];
                // scaled far below any non-zero box distance of interest: only an ordering hint
                dkey = __float_as_uint(1e-30f * __fmaf_rn(mz, mz, __fmaf_rn(my, my, mx * mx)));
            }
        }
        unsigned active = __ballot_sync(CPHB_FULL, dcull <= w.bound);
        if constexpr (LV > 0) {
            while (active) {
                int src = pick_child(active, dkey);
                if (src < 0) break;
                active &= ~(1u << src);
                if (lanes_needing(w, gbox + src)) {
                    Visit<LV - 1, W>::run(ix, group * 32 + src, w);
                    active &= __ballot_sync(CPHB_FULL, dcull <= w.bound);
                }
            }
        } else {
            // leaf level.  A candidate is fetched only if stage 2 says some lane can still improve in it
            // (bounds only tighten, so a leaf rejected now stays rejected); the copy of the next accepted
            // leaf is in flight while the current one is scanned.
            int b = 0;
            int next = -1;
            while (active) {
                const int c = pick_child(active, dkey);
                if (c < 0) { active = 0; break; }
                active &= ~(1u << c);
                if (lanes_needing(w, gbox + c)) { next = c; break; }
            }
            if (next >= 0) issue_leaf(ix, group * 32 + next, w.tile + b * CPHB_LEAF, w.bar + b);
            while (next >= 0) {
                const int cur = next;
                next = -1;
                while (active) {
                    const int c = pick_child(active, dkey);
                    if (c < 0) { active = 0; break; }
                    active &= ~(1u << c);
                    if (lanes_needing(w, gbox + c)) { next = c; break; }
                }
                if (next >= 0) issue_leaf(ix, group * 32 + next, w.tile + (b ^ 1) * CPHB_LEAF, w.bar + (b ^ 1));
                wait_leaf(w, b);
                const unsigned need = lanes_needing(w, gbox + cur);  // bounds may have tightened since the pick
                if (need) {
                    scan_tile(w.tile + b * CPHB_LEAF, w, need);
                    warp_update_bound(w);
                    active &= __ballot_sync(CPHB_FULL, dcull <= w.bound);
                }
                __syncwarp();  // all lanes done with tile b before it is re-armed
                b ^= 1;
            }
        }
    }
};

// top-level entry: TOP is the compile-time depth the kernel was built for; the
// index always has CPHB_LEVELS levels so a deeper kernel on a small cloud only
// walks a few single-child nodes.
template <int TOP, class W>
__device__ __forceinline__ void warp_nn_search(const IndexView &ix, W &w) {
    Visit<TOP, W>::run(ix, 0u, w);
}

// tile: 2*CPHB_LEAF float4, bar: 2 mbarriers (per warp)
template <class W>
__device__ __forceinline__ void warp_search_setup(W &w, float4 *tile, uint64_t *bar) {
    w.tile = tile;
    w.bar = bar;
    w.phase = 0;
    w.warm = false;
    w.tmax = CPHB_TRANSPOSE_MAX;
    if (lane_id() == 0) {
        mbar_init(bar, 1);
        mbar_init(bar + 1, 1);
        fence_mbar_init();
    }
    __syncwarp();
}
#endif  // __CUDACC__
