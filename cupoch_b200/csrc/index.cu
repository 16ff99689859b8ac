// index.cu -- spatial index build (replaces KDTreeFlann::SetRawData + the
// vendored FLANN CUDA kd-tree builder, kdtree_flann.inl:125-144,
// kdtree_cuda_builder.h:401-700).
//
// Build = bounds reduce -> 30-bit 3-D Hilbert keys -> radix sort -> gather to
// float4 (w = original index) -> per-leaf AABBs -> 5 levels of 32-ary AABBs.
// No pointers, no per-level host synchronisation: ~12 launches, all
// stream-ordered.
#include <float.h>
#include <stdarg.h>
#include <string.h>

#include <stdlib.h>

#include "cphb_internal.cuh"

// ---------------------------------------------------------------------------
// library-wide host state
// ---------------------------------------------------------------------------
static thread_local char t_err[512] = "";
unsigned long long g_cphb_launches = 0;

void cphb_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}
extern "C" const char *cphb_last_error(void) { return t_err; }
extern "C" int cphb_version(void) { return CPHB_VERSION; }
extern "C" uint64_t cphb_launch_count(void) { return g_cphb_launches; }
extern "C" int cphb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}
extern "C" int cphb_set_device(int d) {
    CPHB_CUDA(cudaSetDevice(d));
    return CPHB_OK;
}

int cphb_alloc_async(void **p, size_t bytes, cudaStream_t s) {
    static thread_local int pool_ready_dev = -1;
    int dev = 0;
    CPHB_CUDA(cudaGetDevice(&dev));
    if (pool_ready_dev != dev) {
        cudaMemPool_t pool;
        CPHB_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
        uint64_t thr = UINT64_MAX;  // keep freed blocks: no cudaMalloc on later calls
        CPHB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
        pool_ready_dev = dev;
    }
    CPHB_CUDA(cudaMallocAsync(p, bytes ? bytes : 16, s));
    return CPHB_OK;
}
void cphb_free_async(void *p, cudaStream_t s) {
    if (p) cudaFreeAsync(p, s);
}

extern "C" int cphb_reserve_pool(size_t bytes) {
    void *p = nullptr;
    int rc = cphb_alloc_async(&p, bytes, (cudaStream_t)0);  // also sets the pool's release threshold to "never"
    if (rc) return rc;
    CPHB_CUDA(cudaFreeAsync(p, (cudaStream_t)0));
    CPHB_CUDA(cudaStreamSynchronize((cudaStream_t)0));
    return CPHB_OK;
}

// Stream-ordered pool allocation on the default stream: freed blocks stay in the pool (release threshold
// = max), so repeated allocate/free cycles of the API layers cost microseconds instead of cudaMalloc/cudaFree.
extern "C" void *cphb_malloc(size_t bytes) {
    void *p = nullptr;
    if (cphb_alloc_async(&p, bytes ? bytes : 16, (cudaStream_t)0) != CPHB_OK) return nullptr;
    return p;
}
extern "C" void cphb_free(void *p) {
    if (p) cudaFreeAsync(p, (cudaStream_t)0);
}
extern "C" void *cphb_malloc_host(size_t bytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 16) != cudaSuccess) {
        cphb_set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    return p;
}
extern "C" void cphb_free_host(void *p) {
    if (p) cudaFreeHost(p);
}
extern "C" int cphb_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream) {
    CPHB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return CPHB_OK;
}
extern "C" int cphb_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream) {
    CPHB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return CPHB_OK;
}
extern "C" int cphb_memset(void *dst, int value, size_t bytes, void *stream) {
    CPHB_CUDA(cudaMemsetAsync(dst, value, bytes, (cudaStream_t)stream));
    return CPHB_OK;
}
extern "C" int cphb_memcpy_d2d(void *dst, const void *src, size_t bytes, void *stream) {
    CPHB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return CPHB_OK;
}
extern "C" void *cphb_event_create(void) {
    cudaEvent_t e = nullptr;
    if (cudaEventCreate(&e) != cudaSuccess) {
        cphb_set_error("cudaEventCreate: %s", cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    return (void *)e;
}
extern "C" void cphb_event_destroy(void *e) {
    if (e) cudaEventDestroy((cudaEvent_t)e);
}
extern "C" int cphb_event_record(void *e, void *stream) {
    CPHB_CUDA(cudaEventRecord((cudaEvent_t)e, (cudaStream_t)stream));
    return CPHB_OK;
}
extern "C" int cphb_event_elapsed_ms(void *start, void *stop, float *h_ms) {
    CPHB_CUDA(cudaEventSynchronize((cudaEvent_t)stop));
    CPHB_CUDA(cudaEventElapsedTime(h_ms, (cudaEvent_t)start, (cudaEvent_t)stop));
    return CPHB_OK;
}
extern "C" int cphb_stream_synchronize(void *stream) {
    CPHB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return CPHB_OK;
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
__global__ void bounds_init_kernel(unsigned *b) {
    if (threadIdx.x < 3) b[threadIdx.x] = 0xffffffffu;
    else if (threadIdx.x < 6) b[threadIdx.x] = 0u;
}

// element-wise min / max (eigen.inl:197-221); order independent, exact.
__global__ void __launch_bounds__(256) bounds_kernel(const float *__restrict__ xyz, size_t n, unsigned *b) {
    unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            unsigned o = f2ord(xyz[3 * i + a]);
            lo[a] = min(lo[a], o);
            hi[a] = max(hi[a], o);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_min_sync(CPHB_FULL, lo[a]);
        hi[a] = __reduce_max_sync(CPHB_FULL, hi[a]);
    }
    // block-level combine first: one set of same-address global atomics per warp (~10k at 1 M points) would serialise
    __shared__ unsigned s_lo[8][3], s_hi[8][3];
    const int warp = threadIdx.x >> 5;
    if (lane_id() == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { s_lo[warp][a] = lo[a]; s_hi[warp][a] = hi[a]; }
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        const int a = threadIdx.x;
        unsigned l = s_lo[0][a], h = s_hi[0][a];
        for (int w2 = 1; w2 < (int)(blockDim.x >> 5); ++w2) { l = min(l, s_lo[w2][a]); h = max(h, s_hi[w2][a]); }
        atomicMin(&b[a], l);
        atomicMax(&b[3 + a], h);
    }
}

__global__ void __launch_bounds__(256) hilbert_key_kernel(const float *__restrict__ xyz, size_t n,
                                                          const unsigned *__restrict__ b, int shift, uint32_t *keys,
                                                          uint32_t *vals) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float mn[3] = {ord2f(b[0]), ord2f(b[1]), ord2f(b[2])};
    float ext = fmaxf(fmaxf(ord2f(b[3]) - mn[0], ord2f(b[4]) - mn[1]), ord2f(b[5]) - mn[2]);
    float scale = (ext > 0.f && ext < FLT_MAX) ? 1023.999f / ext : 0.f;
    uint32_t c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float v = (xyz[3 * i + a] - mn[a]) * scale;
        c[a] = (uint32_t)fminf(fmaxf(v, 0.f), 1023.f);
    }
    keys[i] = hilbert30(c[0], c[1], c[2]) >> shift;  // the leading 3 * levels bits ARE the coarser curve's index
    vals[i] = (uint32_t)i;
}

// pts[pos] = (xyz[perm[pos]], perm[pos]); tail padding = (FLT_MAX x3, -1); inv[perm[pos]] = pos
__global__ void __launch_bounds__(256) gather_points_kernel(const float *__restrict__ xyz,
                                                            const uint32_t *__restrict__ perm, size_t n,
                                                            size_t n_pad, float4 *pts, uint32_t *inv) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    float4 p;
    if (i < n) {
        uint32_t j = perm[i];
        inv[j] = (uint32_t)i;
        p.x = xyz[3 * (size_t)j];
        p.y = xyz[3 * (size_t)j + 1];
        p.z = xyz[3 * (size_t)j + 2];
        p.w = __uint_as_float(j);
    } else {
        p.x = p.y = p.z = FLT_MAX;
        p.w = __uint_as_float(0xffffffffu);
    }
    pts[i] = p;
}

// ---------------------------------------------------------------------------
// kd refinement of the Hilbert order.  Runs of 32 Hilbert-consecutive points are compact but irregular,
// so their AABBs overlap heavily (a query typically lies inside 2-3 leaf boxes and every one of them has
// to be scanned).  Each group of 1024 consecutive points (= one level-1 node) is therefore re-partitioned
// in shared memory by 5 exact median splits along the widest axis of each segment: the 32 leaves of a
// group become kd cells with pairwise disjoint boxes.  Implicit layout, leaf size and upper levels are
// unchanged; only the order of points inside a group changes.
// One block per group; segmented bitonic sorts (segment = 1024 >> level) of (key, point) pairs.
// ---------------------------------------------------------------------------
#define KD_GROUP 1024
#define KD_THREADS 256
#define KD_QBITS 14 /* coordinate quantisation inside a segment's bbox; ties broken by position */
// Per level: bbox per segment -> widest axis -> 24-bit key (14-bit quantised coordinate, 10-bit position:
// unique) -> radix select of the median key per segment (3 passes of 8 bits, 256-bin histograms in shared
// memory) -> stable partition around it.  The split only has to be a valid partition (search correctness
// never depends on it); quantisation can make sibling boxes overlap by at most 2^-14 of the extent.
struct KdSmem {
    float4 p[KD_GROUP];  // partitioned in place: every thread holds its 4 elements in registers across the barrier
    unsigned key[KD_GROUP];
    unsigned hist[16][256];
    unsigned lo[16][3], hi[16][3];
    unsigned prefix[16], rank[16], pivot[16];
    int axis[16];
    unsigned scan[KD_GROUP + 1];
    unsigned warp_tot[KD_THREADS / 32];
};
__global__ void __launch_bounds__(KD_THREADS) kd_refine_kernel(float4 *pts, size_t n_pad) {
    extern __shared__ __align__(16) unsigned char kd_raw[];
    KdSmem &m = *reinterpret_cast<KdSmem *>(kd_raw);
    const size_t base = (size_t)blockIdx.x * KD_GROUP;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int e = tid; e < KD_GROUP; e += KD_THREADS) {
        size_t i = base + e;
        m.p[e] = (i < n_pad) ? pts[i] : make_float4(FLT_MAX, FLT_MAX, FLT_MAX, __uint_as_float(0xffffffffu));
    }
    __syncthreads();
    for (int level = 0; level < 5; ++level) {
        const int S = KD_GROUP >> level, n_seg = 1 << level, half = S >> 1;
        const float4 *src = m.p;
        float4 *dst = m.p;
        if (tid < n_seg) {
#pragma unroll
            for (int a = 0; a < 3; ++a) { m.lo[tid][a] = 0xffffffffu; m.hi[tid][a] = 0u; }
            m.prefix[tid] = 0u;
            m.rank[tid] = (unsigned)half;  // 0-based rank of the pivot = first element of the upper half
        }
        __syncthreads();
        for (int e = tid; e < KD_GROUP; e += KD_THREADS) {
            // a warp's 32 consecutive elements lie in ONE segment (segments are aligned runs of >= 64 elements):
            // warp-wide REDUX first, then one set of shared-memory atomics per warp instead of one per point (at level 0
            // all 1024 points of the group hit the same six words)
            const float4 q = src[e];
            const bool real = __float_as_uint(q.w) != 0xffffffffu;
            unsigned lo3[3], hi3[3];
            lo3[0] = real ? f2ord(q.x) : 0xffffffffu; hi3[0] = real ? f2ord(q.x) : 0u;
            lo3[1] = real ? f2ord(q.y) : 0xffffffffu; hi3[1] = real ? f2ord(q.y) : 0u;
            lo3[2] = real ? f2ord(q.z) : 0xffffffffu; hi3[2] = real ? f2ord(q.z) : 0u;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                lo3[a] = __reduce_min_sync(CPHB_FULL, lo3[a]);
                hi3[a] = __reduce_max_sync(CPHB_FULL, hi3[a]);
            }
            if (lane < 3) {
                const int sg = e / S;  // (same for the whole warp)
                const unsigned l = lane == 0 ? lo3[0] : lane == 1 ? lo3[1] : lo3[2];
                const unsigned h = lane == 0 ? hi3[0] : lane == 1 ? hi3[1] : hi3[2];
                atomicMin(&m.lo[sg][lane], l);
                atomicMax(&m.hi[sg][lane], h);
            }
        }
        __syncthreads();
        if (tid < n_seg) {
            float ex[3];
#pragma unroll
            for (int a = 0; a < 3; ++a)
                ex[a] = (m.lo[tid][a] <= m.hi[tid][a]) ? ord2f(m.hi[tid][a]) - ord2f(m.lo[tid][a]) : 0.f;
            int ax = 0;
            if (ex[1] > ex[ax]) ax = 1;
            if (ex[2] > ex[ax]) ax = 2;
            m.axis[tid] = ax;
        }
        __syncthreads();
        for (int e = tid; e < KD_GROUP; e += KD_THREADS) {
            const float4 q = src[e];
            const int sg = e / S, ax = m.axis[sg];
            unsigned qk = (1u << KD_QBITS) - 1u;  // padding sorts last
            if (__float_as_uint(q.w) != 0xffffffffu) {
                const float c = (ax == 0) ? q.x : (ax == 1) ? q.y : q.z;
                const float lo = ord2f(m.lo[sg][ax]), hi = ord2f(m.hi[sg][ax]);
                const float t = (hi > lo) ? (c - lo) / (hi - lo) : 0.f;
                qk = (unsigned)fminf(fmaxf(t * (float)((1u << KD_QBITS) - 2u), 0.f), (float)((1u << KD_QBITS) - 2u));
            }
            m.key[e] = (qk << 10) | (unsigned)(e & (S - 1)) | 0u;  // 24 bits, unique inside a segment
        }
        __syncthreads();
        // ---- radix select of the element of rank `half` per segment: 3 passes of 8 bits, MSB first ----
        for (int pass = 0; pass < 3; ++pass) {
            const int shift = 16 - 8 * pass;
            for (int e = tid; e < n_seg * 256; e += KD_THREADS) (&m.hist[0][0])[e] = 0u;
            __syncthreads();
            for (int e = tid; e < KD_GROUP; e += KD_THREADS) {
                const int sg = e / S;
                const unsigned k = m.key[e];
                // elements whose higher digits equal the prefix found so far
                if (pass == 0 || (k >> (shift + 8)) == m.prefix[sg]) atomicAdd(&m.hist[sg][(k >> shift) & 255u], 1u);
            }
            __syncthreads();
            for (int sg = warp; sg < n_seg; sg += KD_THREADS / 32) {
                // lane owns bins [8*lane, 8*lane+8): find the bin where the cumulative count passes rank
                unsigned c[8], tot = 0;
#pragma unroll
                for (int b8 = 0; b8 < 8; ++b8) { c[b8] = m.hist[sg][8 * lane + b8]; tot += c[b8]; }
                unsigned incl = tot;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    unsigned y = __shfl_up_sync(CPHB_FULL, incl, o);
                    if (lane >= o) incl += y;
                }
                const unsigned excl = incl - tot, r = m.rank[sg], pf = m.prefix[sg];
                __syncwarp();  // every lane has read rank/prefix before the winning lane overwrites them
                if (r >= excl && r < incl) {  // exactly one lane
                    unsigned acc = excl;
                    int bin = 8 * lane;
#pragma unroll
                    for (int b8 = 0; b8 < 8; ++b8) {
                        if (r >= acc + c[b8]) { acc += c[b8]; bin = 8 * lane + b8 + 1; }
                        else break;
                    }
                    m.prefix[sg] = (pf << 8) | (unsigned)bin;
                    m.rank[sg] = r - acc;
                }
            }
            __syncthreads();
        }
        // prefix[sg] is now the full 24-bit key of the pivot: lower half = keys < pivot (exactly `half` of them)
        // ---- stable partition: exclusive scan of is_lower over the group in position order ----
        {
            unsigned f[4], cnt = 0;
#pragma unroll
            for (int r4 = 0; r4 < 4; ++r4) {
                const int e = 4 * tid + r4;
                f[r4] = (m.key[e] < m.prefix[e / S]) ? 1u : 0u;
                cnt += f[r4];
            }
            unsigned incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                unsigned y = __shfl_up_sync(CPHB_FULL, incl, o);
                if (lane >= o) incl += y;
            }
            if (lane == 31) m.warp_tot[warp] = incl;
            __syncthreads();
            unsigned wbase = 0;
            for (int w2 = 0; w2 < warp; ++w2) wbase += m.warp_tot[w2];
            unsigned run = wbase + incl - cnt;
#pragma unroll
            for (int r4 = 0; r4 < 4; ++r4) {
                m.scan[4 * tid + r4] = run;
                run += f[r4];
            }
            if (tid == KD_THREADS - 1) m.scan[KD_GROUP] = run;
            float4 mine[4];
#pragma unroll
            for (int r4 = 0; r4 < 4; ++r4) mine[r4] = src[4 * tid + r4];
            __syncthreads();  // scan complete AND every element is in a register: the array may be overwritten
#pragma unroll
            for (int r4 = 0; r4 < 4; ++r4) {
                const int e = 4 * tid + r4;
                const int sg = e / S, s0 = sg * S;
                const unsigned lower_before = m.scan[e] - m.scan[s0];
                const unsigned pos_in_seg = (unsigned)(e - s0);
                const unsigned d = f[r4] ? (unsigned)s0 + lower_before : (unsigned)s0 + (unsigned)half + (pos_in_seg - lower_before);
                dst[d] = mine[r4];
            }
        }
        __syncthreads();
    }
    for (int e = tid; e < KD_GROUP; e += KD_THREADS) {
        size_t i = base + e;
        if (i < n_pad) pts[i] = m.p[e];
    }
}

// inv[original index] = final position
__global__ void __launch_bounds__(256) inverse_perm_kernel(const float4 *__restrict__ pts, size_t n_pad, uint32_t *inv) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    const unsigned j = __float_as_uint(pts[i].w);
    if (j != 0xffffffffu) inv[j] = (uint32_t)i;
}

// one warp per leaf (CPHB_LEAF == 32): AABB of its real points
__global__ void __launch_bounds__(256) leaf_box_kernel(const float4 *__restrict__ pts, size_t n,
                                                       size_t n_boxes_pad, Box *boxes) {
    size_t leaf = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    if (leaf >= n_boxes_pad) return;
    size_t i = leaf * CPHB_LEAF + lane_id();
    unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    if (i < n) {  // real points are a prefix of pts (padding sorts last at every refinement level)
        float4 p = pts[i];
        lo[0] = hi[0] = f2ord(p.x);
        lo[1] = hi[1] = f2ord(p.y);
        lo[2] = hi[2] = f2ord(p.z);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_min_sync(CPHB_FULL, lo[a]);
        hi[a] = __reduce_max_sync(CPHB_FULL, hi[a]);
    }
    if (lane_id() == 0) {
        Box b;
        bool empty = lo[0] == 0xffffffffu && hi[0] == 0u;
        b.lo = empty ? make_float4(INFINITY, INFINITY, INFINITY, 0.f)
                     : make_float4(ord2f(lo[0]), ord2f(lo[1]), ord2f(lo[2]), 0.f);
        b.hi = empty ? make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f)
                     : make_float4(ord2f(hi[0]), ord2f(hi[1]), ord2f(hi[2]), 0.f);
        boxes[leaf] = b;
    }
}

// one warp per parent: union of its 32 children (children array is padded with
// empty boxes, so no bounds logic is needed beyond the parent count)
__global__ void __launch_bounds__(256) upper_box_kernel(const Box *__restrict__ child, size_t n_child,
                                                        size_t n_parent_pad, Box *parent) {
    size_t p = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    if (p >= n_parent_pad) return;
    size_t c = p * 32 + lane_id();
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    if (c < n_child) {
        lo = child[c].lo;
        hi = child[c].hi;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(CPHB_FULL, lo.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(CPHB_FULL, lo.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(CPHB_FULL, lo.z, o));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(CPHB_FULL, hi.x, o));
        hi.y = fmaxf(hi.y, __shfl_xor_sync(CPHB_FULL, hi.y, o));
        hi.z = fmaxf(hi.z, __shfl_xor_sync(CPHB_FULL, hi.z, o));
    }
    if (lane_id() == 0) {
        Box b;
        b.lo = lo;
        b.hi = hi;
        parent[p] = b;
    }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
int cphb_hilbert_order(const float *xyz, size_t n, uint32_t *perm_out, float *bounds_dev6, int bounds_given,
                       cudaStream_t s) {
    return cphb_hilbert_order_n(xyz, n, perm_out, bounds_dev6, bounds_given, n, s);
}
// resolution of the curve chosen for `n_ref` points instead of n: queries are ordered only to make every warp's 32
// queries a compact cluster RELATIVE TO THE TARGET'S LEAVES, so the target's size decides how fine the curve has to be
// (10 M queries against 2 M targets: 24-bit keys = 3 radix passes instead of 4)
int cphb_hilbert_order_n(const float *xyz, size_t n, uint32_t *perm_out, float *bounds_dev6, int bounds_given,
                         size_t n_ref, cudaStream_t s) {
    if (n == 0) return CPHB_OK;
    unsigned *b = (unsigned *)bounds_dev6;
    if (!b) bounds_given = 0;
    void *own = nullptr;
    if (!b) {
        int rc = cphb_alloc_async(&own, 32, s);
        if (rc) return rc;
        b = (unsigned *)own;
    }
    uint32_t *scratch = nullptr;
    int rc = cphb_alloc_async((void **)&scratch, sizeof(uint32_t) * 3 * n, s);
    if (rc) return rc;
    uint32_t *keys = scratch, *keys2 = scratch + n, *vals = scratch + 2 * n;
    if (!bounds_given) {
        CPHB_LAUNCH(bounds_init_kernel, 1, 32, 0, s, b);
        int grid = (int)((n + 255) / 256);
        if (grid > CPHB_SMS * 8) grid = CPHB_SMS * 8;
        CPHB_LAUNCH(bounds_kernel, grid, 256, 0, s, xyz, n, b);
    }
    // Curve resolution by cloud size: ceil(log2(n) / 3) + 1 levels (3 bits each), i.e. >= 8 curve cells per point of a
    // volume-filling cloud; 1 M points -> 8 levels = 24-bit keys = 3 radix passes instead of 4.  The order only has to
    // cluster (every search is exact whatever the order; groups of 1024 are kd-refined afterwards), equal keys keep their
    // original order (stable sort).  CPHB_HILBERT_LEVELS overrides (tuning hook).
    int levels = 1;
    while (levels < 10 && ((size_t)1 << (3 * levels)) < (n_ref ? n_ref : n)) ++levels;
    levels = levels + 1 > 10 ? 10 : levels + 1;
    if (levels < 4) levels = 4;
    if (const char *e = getenv("CPHB_HILBERT_LEVELS")) { int v = atoi(e); if (v >= 1 && v <= 10) levels = v; }
    CPHB_LAUNCH(hilbert_key_kernel, (unsigned)((n + 255) / 256), 256, 0, s, xyz, n, b, 30 - 3 * levels, keys, vals);
    CPHB_CHECK_LAUNCH();
    rc = cphb_sort_pairs_u32(keys, keys2, vals, perm_out, n, 3 * levels, s);
    cphb_free_async(scratch, s);
    cphb_free_async(own, s);
    return rc;
}

extern "C" int cphb_index_create(const float *xyz, size_t n, void *stream, cphb_index **out) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!out || (n && !xyz)) {
        cphb_set_error("cphb_index_create: null argument");
        return CPHB_ERR_INVALID;
    }
    if (n > (size_t)0x7fffffff) {
        cphb_set_error("cphb_index_create: n=%zu exceeds int32 indices", n);
        return CPHB_ERR_INVALID;
    }
    cphb_index *ix = new cphb_index();
    memset(ix, 0, sizeof(*ix));
    CPHB_CUDA(cudaGetDevice(&ix->device));
    ix->stream = s;
    size_t count[CPHB_LEVELS], pad[CPHB_LEVELS];
    count[0] = (n + CPHB_LEAF - 1) / CPHB_LEAF;
    for (int l = 0; l < CPHB_LEVELS; ++l) {
        if (l) count[l] = (count[l - 1] + 31) / 32;
        pad[l] = cphb_align(count[l] ? count[l] : 1, 32);
    }
    if (count[CPHB_LEVELS - 1] > 32) {
        cphb_set_error("cphb_index_create: n=%zu too large for %d levels", n, CPHB_LEVELS);
        delete ix;
        return CPHB_ERR_INVALID;
    }
    size_t n_pad = (count[0] ? count[0] : 1) * CPHB_LEAF;
    size_t off_pts = 0;
    size_t off = cphb_align(n_pad * sizeof(float4), 256);
    size_t off_box[CPHB_LEVELS];
    for (int l = 0; l < CPHB_LEVELS; ++l) {
        off_box[l] = off;
        off = cphb_align(off + pad[l] * sizeof(Box), 256);
    }
    size_t off_bounds = off;
    off += 256;
    size_t off_perm = off;
    off = cphb_align(off + sizeof(uint32_t) * (n ? n : 1), 256);
    size_t off_inv = off;
    off = cphb_align(off + sizeof(uint32_t) * (n ? n : 1), 256);
    ix->arena_bytes = off;
    int rc = cphb_alloc_async(&ix->arena, off, s);
    if (rc) {
        delete ix;
        return rc;
    }
    char *base = (char *)ix->arena;
    float4 *pts = (float4 *)(base + off_pts);
    Box *boxes[CPHB_LEVELS];
    for (int l = 0; l < CPHB_LEVELS; ++l) boxes[l] = (Box *)(base + off_box[l]);
    ix->bounds = (float *)(base + off_bounds);
    uint32_t *perm = (uint32_t *)(base + off_perm);
    uint32_t *inv = (uint32_t *)(base + off_inv);

    if (n) {
        rc = cphb_hilbert_order(xyz, n, perm, ix->bounds, 0, s);
        if (rc) {
            cphb_free_async(ix->arena, s);
            delete ix;
            return rc;
        }
    } else {
        CPHB_LAUNCH(bounds_init_kernel, 1, 32, 0, s, (unsigned *)ix->bounds);
    }
    CPHB_LAUNCH(gather_points_kernel, (unsigned)((n_pad + 255) / 256), 256, 0, s, xyz, perm, n, n_pad, pts, inv);
    if (n > KD_GROUP / 2) {  // tiny clouds: nothing to gain
        CPHB_CUDA(cudaFuncSetAttribute(kd_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(KdSmem)));
        CPHB_LAUNCH(kd_refine_kernel, (unsigned)((n_pad + KD_GROUP - 1) / KD_GROUP), KD_THREADS, sizeof(KdSmem), s, pts, n_pad);
        CPHB_LAUNCH(inverse_perm_kernel, (unsigned)((n_pad + 255) / 256), 256, 0, s, pts, n_pad, inv);
    }
    CPHB_LAUNCH(leaf_box_kernel, (unsigned)((pad[0] * 32 + 255) / 256), 256, 0, s, pts, n, pad[0], boxes[0]);
    for (int l = 1; l < CPHB_LEVELS; ++l)
        CPHB_LAUNCH(upper_box_kernel, (unsigned)((pad[l] * 32 + 255) / 256), 256, 0, s, boxes[l - 1], count[l - 1],
                    pad[l], boxes[l]);
    CPHB_CHECK_LAUNCH();

    ix->v.pts = pts;
    ix->v.inv = inv;
    for (int l = 0; l < CPHB_LEVELS; ++l) ix->v.boxes[l] = boxes[l];
    ix->v.n = n;
    ix->v.n_leaves = (unsigned)count[0];
    int top = 0;
    while (count[top] > 32) ++top;
    ix->v.top = top;
    *out = ix;
    return CPHB_OK;
}

extern "C" void cphb_index_destroy(cphb_index *ix) {
    if (!ix) return;
    if (ix->arena) cudaFreeAsync(ix->arena, ix->stream);
    delete ix;
}
extern "C" size_t cphb_index_size(const cphb_index *ix) { return ix ? (size_t)ix->v.n : 0; }

extern "C" int cphb_min_max_bound(const float *points, size_t n, float h_min[3], float h_max[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    for (int a = 0; a < 3; ++a) h_min[a] = h_max[a] = 0.f;  // reference: Zero() for an empty cloud
    if (n == 0) return CPHB_OK;
    unsigned *b = nullptr;
    int rc = cphb_alloc_async((void **)&b, 32, s);
    if (rc) return rc;
    CPHB_LAUNCH(bounds_init_kernel, 1, 32, 0, s, b);
    int grid = (int)((n + 255) / 256);
    if (grid > CPHB_SMS * 8) grid = CPHB_SMS * 8;
    CPHB_LAUNCH(bounds_kernel, grid, 256, 0, s, points, n, b);
    CPHB_CHECK_LAUNCH();
    unsigned h[6];
    CPHB_CUDA(cudaMemcpyAsync(h, b, sizeof(h), cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    cphb_free_async(b, s);
    for (int a = 0; a < 3; ++a) {
        h_min[a] = ord2f(h[a]);
        h_max[a] = ord2f(h[3 + a]);
    }
    return CPHB_OK;
}
