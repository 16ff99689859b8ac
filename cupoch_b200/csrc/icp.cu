// icp.cu -- fused ICP iteration (one launch per iteration) + device-side 6x6
// solve / Kabsch / convergence logic + the RegistrationICP driver.
//
// Replaces, per iteration, the reference's ~13 thrust launches and >= 2 host
// synchronisations (SURVEY.md 2.4, K1 K3-K11):
//   pcd.Transform(update)                      registration.cu:160, geometry_utils.cu:34-54,257-265
//   kdtree.SearchRadius(.., 1, ..)             registration.cu:47, kdtree_cuda_3d_index.cu:52-154
//   error2 / correspondence list               registration.cu:50-69
//   ComputeJTJandJTr / Kabsch sums             eigen.inl:92-145, kabsch.cu:48-104
//   SolveJacobianSystemAndObtainExtrinsicMatrix eigen.cu:75-122 (host Eigen LDLT in the reference)
//   transformation = update * transformation   registration.cu:159
//   convergence test                           registration.cu:165-170
//
// Arithmetic contract (DESIGN.md): per-row float32 arithmetic in the stated
// order with explicit FMAs (this file is compiled with -fmad=false, so only
// the __fmaf_rn/fma calls below fuse); sums of exact float*float products in
// float64, reduced in a fixed order (warp -> block -> grid), rounded once to
// float32; the 6x6 LDLT, se(3) exponential and 4x4 composition use unfused
// float32 like the reference's host code.
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdlib.h>
#include <time.h>
#include <string.h>

#include "cphb_internal.cuh"
#include <vector>
#include "cphb_eigen3.cuh"

#include "icp_types.cuh"
#include "icp_solve.cuh"
#include "icp_rows.cuh"
#include "icp_kernels.cuh"
#include "icp_estimate.cuh"
#include "icp_aux.cuh"

// ===========================================================================
// host driver
// ===========================================================================

struct cphb_icp {
    cphb_index *index;
    cphb_icp_params prm;
    cphb_cloud tgt;
    unsigned n_src, n_pad;
    unsigned n_full;   // size of the source as passed (== n_src unless the library shards it)
    void *arena;
    size_t arena_bytes;
    float4 *pristine_xyz, *pristine_nrm, *pristine_cov;  // Hilbert-ordered source as given
    float4 *work_xyz, *work_nrm, *work_cov;
    float4 *src_col;
    float4 *tix_nrm, *tix_grad, *tix_cov;  // target attributes in index order (icp_types.cuh)
    float4 *alt_xyz, *alt_nrm, *alt_cov, *alt_col, *cur_col;  // re-tiling ping-pong buffers
    int2 *alt_prev;
    uint32_t *rt_keys, *rt_keys2, *rt_vals, *rt_order;
    IcpState *st;
    IcpState *h_st;  // pinned
    bool owns_host;
    cudaEvent_t ev0, ev1;
    double *partials;
    int32_t *corr_index;
    unsigned *cmp_counts;
    unsigned *cmp_total;
    double *tile_sums;
    unsigned *flag_bits;
    unsigned flag_words;
    int2 *prev;
    unsigned *dbg = nullptr;  // CPHB_DEBUG_CERT statistics
    cudaEvent_t *dbg_ev = nullptr;  // CPHB_DEBUG_EVENTS: 3 events per launch (before, between, after)
    unsigned grid_search;  // ROLE 0 launch (searching regime)
    unsigned grid;         // ROLE 1 launch (certified regime / sum of a searching launch's tile sums + solve)
    unsigned reduce_grid;  // blocks of the ROLE 1 launch that take part in that sum
    cudaStream_t stream;
};

// per-thread cached pinned staging buffer + events: cudaMallocHost / cudaEventCreate cost milliseconds,
// far more than a 1M-point registration's launch loop.
struct HostCache {
    IcpState *h_st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool in_use = false;
};
static thread_local HostCache t_cache;
// cphb_registration_icp_host: the source arrays are still being uploaded on another stream while the target index is
// built; cphb_icp_create waits for this event right before it first reads them
static thread_local cudaEvent_t t_source_ready = nullptr;
// side stream on which cphb_icp_create orders the source while the target index is built
struct SideStream {
    cudaStream_t stream = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    int device = -1;
};
static thread_local SideStream t_side;

static bool is_identity4(const float *T) {  // Eigen isIdentity(1e-5), registration.cu:148
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float v = T[4 * i + j];
            if (i == j) { if (fabsf(v - 1.f) > 1e-5f) return false; }
            else if (fabsf(v) > 1e-5f) return false;
        }
    return true;
}

// resident blocks / SM of the two instances of the iteration kernel (register-limited)
template <int KIND, int ROLE>
static int iteration_occupancy(bool top3) {
    int nb = 0;
    cudaError_t e = top3 ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, icp_iteration_kernel<KIND, 3, ROLE>, ICP_SEARCH_WARPS * 32, 0)
                         : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, icp_iteration_kernel<KIND, 5, ROLE>, ICP_SEARCH_WARPS * 32, 0);
    if (e != cudaSuccess) { cudaGetLastError(); return 0; }
    return nb;
}
template <int ROLE>
static int iteration_occupancy_kind(int kind, bool top3) {
    static int cache[8][2] = {};  // 0 = not queried yet
    int &c = cache[kind & 7][top3 ? 0 : 1];
    if (c == 0) {
        switch (kind) {
            case CPHB_EST_POINT_TO_POINT: c = iteration_occupancy<CPHB_EST_POINT_TO_POINT, ROLE>(top3); break;
            case CPHB_EST_POINT_TO_PLANE: c = iteration_occupancy<CPHB_EST_POINT_TO_PLANE, ROLE>(top3); break;
            case CPHB_EST_SYMMETRIC: c = iteration_occupancy<CPHB_EST_SYMMETRIC, ROLE>(top3); break;
            case CPHB_EST_COLORED_ICP: c = iteration_occupancy<CPHB_EST_COLORED_ICP, ROLE>(top3); break;
            case CPHB_EST_GENERALIZED_ICP: c = iteration_occupancy<CPHB_EST_GENERALIZED_ICP, ROLE>(top3); break;
        }
        if (c <= 0) c = -1;
    }
    return c;
}

#if CPHB_PDL
// launch with stream serialisation relaxed (programmatic dependent launch): the kernel may start while its
// predecessor drains and synchronises on it with griddepcontrol.wait
template <class K>
static void launch_pdl(K kernel, unsigned grid, unsigned block, cudaStream_t s, const IcpArgs &a) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, a);
    ++g_cphb_launches;
    if (e != cudaSuccess) cphb_set_error("PDL launch failed: %s", cudaGetErrorString(e));
}
#endif

template <int KIND>
static void launch_iteration(const cphb_icp *icp, const IcpArgs &a, cudaStream_t s) {
#if CPHB_PDL
    static const bool pdl = getenv("CPHB_NO_PDL") == nullptr;
    // two launches per iteration: the searching-regime instance, then the certified-regime instance (which also sums and
    // solves after a searching launch); the regime is decided on the device, the instance it does not concern returns
    // at its first instructions (icp_kernels.cuh)
    const bool top3 = icp->index->v.top <= 3;
    if (pdl && !a.defer_finalize && !a.step_mode && !icp->dbg_ev) {
        if (top3) launch_pdl(icp_iteration_kernel<KIND, 3, 0>, icp->grid_search, ICP_SEARCH_WARPS * 32, s, a);
        else launch_pdl(icp_iteration_kernel<KIND, 5, 0>, icp->grid_search, ICP_SEARCH_WARPS * 32, s, a);
        if (top3) launch_pdl(icp_iteration_kernel<KIND, 3, 1>, icp->grid, ICP_SEARCH_WARPS * 32, s, a);
        else launch_pdl(icp_iteration_kernel<KIND, 5, 1>, icp->grid, ICP_SEARCH_WARPS * 32, s, a);
        return;
    }
#endif
    if (icp->index->v.top <= 3) CPHB_LAUNCH((icp_iteration_kernel<KIND, 3, 0>), icp->grid_search, ICP_SEARCH_WARPS * 32, 0, s, a);
    else CPHB_LAUNCH((icp_iteration_kernel<KIND, 5, 0>), icp->grid_search, ICP_SEARCH_WARPS * 32, 0, s, a);
    if (icp->dbg_ev) cudaEventRecord(icp->dbg_ev[3 * a.launch_idx + 1], s);
    if (icp->index->v.top <= 3) CPHB_LAUNCH((icp_iteration_kernel<KIND, 3, 1>), icp->grid, ICP_SEARCH_WARPS * 32, 0, s, a);
    else CPHB_LAUNCH((icp_iteration_kernel<KIND, 5, 1>), icp->grid, ICP_SEARCH_WARPS * 32, 0, s, a);
}
static void launch_iteration_kind(const cphb_icp *icp, const IcpArgs &a, cudaStream_t s) {
    switch (icp->prm.estimation) {
        case CPHB_EST_POINT_TO_POINT: launch_iteration<CPHB_EST_POINT_TO_POINT>(icp, a, s); break;
        case CPHB_EST_POINT_TO_PLANE: launch_iteration<CPHB_EST_POINT_TO_PLANE>(icp, a, s); break;
        case CPHB_EST_SYMMETRIC: launch_iteration<CPHB_EST_SYMMETRIC>(icp, a, s); break;
        case CPHB_EST_COLORED_ICP: launch_iteration<CPHB_EST_COLORED_ICP>(icp, a, s); break;
        case CPHB_EST_GENERALIZED_ICP: launch_iteration<CPHB_EST_GENERALIZED_ICP>(icp, a, s); break;
    }
}
static void launch_finalize_kind(const cphb_icp *icp, const IcpArgs &a, cudaStream_t s) {
    switch (icp->prm.estimation) {
        case CPHB_EST_POINT_TO_POINT: CPHB_LAUNCH(icp_finalize_kernel<CPHB_EST_POINT_TO_POINT>, 1, 32, 0, s, a); break;
        case CPHB_EST_POINT_TO_PLANE: CPHB_LAUNCH(icp_finalize_kernel<CPHB_EST_POINT_TO_PLANE>, 1, 32, 0, s, a); break;
        case CPHB_EST_SYMMETRIC: CPHB_LAUNCH(icp_finalize_kernel<CPHB_EST_SYMMETRIC>, 1, 32, 0, s, a); break;
        case CPHB_EST_COLORED_ICP: CPHB_LAUNCH(icp_finalize_kernel<CPHB_EST_COLORED_ICP>, 1, 32, 0, s, a); break;
        case CPHB_EST_GENERALIZED_ICP: CPHB_LAUNCH(icp_finalize_kernel<CPHB_EST_GENERALIZED_ICP>, 1, 32, 0, s, a); break;
    }
}

extern "C" int cphb_icp_create(const cphb_cloud *source, const cphb_cloud *target, const cphb_icp_params *params,
                               void *stream, cphb_icp **out) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!source || !target || !params || !out) {
        cphb_set_error("cphb_icp_create: null argument");
        return CPHB_ERR_INVALID;
    }
    if (params->estimation < CPHB_EST_POINT_TO_POINT || params->estimation > CPHB_EST_GENERALIZED_ICP) {
        cphb_set_error("cphb_icp_create: estimation %d has no fused path (use the facade's generic loop)",
                       params->estimation);
        return CPHB_ERR_UNSUPPORTED;
    }
    if (source->n > 0x7fffff00ull || target->n > 0x7fffffffull) {
        cphb_set_error("cphb_icp_create: cloud exceeds int32 indices");
        return CPHB_ERR_INVALID;
    }
    cphb_icp *icp = new cphb_icp();
    memset(icp, 0, sizeof(*icp));
    uint32_t *perm_side = nullptr;
    // one exit for CUDA errors after this point: the half-built context (index, arena, host staging) is released
#define CREATE_TRY(call)                                                                                 \
    do {                                                                                                 \
        cudaError_t e__ = (call);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            cphb_set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));          \
            if (perm_side) cphb_free_async(perm_side, t_side.stream);                                    \
            cphb_icp_destroy(icp);                                                                       \
            return CPHB_ERR_CUDA;                                                                        \
        }                                                                                                \
    } while (0)
    icp->prm = *params;
    icp->tgt = *target;
    icp->stream = s;
    const unsigned n_full = (unsigned)source->n;
    // The source's Hilbert ordering (bounds, keys, radix sort) does not depend on the target index: it runs on a side
    // stream, concurrently with the index build (both are short chains of small kernels), and joins right before the
    // source is gathered.
    int cur_dev = 0;
    cudaGetDevice(&cur_dev);
    if (!t_side.stream || t_side.device != cur_dev) {  // (a thread that moved to another device gets a new one)
        t_side.device = cur_dev;
        CREATE_TRY(cudaStreamCreateWithFlags(&t_side.stream, cudaStreamNonBlocking));
        CREATE_TRY(cudaEventCreateWithFlags(&t_side.fork, cudaEventDisableTiming));
        CREATE_TRY(cudaEventCreateWithFlags(&t_side.join, cudaEventDisableTiming));
    }
    int rc = CPHB_OK;
    if (n_full) {
        CREATE_TRY(cudaEventRecord(t_side.fork, s));
        CREATE_TRY(cudaStreamWaitEvent(t_side.stream, t_side.fork, 0));
        if (t_source_ready) {  // (host-buffer call: the source upload is still in flight on the copy stream)
            cudaStreamWaitEvent(t_side.stream, t_source_ready, 0);
            t_source_ready = nullptr;
        }
        rc = cphb_alloc_async((void **)&perm_side, sizeof(uint32_t) * n_full, t_side.stream);
        if (!rc) rc = cphb_hilbert_order(source->points, n_full, perm_side, nullptr, 0, t_side.stream);
        if (rc) { cphb_free_async(perm_side, t_side.stream); delete icp; return rc; }
        CREATE_TRY(cudaEventRecord(t_side.join, t_side.stream));
    }
    rc = cphb_index_create(target->points, target->n, s, &icp->index);
    if (rc) {
        if (perm_side) { cudaStreamWaitEvent(s, t_side.join, 0); cphb_free_async(perm_side, s); }
        delete icp;
        return rc;
    }
    unsigned lo = 0, n = n_full;
    if (params->shard_world > 1) {
        if (params->shard_rank < 0 || params->shard_rank >= params->shard_world) {
            cphb_set_error("cphb_icp_create: shard_rank %d outside [0,%d)", params->shard_rank, params->shard_world);
            cphb_index_destroy(icp->index);
            delete icp;
            return CPHB_ERR_INVALID;
        }
        lo = (unsigned)(((unsigned long long)n_full * params->shard_rank) / params->shard_world);
        unsigned hi = (unsigned)(((unsigned long long)n_full * (params->shard_rank + 1)) / params->shard_world);
        n = hi - lo;
    }
    icp->n_full = n_full;
    const unsigned n_pad = (unsigned)cphb_align(n ? n : 1, ICP_BLOCK);
    icp->n_src = n;
    icp->n_pad = n_pad;
    {
        int dev = 0, sms = CPHB_SMS;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const unsigned n_tiles = n_pad / 32;
        unsigned want = (n_tiles + ICP_SEARCH_WARPS - 1) / ICP_SEARCH_WARPS;
        // every block must be resident: warps start on a static tile, and a block waiting for an SM slot
        // would hold its four tiles back until the dynamic queue has drained
        auto grid_for = [&](int occ, const char *hook) {
            unsigned per_sm = 9u;
            if (occ > 0 && (unsigned)occ < per_sm) per_sm = (unsigned)occ;
            if (const char *e = getenv(hook)) {  // tuning hook
                int v = atoi(e);
                if (v >= 1 && v <= 32) per_sm = (unsigned)v;
            }
            const unsigned cap = (unsigned)sms * per_sm;
            return want < cap ? want : cap;
        };
        icp->grid_search = grid_for(iteration_occupancy_kind<0>(params->estimation, icp->index->v.top <= 3), "CPHB_ICP_SEARCH_BLOCKS_PER_SM");
        icp->grid = grid_for(iteration_occupancy_kind<1>(params->estimation, icp->index->v.top <= 3), "CPHB_ICP_BLOCKS_PER_SM");
        unsigned rg = (n_tiles + 63) / 64;
        unsigned rg_cap = (unsigned)sms;
        if (const char *e = getenv("CPHB_REDUCE_BLOCKS_PER_SM")) {  // tuning hook: more, shorter chains of tile sums
            int v = atoi(e);
            if (v >= 1 && v <= 8) rg_cap = (unsigned)sms * (unsigned)v;
        }
        icp->reduce_grid = rg < 1 ? 1 : (rg > rg_cap ? rg_cap : rg);
        if (icp->reduce_grid > icp->grid) icp->reduce_grid = icp->grid;  // the sum runs on blocks of the ROLE 1 launch
    }
    const bool want_nrm = params->estimation == CPHB_EST_SYMMETRIC && source->normals;
    const bool want_col = params->estimation == CPHB_EST_COLORED_ICP && source->colors;
    const bool want_cov = params->estimation == CPHB_EST_GENERALIZED_ICP && source->covariances;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = cphb_align(off + bytes, 256); return o; };
    size_t o_pxyz = take(sizeof(float4) * n_pad), o_wxyz = take(sizeof(float4) * n_pad);
    size_t o_pnrm = want_nrm ? take(sizeof(float4) * n_pad) : 0, o_wnrm = want_nrm ? take(sizeof(float4) * n_pad) : 0;
    size_t o_pcov = want_cov ? take(sizeof(float4) * 3 * n_pad) : 0, o_wcov = want_cov ? take(sizeof(float4) * 3 * n_pad) : 0;
    size_t o_col = want_col ? take(sizeof(float4) * n_pad) : 0;
    size_t o_st = take(sizeof(IcpState));
    size_t o_part = take(sizeof(double) * 32 * (icp->reduce_grid > icp->grid ? icp->reduce_grid : icp->grid));
    // private copies of the target attributes in index order (nothing of the caller's target is retained)
    const size_t nt_pad = (size_t)icp->index->v.n_leaves * CPHB_LEAF;
    const int est = params->estimation;
    const bool t_nrm = target->normals && (est == CPHB_EST_POINT_TO_PLANE || est == CPHB_EST_SYMMETRIC || est == CPHB_EST_COLORED_ICP);
    const bool t_grad = target->color_gradient && est == CPHB_EST_COLORED_ICP;
    const bool t_cov = target->covariances && est == CPHB_EST_GENERALIZED_ICP;
    size_t o_tn = t_nrm ? take(sizeof(float4) * (nt_pad ? nt_pad : 1)) : 0, o_tg = t_grad ? take(sizeof(float4) * (nt_pad ? nt_pad : 1)) : 0;
    size_t o_tc = t_cov ? take(sizeof(float4) * 3 * (nt_pad ? nt_pad : 1)) : 0;
    size_t o_ts = take(sizeof(double) * n_pad);
    const unsigned flag_words = n_pad / 1024 + 1;
    size_t o_fb = take(sizeof(unsigned) * 2 * flag_words);
    size_t o_prev = take(sizeof(int2) * n_pad);
    size_t o_axyz = take(sizeof(float4) * n_pad), o_aprev = take(sizeof(int2) * n_pad);
    size_t o_anrm = want_nrm ? take(sizeof(float4) * n_pad) : 0, o_acov = want_cov ? take(sizeof(float4) * 3 * n_pad) : 0;
    size_t o_acol = want_col ? take(sizeof(float4) * n_pad) : 0, o_ccol = want_col ? take(sizeof(float4) * n_pad) : 0;
    size_t o_rt = take(sizeof(uint32_t) * 4 * n_pad);
    const unsigned nf_pad = (unsigned)cphb_align(n_full ? n_full : 1, ICP_BLOCK);
    size_t o_ci = take(sizeof(int32_t) * nf_pad);
    unsigned cmp_blocks = (nf_pad + CMP_BLOCK - 1) / CMP_BLOCK;
    size_t o_cc = take(sizeof(unsigned) * (cmp_blocks + 1));
    size_t o_ct = take(16);
    icp->arena_bytes = off;
    rc = cphb_alloc_async(&icp->arena, off, s);
    if (rc) { cphb_index_destroy(icp->index); delete icp; return rc; }
    char *b = (char *)icp->arena;
    icp->pristine_xyz = (float4 *)(b + o_pxyz);
    icp->work_xyz = (float4 *)(b + o_wxyz);
    icp->pristine_nrm = want_nrm ? (float4 *)(b + o_pnrm) : nullptr;
    icp->work_nrm = want_nrm ? (float4 *)(b + o_wnrm) : nullptr;
    icp->pristine_cov = want_cov ? (float4 *)(b + o_pcov) : nullptr;
    icp->work_cov = want_cov ? (float4 *)(b + o_wcov) : nullptr;
    icp->src_col = want_col ? (float4 *)(b + o_col) : nullptr;
    icp->st = (IcpState *)(b + o_st);
    icp->partials = (double *)(b + o_part);
    icp->tix_nrm = t_nrm ? (float4 *)(b + o_tn) : nullptr;
    icp->tix_grad = t_grad ? (float4 *)(b + o_tg) : nullptr;
    icp->tix_cov = t_cov ? (float4 *)(b + o_tc) : nullptr;
    icp->tile_sums = (double *)(b + o_ts);
    icp->flag_bits = (unsigned *)(b + o_fb);
    icp->flag_words = flag_words;
    icp->prev = (int2 *)(b + o_prev);
    icp->alt_xyz = (float4 *)(b + o_axyz);
    icp->alt_prev = (int2 *)(b + o_aprev);
    icp->alt_nrm = want_nrm ? (float4 *)(b + o_anrm) : nullptr;
    icp->alt_cov = want_cov ? (float4 *)(b + o_acov) : nullptr;
    icp->alt_col = want_col ? (float4 *)(b + o_acol) : nullptr;
    icp->cur_col = want_col ? (float4 *)(b + o_ccol) : nullptr;
    icp->rt_keys = (uint32_t *)(b + o_rt);
    icp->rt_keys2 = icp->rt_keys + n_pad;
    icp->rt_vals = icp->rt_keys + 2 * (size_t)n_pad;
    icp->rt_order = icp->rt_keys + 3 * (size_t)n_pad;
    icp->corr_index = (int32_t *)(b + o_ci);
    icp->cmp_counts = (unsigned *)(b + o_cc);
    icp->cmp_total = (unsigned *)(b + o_ct);
    if (!t_cache.in_use) {
        if (!t_cache.h_st) {
            CREATE_TRY(cudaMallocHost((void **)&t_cache.h_st, sizeof(IcpState)));
            CREATE_TRY(cudaEventCreate(&t_cache.ev0));
            CREATE_TRY(cudaEventCreate(&t_cache.ev1));
        }
        t_cache.in_use = true;
        icp->owns_host = false;
        icp->h_st = t_cache.h_st;
        icp->ev0 = t_cache.ev0;
        icp->ev1 = t_cache.ev1;
    } else {  // a second live context on this thread gets its own
        icp->owns_host = true;
        CREATE_TRY(cudaMallocHost((void **)&icp->h_st, sizeof(IcpState)));
        CREATE_TRY(cudaEventCreate(&icp->ev0));
        CREATE_TRY(cudaEventCreate(&icp->ev1));
    }
    if (t_source_ready) {  // (n_full == 0)
        cudaStreamWaitEvent(s, t_source_ready, 0);
        t_source_ready = nullptr;
    }
    if (perm_side) cudaStreamWaitEvent(s, t_side.join, 0);
    CPHB_LAUNCH(gather_source_kernel, n_pad / 256, 256, 0, s, source->points, source->normals, source->colors,
                source->covariances, source->cov_col_major, perm_side, lo, n, n_pad, icp->pristine_xyz, icp->pristine_nrm,
                icp->src_col, icp->pristine_cov);
    cphb_free_async(perm_side, s);
    perm_side = nullptr;
    if ((t_nrm || t_grad || t_cov) && nt_pad)
        CPHB_LAUNCH(gather_target_kernel, (unsigned)((nt_pad + 255) / 256), 256, 0, s, icp->index->v.pts, nt_pad, target->normals,
                    (est == CPHB_EST_COLORED_ICP) ? target->colors : nullptr, target->color_gradient, target->covariances,
                    target->cov_col_major, icp->tix_nrm, icp->tix_grad, icp->tix_cov);
    CREATE_TRY(cudaGetLastError());
    *out = icp;
    return CPHB_OK;
}

#undef CREATE_TRY
extern "C" void cphb_icp_destroy(cphb_icp *icp) {
    if (!icp) return;
    if (icp->arena) cudaFreeAsync(icp->arena, icp->stream);
    if (icp->dbg) cudaFree(icp->dbg);
    if (icp->owns_host) {
        if (icp->h_st) cudaFreeHost(icp->h_st);
        if (icp->ev0) cudaEventDestroy(icp->ev0);
        if (icp->ev1) cudaEventDestroy(icp->ev1);
    } else if (icp->h_st == t_cache.h_st) {
        t_cache.in_use = false;
    }
    cphb_index_destroy(icp->index);
    delete icp;
}

static void fill_args(const cphb_icp *icp, IcpArgs &a) {
    memset(&a, 0, sizeof(a));
    a.ix = icp->index->v;
    a.src = icp->work_xyz;
    a.src_nrm = icp->work_nrm;
    a.src_cov = icp->work_cov;
    a.src_col = icp->src_col;
    a.tgt_nrm = icp->tix_nrm;
    a.tgt_grad = icp->tix_grad;
    a.tgt_cov = icp->tix_cov;
    a.has_tgt_col = icp->tgt.colors != nullptr;
    a.st = icp->st;
    a.partials = icp->partials;
    a.tile_sums = icp->tile_sums;
    a.flag_bits = icp->flag_bits;
    a.flag_words = icp->flag_words;
    a.reduce_grid = icp->reduce_grid;
    // certified regime: 1 block in 8 (at least 2 when the grid allows) only runs the tiles that needed a search last time:
    // a search on an otherwise idle SM is one warp's dependent chain, so a helper warp should not get more than one or two
    // of them (config 2 on the H100, profiles/h100_tuning_sweep.txt: 17 / 33 / 132 helper blocks -> 6429 / 7350 / 7330 it/s, the default
    // 66 -> 7145-7381 it/s over three runs)
    a.helper_blocks = icp->grid >= 64 ? (icp->grid / 8 > 2 ? icp->grid / 8 : 2) : 0;
    if (const char *e = getenv("CPHB_HELPER_BLOCKS")) { int v = atoi(e); if (v >= 0 && (unsigned)v < icp->grid / 2) a.helper_blocks = (unsigned)v; }
    a.prev = icp->prev;
    a.n_src = icp->n_src;
    a.n_pad = icp->n_pad;
    a.n_total = icp->n_src;
    float r = icp->prm.max_correspondence_distance;
    a.r2 = (r > 0.f) ? r * r : 0.f;  // registration.cu:40-42: r <= 0 -> no correspondences
    a.rel_fitness = icp->prm.relative_fitness;
    a.rel_rmse = icp->prm.relative_rmse;
    a.det_thresh = icp->prm.det_thresh;
    a.max_iter = icp->prm.max_iteration > 0 ? icp->prm.max_iteration : 0;
    float lg = icp->prm.lambda_geometric;
    if (lg < 0.f || lg > 1.0f) lg = 0.968f;  // colored_icp.cu:48-52
    a.sg = (float)sqrt((double)lg);
    float lp = (float)(1.0 - (double)lg);
    a.sp = (float)sqrt((double)lp);
    a.cert_gain = 4.f;   // config 2 on the H100: gain 2 / 8 -> 7168 / 7187 it/s, 4 -> 7145-7381 (flat; profiles/h100_tuning_sweep.txt)
    a.cert_cap = 0.5f;
    if (const char *e = getenv("CPHB_CERT_GAIN")) a.cert_gain = (float)atof(e);  // tuning hooks; 0 = no certificates
    if (const char *e = getenv("CPHB_CERT_CAP")) a.cert_cap = (float)atof(e);
    a.cert_cap_r = 0.25f * (r > 0.f ? r : 0.f);
    a.r_up = (float)(sqrt((double)a.r2) * 1.00002);
    a.dbg = icp->dbg;
    a.claim_max = 8u;
    if (const char *e = getenv("CPHB_CLAIM_MAX")) { int v = atoi(e); if (v >= 1 && v <= 1024) a.claim_max = (unsigned)v; }
    a.static_sched = 1;  // config 2 on the H100: 7145-7381 it/s vs 6870 with the dynamic schedule (profiles/h100_tuning_sweep.txt)
    if (const char *e = getenv("CPHB_STATIC_SCHED")) a.static_sched = atoi(e) != 0;
    a.tmax = CPHB_TRANSPOSE_MAX;
    if (const char *e = getenv("CPHB_TRANSPOSE_MAX")) {  // tuning hook
        int v = atoi(e);
        if (v >= 0 && v <= 32) a.tmax = v;
    }
}

static int reset_working_copy(cphb_icp *icp, cudaStream_t s) {
    CPHB_CUDA(cudaMemsetAsync(icp->flag_bits, 0, sizeof(unsigned) * 2 * icp->flag_words, s));
    CPHB_CUDA(cudaMemsetAsync(icp->prev, 0xff, sizeof(int2) * icp->n_pad, s));  // no warm start at launch 0
    CPHB_CUDA(cudaMemcpyAsync(icp->work_xyz, icp->pristine_xyz, sizeof(float4) * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    if (icp->work_nrm)
        CPHB_CUDA(cudaMemcpyAsync(icp->work_nrm, icp->pristine_nrm, sizeof(float4) * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    if (icp->work_cov)
        CPHB_CUDA(cudaMemcpyAsync(icp->work_cov, icp->pristine_cov, sizeof(float4) * 3 * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    return CPHB_OK;
}

static int compact_correspondences(cphb_icp *icp, int32_t *corr_out, cudaStream_t s) {
    unsigned n = icp->n_full;
    unsigned nb = (n + CMP_BLOCK - 1) / CMP_BLOCK;
    if (nb == 0) nb = 1;
    CPHB_LAUNCH(compact_count_kernel, nb, CMP_BLOCK, 0, s, icp->corr_index, n, icp->cmp_counts);
    CPHB_LAUNCH(compact_scan_kernel, 1, 1024, 0, s, icp->cmp_counts, nb, icp->cmp_total);
    CPHB_LAUNCH(compact_write_kernel, nb, CMP_BLOCK, 0, s, icp->corr_index, n, icp->cmp_counts, corr_out);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// permute the working arrays referenced by `a` into the alt buffers and swap
static int retile(cphb_icp *icp, IcpArgs &a, cudaStream_t s) {
    const unsigned n_pad = icp->n_pad, grid = n_pad / 256;
    const uint32_t n_tgt_pad = (uint32_t)icp->index->v.n_leaves * CPHB_LEAF;
    CPHB_LAUNCH(retile_key_kernel, grid, 256, 0, s, a.prev, icp->n_src, n_pad, n_tgt_pad, icp->rt_keys, icp->rt_vals);
    CPHB_CHECK_LAUNCH();
    // keys are target LEAVES (< n_tgt_pad / 32) or the two sentinels right above them: the stable radix sort only
    // has to look at the bits that can differ (16 for 1 M points: 2 onesweep passes)
    int bits = 1;
    while (bits < 32 && ((uint64_t)1 << bits) < (uint64_t)(n_tgt_pad >> 5) + 2u) ++bits;
    int rc = cphb_sort_pairs_u32(icp->rt_keys, icp->rt_keys2, icp->rt_vals, icp->rt_order, n_pad, bits, s);
    if (rc) return rc;
    float4 *o_xyz = (a.src == icp->work_xyz) ? icp->alt_xyz : icp->work_xyz;
    int2 *o_prev = (a.prev == icp->prev) ? icp->alt_prev : icp->prev;
    float4 *o_nrm = a.src_nrm ? ((a.src_nrm == icp->work_nrm) ? icp->alt_nrm : icp->work_nrm) : nullptr;
    float4 *o_cov = a.src_cov ? ((a.src_cov == icp->work_cov) ? icp->alt_cov : icp->work_cov) : nullptr;
    float4 *o_col = a.src_col ? ((a.src_col == icp->alt_col) ? icp->cur_col : icp->alt_col) : nullptr;
    CPHB_LAUNCH(retile_gather_kernel, grid, 256, 0, s, icp->rt_order, n_pad, a.src, a.prev, a.src_nrm, a.src_col, a.src_cov,
                o_xyz, o_prev, o_nrm, o_col, o_cov);
    CPHB_CHECK_LAUNCH();
    a.src = o_xyz;
    a.prev = o_prev;
    a.src_nrm = o_nrm;
    a.src_cov = o_cov;
    a.src_col = o_col;
    return CPHB_OK;
}

extern "C" int cphb_icp_run(cphb_icp *icp, const float h_init[16], cphb_comm *comm, cphb_icp_result *h_result,
                            int32_t *corr_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!icp || !h_init || !h_result) {
        cphb_set_error("cphb_icp_run: null argument");
        return CPHB_ERR_INVALID;
    }
    int rc = reset_working_copy(icp, s);
    if (rc) return rc;
    IcpState *h = icp->h_st;
    memset(h, 0, sizeof(*h));
    memcpy(h->T, h_init, 64);
    memcpy(h->U, h_init, 64);
    h->apply_u = is_identity4(h_init) ? 0 : 1;
    CPHB_CUDA(cudaMemcpyAsync(icp->st, h, sizeof(IcpState), cudaMemcpyHostToDevice, s));
    static const bool dbg_cert = getenv("CPHB_DEBUG_CERT") != nullptr;
    if (dbg_cert) {
        if (!icp->dbg) CPHB_CUDA(cudaMalloc(&icp->dbg, sizeof(unsigned) * 256 + 128));
        CPHB_CUDA(cudaMemsetAsync(icp->dbg, 0, sizeof(unsigned) * 256 + 128, s));
        CPHB_CUDA(cudaMemsetAsync(icp->dbg + 256, 0xff, 8, s));  // slot 0 takes a minimum
    }
    IcpArgs a;
    fill_args(icp, a);
    a.corr_index = corr_out ? icp->corr_index : nullptr;
    if (corr_out && icp->n_full != icp->n_src)  // points owned by other ranks have no entry here
        CPHB_CUDA(cudaMemsetAsync(icp->corr_index, 0xff, sizeof(int32_t) * icp->n_full, s));
    unsigned long long n_total = icp->n_src;
    const bool lib_sharded = icp->prm.shard_world > 1;
    if (lib_sharded) n_total = icp->n_full;
    void *nccl_comm = nullptr;
    if (comm && comm->world > 1) {
        // a communicator that cannot exchange would fault (null mailboxes) or hang every peer's GPU: refuse it here
        if (comm->kind == CPHB_COMM_P2P && !comm->connected) {
            cphb_set_error("cphb_icp_run: peer-memory communicator is not connected (cphb_comm_p2p_connect)");
            return CPHB_ERR_INVALID;
        }
        if (comm->kind == CPHB_COMM_NCCL && !comm->nccl) {
            cphb_set_error("cphb_icp_run: NCCL communicator is not initialised");
            return CPHB_ERR_INVALID;
        }
        if (lib_sharded && (comm->world != icp->prm.shard_world || comm->rank != icp->prm.shard_rank)) {
            cphb_set_error("cphb_icp_run: communicator is rank %d of %d but the context was created as shard %d of %d", comm->rank,
                           comm->world, icp->prm.shard_rank, icp->prm.shard_world);
            return CPHB_ERR_INVALID;
        }
    }
    if (comm && comm->world > 1 && lib_sharded) {
        if (comm->kind == CPHB_COMM_NCCL) {
            nccl_comm = comm->nccl;
            a.defer_finalize = 1;
        } else {
            a.use_p2p = 1;
            a.p2p = comm->view;
        }
    } else if (comm && comm->world > 1) {
        // caller-sharded source: global source size by one tiny exchange before the loop
        double *tmp = icp->partials;  // scratch
        double hn = (double)icp->n_src;
        CPHB_CUDA(cudaMemcpyAsync(tmp, &hn, 8, cudaMemcpyHostToDevice, s));
        rc = cphb_comm_allreduce_f64(comm, tmp, 1, s);
        if (rc) return rc;
        CPHB_CUDA(cudaMemcpyAsync(&hn, tmp, 8, cudaMemcpyDeviceToHost, s));
        CPHB_CUDA(cudaStreamSynchronize(s));
        n_total = (unsigned long long)hn;
        if (comm->kind == CPHB_COMM_NCCL) {
            nccl_comm = comm->nccl;
            a.defer_finalize = 1;
        } else {
            a.use_p2p = 1;
            a.p2p = comm->view;
        }
    }
    a.n_total = n_total;
    // launches 0..max_iter: search (+ update).  If the convergence test stops the loop at launch
    // j < max_iter, launch j+1 re-runs that search only to materialise its correspondences;
    // launches after "done" exit at their first instruction.
    const unsigned long long launches0 = g_cphb_launches;
    // Re-tiling (the working copy re-ordered by the target position of every point's current match) after the launches
    // whose bit is set.  It paid for itself while the rows were gathered through the caller's arrays; with the target
    // attributes in index order and the certified regime's cp.async row pipeline a re-tiling is no longer earned back
    // (config 2 on the H100: mask 0x12 / 0x4 -> 7059 / 7135 it/s, none -> 7145-7381; profiles/h100_tuning_sweep.txt), so the default is none.
    unsigned long long retile_mask = 0ull;
    if (const char *e = getenv("CPHB_RETILE_MASK")) retile_mask = strtoull(e, nullptr, 0);  // tuning hook
    static const bool dbg_events = getenv("CPHB_DEBUG_EVENTS") != nullptr;
    std::vector<cudaEvent_t> evs;
    if (dbg_events) {
        evs.resize(3 * (size_t)(a.max_iter + 1));
        for (auto &e : evs) cudaEventCreate(&e);
        icp->dbg_ev = evs.data();
    }
    CPHB_CUDA(cudaEventRecord(icp->ev0, s));
    for (int it = 0; it <= a.max_iter; ++it) {
        a.launch_idx = it;
        if (dbg_events) cudaEventRecord(evs[3 * it], s);
        launch_iteration_kind(icp, a, s);
        if (dbg_events) cudaEventRecord(evs[3 * it + 2], s);
        if (nccl_comm) {
            rc = cphb_nccl_allreduce_f64(nccl_comm, icp->st->local, icp->st->total, 32, s);
            if (rc) return rc;
            launch_finalize_kind(icp, a, s);
        }
        if (!(icp->prm.flags & CPHB_ICP_NO_RETILE) && it < a.max_iter && it < 64 && ((retile_mask >> it) & 1ull) && icp->n_src >= 4096) {
            rc = retile(icp, a, s);
            if (rc) return rc;
        }
    }
    CPHB_CUDA(cudaEventRecord(icp->ev1, s));
    const int loop_launches = (int)(g_cphb_launches - launches0);
    CPHB_CHECK_LAUNCH();
    if (corr_out) {
        rc = compact_correspondences(icp, corr_out, s);
        if (rc) return rc;
    }
    unsigned h_local = 0;
    if (corr_out) CPHB_CUDA(cudaMemcpyAsync(&h->pad_local, icp->cmp_total, 4, cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaMemcpyAsync(h, icp->st, offsetof(IcpState, pad_local), cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    h_local = h->pad_local;
    if (h->comm_timeout) {
        cphb_set_error("cphb_icp_run: the peer-memory exchange timed out waiting for another rank; the result is invalid");
        return CPHB_ERR_CUDA;
    }
    memcpy(h_result->transformation, h->T, 64);
    h_result->fitness = h->fitness;
    h_result->inlier_rmse = h->rmse;
    h_result->n_correspondences = h->n_corr;
    h_result->n_local_correspondences = corr_out ? (long long)h_local : 0;
    h_result->iterations = h->iterations;
    h_result->converged = h->converged;
    h_result->loop_ms = 0.f;
    cudaEventElapsedTime(&h_result->loop_ms, icp->ev0, icp->ev1);
    h_result->loop_launches = loop_launches;
    if (dbg_events) {
        fprintf(stderr, "[cphb] per launch us (search kernel / reduce+solve / until next launch):\n");
        for (int it = 0; it <= a.max_iter; ++it) {
            float t_it = 0.f, t_red = 0.f, t_gap = 0.f;
            cudaEventElapsedTime(&t_it, evs[3 * it], evs[3 * it + 1]);
            cudaEventElapsedTime(&t_red, evs[3 * it + 1], evs[3 * it + 2]);
            if (it < a.max_iter) cudaEventElapsedTime(&t_gap, evs[3 * it + 2], evs[3 * it + 3]);
            fprintf(stderr, " %d:%.1f/%.1f/%.1f", it, 1e3f * t_it, 1e3f * t_red, 1e3f * t_gap);
        }
        fprintf(stderr, "\n");
        for (auto &e : evs) cudaEventDestroy(e);
        icp->dbg_ev = nullptr;
    }
    if (dbg_cert && icp->dbg) {
        unsigned hd[256 + 32];
        CPHB_CUDA(cudaMemcpy(hd, icp->dbg, sizeof(hd), cudaMemcpyDeviceToHost));
        {
            const unsigned long long *tl = reinterpret_cast<const unsigned long long *>(hd + 256);
            if (tl[4] && tl[0] != ~0ull)
                fprintf(stderr, "[cphb] launch 20 timeline (us after the first block started): tile loops done %.1f, last block in %.1f, grid sum done %.1f, "
                        "[state read %.1f, 6x6 solved %.1f, pose composed %.1f] finalize done %.1f\n",
                        (tl[1] - tl[0]) * 1e-3, (tl[2] - tl[0]) * 1e-3, (tl[3] - tl[0]) * 1e-3, (tl[5] - tl[0]) * 1e-3, (tl[6] - tl[0]) * 1e-3,
                        (tl[7] - tl[0]) * 1e-3, (tl[4] - tl[0]) * 1e-3);
            if (tl[4] && tl[0] != ~0ull)
                fprintf(stderr, "[cphb] launch 20 tile loops (us): main warps without an in-line search done %.1f, with one %.1f, helper warps done %.1f, "
                        "last block start %.1f\n", tl[8] ? (tl[8] - tl[0]) * 1e-3 : 0.0, tl[9] ? (tl[9] - tl[0]) * 1e-3 : 0.0,
                        tl[10] ? (tl[10] - tl[0]) * 1e-3 : 0.0, tl[11] ? (tl[11] - tl[0]) * 1e-3 : 0.0);
        }
        fprintf(stderr, "[cphb] certificates (n_src %u, tiles %u): launch: certified lanes / skipped tiles [/ deferred tiles, * = certified regime]\n", icp->n_src, icp->n_pad / 32);
        for (int it = 0; it <= a.max_iter && it < 64; ++it) {
            if (hd[192 + it]) fprintf(stderr, " %d*:%u/%u/%u", it, hd[it], hd[64 + it], hd[128 + it]);
            else fprintf(stderr, " %d:%u/%u", it, hd[it], hd[64 + it]);
        }
        fprintf(stderr, "\n");
    }
    return CPHB_OK;
}

extern "C" int cphb_icp_step(cphb_icp *icp, const float h_T[16], double h_sums[32], int32_t *corr_index, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!icp || !h_T || !h_sums) {
        cphb_set_error("cphb_icp_step: null argument");
        return CPHB_ERR_INVALID;
    }
    int rc = reset_working_copy(icp, s);
    if (rc) return rc;
    IcpState *h = icp->h_st;
    memset(h, 0, sizeof(*h));
    memcpy(h->T, h_T, 64);
    memcpy(h->U, h_T, 64);
    h->apply_u = 1;
    CPHB_CUDA(cudaMemcpyAsync(icp->st, h, sizeof(IcpState), cudaMemcpyHostToDevice, s));
    IcpArgs a;
    fill_args(icp, a);
    a.step_mode = 1;
    a.corr_index = icp->corr_index;
    CPHB_CUDA(cudaMemsetAsync(icp->corr_index, 0xff, sizeof(int32_t) * icp->n_full, s));
    launch_iteration_kind(icp, a, s);
    CPHB_CHECK_LAUNCH();
    if (corr_index)
        CPHB_CUDA(cudaMemcpyAsync(corr_index, icp->corr_index, sizeof(int32_t) * icp->n_full, cudaMemcpyDeviceToDevice, s));
    CPHB_CUDA(cudaMemcpyAsync(h, icp->st, sizeof(IcpState), cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    memcpy(h_sums, h->total, sizeof(double) * 32);
    return CPHB_OK;
}

extern "C" int cphb_registration_icp(const cphb_cloud *source, const cphb_cloud *target, const float h_init[16],
                                     const cphb_icp_params *params, cphb_comm *comm, cphb_icp_result *h_result,
                                     int32_t *corr_out, void *stream) {
    static const bool dbg = getenv("CPHB_DEBUG_TIMING") != nullptr;
    struct timespec t0, t1, t2, t3;
    if (dbg) clock_gettime(CLOCK_MONOTONIC, &t0);
    cphb_icp *icp = nullptr;
    int rc = cphb_icp_create(source, target, params, stream, &icp);
    if (rc) return rc;
    if (dbg) clock_gettime(CLOCK_MONOTONIC, &t1);
    rc = cphb_icp_run(icp, h_init, comm, h_result, corr_out, stream);
    if (dbg) clock_gettime(CLOCK_MONOTONIC, &t2);
    cphb_icp_destroy(icp);
    if (dbg) {
        clock_gettime(CLOCK_MONOTONIC, &t3);
        auto ms = [](const timespec &a, const timespec &b) { return (b.tv_sec - a.tv_sec) * 1e3 + (b.tv_nsec - a.tv_nsec) * 1e-6; };
        fprintf(stderr, "[cphb] registration_icp host ms: create %.3f run %.3f destroy %.3f (loop device %.3f)\n", ms(t0, t1),
                ms(t1, t2), ms(t2, t3), h_result->loop_ms);
    }
    return rc;
}

// One-shot registration from HOST buffers (pinned or pageable): the uploads run on a separate stream and overlap the
// target index build and the source ordering -- target points first (the index needs nothing else), then the
// source, then the target attributes that only the first iteration reads.  The clouds' pointers are host pointers;
// h_corr_out (optional, host, 2 * source.n int32) receives the (i, j) pairs.  Everything is complete on return.
struct HostUploadCache {
    cudaStream_t copy = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
};
static thread_local HostUploadCache t_up;

extern "C" int cphb_registration_icp_host(const cphb_cloud *h_source, const cphb_cloud *h_target, const float h_init[16],
                                          const cphb_icp_params *params, cphb_comm *comm, cphb_icp_result *h_result,
                                          int32_t *h_corr_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_source || !h_target || !params || !h_result || !h_init) {
        cphb_set_error("cphb_registration_icp_host: null argument");
        return CPHB_ERR_INVALID;
    }
    if (!t_up.copy) {
        CPHB_CUDA(cudaStreamCreateWithFlags(&t_up.copy, cudaStreamNonBlocking));
        for (auto &e : t_up.ev) CPHB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    const size_t ns = h_source->n, nt = h_target->n;
    // device arena: [tgt points | src points, normals, colors, covariances | tgt normals, colors, covariances, gradient | pairs]
    size_t off = 0;
    auto take = [&](const void *hp, size_t bytes) { size_t o = off; if (hp) off = cphb_align(off + bytes, 256); return hp ? o : (size_t)-1; };
    const size_t o_tp = take(h_target->points, 12 * nt);
    const size_t o_sp = take(h_source->points, 12 * ns), o_sn = take(h_source->normals, 12 * ns), o_sc = take(h_source->colors, 12 * ns),
                 o_sv = take(h_source->covariances, 36 * ns);
    const size_t o_tn = take(h_target->normals, 12 * nt), o_tc = take(h_target->colors, 12 * nt),
                 o_tv = take(h_target->covariances, 36 * nt), o_tg = take(h_target->color_gradient, 12 * nt);
    const size_t o_pairs = take(h_corr_out, 8 * ns);
    char *base = nullptr;
    int rc = cphb_alloc_async((void **)&base, off ? off : 256, s);
    if (rc) return rc;
    auto dp = [&](size_t o) { return o == (size_t)-1 ? (float *)nullptr : (float *)(base + o); };
    cudaStream_t c = t_up.copy;
    // one exit for CUDA errors: no upload may still be reading the caller's buffers, and the arena goes back to the pool
#define HOST_TRY(call)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (call);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            cphb_set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));          \
            cudaStreamSynchronize(c);                                                                    \
            cphb_free_async(base, s);                                                                    \
            return CPHB_ERR_CUDA;                                                                        \
        }                                                                                                \
    } while (0)
    HOST_TRY(cudaEventRecord(t_up.ev[0], s));            // the arena exists from here on in stream order
    HOST_TRY(cudaStreamWaitEvent(c, t_up.ev[0], 0));
    auto up = [&](size_t o, const void *hp, size_t bytes) {
        if (hp && bytes) cudaMemcpyAsync(base + o, hp, bytes, cudaMemcpyHostToDevice, c);
    };
    up(o_tp, h_target->points, 12 * nt);
    HOST_TRY(cudaEventRecord(t_up.ev[1], c));            // target points: all the index build needs
    up(o_sp, h_source->points, 12 * ns);
    up(o_sn, h_source->normals, 12 * ns);
    up(o_sc, h_source->colors, 12 * ns);
    up(o_sv, h_source->covariances, 36 * ns);
    HOST_TRY(cudaEventRecord(t_up.ev[2], c));            // source: first read by the Hilbert ordering
    up(o_tn, h_target->normals, 12 * nt);
    up(o_tc, h_target->colors, 12 * nt);
    up(o_tv, h_target->covariances, 36 * nt);
    up(o_tg, h_target->color_gradient, 12 * nt);
    HOST_TRY(cudaEventRecord(t_up.ev[3], c));            // target attributes: first read by the first iteration
    cphb_cloud ds = *h_source, dt = *h_target;
    ds.points = dp(o_sp); ds.normals = dp(o_sn); ds.colors = dp(o_sc); ds.covariances = dp(o_sv); ds.color_gradient = nullptr;
    dt.points = dp(o_tp); dt.normals = dp(o_tn); dt.colors = dp(o_tc); dt.covariances = dp(o_tv); dt.color_gradient = dp(o_tg);
    HOST_TRY(cudaStreamWaitEvent(s, t_up.ev[1], 0));
#undef HOST_TRY
    t_source_ready = t_up.ev[2];
    cphb_icp *icp = nullptr;
    rc = cphb_icp_create(&ds, &dt, params, stream, &icp);
    t_source_ready = nullptr;
    if (!rc) {
        cudaStreamWaitEvent(s, t_up.ev[2], 0);            // (already waited inside create; harmless if it returned early)
        cudaStreamWaitEvent(s, t_up.ev[3], 0);
        int32_t *d_pairs = (int32_t *)dp(o_pairs);
        rc = cphb_icp_run(icp, h_init, comm, h_result, d_pairs, stream);
        if (!rc && h_corr_out && h_result->n_local_correspondences > 0) {
            cudaError_t e = cudaMemcpyAsync(h_corr_out, d_pairs, sizeof(int32_t) * 2 * (size_t)h_result->n_local_correspondences,
                                            cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e != cudaSuccess) { cphb_set_error("cphb_registration_icp_host: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
        }
        cphb_icp_destroy(icp);
    }
    cudaStreamSynchronize(c);                              // no upload may outlive the host buffers or the arena
    cphb_free_async(base, s);
    cudaStreamSynchronize(s);
    return rc;
}

extern "C" int cphb_evaluate_registration(const cphb_cloud *source, const cphb_cloud *target,
                                          float max_correspondence_distance, const float h_T[16],
                                          cphb_icp_result *h_result, int32_t *corr_out, void *stream) {
    cphb_icp_params p;
    memset(&p, 0, sizeof(p));
    p.estimation = CPHB_EST_POINT_TO_POINT;
    p.max_correspondence_distance = max_correspondence_distance;
    p.max_iteration = 0;
    cphb_cloud src = *source, tgt = *target;
    src.normals = src.colors = src.covariances = nullptr;
    tgt.normals = tgt.colors = tgt.covariances = tgt.color_gradient = nullptr;
    return cphb_registration_icp(&src, &tgt, h_T, &p, nullptr, h_result, corr_out, stream);
}

extern "C" int cphb_transform(float *points, float *normals, float *covariances, int cov_col_major, size_t n,
                              const float h_T[16], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return CPHB_OK;
    float *Td = nullptr;
    int rc = cphb_alloc_async((void **)&Td, 64, s);
    if (rc) return rc;
    CPHB_CUDA(cudaMemcpyAsync(Td, h_T, 64, cudaMemcpyHostToDevice, s));
    CPHB_LAUNCH(transform_kernel, (unsigned)((n + 255) / 256), 256, 0, s, points, normals, covariances, cov_col_major, n, Td);
    CPHB_CHECK_LAUNCH();
    cphb_free_async(Td, s);
    return CPHB_OK;
}

// ---------------------------------------------------------------------------
// standalone estimator entry points
// ---------------------------------------------------------------------------
static int run_estimate(int estimation, const cphb_cloud *source, const cphb_cloud *target, const int32_t *corr,
                        size_t n_corr, const cphb_icp_params *params, double h_S[32], float h_T[16], cudaStream_t s) {
    if (!source || !target || (n_corr && !corr)) {
        cphb_set_error("estimate: null argument");
        return CPHB_ERR_INVALID;
    }
    if (estimation < CPHB_EST_POINT_TO_POINT || estimation > CPHB_EST_GENERALIZED_ICP) {
        cphb_set_error("estimate: estimation %d unsupported", estimation);
        return CPHB_ERR_UNSUPPORTED;
    }
    for (int i = 0; i < 32; ++i) h_S[i] = 0.0;
    if (h_T) for (int i = 0; i < 16; ++i) h_T[i] = (i % 5 == 0) ? 1.f : 0.f;
    if (n_corr == 0) return CPHB_OK;
    EstArgs a;
    memset(&a, 0, sizeof(a));
    float lg = params ? params->lambda_geometric : 0.968f;
    if (lg < 0.f || lg > 1.0f) lg = 0.968f;
    a.ta.tgt_xyz = target->points; a.ta.tgt_nrm = target->normals; a.ta.tgt_col = target->colors;
    a.ta.tgt_grad = target->color_gradient; a.ta.tgt_cov = target->covariances;
    a.ta.tgt_cov_col_major = target->cov_col_major;
    a.ta.sg = (float)sqrt((double)lg);
    a.ta.sp = (float)sqrt((double)(float)(1.0 - (double)lg));
    a.ta.src_nrm = source->normals != nullptr; a.ta.src_col = source->colors != nullptr;
    a.ta.src_cov = source->covariances != nullptr;
    a.src_xyz = source->points; a.src_nrm = source->normals; a.src_col = source->colors;
    a.src_cov = source->covariances; a.src_cov_col_major = source->cov_col_major;
    a.corr = corr;
    a.n_corr = (unsigned)n_corr;
    unsigned grid = (unsigned)((n_corr + ICP_BLOCK - 1) / ICP_BLOCK);
    char *buf = nullptr;
    size_t bytes = cphb_align(sizeof(double) * 32 * grid, 256) + 256 + 256 + 64;
    int rc = cphb_alloc_async((void **)&buf, bytes, s);
    if (rc) return rc;
    a.partials = (double *)buf;
    a.total = (double *)(buf + cphb_align(sizeof(double) * 32 * grid, 256));
    a.ticket = (unsigned *)((char *)a.total + 256);
    float *Td = (float *)((char *)a.total + 512);
    CPHB_CUDA(cudaMemsetAsync(a.ticket, 0, 4, s));
    bool have = true;
    switch (estimation) {
        case CPHB_EST_POINT_TO_POINT: CPHB_LAUNCH(estimate_kernel<CPHB_EST_POINT_TO_POINT>, grid, ICP_BLOCK, 0, s, a); break;
        case CPHB_EST_POINT_TO_PLANE: have = target->normals; CPHB_LAUNCH(estimate_kernel<CPHB_EST_POINT_TO_PLANE>, grid, ICP_BLOCK, 0, s, a); break;
        case CPHB_EST_SYMMETRIC: have = target->normals && source->normals; CPHB_LAUNCH(estimate_kernel<CPHB_EST_SYMMETRIC>, grid, ICP_BLOCK, 0, s, a); break;
        case CPHB_EST_COLORED_ICP: have = target->normals && target->colors && source->colors; CPHB_LAUNCH(estimate_kernel<CPHB_EST_COLORED_ICP>, grid, ICP_BLOCK, 0, s, a); break;
        case CPHB_EST_GENERALIZED_ICP: have = target->covariances && source->covariances; CPHB_LAUNCH(estimate_kernel<CPHB_EST_GENERALIZED_ICP>, grid, ICP_BLOCK, 0, s, a); break;
    }
    if (h_T) {
        float dt = params ? params->det_thresh : 1e-6f;
        unsigned long long nm = source->n;
        switch (estimation) {
            case CPHB_EST_POINT_TO_POINT: CPHB_LAUNCH(estimate_solve_kernel<CPHB_EST_POINT_TO_POINT>, 1, 32, 0, s, a.total, nm, dt, have, Td); break;
            case CPHB_EST_POINT_TO_PLANE: CPHB_LAUNCH(estimate_solve_kernel<CPHB_EST_POINT_TO_PLANE>, 1, 32, 0, s, a.total, nm, dt, have, Td); break;
            case CPHB_EST_SYMMETRIC: CPHB_LAUNCH(estimate_solve_kernel<CPHB_EST_SYMMETRIC>, 1, 32, 0, s, a.total, nm, dt, have, Td); break;
            case CPHB_EST_COLORED_ICP: CPHB_LAUNCH(estimate_solve_kernel<CPHB_EST_COLORED_ICP>, 1, 32, 0, s, a.total, nm, dt, have, Td); break;
            case CPHB_EST_GENERALIZED_ICP: CPHB_LAUNCH(estimate_solve_kernel<CPHB_EST_GENERALIZED_ICP>, 1, 32, 0, s, a.total, nm, dt, have, Td); break;
        }
        CPHB_CUDA(cudaMemcpyAsync(h_T, Td, 64, cudaMemcpyDeviceToHost, s));
    }
    CPHB_CHECK_LAUNCH();
    CPHB_CUDA(cudaMemcpyAsync(h_S, a.total, sizeof(double) * 32, cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    cphb_free_async(buf, s);
    return CPHB_OK;
}

extern "C" int cphb_compute_transformation(int estimation, const cphb_cloud *source, const cphb_cloud *target,
                                           const int32_t *corr, size_t n_corr, const cphb_icp_params *params,
                                           float h_T[16], void *stream) {
    double S[32];
    return run_estimate(estimation, source, target, corr, n_corr, params, S, h_T, (cudaStream_t)stream);
}

extern "C" int cphb_compute_rmse(int estimation, const cphb_cloud *source, const cphb_cloud *target, const int32_t *corr,
                                 size_t n_corr, const cphb_icp_params *params, float *h_rmse, void *stream) {
    double S[32];
    *h_rmse = 0.f;
    int rc = run_estimate(estimation, source, target, corr, n_corr, params, S, nullptr, (cudaStream_t)stream);
    if (rc || n_corr == 0) return rc;
    const float C = (float)n_corr;
    switch (estimation) {
        case CPHB_EST_POINT_TO_POINT: *h_rmse = sqrtf((float)S[28] / C); break;                      // transformation_estimation.cu:92-116
        case CPHB_EST_POINT_TO_PLANE: *h_rmse = target->normals ? sqrtf((float)S[27] / C) : 0.f; break;  // :118-166
        case CPHB_EST_SYMMETRIC: *h_rmse = (target->normals && source->normals) ? sqrtf((float)S[28] / C) : 0.f; break;  // :224-287
        case CPHB_EST_GENERALIZED_ICP: *h_rmse = sqrtf((float)S[28] / C); break;                     // generalized_icp.cu:134-151
        case CPHB_EST_COLORED_ICP: *h_rmse = (float)S[27]; break;  // colored_icp.cu:303-327 returns the plain sum (quirk)
    }
    return CPHB_OK;
}

// registration::Kabsch(model, target[, corres]) (kabsch.h:30-49); corr == NULL pairs i<->i
__global__ void __launch_bounds__(256) iota_pairs_kernel(int32_t *p, unsigned n) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { p[2 * (size_t)i] = (int32_t)i; p[2 * (size_t)i + 1] = (int32_t)i; }
}
extern "C" int cphb_kabsch(const float *model, size_t n_model, const float *target, const int32_t *corr, size_t n_corr,
                           float h_T[16], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    cphb_cloud src, tgt;
    memset(&src, 0, sizeof(src));
    memset(&tgt, 0, sizeof(tgt));
    src.points = model; src.n = n_model;
    tgt.points = target; tgt.n = n_model;
    int32_t *tmp = nullptr;
    if (!corr) {
        n_corr = n_model;
        int rc = cphb_alloc_async((void **)&tmp, sizeof(int32_t) * 2 * (n_model ? n_model : 1), s);
        if (rc) return rc;
        if (n_model) CPHB_LAUNCH(iota_pairs_kernel, (unsigned)((n_model + 255) / 256), 256, 0, s, tmp, (unsigned)n_model);
        corr = tmp;
    }
    int rc = cphb_compute_transformation(CPHB_EST_POINT_TO_POINT, &src, &tgt, corr, n_corr, nullptr, h_T, stream);
    cphb_free_async(tmp, s);
    return rc;
}
