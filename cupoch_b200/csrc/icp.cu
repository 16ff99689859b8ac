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
#include <memory>
#include <type_traits>
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
    cphb_arena arena;  // every device buffer below but dbg
    cphb_index *index = nullptr;
    cphb_icp_params prm = {};
    cphb_cloud tgt = {};
    unsigned n_src = 0, n_pad = 0;
    unsigned n_full = 0;  // size of the source as passed (== n_src unless the library shards it)
    float4 *pristine_xyz = nullptr, *pristine_nrm = nullptr, *pristine_cov = nullptr;  // Hilbert-ordered source as given
    float4 *work_xyz = nullptr, *work_nrm = nullptr, *work_cov = nullptr;
    float4 *src_col = nullptr;
    float4 *tix_nrm = nullptr, *tix_grad = nullptr, *tix_cov = nullptr;  // target attributes in index order (icp_types.cuh)
    IcpState *st = nullptr;
    IcpState *h_st = nullptr;  // pinned
    bool owns_host = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    double *partials = nullptr;
    int32_t *corr_index = nullptr;
    unsigned *cmp_counts = nullptr;
    unsigned *cmp_total = nullptr;
    double *tile_sums = nullptr;
    unsigned *flag_bits = nullptr;
    unsigned flag_words = 0;
    int2 *prev = nullptr;
    unsigned *dbg = nullptr;  // CPHB_DEBUG_CERT statistics
    cudaEvent_t *dbg_ev = nullptr;  // CPHB_DEBUG_EVENTS: 3 events per launch (before, between, after)
    unsigned grid_search = 0;  // ROLE 0 launch (searching regime)
    unsigned grid = 0;         // ROLE 1 launch (certified regime / sum of a searching launch's tile sums + solve)
    unsigned reduce_grid = 0;  // blocks of the ROLE 1 launch that take part in that sum
    ~cphb_icp();
};

// per-thread cached pinned staging buffer + events: cudaMallocHost / cudaEventCreate cost milliseconds,
// far more than a 1M-point registration's launch loop.
struct HostCache {
    IcpState *h_st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool in_use = false;
};
static thread_local HostCache t_cache;

cphb_icp::~cphb_icp() {
    if (dbg) cudaFree(dbg);
    if (owns_host) {
        if (h_st) cudaFreeHost(h_st);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    } else if (h_st == t_cache.h_st) {
        t_cache.in_use = false;
    }
    cphb_index_destroy(index);
}

// runs f when it leaves scope
template <class F>
struct scope_exit {
    F f;
    ~scope_exit() { f(); }
};
template <class F>
scope_exit(F) -> scope_exit<F>;

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

// f(std::integral_constant<int, KIND>{}) for a fused estimator (the callers have validated `kind`): one switch selects
// the kernel instances of every launch site
template <class F>
static void with_kind(int kind, F &&f) {
    switch (kind) {
        case CPHB_EST_POINT_TO_POINT: f(std::integral_constant<int, CPHB_EST_POINT_TO_POINT>{}); break;
        case CPHB_EST_POINT_TO_PLANE: f(std::integral_constant<int, CPHB_EST_POINT_TO_PLANE>{}); break;
        case CPHB_EST_SYMMETRIC: f(std::integral_constant<int, CPHB_EST_SYMMETRIC>{}); break;
        case CPHB_EST_COLORED_ICP: f(std::integral_constant<int, CPHB_EST_COLORED_ICP>{}); break;
        case CPHB_EST_GENERALIZED_ICP: f(std::integral_constant<int, CPHB_EST_GENERALIZED_ICP>{}); break;
    }
}
// f(std::integral_constant<int, TOP>{}): the iteration kernel is compiled for traversal depths 3 and 5; an index whose
// top level is at most 3 takes the shallow instance
template <class F>
static void with_top(int top, F &&f) {
    if (top <= 3) f(std::integral_constant<int, 3>{});
    else f(std::integral_constant<int, 5>{});
}

// resident blocks / SM of the two instances of the iteration kernel (register-limited)
template <int ROLE>
static int iteration_occupancy_kind(int kind, int top) {
    static int cache[8][2] = {};  // 0 = not queried yet
    int &c = cache[kind & 7][top <= 3 ? 0 : 1];
    if (c == 0) {
        with_kind(kind, [&](auto k) {
            with_top(top, [&](auto t) {
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, icp_iteration_kernel<decltype(k)::value, decltype(t)::value, ROLE>,
                                                                  ICP_SEARCH_WARPS * 32, 0) != cudaSuccess) {
                    cudaGetLastError();
                    c = 0;
                }
            });
        });
        if (c <= 0) c = -1;
    }
    return c;
}

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

// two launches per iteration: the searching-regime instance, then the certified-regime instance (which also sums and
// solves after a searching launch); the regime is decided on the device, the instance it does not concern returns
// at its first instructions (icp_kernels.cuh)
static void launch_iteration(const cphb_icp *icp, const IcpArgs &a, cudaStream_t s) {
    // plain stream-ordered launches where the host has work between or right after them: step mode, the NCCL
    // all-reduce + finalize, the CPHB_DEBUG_EVENTS event between the two instances
    const bool pdl = !a.defer_finalize && !a.step_mode && !icp->dbg_ev;
    with_kind(icp->prm.estimation, [&](auto k) {
        with_top(icp->index->v.top, [&](auto t) {
            constexpr int KIND = decltype(k)::value, TOP = decltype(t)::value;
            if (pdl) {
                launch_pdl(icp_iteration_kernel<KIND, TOP, 0>, icp->grid_search, ICP_SEARCH_WARPS * 32, s, a);
                launch_pdl(icp_iteration_kernel<KIND, TOP, 1>, icp->grid, ICP_SEARCH_WARPS * 32, s, a);
                return;
            }
            CPHB_LAUNCH((icp_iteration_kernel<KIND, TOP, 0>), icp->grid_search, ICP_SEARCH_WARPS * 32, 0, s, a);
            if (icp->dbg_ev) cudaEventRecord(icp->dbg_ev[3 * a.launch_idx + 1], s);
            CPHB_LAUNCH((icp_iteration_kernel<KIND, TOP, 1>), icp->grid, ICP_SEARCH_WARPS * 32, 0, s, a);
        });
    });
}
static void launch_finalize(const cphb_icp *icp, const IcpArgs &a, cudaStream_t s) {
    with_kind(icp->prm.estimation, [&](auto k) { CPHB_LAUNCH(icp_finalize_kernel<decltype(k)::value>, 1, 32, 0, s, a); });
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
    if (params->shard_world > 1 && (params->shard_rank < 0 || params->shard_rank >= params->shard_world)) {
        cphb_set_error("cphb_icp_create: shard_rank %d outside [0,%d)", params->shard_rank, params->shard_world);
        return CPHB_ERR_INVALID;
    }
    std::unique_ptr<cphb_icp> icp(new cphb_icp());
    icp->prm = *params;
    icp->tgt = *target;
    const unsigned n_full = (unsigned)source->n;
    // The source's Hilbert ordering (bounds, keys, radix sort) does not depend on the target index: it runs on a side
    // stream, concurrently with the index build (both are short chains of small kernels), and joins right before the
    // source is gathered.
    int cur_dev = 0;
    cudaGetDevice(&cur_dev);
    if (!t_side.stream || t_side.device != cur_dev) {  // (a thread that moved to another device gets a new one)
        t_side.device = cur_dev;
        CPHB_CUDA(cudaStreamCreateWithFlags(&t_side.stream, cudaStreamNonBlocking));
        CPHB_CUDA(cudaEventCreateWithFlags(&t_side.fork, cudaEventDisableTiming));
        CPHB_CUDA(cudaEventCreateWithFlags(&t_side.join, cudaEventDisableTiming));
    }
    cphb_arena side;  // the source permutation, allocated on the side stream
    uint32_t *perm_side = nullptr;
    // it goes back to the pool on the side stream, which first waits for s: the gather on s reads it
    scope_exit side_waits{[&] {
        if (!perm_side) return;
        cudaEventRecord(t_side.fork, s);
        cudaStreamWaitEvent(t_side.stream, t_side.fork, 0);
    }};
    int rc = CPHB_OK;
    if (n_full) {
        CPHB_CUDA(cudaEventRecord(t_side.fork, s));
        CPHB_CUDA(cudaStreamWaitEvent(t_side.stream, t_side.fork, 0));
        if (t_source_ready) {  // (host-buffer call: the source upload is still in flight on the copy stream)
            cudaStreamWaitEvent(t_side.stream, t_source_ready, 0);
            t_source_ready = nullptr;
        }
        side.slice(&perm_side, n_full);
        rc = side.alloc(t_side.stream);
        if (!rc) rc = cphb_hilbert_order(source->points, n_full, perm_side, nullptr, 0, t_side.stream);
        if (rc) return rc;
        CPHB_CUDA(cudaEventRecord(t_side.join, t_side.stream));
    }
    rc = cphb_index_create(target->points, target->n, s, &icp->index);
    if (rc) return rc;
    unsigned lo = 0, n = n_full;
    if (params->shard_world > 1) {
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
        auto grid_for = [&](int occ) {
            unsigned per_sm = 9u;
            if (occ > 0 && (unsigned)occ < per_sm) per_sm = (unsigned)occ;
            const unsigned cap = (unsigned)sms * per_sm;
            return want < cap ? want : cap;
        };
        icp->grid_search = grid_for(iteration_occupancy_kind<0>(params->estimation, icp->index->v.top));
        icp->grid = grid_for(iteration_occupancy_kind<1>(params->estimation, icp->index->v.top));
        const unsigned rg = (n_tiles + 63) / 64;
        icp->reduce_grid = rg < 1 ? 1 : (rg > (unsigned)sms ? (unsigned)sms : rg);
        if (icp->reduce_grid > icp->grid) icp->reduce_grid = icp->grid;  // the sum runs on blocks of the ROLE 1 launch
    }
    const bool want_nrm = params->estimation == CPHB_EST_SYMMETRIC && source->normals;
    const bool want_col = params->estimation == CPHB_EST_COLORED_ICP && source->colors;
    const bool want_cov = params->estimation == CPHB_EST_GENERALIZED_ICP && source->covariances;
    // private copies of the target attributes in index order (nothing of the caller's target is retained)
    const size_t nt_pad = (size_t)icp->index->v.n_leaves * CPHB_LEAF, nt_slice = nt_pad ? nt_pad : 1;
    const int est = params->estimation;
    const bool t_nrm = target->normals && (est == CPHB_EST_POINT_TO_PLANE || est == CPHB_EST_SYMMETRIC || est == CPHB_EST_COLORED_ICP);
    const bool t_grad = target->color_gradient && est == CPHB_EST_COLORED_ICP;
    const bool t_cov = target->covariances && est == CPHB_EST_GENERALIZED_ICP;
    const unsigned nf_pad = (unsigned)cphb_align(n_full ? n_full : 1, ICP_BLOCK);
    icp->flag_words = n_pad / 1024 + 1;
    cphb_arena &ar = icp->arena;
    ar.slice(&icp->pristine_xyz, n_pad);
    ar.slice(&icp->work_xyz, n_pad);
    ar.slice(&icp->pristine_nrm, n_pad, want_nrm);
    ar.slice(&icp->work_nrm, n_pad, want_nrm);
    ar.slice(&icp->pristine_cov, 3 * n_pad, want_cov);
    ar.slice(&icp->work_cov, 3 * n_pad, want_cov);
    ar.slice(&icp->src_col, n_pad, want_col);
    ar.slice(&icp->st, 1);
    ar.slice(&icp->partials, 32 * (icp->reduce_grid > icp->grid ? icp->reduce_grid : icp->grid));
    ar.slice(&icp->tix_nrm, nt_slice, t_nrm);
    ar.slice(&icp->tix_grad, nt_slice, t_grad);
    ar.slice(&icp->tix_cov, 3 * nt_slice, t_cov);
    ar.slice(&icp->tile_sums, n_pad);
    ar.slice(&icp->flag_bits, 2 * icp->flag_words);
    ar.slice(&icp->prev, n_pad);
    ar.slice(&icp->corr_index, nf_pad);
    ar.slice(&icp->cmp_counts, (nf_pad + CMP_BLOCK - 1) / CMP_BLOCK + 1);
    ar.slice(&icp->cmp_total, 4);
    rc = ar.alloc(s);
    if (rc) return rc;
    if (!t_cache.in_use) {
        if (!t_cache.h_st) CPHB_CUDA(cudaMallocHost((void **)&t_cache.h_st, sizeof(IcpState)));
        if (!t_cache.ev0) CPHB_CUDA(cudaEventCreate(&t_cache.ev0));
        if (!t_cache.ev1) CPHB_CUDA(cudaEventCreate(&t_cache.ev1));
        t_cache.in_use = true;
        icp->h_st = t_cache.h_st;
        icp->ev0 = t_cache.ev0;
        icp->ev1 = t_cache.ev1;
    } else {  // a second live context on this thread gets its own
        icp->owns_host = true;
        CPHB_CUDA(cudaMallocHost((void **)&icp->h_st, sizeof(IcpState)));
        CPHB_CUDA(cudaEventCreate(&icp->ev0));
        CPHB_CUDA(cudaEventCreate(&icp->ev1));
    }
    if (t_source_ready) {  // (n_full == 0)
        cudaStreamWaitEvent(s, t_source_ready, 0);
        t_source_ready = nullptr;
    }
    if (perm_side) cudaStreamWaitEvent(s, t_side.join, 0);
    CPHB_LAUNCH(gather_source_kernel, n_pad / 256, 256, 0, s, source->points, source->normals, source->colors,
                source->covariances, source->cov_col_major, perm_side, lo, n, n_pad, icp->pristine_xyz, icp->pristine_nrm,
                icp->src_col, icp->pristine_cov);
    if ((t_nrm || t_grad || t_cov) && nt_pad)
        CPHB_LAUNCH(gather_target_kernel, (unsigned)((nt_pad + 255) / 256), 256, 0, s, icp->index->v.pts, nt_pad, target->normals,
                    (est == CPHB_EST_COLORED_ICP) ? target->colors : nullptr, target->color_gradient, target->covariances,
                    target->cov_col_major, icp->tix_nrm, icp->tix_grad, icp->tix_cov);
    CPHB_CUDA(cudaGetLastError());
    *out = icp.release();
    return CPHB_OK;
}

extern "C" void cphb_icp_destroy(cphb_icp *icp) { delete icp; }

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
    a.static_sched = 1;  // config 2 on the H100: 7145-7381 it/s vs 6870 with the dynamic schedule (profiles/h100_tuning_sweep.txt)
    if (const char *e = getenv("CPHB_STATIC_SCHED")) a.static_sched = atoi(e) != 0;
    a.tmax = CPHB_TRANSPOSE_MAX;
}

// the opening of a run or a step: the working copy back to the pristine source, and a fresh state at pose T (U = T) on
// the device
static int reset_state(cphb_icp *icp, const float T[16], int apply_u, cudaStream_t s) {
    CPHB_CUDA(cudaMemsetAsync(icp->flag_bits, 0, sizeof(unsigned) * 2 * icp->flag_words, s));
    CPHB_CUDA(cudaMemsetAsync(icp->prev, 0xff, sizeof(int2) * icp->n_pad, s));  // no warm start at launch 0
    CPHB_CUDA(cudaMemcpyAsync(icp->work_xyz, icp->pristine_xyz, sizeof(float4) * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    if (icp->work_nrm)
        CPHB_CUDA(cudaMemcpyAsync(icp->work_nrm, icp->pristine_nrm, sizeof(float4) * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    if (icp->work_cov)
        CPHB_CUDA(cudaMemcpyAsync(icp->work_cov, icp->pristine_cov, sizeof(float4) * 3 * icp->n_pad, cudaMemcpyDeviceToDevice, s));
    IcpState *h = icp->h_st;
    memset(h, 0, sizeof(*h));
    memcpy(h->T, T, 64);
    memcpy(h->U, T, 64);
    h->apply_u = apply_u;
    CPHB_CUDA(cudaMemcpyAsync(icp->st, h, sizeof(IcpState), cudaMemcpyHostToDevice, s));
    return CPHB_OK;
}

static int compact_correspondences(cphb_icp *icp, int32_t *corr_out, cudaStream_t s) {
    unsigned n = icp->n_full;
    unsigned nb = (n + CMP_BLOCK - 1) / CMP_BLOCK;
    if (nb == 0) nb = 1;
    CPHB_LAUNCH(compact_count_kernel, nb, CMP_BLOCK, 0, s, icp->corr_index, n, icp->cmp_counts);
    cphb_scan_block_counts(icp->cmp_counts, nb, icp->cmp_total, s);
    CPHB_LAUNCH(compact_write_kernel, nb, CMP_BLOCK, 0, s, icp->corr_index, n, icp->cmp_counts, corr_out);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

extern "C" int cphb_icp_run(cphb_icp *icp, const float h_init[16], cphb_comm *comm, cphb_icp_result *h_result,
                            int32_t *corr_out, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!icp || !h_init || !h_result) {
        cphb_set_error("cphb_icp_run: null argument");
        return CPHB_ERR_INVALID;
    }
    int rc = reset_state(icp, h_init, is_identity4(h_init) ? 0 : 1, s);
    if (rc) return rc;
    IcpState *h = icp->h_st;
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
        if (!lib_sharded) {
            // caller-sharded source: global source size by one tiny exchange before the loop
            double *tmp = icp->partials;  // scratch
            double hn = (double)icp->n_src;
            CPHB_CUDA(cudaMemcpyAsync(tmp, &hn, 8, cudaMemcpyHostToDevice, s));
            rc = cphb_comm_allreduce_f64(comm, tmp, 1, s);
            if (rc) return rc;
            CPHB_CUDA(cudaMemcpyAsync(&hn, tmp, 8, cudaMemcpyDeviceToHost, s));
            CPHB_CUDA(cudaStreamSynchronize(s));
            n_total = (unsigned long long)hn;
        }
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
        launch_iteration(icp, a, s);
        if (dbg_events) cudaEventRecord(evs[3 * it + 2], s);
        if (nccl_comm) {
            rc = cphb_nccl_allreduce_f64(nccl_comm, icp->st->local, icp->st->total, 32, s);
            if (rc) return rc;
            launch_finalize(icp, a, s);
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
    int rc = reset_state(icp, h_T, 1, s);
    if (rc) return rc;
    IcpState *h = icp->h_st;
    IcpArgs a;
    fill_args(icp, a);
    a.step_mode = 1;
    a.corr_index = icp->corr_index;
    CPHB_CUDA(cudaMemsetAsync(icp->corr_index, 0xff, sizeof(int32_t) * icp->n_full, s));
    launch_iteration(icp, a, s);
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
    cudaStream_t c = t_up.copy;
    scope_exit all_done{[&] { cudaStreamSynchronize(s); }};  // everything is complete on return, the arena's release included
    // the clouds on the device, in one arena: [tgt points | src points, normals, colors, covariances | tgt normals, colors,
    // covariances, gradient | pairs]
    cphb_cloud ds = *h_source, dt = *h_target;
    int32_t *d_pairs = nullptr;
    cphb_arena arena;
    arena.slice(&dt.points, 3 * nt, h_target->points);
    arena.slice(&ds.points, 3 * ns, h_source->points);
    arena.slice(&ds.normals, 3 * ns, h_source->normals);
    arena.slice(&ds.colors, 3 * ns, h_source->colors);
    arena.slice(&ds.covariances, 9 * ns, h_source->covariances);
    arena.slice(&dt.normals, 3 * nt, h_target->normals);
    arena.slice(&dt.colors, 3 * nt, h_target->colors);
    arena.slice(&dt.covariances, 9 * nt, h_target->covariances);
    arena.slice(&dt.color_gradient, 3 * nt, h_target->color_gradient);
    arena.slice(&d_pairs, 2 * ns, h_corr_out);
    ds.color_gradient = nullptr;
    int rc = arena.alloc(s);
    if (rc) return rc;
    // declared after the arena, so it runs first: no upload may still be reading the caller's buffers, or writing into
    // the arena, when the arena is freed
    scope_exit uploads_done{[&] { cudaStreamSynchronize(c); }};
    CPHB_CUDA(cudaEventRecord(t_up.ev[0], s));            // the arena exists from here on in stream order
    CPHB_CUDA(cudaStreamWaitEvent(c, t_up.ev[0], 0));
    auto up = [&](const float *d, const float *h, size_t floats) {
        return h && floats ? cudaMemcpyAsync((void *)d, h, sizeof(float) * floats, cudaMemcpyHostToDevice, c) : cudaSuccess;
    };
    CPHB_CUDA(up(dt.points, h_target->points, 3 * nt));
    CPHB_CUDA(cudaEventRecord(t_up.ev[1], c));            // target points: all the index build needs
    CPHB_CUDA(up(ds.points, h_source->points, 3 * ns));
    CPHB_CUDA(up(ds.normals, h_source->normals, 3 * ns));
    CPHB_CUDA(up(ds.colors, h_source->colors, 3 * ns));
    CPHB_CUDA(up(ds.covariances, h_source->covariances, 9 * ns));
    CPHB_CUDA(cudaEventRecord(t_up.ev[2], c));            // source: first read by the Hilbert ordering
    CPHB_CUDA(up(dt.normals, h_target->normals, 3 * nt));
    CPHB_CUDA(up(dt.colors, h_target->colors, 3 * nt));
    CPHB_CUDA(up(dt.covariances, h_target->covariances, 9 * nt));
    CPHB_CUDA(up(dt.color_gradient, h_target->color_gradient, 3 * nt));
    CPHB_CUDA(cudaEventRecord(t_up.ev[3], c));            // target attributes: first read by the first iteration
    CPHB_CUDA(cudaStreamWaitEvent(s, t_up.ev[1], 0));
    t_source_ready = t_up.ev[2];
    cphb_icp *icp = nullptr;
    rc = cphb_icp_create(&ds, &dt, params, stream, &icp);
    t_source_ready = nullptr;
    if (rc) return rc;
    cudaStreamWaitEvent(s, t_up.ev[2], 0);            // (already waited inside create; harmless if it returned early)
    cudaStreamWaitEvent(s, t_up.ev[3], 0);
    rc = cphb_icp_run(icp, h_init, comm, h_result, d_pairs, stream);
    if (!rc && h_corr_out && h_result->n_local_correspondences > 0) {
        cudaError_t e = cudaMemcpyAsync(h_corr_out, d_pairs, sizeof(int32_t) * 2 * (size_t)h_result->n_local_correspondences,
                                        cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { cphb_set_error("cphb_registration_icp_host: %s", cudaGetErrorString(e)); rc = CPHB_ERR_CUDA; }
    }
    cphb_icp_destroy(icp);
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
    cphb_scratch sc(s);
    float *Td = nullptr;
    int rc = sc.alloc(&Td, 16);
    if (rc) return rc;
    CPHB_CUDA(cudaMemcpyAsync(Td, h_T, 64, cudaMemcpyHostToDevice, s));
    CPHB_LAUNCH(transform_kernel, (unsigned)((n + 255) / 256), 256, 0, s, points, normals, covariances, cov_col_major, n, Td);
    CPHB_CHECK_LAUNCH();
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
    cphb_arena arena;
    float *Td;
    arena.slice(&a.partials, 32 * (size_t)grid);
    arena.slice(&a.total, 32);
    arena.slice(&a.ticket, 1);
    arena.slice(&Td, 16);
    int rc = arena.alloc(s);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(a.ticket, 0, 4, s));
    // the inputs the estimator needs are present (otherwise the solve leaves the identity)
    const bool have = estimation == CPHB_EST_POINT_TO_PLANE ? target->normals != nullptr
                      : estimation == CPHB_EST_SYMMETRIC    ? target->normals && source->normals
                      : estimation == CPHB_EST_COLORED_ICP  ? target->normals && target->colors && source->colors
                      : estimation == CPHB_EST_GENERALIZED_ICP ? target->covariances && source->covariances
                                                               : true;
    const float dt = params ? params->det_thresh : 1e-6f;
    const unsigned long long nm = source->n;
    with_kind(estimation, [&](auto k) {
        CPHB_LAUNCH(estimate_kernel<decltype(k)::value>, grid, ICP_BLOCK, 0, s, a);
        if (h_T) CPHB_LAUNCH(estimate_solve_kernel<decltype(k)::value>, 1, 32, 0, s, a.total, nm, dt, have, Td);
    });
    if (h_T) CPHB_CUDA(cudaMemcpyAsync(h_T, Td, 64, cudaMemcpyDeviceToHost, s));
    return cphb_read_back(h_S, a.total, sizeof(double) * 32, s, "estimate");
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
    cphb_scratch sc(s);
    if (!corr) {
        n_corr = n_model;
        int32_t *tmp = nullptr;
        const int rc = sc.alloc(&tmp, 2 * (n_model ? n_model : 1));
        if (rc) return rc;
        if (n_model) CPHB_LAUNCH(iota_pairs_kernel, (unsigned)((n_model + 255) / 256), 256, 0, s, tmp, (unsigned)n_model);
        corr = tmp;
    }
    return cphb_compute_transformation(CPHB_EST_POINT_TO_POINT, &src, &tgt, corr, n_corr, nullptr, h_T, stream);
}
