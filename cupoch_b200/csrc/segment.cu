// segment.cu -- PointCloud::SegmentPlane (segmentation.cu:36-267): RANSAC plane segmentation.
//
// The reference repeats per iteration: tabulate n random keys, a full sort_by_key of n pairs, three points to the
// host, a plane built there, then copy_if + reduce over the cloud with host synchronisations.  The hypotheses do not
// depend on the data (iteration t's sample depends only on its seed and the earlier sorts), so here
//   sampling : T x (key kernel + stable CUB radix sort of (key, card)) back to back, no host synchronisation;
//   planes   : one kernel builds the T triangle planes;
//   scoring  : ONE pass over the cloud scores all T planes (seg_score_kernel), then the tile partials are added per
//              hypothesis and the reference's selection rule runs sequentially over t, on the device;
//   final    : one flag pass, the shared compaction (the host learns the inlier count), the refit sums and a one-thread
//              finalize.
//
// Arithmetic (oracle/segment_plane.c restates it; DESIGN.md arithmetic contract):
//   - keys: thrust's random_functor exactly (minstd_rand jump-ahead + uniform_int_distribution computed in double);
//   - triangle plane, fitness, rmse, centroid division and the refit's determinant / normalisation are host code in
//     the reference (no FMA): unfused float32 here, sqrtf and division correctly rounded;
//   - distance |dot3(n, p) + d| (device code in the reference: the contract's dot3);
//   - every sum over points / inliers: tiles of SEG_TILE consecutive elements summed sequentially in double from 0,
//     then the tile sums in tile order, rounded to float once.  The order is part of the answer: the refit's
//     determinant cancels badly for axis-aligned planes.
#include <math.h>

#include "cphb_internal.cuh"
#include "minstd.cuh"

#define SEG_TILE 1024      // summation tile, also the scoring kernel's shared-memory tile (12 KB of points)
#define SEG_KEY_STEPS 16   // key-kernel positions per thread

struct SegState {
    float4 plane;  // best hypothesis, then the refit
    float centroid[3];
    int best;
    float fitness, rmse;
};

__device__ __forceinline__ float seg_dist(float4 pl, float x, float y, float z) {
    return fabsf(__fadd_rn(dot3(pl.x, pl.y, pl.z, x, y, z), pl.w));
}

// ---- sampling ---------------------------------------------------------------
// keys[p] = random_functor(seed, n)(p): the draw after discard(p) is x_{p+1} = a^(p+1) x0 mod m.  Lane l of a warp owns
// positions first + 32 i (coalesced stores): one jump-ahead by a^(first+1) from the table, then steps of a^32.
__global__ void __launch_bounds__(256) seg_keys_kernel(uint32_t x0, uint32_t n, cphb_minstd_pow pw, uint32_t *__restrict__ keys) {
    const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    const size_t first = warp * (32 * SEG_KEY_STEPS) + lane_id();
    if (first >= n) return;
    const uint64_t e = first + 1;
    uint32_t x = cphb_minstd_jump(x0, e, pw);
    const uint32_t a32 = pw.p[5];
    const double span = (double)(n - 1u) + 1.0;  // uniform_real_distribution(0, (n-1) + 1)
#pragma unroll 4
    for (int i = 0; i < SEG_KEY_STEPS; ++i) {
        const size_t p = first + 32 * (size_t)i;
        if (p >= n) break;
        keys[p] = (uint32_t)(int)__dmul_rn(__ddiv_rn((double)(x - 1u), 2147483646.0), span);
        x = cphb_minstd_mulmod(x, a32);
    }
}

__global__ void __launch_bounds__(256) seg_iota_kernel(uint32_t *__restrict__ cards, size_t n) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) cards[i] = (uint32_t)i;
}

__global__ void seg_take_kernel(const uint32_t *__restrict__ cards, int32_t *__restrict__ sample) {
    if (threadIdx.x < 3) sample[threadIdx.x] = (int32_t)cards[threadIdx.x];
}

// ComputeTrianglePlane (:60-74), host code there: unfused float32; zero plane for collinear points
__global__ void __launch_bounds__(128) seg_planes_kernel(const float *__restrict__ pts, const int32_t *__restrict__ samples, int T,
                                                         float4 *__restrict__ planes) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const float *p0 = pts + 3 * (size_t)samples[3 * t], *p1 = pts + 3 * (size_t)samples[3 * t + 1],
                *p2 = pts + 3 * (size_t)samples[3 * t + 2];
    const float e0x = __fsub_rn(p1[0], p0[0]), e0y = __fsub_rn(p1[1], p0[1]), e0z = __fsub_rn(p1[2], p0[2]);
    const float e1x = __fsub_rn(p2[0], p0[0]), e1y = __fsub_rn(p2[1], p0[1]), e1z = __fsub_rn(p2[2], p0[2]);
    float a = __fsub_rn(__fmul_rn(e0y, e1z), __fmul_rn(e0z, e1y));
    float b = __fsub_rn(__fmul_rn(e0z, e1x), __fmul_rn(e0x, e1z));
    float c = __fsub_rn(__fmul_rn(e0x, e1y), __fmul_rn(e0y, e1x));
    const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c)));
    if (norm == 0.f) {
        planes[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    a = __fdiv_rn(a, norm);
    b = __fdiv_rn(b, norm);
    c = __fdiv_rn(c, norm);
    const float d = -__fadd_rn(__fadd_rn(__fmul_rn(a, p0[0]), __fmul_rn(b, p0[1])), __fmul_rn(c, p0[2]));
    planes[t] = make_float4(a, b, c, d);
}

// ---- scoring: every hypothesis in one pass over the cloud --------------------
// Block (tile, chunk of hypotheses): the tile's points are staged in shared memory, one thread per hypothesis walks
// them in index order (broadcast reads, no divergence, no shuffles) keeping an int count and a sequential double sum.
__global__ void __launch_bounds__(256) seg_score_kernel(const float *__restrict__ pts, size_t n, const float4 *__restrict__ planes,
                                                        int T, float thr, int *__restrict__ pcnt, double *__restrict__ psum) {
    __shared__ float s_p[3 * SEG_TILE];
    const size_t tile = blockIdx.x;
    const size_t base = tile * SEG_TILE;
    const int len = (int)min((size_t)SEG_TILE, n - base);
    const float *src = pts + 3 * base;
    for (int i = threadIdx.x; i < 3 * len; i += blockDim.x) s_p[i] = src[i];
    __syncthreads();
    const int h = blockIdx.y * blockDim.x + threadIdx.x;
    if (h >= T) return;
    const float4 pl = planes[h];
    int c = 0;
    double s = 0.0;
#pragma unroll 4
    for (int i = 0; i < len; ++i) {
        const float d = seg_dist(pl, s_p[3 * i], s_p[3 * i + 1], s_p[3 * i + 2]);
        if (d < thr) {
            ++c;
            s = __dadd_rn(s, (double)d);
        }
    }
    pcnt[tile * T + h] = c;
    psum[tile * T + h] = s;
}

// per hypothesis: the tile partials in tile order -> (fitness, "rmse") as EvaluateRANSACBasedOnDistance (:94-128)
__global__ void __launch_bounds__(128) seg_total_kernel(const int *__restrict__ pcnt, const double *__restrict__ psum, size_t n_tiles,
                                                        int T, size_t n, float2 *__restrict__ fr) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= T) return;
    unsigned long long c = 0;
    double s = 0.0;
    for (size_t t = 0; t < n_tiles; ++t) {
        c += (unsigned)pcnt[t * T + h];
        s = __dadd_rn(s, psum[t * T + h]);
    }
    float fit = 0.f, rmse = 0.f;
    if (c) {
        fit = __fdiv_rn((float)c, (float)n);
        rmse = __fdiv_rn((float)s, __fsqrt_rn((float)c));
    }
    fr[h] = make_float2(fit, rmse);
}

// the reference's selection (:237-242), sequentially over t: skipped (zero-plane) iterations do not compete
__global__ void seg_select_kernel(const float4 *__restrict__ planes, const float2 *__restrict__ fr, int T, SegState *st) {
    if (threadIdx.x != 0) return;
    float bf = 0.f, br = 0.f;
    int best = -1;
    for (int t = 0; t < T; ++t) {
        const float4 p = planes[t];
        if (p.x == 0.f && p.y == 0.f && p.z == 0.f && p.w == 0.f) continue;  // isZero(0)
        const float2 r = fr[t];
        if (r.x > bf || (r.x == bf && r.y < br)) {
            bf = r.x;
            br = r.y;
            best = t;
        }
    }
    st->best = best;
    st->fitness = bf;
    st->rmse = br;
    st->plane = best >= 0 ? planes[best] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- final inliers and the refit (GetPlaneFromPoints, :135-185) --------------
__global__ void __launch_bounds__(256) seg_flag_kernel(const float *__restrict__ pts, size_t n, const SegState *__restrict__ st, float thr,
                                                       uint8_t *__restrict__ keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    keep[i] = seg_dist(st->plane, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]) < thr ? 1 : 0;
}

// one thread per tile of the inlier list: pass 0 the coordinate sums, pass 1 the six second moments of p - centroid
// (float32 products, as the reference's device functor forms them)
__global__ void __launch_bounds__(128) seg_refit_partial_kernel(const float *__restrict__ pts, const int32_t *__restrict__ idx, size_t m,
                                                                int pass, const SegState *__restrict__ st, double *__restrict__ partial) {
    const size_t tile = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t base = tile * SEG_TILE;
    if (base >= m) return;
    const size_t end = min(base + SEG_TILE, m);
    double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (pass == 0) {
        for (size_t k = base; k < end; ++k) {
            const float *p = pts + 3 * (size_t)idx[k];
#pragma unroll
            for (int a = 0; a < 3; ++a) s[a] = __dadd_rn(s[a], (double)p[a]);
        }
    } else {
        const float cx = st->centroid[0], cy = st->centroid[1], cz = st->centroid[2];
        for (size_t k = base; k < end; ++k) {
            const float *p = pts + 3 * (size_t)idx[k];
            const float r0 = __fsub_rn(p[0], cx), r1 = __fsub_rn(p[1], cy), r2 = __fsub_rn(p[2], cz);
            const float prod[6] = {__fmul_rn(r0, r0), __fmul_rn(r0, r1), __fmul_rn(r0, r2),
                                   __fmul_rn(r1, r1), __fmul_rn(r1, r2), __fmul_rn(r2, r2)};
#pragma unroll
            for (int j = 0; j < 6; ++j) s[j] = __dadd_rn(s[j], (double)prod[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) partial[6 * tile + j] = s[j];
}

// lane j adds component j over the tiles in order; lane 0 then runs the host arithmetic of the reference
__global__ void __launch_bounds__(32) seg_refit_final_kernel(const double *__restrict__ partial, size_t n_tiles, size_t m, int pass,
                                                             SegState *st) {
    __shared__ float s_v[6];
    const int j = threadIdx.x;
    if (j < (pass == 0 ? 3 : 6)) {
        double s = 0.0;
        for (size_t t = 0; t < n_tiles; ++t) s = __dadd_rn(s, partial[6 * t + j]);
        s_v[j] = (float)s;
    }
    __syncthreads();
    if (j != 0) return;
    if (pass == 0) {  // centroid /= float(inliers.size()); m == 0 gives NaN, unused: the moments are then zero
        for (int a = 0; a < 3; ++a) st->centroid[a] = __fdiv_rn(s_v[a], (float)m);
        return;
    }
    const float *mu = s_v;
    const float det_x = __fsub_rn(__fmul_rn(mu[3], mu[5]), __fmul_rn(mu[4], mu[4]));
    const float det_y = __fsub_rn(__fmul_rn(mu[0], mu[5]), __fmul_rn(mu[2], mu[2]));
    const float det_z = __fsub_rn(__fmul_rn(mu[0], mu[3]), __fmul_rn(mu[1], mu[1]));
    const float u = __fsub_rn(__fmul_rn(mu[2], mu[4]), __fmul_rn(mu[1], mu[5]));
    const float v = __fsub_rn(__fmul_rn(mu[1], mu[4]), __fmul_rn(mu[2], mu[3]));
    const float w = __fsub_rn(__fmul_rn(mu[1], mu[2]), __fmul_rn(mu[4], mu[0]));
    float a, b, c;
    if (det_x > det_y && det_x > det_z) {
        a = det_x; b = u; c = v;
    } else if (det_y > det_z) {
        a = u; b = det_y; c = w;
    } else {
        a = v; b = w; c = det_z;
    }
    const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c)));
    if (norm == 0.f) {
        st->plane = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    a = __fdiv_rn(a, norm);
    b = __fdiv_rn(b, norm);
    c = __fdiv_rn(c, norm);
    const float d = -__fadd_rn(__fadd_rn(__fmul_rn(a, st->centroid[0]), __fmul_rn(b, st->centroid[1])), __fmul_rn(c, st->centroid[2]));
    st->plane = make_float4(a, b, c, d);
}

// ---- the C ABI --------------------------------------------------------------
extern "C" int cphb_segment_plane(const float *points, size_t n, float distance_threshold, int ransac_n, int num_iterations,
                                  const int32_t *h_seeds, float h_plane[4], int32_t *inliers_out, size_t *h_n_out,
                                  int32_t *h_best_iteration, float h_fitness_rmse[2], float h_phase_ms[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!h_plane || !h_n_out) {
        cphb_set_error("cphb_segment_plane: null argument");
        return CPHB_ERR_INVALID;
    }
    h_plane[0] = h_plane[1] = h_plane[2] = h_plane[3] = 0.f;
    *h_n_out = 0;
    if (h_best_iteration) *h_best_iteration = -1;
    if (h_fitness_rmse) h_fitness_rmse[0] = h_fitness_rmse[1] = 0.f;
    if (h_phase_ms) h_phase_ms[0] = h_phase_ms[1] = h_phase_ms[2] = 0.f;
    if (num_iterations < 0 || n > (size_t)INT32_MAX) {
        cphb_set_error("cphb_segment_plane: num_iterations = %d, n = %zu (need num_iterations >= 0, n <= 2^31-1)", num_iterations, n);
        return CPHB_ERR_INVALID;
    }
    if (ransac_n < 3 || n < (size_t)ransac_n) return CPHB_OK;  // :204-212: logged by the caller, zero plane, no inliers
    if (!points || !inliers_out || (num_iterations > 0 && !h_seeds)) {
        cphb_set_error("cphb_segment_plane: null argument");
        return CPHB_ERR_INVALID;
    }
    const int T = num_iterations;
    const size_t n_tiles = (n + SEG_TILE - 1) / SEG_TILE;
    int bits = 1;
    while (((size_t)1 << bits) < n) ++bits;  // keys lie in [0, n)
    cphb_minstd_pow pw;
    cphb_minstd_table(&pw);

    uint32_t *keys = nullptr, *keys_out = nullptr, *cards = nullptr, *cards_alt = nullptr;
    int32_t *samples = nullptr;
    float4 *planes = nullptr;
    float2 *fr = nullptr;
    int *pcnt = nullptr;
    double *psum = nullptr, *partial = nullptr;
    uint8_t *keep = nullptr;
    SegState *st = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    const size_t Tz = T > 0 ? (size_t)T : 1;
    cphb_scratch sc(s);
    int rc = CPHB_OK;
    if (T > 0) {
        rc = sc.alloc(&keys, n);
        if (!rc) rc = sc.alloc(&keys_out, n);
        if (!rc) rc = sc.alloc(&cards, n);
        if (!rc) rc = sc.alloc(&cards_alt, n);
        if (!rc) rc = sc.alloc(&pcnt, n_tiles * Tz);
        if (!rc) rc = sc.alloc(&psum, n_tiles * Tz);
    }
    if (!rc) rc = sc.alloc(&samples, 3 * Tz);
    if (!rc) rc = sc.alloc(&planes, Tz);
    if (!rc) rc = sc.alloc(&fr, Tz);
    if (!rc) rc = sc.alloc(&partial, 6 * n_tiles);
    if (!rc) rc = sc.alloc(&keep, n);
    if (!rc) rc = sc.alloc(&st, 1);
    if (!rc && h_phase_ms) {
        for (int k = 0; k < 4 && !rc; ++k)
            if (cudaEventCreate(&ev[k]) != cudaSuccess) {
                cphb_set_error("cphb_segment_plane: cudaEventCreate failed");
                rc = CPHB_ERR_CUDA;
            }
    }
    if (!rc && ev[0]) cudaEventRecord(ev[0], s);
    if (!rc && T > 0) {
        // sampling: d_cards = 0..n-1 once (:214-216), then T stable sorts; the sample is d_cards[0..2] after each
        CPHB_LAUNCH(seg_iota_kernel, (unsigned)((n + 255) / 256), 256, 0, s, cards, n);
        const size_t key_threads = (n + SEG_KEY_STEPS * 32 - 1) / (SEG_KEY_STEPS * 32) * 32;
        const unsigned key_blocks = (unsigned)((key_threads + 255) / 256);
        for (int t = 0; t < T && !rc; ++t) {
            uint32_t x0 = (uint32_t)h_seeds[t] % CPHB_MINSTD_M;  // the int seed as the engine's uint32_t, mod m, 0 -> 1
            if (x0 == 0) x0 = 1;
            CPHB_LAUNCH(seg_keys_kernel, key_blocks, 256, 0, s, x0, (uint32_t)n, pw, keys);
            rc = cphb_sort_pairs_u32(keys, keys_out, cards, cards_alt, n, bits, s);
            uint32_t *sw = cards;
            cards = cards_alt;
            cards_alt = sw;
            CPHB_LAUNCH(seg_take_kernel, 1, 32, 0, s, cards, samples + 3 * (size_t)t);
        }
        if (!rc && ev[1]) cudaEventRecord(ev[1], s);
        if (!rc) {
            CPHB_LAUNCH(seg_planes_kernel, (unsigned)((T + 127) / 128), 128, 0, s, points, samples, T, planes);
            const int hb = T >= 256 ? 256 : (T + 31) / 32 * 32;
            const dim3 grid((unsigned)n_tiles, (unsigned)((T + hb - 1) / hb));
            CPHB_LAUNCH(seg_score_kernel, grid, hb, 0, s, points, n, planes, T, distance_threshold, pcnt, psum);
            CPHB_LAUNCH(seg_total_kernel, (unsigned)((T + 127) / 128), 128, 0, s, pcnt, psum, n_tiles, T, n, fr);
        }
    } else if (!rc && ev[1]) {
        cudaEventRecord(ev[1], s);
    }
    size_t m = 0;
    if (!rc) {
        CPHB_LAUNCH(seg_select_kernel, 1, 32, 0, s, planes, fr, T, st);
        if (ev[2]) cudaEventRecord(ev[2], s);
        CPHB_LAUNCH(seg_flag_kernel, (unsigned)((n + 255) / 256), 256, 0, s, points, n, st, distance_threshold, keep);
        rc = cphb_compact_flags(keep, n, inliers_out, &m, s);
    }
    if (!rc) {
        const size_t m_tiles = (m + SEG_TILE - 1) / SEG_TILE;
        const unsigned g = (unsigned)(m_tiles ? (m_tiles + 127) / 128 : 1);
        for (int pass = 0; pass < 2; ++pass) {
            CPHB_LAUNCH(seg_refit_partial_kernel, g, 128, 0, s, points, inliers_out, m, pass, st, partial);
            CPHB_LAUNCH(seg_refit_final_kernel, 1, 32, 0, s, partial, m_tiles, m, pass, st);
        }
        if (ev[3]) cudaEventRecord(ev[3], s);
        SegState h;
        rc = cphb_read_back(&h, st, sizeof(h), s, "cphb_segment_plane");
        if (!rc) {
            h_plane[0] = h.plane.x;
            h_plane[1] = h.plane.y;
            h_plane[2] = h.plane.z;
            h_plane[3] = h.plane.w;
            *h_n_out = m;
            if (h_best_iteration) *h_best_iteration = h.best;
            if (h_fitness_rmse) {
                h_fitness_rmse[0] = h.fitness;
                h_fitness_rmse[1] = h.rmse;
            }
            if (h_phase_ms) {
                cudaEventElapsedTime(&h_phase_ms[0], ev[0], ev[1]);
                cudaEventElapsedTime(&h_phase_ms[1], ev[1], ev[2]);
                cudaEventElapsedTime(&h_phase_ms[2], ev[2], ev[3]);
            }
        }
    }
    sc.release();
    cudaStreamSynchronize(s);
    for (int k = 0; k < 4; ++k)
        if (ev[k]) cudaEventDestroy(ev[k]);
    return rc;
}
