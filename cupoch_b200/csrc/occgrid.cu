// occgrid.cu -- geometry::OccupancyGrid (occupancygrid.h, occupancygrid.cu): a dense log-odds grid.  SURVEY 8f rank 2.
//
// The reference builds, per Insert, a buffer of (n_div + 1) * 3 voxel indices PER RAY (Vector3i, 12 B each), removes the
// out-of-range ones, sorts and uniques them (twice: free and occupied), takes a set difference and only then touches the
// grid (occupancygrid.cu:152-184,224-244,462-526).  Here the grid itself deduplicates: one bit per cell and per role
// (occupied / free) is raised with atomicOr while the rays are walked, and the thread that raises a bit FIRST applies the
// cell's single update -- no voxel lists, no sort, no unique, no set difference, and every cell still changes exactly
// once per Insert, by the same amount, whichever thread got there first (the result is deterministic).
//
// Storage: prob_log[res^3] float (NaN = unknown, OccupancyVoxel's default) + 1 bit per cell "grid_index_ was written"
// (SetFreeArea does not write it, occupancygrid.cu:441-446, so extracted voxels of such cells carry (0,0,0) like the
// reference's) instead of the reference's 24-byte voxels (grid index, colour, prob): 4.1 B per cell instead of 24.
#include <float.h>
#include <math.h>
#include <string.h>

#include "cphb_internal.cuh"

struct cphb_occgrid {
    float voxel_size;
    int res;
    float origin[3];
    cphb_occgrid_params prm;
    size_t cells, words;
    float *prob;
    unsigned *occ_bits, *free_bits, *idx_bits;
    unsigned *bounds;  // device u32[6]: min_bound_ xyz, max_bound_ xyz (grid indices)
    unsigned *scratch; // device u32[4]: max ranged distance (float bits), counters
};

__device__ __forceinline__ long long occ_index_of(int x, int y, int z, int res) {  // utility/helper.h:422-424
    return (long long)(x * res * res + y * res + z);
}
__device__ __forceinline__ bool occ_in_range(int x, int y, int z, int res) {  // occupancygrid.cu:173-178
    return !(x < 0 || y < 0 || z < 0 || x >= res || y >= res || z >= res);
}

__global__ void __launch_bounds__(256) occ_fill_kernel(float *prob, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const float nan = __int_as_float(0x7fc00000);
    for (; i < n; i += (size_t)gridDim.x * blockDim.x) prob[i] = nan;
}
__global__ void occ_bounds_init_kernel(unsigned *b, unsigned half) {
    if (threadIdx.x < 6) b[threadIdx.x] = half;
}

// add_occupancy_functor (occupancygrid.cu:246-275) applied by the one thread that owns the cell in this launch
__device__ __forceinline__ void occ_apply(float *prob, unsigned *idx_bits, long long idx, float inc, float cmin, float cmax) {
    float p = prob[idx];
    p = (p != p) ? 0.f : p;
    p = __fadd_rn(p, inc);
    prob[idx] = fminf(fmaxf(p, cmin), cmax);
    atomicOr(&idx_bits[idx >> 5], 1u << (idx & 31));
}
__device__ __forceinline__ void occ_bounds_commit(unsigned *bounds, int lo[3], int hi[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const int l = __reduce_min_sync(CPHB_FULL, lo[a]);
        const int h = __reduce_max_sync(CPHB_FULL, hi[a]);
        if (lane_id() == 0 && l <= h) {  // AddVoxels (:585-592): the u16 casts of the list's extremes
            atomicMin(&bounds[a], (unsigned)(unsigned short)l);
            atomicMax(&bounds[3 + a], (unsigned)(unsigned short)h);
        }
    }
}

// Insert step 1 (occupancygrid.cu:471-489): the point cut at max_range, its hit flag, the largest |component| of
// (ranged point - viewpoint) over the cloud
__global__ void __launch_bounds__(256) occ_range_kernel(const float *__restrict__ pts, size_t n, float vx, float vy, float vz,
                                                        float max_range, float *__restrict__ ranged, unsigned char *__restrict__ hit,
                                                        unsigned *max_bits) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    float m = 0.f;
    if (i < n) {
        const float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        const float v[3] = {vx, vy, vz};
        const float d[3] = {p[0] - vx, p[1] - vy, p[2] - vz};
        const float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
        const bool is_hit = max_range < 0 || dist <= max_range;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float r = is_hit ? p[a] : ((dist == 0) ? v[a] : __fadd_rn(v[a], __fmul_rn(__fdiv_rn(d[a], dist), max_range)));
            ranged[3 * i + a] = r;
            m = fmaxf(m, fabsf(r - v[a]));
        }
        hit[i] = is_hit ? 1 : 0;
    }
    const unsigned mb = __reduce_max_sync(CPHB_FULL, __float_as_uint(m));  // m >= 0: the bit patterns order like the values
    if (lane_id() == 0 && mb) atomicMax(max_bits, mb);
}

__device__ __forceinline__ bool occ_hit_voxel(const float *ranged, size_t i, const float (&o)[3], float vs, int half, int res,
                                              int (&v)[3]) {  // create_occupancy_voxels_functor (:198-217)
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = (int)floorf(__fdiv_rn(ranged[3 * i + a] - o[a], vs)) + half;
    return occ_in_range(v[0], v[1], v[2], res);
}
// Insert step 2: raise the occupied bit of every hit point's voxel
__global__ void __launch_bounds__(256) occ_mark_kernel(const float *__restrict__ ranged, const unsigned char *__restrict__ hit, size_t n,
                                                       float ox, float oy, float oz, float vs, int res, unsigned *occ_bits) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n || !hit[i]) return;
    const float o[3] = {ox, oy, oz};
    int v[3];
    if (!occ_hit_voxel(ranged, i, o, vs, res / 2, res, v)) return;
    const long long idx = occ_index_of(v[0], v[1], v[2], res);
    atomicOr(&occ_bits[idx >> 5], 1u << (idx & 31));
}
// Insert step 3: VoxelTraversal (occupancygrid.cu:57-132) of every ray, with the first boundary on the face of the start
// cell (DESIGN §4 item 27); a cell that is not occupied and whose free bit this thread raises first gets prob_miss_log.
// The end voxel of a ray is never part of its free list (:119-121) unless it is also the start voxel.
__global__ void __launch_bounds__(128) occ_traverse_kernel(const float *__restrict__ ranged, size_t n, float sx, float sy, float sz,
                                                           float ox, float oy, float oz, float vs, int res, int n_buffer,
                                                           const unsigned *__restrict__ occ_bits, unsigned *free_bits, float *prob,
                                                           unsigned *idx_bits, unsigned *bounds, float miss, float cmin, float cmax) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1};
    if (i < n) {
        const int half = res / 2;
        const float start[3] = {sx, sy, sz};  // viewpoint - origin
        const float end[3] = {ranged[3 * i] - ox, ranged[3 * i + 1] - oy, ranged[3 * i + 2] - oz};
        float ray[3] = {end[0] - start[0], end[1] - start[1], end[2] - start[2]};
        const float length = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ray[0], ray[0]), __fmul_rn(ray[1], ray[1])), __fmul_rn(ray[2], ray[2])));
        if (length != 0 && n_buffer > 0) {
            int cur[3], last[3];
            float step[3], tmax[3], tdelta[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                ray[a] = __fdiv_rn(ray[a], length);
                cur[a] = (int)floorf(__fdiv_rn(start[a], vs));
                last[a] = (int)floorf(__fdiv_rn(end[a], vs));
                step[a] = (ray[a] > 0) ? 1.f : ((ray[a] < 0) ? -1.f : 0.f);
                // the face the ray leaves cell cur = [cur vs, (cur + 1) vs) through (DESIGN §4 item 27: the reference's
                // (cur + 0.5 step) vs is half a voxel off it)
                const float boundary = (float)(((double)cur[a] + ((step[a] > 0) ? 1.0 : 0.0)) * (double)vs);
                tmax[a] = (step[a] != 0) ? __fdiv_rn(boundary - start[a], ray[a]) : INFINITY;
                tdelta[a] = (step[a] != 0) ? __fdiv_rn(vs, fabsf(ray[a])) : INFINITY;
            }
            int count = 0;
            for (;;) {
                // the current voxel joins the ray's list
                const int v[3] = {cur[0] + half, cur[1] + half, cur[2] + half};
                if (occ_in_range(v[0], v[1], v[2], res)) {
                    const long long idx = occ_index_of(v[0], v[1], v[2], res);
                    const unsigned bit = 1u << (idx & 31);
                    if (!(__ldg(&occ_bits[idx >> 5]) & bit)) {  // free \ occupied (:516-520)
                        const unsigned old = atomicOr(&free_bits[idx >> 5], bit);
                        if (!(old & bit)) {
                            occ_apply(prob, idx_bits, idx, miss, cmin, cmax);
#pragma unroll
                            for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], v[a]); hi[a] = max(hi[a], v[a]); }
                        }
                    }
                }
                if (++count >= n_buffer) break;
                int ax;
                if (tmax[0] < tmax[1]) ax = (tmax[0] < tmax[2]) ? 0 : 2;
                else ax = (tmax[1] < tmax[2]) ? 1 : 2;
                // (selected by predication: indexing the small arrays dynamically would put them in local memory)
#pragma unroll
                for (int a = 0; a < 3; ++a)
                    if (a == ax) { cur[a] = (int)__fadd_rn((float)cur[a], step[a]); tmax[a] = __fadd_rn(tmax[a], tdelta[a]); }
                if (last[0] == cur[0] && last[1] == cur[1] && last[2] == cur[2]) break;
                if (fminf(fminf(tmax[0], tmax[1]), tmax[2]) > length) break;
            }
        }
    }
    occ_bounds_commit(bounds, lo, hi);
}
// Insert step 4: the thread that LOWERS a cell's occupied bit applies prob_hit_log (also leaves the bitmap clean)
__global__ void __launch_bounds__(256) occ_apply_hit_kernel(const float *__restrict__ ranged, const unsigned char *__restrict__ hit, size_t n,
                                                            float ox, float oy, float oz, float vs, int res, unsigned *occ_bits,
                                                            float *prob, unsigned *idx_bits, unsigned *bounds, float inc, float cmin,
                                                            float cmax) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1};
    if (i < n && hit[i]) {
        const float o[3] = {ox, oy, oz};
        int v[3];
        if (occ_hit_voxel(ranged, i, o, vs, res / 2, res, v)) {
            const long long idx = occ_index_of(v[0], v[1], v[2], res);
            const unsigned bit = 1u << (idx & 31);
            const unsigned old = atomicAnd(&occ_bits[idx >> 5], ~bit);
            if (old & bit) {
                occ_apply(prob, idx_bits, idx, inc, cmin, cmax);
#pragma unroll
                for (int a = 0; a < 3; ++a) { lo[a] = v[a]; hi[a] = v[a]; }
            }
        }
    }
    occ_bounds_commit(bounds, lo, hi);
}

// AddVoxels (occupancygrid.cu:579-600): the list may name a voxel several times; every occurrence adds its increment
// (one atomic compare-and-swap per occurrence, so the clamped result is that of the sequential loop whatever the order)
__global__ void __launch_bounds__(256) occ_add_voxels_kernel(const int32_t *__restrict__ vox, size_t n, int res, float *prob,
                                                             unsigned *idx_bits, unsigned *bounds, float inc, float cmin, float cmax) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1};
    if (i < n) {
        const int v[3] = {vox[3 * i], vox[3 * i + 1], vox[3 * i + 2]};
        const long long idx = occ_index_of(v[0], v[1], v[2], res);
        unsigned *w = reinterpret_cast<unsigned *>(prob + idx);
        unsigned old = *w, assumed;
        do {
            assumed = old;
            float p = __uint_as_float(assumed);
            p = (p != p) ? 0.f : p;
            p = fminf(fmaxf(__fadd_rn(p, inc), cmin), cmax);
            old = atomicCAS(w, assumed, __float_as_uint(p));
        } while (old != assumed);
        atomicOr(&idx_bits[idx >> 5], 1u << (idx & 31));
#pragma unroll
        for (int a = 0; a < 3; ++a) { lo[a] = v[a]; hi[a] = v[a]; }
    }
    occ_bounds_commit(bounds, lo, hi);
}

// SetFreeArea (occupancygrid.cu:415-460): box cells get + prob_miss_log, no clamping, grid_index_ untouched
__global__ void __launch_bounds__(256) occ_free_area_kernel(float *prob, int res, int x0, int y0, int z0, int dx, int dy, int dz, float miss) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= (size_t)dx * dy * dz) return;
    const int x = (int)(i / ((size_t)dy * dz)), yz = (int)(i % ((size_t)dy * dz));
    const long long idx = occ_index_of(x0 + x, y0 + yz / dz, z0 + yz % dz, res);
    float p = prob[idx];
    p = (p != p) ? 0.f : p;
    prob[idx] = __fadd_rn(p, miss);
}

// ExtractBoundVoxels (occupancygrid.cu:358-408): predicate over the bound box, box order (x slowest)
__global__ void __launch_bounds__(256) occ_extract_flag_kernel(const float *__restrict__ prob, int res, int x0, int y0, int z0, int dx, int dy,
                                                               int dz, float thres, int which, unsigned char *keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= (size_t)dx * dy * dz) return;
    const int x = (int)(i / ((size_t)dy * dz)), yz = (int)(i % ((size_t)dy * dz));
    const float p = prob[occ_index_of(x0 + x, y0 + yz / dz, z0 + yz % dz, res)];
    keep[i] = cphb_occ_keep(p, thres, which) ? 1 : 0;
}
__global__ void __launch_bounds__(256) occ_extract_write_kernel(const float *__restrict__ prob, const unsigned *__restrict__ idx_bits, int res,
                                                                int x0, int y0, int z0, int dy, int dz, const int32_t *__restrict__ sel, size_t m,
                                                                int32_t *out_index, float *out_prob) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k >= m) return;
    const size_t i = (size_t)sel[k];
    const int x = x0 + (int)(i / ((size_t)dy * dz)), yz = (int)(i % ((size_t)dy * dz));
    const int y = y0 + yz / dz, z = z0 + yz % dz;
    const long long idx = occ_index_of(x, y, z, res);
    const bool w = (idx_bits[idx >> 5] >> (idx & 31)) & 1u;
    if (out_index) { out_index[3 * k] = w ? x : 0; out_index[3 * k + 1] = w ? y : 0; out_index[3 * k + 2] = w ? z : 0; }
    if (out_prob) out_prob[k] = prob[idx];
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
extern "C" void cphb_occgrid_default_params(cphb_occgrid_params *p) {  // occupancygrid.h:139-143
    if (!p) return;
    p->clamping_thres_min = -2.0f;
    p->clamping_thres_max = 3.5f;
    p->prob_hit_log = 0.85f;
    p->prob_miss_log = -0.4f;
    p->occ_prob_thres_log = 0.0f;
}

static void occ_reset(cphb_occgrid *g, cudaStream_t s) {
    CPHB_LAUNCH(occ_fill_kernel, CPHB_SMS * 8, 256, 0, s, g->prob, g->cells);
    cudaMemsetAsync(g->occ_bits, 0, sizeof(unsigned) * 3 * g->words + 64, s);  // occ | free | idx bitmaps + scratch (contiguous)
    CPHB_LAUNCH(occ_bounds_init_kernel, 1, 32, 0, s, g->bounds, (unsigned)(g->res / 2));
}

extern "C" int cphb_occgrid_create(float voxel_size, int resolution, const float origin[3], void *stream, cphb_occgrid **out) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!out || resolution < 2 || resolution > 1290) {  // res^3 must fit the reference's int index (helper.h:422-424)
        cphb_set_error("cphb_occgrid_create: resolution %d outside [2, 1290]", resolution);
        return CPHB_ERR_INVALID;
    }
    cphb_occgrid *g = new cphb_occgrid();
    memset(g, 0, sizeof(*g));
    g->voxel_size = voxel_size;
    g->res = resolution;
    for (int a = 0; a < 3; ++a) g->origin[a] = origin ? origin[a] : 0.f;
    cphb_occgrid_default_params(&g->prm);
    g->cells = (size_t)resolution * resolution * resolution;
    g->words = (g->cells + 31) / 32;
    int rc = cphb_alloc_async((void **)&g->prob, sizeof(float) * g->cells, s);
    if (!rc) rc = cphb_alloc_async((void **)&g->occ_bits, sizeof(unsigned) * 3 * g->words + 64, s);
    if (rc) { cphb_free_async(g->prob, s); delete g; return rc; }
    g->free_bits = g->occ_bits + g->words;
    g->idx_bits = g->free_bits + g->words;
    g->scratch = g->idx_bits + g->words;  // 16 u32: [0..5] bounds, [8] max distance bits
    g->bounds = g->scratch;
    occ_reset(g, s);
    CPHB_CHECK_LAUNCH();
    *out = g;
    return CPHB_OK;
}
extern "C" void cphb_occgrid_destroy(cphb_occgrid *g) {
    if (!g) return;
    cudaFreeAsync(g->prob, 0);
    cudaFreeAsync(g->occ_bits, 0);
    delete g;
}
extern "C" int cphb_occgrid_clear(cphb_occgrid *g, void *stream) {  // OccupancyGrid::Clear (occupancygrid.cu:310-315)
    if (!g) { cphb_set_error("cphb_occgrid_clear: null grid"); return CPHB_ERR_INVALID; }
    occ_reset(g, (cudaStream_t)stream);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}
extern "C" int cphb_occgrid_set_params(cphb_occgrid *g, const cphb_occgrid_params *p) {
    if (!g || !p) { cphb_set_error("cphb_occgrid_set_params: null argument"); return CPHB_ERR_INVALID; }
    g->prm = *p;
    return CPHB_OK;
}
extern "C" int cphb_occgrid_get_params(const cphb_occgrid *g, cphb_occgrid_params *p) {
    if (!g || !p) { cphb_set_error("cphb_occgrid_get_params: null argument"); return CPHB_ERR_INVALID; }
    *p = g->prm;
    return CPHB_OK;
}
void cphb_occgrid_geometry(const cphb_occgrid *g, float *voxel_size, float origin[3]) {
    *voxel_size = g->voxel_size;
    for (int a = 0; a < 3; ++a) origin[a] = g->origin[a];
}
void cphb_occgrid_view_of(const cphb_occgrid *g, cphb_occgrid_view *v) {
    v->prob = g->prob;
    v->bounds = g->bounds;
    v->res = g->res;
    v->thres = g->prm.occ_prob_thres_log;
}
extern "C" int cphb_occgrid_set_geometry(cphb_occgrid *g, float voxel_size, const float origin[3]) {
    if (!g) { cphb_set_error("cphb_occgrid_set_geometry: null grid"); return CPHB_ERR_INVALID; }
    g->voxel_size = voxel_size;  // the reference exposes voxel_size_ / origin_ as plain members (its tests assign them)
    if (origin) for (int a = 0; a < 3; ++a) g->origin[a] = origin[a];
    return CPHB_OK;
}
extern "C" const float *cphb_occgrid_data(const cphb_occgrid *g) { return g ? g->prob : nullptr; }
extern "C" int cphb_occgrid_resolution(const cphb_occgrid *g) { return g ? g->res : 0; }

extern "C" int cphb_occgrid_insert(cphb_occgrid *g, const float *points, size_t n, const float viewpoint[3], float max_range,
                                   void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !viewpoint || (n && !points)) { cphb_set_error("cphb_occgrid_insert: null argument"); return CPHB_ERR_INVALID; }
    if (n == 0) return CPHB_OK;  // occupancygrid.cu:465
    cphb_scratch sc(s);
    float *ranged = nullptr;
    unsigned char *hit = nullptr;
    int rc = sc.alloc(&ranged, 3 * n);
    if (!rc) rc = sc.alloc(&hit, n);
    if (rc) return rc;
    unsigned *max_bits = g->scratch + 8;
    CPHB_CUDA(cudaMemsetAsync(max_bits, 0, 4, s));
    const unsigned grid = (unsigned)((n + 255) / 256);
    CPHB_LAUNCH(occ_range_kernel, grid, 256, 0, s, points, n, viewpoint[0], viewpoint[1], viewpoint[2], max_range, ranged, hit, max_bits);
    unsigned h_bits = 0;
    rc = cphb_read_back(&h_bits, max_bits, 4, s, "cphb_occgrid_insert");  // the reference reads max_element back too (:490-492)
    if (rc) return rc;
    float max_dist;
    memcpy(&max_dist, &h_bits, 4);
    const int n_div = (int)ceilf(max_dist / g->voxel_size);
    const float *o = g->origin;
    CPHB_LAUNCH(occ_mark_kernel, grid, 256, 0, s, ranged, hit, n, o[0], o[1], o[2], g->voxel_size, g->res, g->occ_bits);
    if (n_div > 0) {
        const int n_buffer = (n_div + 1) * 3;  // ComputeFreeVoxels(.., n_div + 1, ..) -> n_div * 3 entries per ray (:161-166)
        CPHB_LAUNCH(occ_traverse_kernel, (unsigned)((n + 127) / 128), 128, 0, s, ranged, n, viewpoint[0] - o[0], viewpoint[1] - o[1],
                    viewpoint[2] - o[2], o[0], o[1], o[2], g->voxel_size, g->res, n_buffer, g->occ_bits, g->free_bits, g->prob, g->idx_bits,
                    g->bounds, g->prm.prob_miss_log, g->prm.clamping_thres_min, g->prm.clamping_thres_max);
        CPHB_CUDA(cudaMemsetAsync(g->free_bits, 0, sizeof(unsigned) * g->words, s));
    }
    CPHB_LAUNCH(occ_apply_hit_kernel, grid, 256, 0, s, ranged, hit, n, o[0], o[1], o[2], g->voxel_size, g->res, g->occ_bits, g->prob,
                g->idx_bits, g->bounds, g->prm.prob_hit_log, g->prm.clamping_thres_min, g->prm.clamping_thres_max);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

extern "C" int cphb_occgrid_add_voxels(cphb_occgrid *g, const int32_t *voxels, size_t n, int occupied, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || (n && !voxels)) { cphb_set_error("cphb_occgrid_add_voxels: null argument"); return CPHB_ERR_INVALID; }
    if (n == 0) return CPHB_OK;
    CPHB_LAUNCH(occ_add_voxels_kernel, (unsigned)((n + 255) / 256), 256, 0, s, voxels, n, g->res, g->prob, g->idx_bits, g->bounds,
                occupied ? g->prm.prob_hit_log : g->prm.prob_miss_log, g->prm.clamping_thres_min, g->prm.clamping_thres_max);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// OccupancyGrid::AddVoxel (occupancygrid.cu:554-577): one voxel from the host, range-checked on its LINEAR index
extern "C" int cphb_occgrid_add_voxel(cphb_occgrid *g, const int32_t voxel[3], int occupied, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !voxel) { cphb_set_error("cphb_occgrid_add_voxel: null argument"); return CPHB_ERR_INVALID; }
    const long long idx = (long long)voxel[0] * g->res * g->res + (long long)voxel[1] * g->res + voxel[2];
    if (idx < 0 || idx >= (long long)g->cells || voxel[0] < 0 || voxel[1] < 0 || voxel[2] < 0 || voxel[0] >= g->res ||
        voxel[1] >= g->res || voxel[2] >= g->res) {
        cphb_set_error("[OccupancyGrid] a provided voxel is not in the occupancy grid range.");
        return CPHB_ERR_INVALID;
    }
    cphb_scratch sc(s);
    int32_t *d = nullptr;
    int rc = sc.alloc(&d, 4);
    if (rc) return rc;
    CPHB_CUDA(cudaMemcpyAsync(d, voxel, 12, cudaMemcpyHostToDevice, s));
    rc = cphb_occgrid_add_voxels(g, d, 1, occupied, stream);
    CPHB_CUDA(cudaStreamSynchronize(s));  // (the host array may go out of scope)
    return rc;
}

static int occ_read_bounds(const cphb_occgrid *g, int lo[3], int hi[3], cudaStream_t s) {
    unsigned h[6];
    CPHB_CUDA(cudaMemcpyAsync(h, g->bounds, sizeof(h), cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    for (int a = 0; a < 3; ++a) { lo[a] = (int)h[a]; hi[a] = (int)h[3 + a]; }
    return CPHB_OK;
}
extern "C" int cphb_occgrid_bounds(const cphb_occgrid *g, int32_t h_min[3], int32_t h_max[3], void *stream) {
    if (!g || !h_min || !h_max) { cphb_set_error("cphb_occgrid_bounds: null argument"); return CPHB_ERR_INVALID; }
    int lo[3], hi[3];
    int rc = occ_read_bounds(g, lo, hi, (cudaStream_t)stream);
    if (rc) return rc;
    for (int a = 0; a < 3; ++a) { h_min[a] = lo[a]; h_max[a] = hi[a]; }
    return CPHB_OK;
}

extern "C" int cphb_occgrid_set_free_area(cphb_occgrid *g, const float min_bound[3], const float max_bound[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !min_bound || !max_bound) { cphb_set_error("cphb_occgrid_set_free_area: null argument"); return CPHB_ERR_INVALID; }
    const int half = g->res / 2;
    int lo[3], hi[3];
    unsigned h[6];
    for (int a = 0; a < 3; ++a) {
        const int imin = (int)floorf((min_bound[a] - g->origin[a]) / g->voxel_size) + half;
        const int imax = (int)floorf((max_bound[a] - g->origin[a]) / g->voxel_size) + half;
        lo[a] = imin > 0 ? imin : 0;
        hi[a] = imax < g->res - 1 ? imax : g->res - 1;
        h[a] = (unsigned)(unsigned short)lo[a];
        h[3 + a] = (unsigned)(unsigned short)hi[a];
    }
    CPHB_CUDA(cudaMemcpyAsync(g->bounds, h, sizeof(h), cudaMemcpyHostToDevice, s));  // REPLACES the bounds (:429-436)
    CPHB_CUDA(cudaStreamSynchronize(s));
    if (hi[0] < lo[0] || hi[1] < lo[1] || hi[2] < lo[2]) return CPHB_OK;
    const int dx = hi[0] - lo[0] + 1, dy = hi[1] - lo[1] + 1, dz = hi[2] - lo[2] + 1;
    const size_t m = (size_t)dx * dy * dz;
    CPHB_LAUNCH(occ_free_area_kernel, (unsigned)((m + 255) / 256), 256, 0, s, g->prob, g->res, lo[0], lo[1], lo[2], dx, dy, dz,
                g->prm.prob_miss_log);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// which: 0 known, 1 free, 2 occupied.  out_index [capacity][3] / out_prob [capacity] (device, either may be null);
// *h_count receives the number of voxels that satisfy the predicate (call with capacity 0 to size the outputs).
extern "C" int cphb_occgrid_extract(const cphb_occgrid *g, int which, int32_t *out_index, float *out_prob, size_t capacity,
                                    size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !h_count || which < 0 || which > 2) { cphb_set_error("cphb_occgrid_extract: invalid argument"); return CPHB_ERR_INVALID; }
    int lo[3], hi[3];
    int rc = occ_read_bounds(g, lo, hi, s);
    if (rc) return rc;
    *h_count = 0;
    if (hi[0] < lo[0] || hi[1] < lo[1] || hi[2] < lo[2]) return CPHB_OK;
    const int dx = hi[0] - lo[0] + 1, dy = hi[1] - lo[1] + 1, dz = hi[2] - lo[2] + 1;
    const size_t m = (size_t)dx * dy * dz;
    cphb_scratch sc(s);
    unsigned char *keep = nullptr;
    int32_t *sel = nullptr;
    rc = sc.alloc(&keep, m);
    if (!rc) rc = sc.alloc(&sel, m);
    if (rc) return rc;
    CPHB_LAUNCH(occ_extract_flag_kernel, (unsigned)((m + 255) / 256), 256, 0, s, g->prob, g->res, lo[0], lo[1], lo[2], dx, dy, dz,
                g->prm.occ_prob_thres_log, which, keep);
    size_t cnt = 0;
    rc = cphb_compact_flags(keep, m, sel, &cnt, s);
    if (rc) return rc;
    *h_count = cnt;
    const size_t w = cnt < capacity ? cnt : capacity;
    if (w && (out_index || out_prob))
        CPHB_LAUNCH(occ_extract_write_kernel, (unsigned)((w + 255) / 256), 256, 0, s, g->prob, g->idx_bits, g->res, lo[0], lo[1], lo[2], dy,
                    dz, sel, w, out_index, out_prob);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// DenseGrid::GetVoxelIndex + OccupancyGrid::GetVoxel (densegrid.inl:137-146, occupancygrid.cu:351-356): *h_known = the cell
// exists and is not NaN; *h_prob_log its value (NaN when unknown); h_grid_index the stored grid_index_.  Returns
// CPHB_OK also for points outside the grid (known = 0), like the reference's (false, OccupancyVoxel()).
extern "C" int cphb_occgrid_get_voxel(const cphb_occgrid *g, const float point[3], int *h_known, float *h_prob_log,
                                      int32_t h_grid_index[3], void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !point || !h_known) { cphb_set_error("cphb_occgrid_get_voxel: null argument"); return CPHB_ERR_INVALID; }
    const int half = g->res / 2;
    int v[3];
    for (int a = 0; a < 3; ++a) v[a] = (int)floorf((point[a] - g->origin[a]) / g->voxel_size) + half;
    const int idx = v[0] * g->res * g->res + v[1] * g->res + v[2];  // (int arithmetic and linear-only check as in the reference)
    *h_known = 0;
    if (h_prob_log) *h_prob_log = NAN;
    if (h_grid_index) h_grid_index[0] = h_grid_index[1] = h_grid_index[2] = 0;
    if (idx < 0 || (size_t)idx >= g->cells) return CPHB_OK;
    float p;
    unsigned w;
    CPHB_CUDA(cudaMemcpyAsync(&p, g->prob + idx, 4, cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaMemcpyAsync(&w, g->idx_bits + (idx >> 5), 4, cudaMemcpyDeviceToHost, s));
    CPHB_CUDA(cudaStreamSynchronize(s));
    *h_known = !(p != p);
    if (h_prob_log) *h_prob_log = p;
    if (h_grid_index && ((w >> (idx & 31)) & 1u)) {
        h_grid_index[0] = idx / (g->res * g->res);
        h_grid_index[1] = (idx / g->res) % g->res;
        h_grid_index[2] = idx % g->res;
    }
    return CPHB_OK;
}
