// edt.cu -- geometry::DistanceTransform (distancetransform.h, distancetransform.cu): an exact Euclidean distance field
// over a dense resolution^3 grid.  SURVEY 8f rank 8.
//
// Each cell stores its nearest site (the Voronoi site) and the distance to it.  The reference runs PBA-style passes as
// thrust functors over 12-byte structs, one thread per column with uncoalesced loads, and keeps two full grids of
// 24 B per cell.  Here a compute is a fixed sequence of launches whatever the resolution or the site count:
//   stamp    the sites become one bit per cell (duplicates collapse; sites outside the grid are dropped);
//   sweep z  one warp per (x, y) line: the nearest site of the line at or below / at or above each cell from ballots
//            and shuffles -- the smaller z wins a tie;
//   sweep y  one thread per (x, z) line, threads of a warp on consecutive z (every load and store is coalesced): the
//            lower envelope of the line's candidates (x, y', z*(y')) under (y - y')^2 + (z* - z)^2, in exact integers;
//   sweep x  the same over (., y, z) lines with (y* - y)^2 + (z* - z)^2, fused with the distance.
// In every envelope the earlier candidate (the smaller coordinate along the line) wins a tie, so z, then y, then x
// yields the lexicographically smallest of the equidistant sites (DESIGN.md, parity hazard 13).
//
// Storage (DESIGN.md section 3): nearest u32[res^3] (x << 20 | y << 10 | z, bit 30 = NotSite) + distance f32[res^3],
// 8 B per cell.  A compute borrows the distance array for the site bitmap and takes u32[res^3] of scratch for the
// envelope stacks, which live at the line's own cells; nothing is held in per-thread arrays.
//
// Arithmetic: every squared distance is an integer below 3 * 1023^2 < 2^22 and every envelope numerator is below 2^23,
// so 32-bit integers are exact and (float)d2 is exact; distance = __fsqrt_rn((float)d2) * voxel_size.
#include <float.h>
#include <math.h>
#include <string.h>

#include "cphb_internal.cuh"

#define EDT_MAX_RES 1024
#define EDT_NOT_SITE (1u << 30) /* DistanceVoxel::NotSite; also "no candidate" between the sweeps */
#define EDT_PREFETCH 4

struct cphb_dt {
    float voxel_size;
    int res;
    float origin[3];
    size_t cells;
    uint32_t *nearest;
    float *dist;
};

__host__ __device__ __forceinline__ uint32_t edt_pack(int x, int y, int z) {
    return ((uint32_t)x << 20) | ((uint32_t)y << 10) | (uint32_t)z;
}
__device__ __forceinline__ int edt_cx(uint32_t p) { return (int)((p >> 20) & 1023u); }
__device__ __forceinline__ int edt_cy(uint32_t p) { return (int)((p >> 10) & 1023u); }
__device__ __forceinline__ int edt_cz(uint32_t p) { return (int)(p & 1023u); }

// default voxels (nearest (0,0,0), NotSite, distance 0) on [from, n)
__global__ void __launch_bounds__(256) edt_fill_kernel(uint32_t *nearest, float *dist, size_t from, size_t n) {
    for (size_t i = from + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        nearest[i] = EDT_NOT_SITE;
        dist[i] = 0.f;
    }
}

// Stamp grid cells ([n][3] int32).  map != 0: they are VoxelGrid keys, mapped as compute_obstacle_cells_functor does
// (distancetransform.cu:254-260): floor(((k * vs + o_vg) - o_dt) / vs) + res / 2, each operation rounded on its own.
__global__ void __launch_bounds__(256) edt_stamp_kernel(const int32_t *__restrict__ cells, size_t n, int res, int map, float vs,
                                                         float gx, float gy, float gz, float ox, float oy, float oz,
                                                         unsigned *bits) {
    const float og[3] = {gx, gy, gz}, od[3] = {ox, oy, oz};
    const int half = res / 2;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        int c[3];
        bool in = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int k = cells[3 * i + a];
            if (map) {
                const float f = floorf(__fdiv_rn(__fsub_rn(__fadd_rn(__fmul_rn((float)k, vs), og[a]), od[a]), vs));
                in = in && f >= (float)-half && f < (float)(res - half);  // (also false for NaN)
                c[a] = in ? (int)f + half : 0;
            } else {
                in = in && k >= 0 && k < res;
                c[a] = k;
            }
        }
        if (!in) continue;
        const size_t idx = ((size_t)c[0] * res + c[1]) * res + c[2];
        atomicOr(&bits[idx >> 5], 1u << (idx & 31));
    }
}

// Stamp the occupied cells of an OccupancyGrid's dense log-odds array: !isnan(p) && p > thres.  Each warp writes whole
// bitmap words, so no clear is needed.
__global__ void __launch_bounds__(256) edt_stamp_occ_kernel(const float *__restrict__ prob, size_t cells, float thres, unsigned *bits) {
    const size_t words = (cells + 31) / 32;
    for (size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; w < words; w += ((size_t)gridDim.x * blockDim.x) >> 5) {
        const size_t i = w * 32 + lane_id();
        const float p = i < cells ? prob[i] : 0.f;
        const unsigned m = __ballot_sync(CPHB_FULL, i < cells && !(p != p) && p > thres);
        if (lane_id() == 0) bits[w] = m;
    }
}

// Sweep z: one warp per (x, y) line.  Lane c first keeps the site mask of chunk c (z in [32c, 32c + 32)), then the
// warp scans the chunks' highest / lowest sites to carry the nearest site below / above each chunk.
__global__ void __launch_bounds__(256) edt_sweep_z_kernel(const unsigned *__restrict__ bits, int res, uint32_t *__restrict__ nearest) {
    const size_t line = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    if (line >= (size_t)res * res) return;  // warp-uniform
    const int lane = lane_id();
    const int x = (int)(line / res), y = (int)(line % res);
    const size_t base = line * res;
    const int chunks = (res + 31) >> 5;
    unsigned mine = 0;
    for (int c = 0; c < chunks; ++c) {
        const int z = c * 32 + lane;
        bool site = false;
        if (z < res) {
            const size_t b = base + z;
            site = (__ldg(&bits[b >> 5]) >> (b & 31)) & 1u;
        }
        const unsigned m = __ballot_sync(CPHB_FULL, site);
        if (lane == c) mine = m;
    }
    const int none_hi = -1, none_lo = 1 << 20;
    int hi = mine ? lane * 32 + 31 - __clz(mine) : none_hi;  // highest site of chunk `lane`
    int lo = mine ? lane * 32 + __ffs(mine) - 1 : none_lo;   // lowest
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {  // inclusive prefix max of hi, inclusive suffix min of lo
        const int h = __shfl_up_sync(CPHB_FULL, hi, d), l = __shfl_down_sync(CPHB_FULL, lo, d);
        if (lane >= d) hi = max(hi, h);
        if (lane + d < 32) lo = min(lo, l);
    }
    int below = __shfl_up_sync(CPHB_FULL, hi, 1), above = __shfl_down_sync(CPHB_FULL, lo, 1);
    if (lane == 0) below = none_hi;
    if (lane == 31) above = none_lo;
    for (int c = 0; c < chunks; ++c) {
        const unsigned m = __shfl_sync(CPHB_FULL, mine, c);
        const int carry_lo = __shfl_sync(CPHB_FULL, below, c), carry_hi = __shfl_sync(CPHB_FULL, above, c);
        const int z = c * 32 + lane;
        const unsigned at_or_below = m & (0xffffffffu >> (31 - lane)), at_or_above = m & (0xffffffffu << lane);
        const int prev = at_or_below ? c * 32 + 31 - __clz(at_or_below) : carry_lo;
        const int next = at_or_above ? c * 32 + __ffs(at_or_above) - 1 : carry_hi;
        uint32_t v = EDT_NOT_SITE;
        if (prev >= 0 && (next >= none_lo || z - prev <= next - z)) v = edt_pack(x, y, prev);
        else if (next < none_lo) v = edt_pack(x, y, next);
        if (z < res) nearest[base + z] = v;
    }
}

// Sweeps y (AXIS 1, lines (x, ., z)) and x (AXIS 0, lines (., y, z)).  A candidate at line position q is the packed
// site found by the previous sweep; F is its squared distance to the line in the two axes already swept, and
// f(t) = (t - q)^2 + F its squared distance to the cell at position t.  first_win(a, b) is the first position at
// which the later candidate b is strictly nearer than a (a wins the tie before it).
template <int AXIS>
struct EdtLine {
    int a, z;  // the line's fixed coordinates: AXIS 1: x = a; AXIS 0: y = a
    __device__ __forceinline__ int q(uint32_t p) const { return AXIS == 1 ? edt_cy(p) : edt_cx(p); }
    __device__ __forceinline__ int F(uint32_t p) const {
        const int dz = edt_cz(p) - z;
        if (AXIS == 1) return dz * dz;
        const int dy = edt_cy(p) - a;
        return dy * dy + dz * dz;
    }
    __device__ __forceinline__ int f(uint32_t p, int t) const { const int d = t - q(p); return d * d + F(p); }
    __device__ __forceinline__ int first_win(uint32_t pa, uint32_t pb) const {
        const int qa = q(pa), qb = q(pb);
        const int num = F(pb) - F(pa) + qb * qb - qa * qa, den = 2 * (qb - qa);  // den > 0
        const int fl = num >= 0 ? num / den : -((-num + den - 1) / den);
        return fl + 1;
    }
};

template <int AXIS>
__global__ void __launch_bounds__(128) edt_sweep_kernel(uint32_t *nearest, uint32_t *stack, float *dist, int res, float vs,
                                                        int with_distance) {
    const size_t line = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (line >= (size_t)res * res) return;
    EdtLine<AXIS> L;
    L.a = (int)(line / res);
    L.z = (int)(line % res);
    const size_t rr = (size_t)res * res;
    const size_t base = AXIS == 1 ? (size_t)L.a * rr + L.z : (size_t)L.a * res + L.z;
    const size_t step = AXIS == 1 ? (size_t)res : rr;

    // lower envelope: stack[0 .. k) at the line's own cells, top and below it also in registers, st = top's first cell
    int k = 0, st = 0;
    uint32_t top = 0, below = 0;
    for (int t0 = 0; t0 < res; t0 += EDT_PREFETCH) {
        uint32_t v[EDT_PREFETCH];
#pragma unroll
        for (int u = 0; u < EDT_PREFETCH; ++u) v[u] = (t0 + u < res) ? nearest[base + (size_t)(t0 + u) * step] : EDT_NOT_SITE;
#pragma unroll
        for (int u = 0; u < EDT_PREFETCH; ++u) {
            const uint32_t c = v[u];
            if (c & EDT_NOT_SITE) continue;
            int s = 0;
            while (k > 0) {
                s = L.first_win(top, c);
                if (s > st) break;
                --k;  // c is nearer than top wherever top was nearest: top never wins
                top = below;
                if (k >= 2) below = stack[base + (size_t)(k - 2) * step];
                st = k >= 2 ? L.first_win(below, top) : 0;
                s = 0;
            }
            if (k > 0 && s >= res) continue;  // c never wins inside the grid
            stack[base + (size_t)k * step] = c;
            ++k;
            below = top;
            top = c;
            st = s;
        }
    }
    // the envelope read back from the last cell down: the nearest candidate moves to earlier stack entries only
    int j = k - 1;
    uint32_t cur = top, prv = below;
    for (int t = res - 1; t >= 0; --t) {
        const size_t id = base + (size_t)t * step;
        if (k == 0) {  // no site on the line: for AXIS 0 none in the whole grid
            nearest[id] = EDT_NOT_SITE;
            if (AXIS == 0) {
                const int d2 = t * t + L.a * L.a + L.z * L.z;  // |cell - (0,0,0)|^2
                dist[id] = with_distance ? __fmul_rn(__fsqrt_rn((float)d2), vs) : 0.f;
            }
            continue;
        }
        while (j > 0 && L.f(prv, t) <= L.f(cur, t)) {
            cur = prv;
            --j;
            if (j > 0) prv = stack[base + (size_t)(j - 1) * step];
        }
        nearest[id] = cur;
        if (AXIS == 0) dist[id] = with_distance ? __fmul_rn(__fsqrt_rn((float)L.f(cur, t)), vs) : 0.f;
    }
}

// get_distances (distancetransform.cu:263-279, 421-435): floor(((q - origin) + (0.5 * vs) * res) / vs) per axis; a
// query outside the grid or with a NaN coordinate reads 0
__global__ void __launch_bounds__(256) edt_query_kernel(const float *__restrict__ pts, size_t n, const float *__restrict__ dist, int res,
                                                         float vs, float ox, float oy, float oz, float *__restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float o[3] = {ox, oy, oz};
    const float shift = __fmul_rn(__fmul_rn(0.5f, vs), (float)res);
    size_t idx = 0;
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float f = floorf(__fdiv_rn(__fadd_rn(__fsub_rn(pts[3 * i + a], o[a]), shift), vs));
        in = in && f >= 0.f && f < (float)res;
        idx = idx * res + (in ? (size_t)f : 0);
    }
    out[i] = in ? dist[idx] : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
static unsigned edt_blocks(size_t n, unsigned threads, unsigned cap) {
    const size_t b = (n + threads - 1) / threads;
    return (unsigned)(b == 0 ? 1 : (b < cap ? b : cap));
}

static int edt_alloc_grid(cphb_dt *g, int res, uint32_t **nearest, float **dist, cudaStream_t s) {
    const size_t cells = (size_t)res * res * res;
    *nearest = nullptr;
    *dist = nullptr;
    int rc = cphb_alloc_async((void **)nearest, sizeof(uint32_t) * cells, s);
    if (!rc) rc = cphb_alloc_async((void **)dist, sizeof(float) * cells, s);
    if (rc) { cphb_free_async(*nearest, s); *nearest = nullptr; }
    return rc;
}

static bool edt_res_ok(int res, const char *who) {
    if (res >= 1 && res <= EDT_MAX_RES) return true;
    cphb_set_error("%s: resolution %d outside [1, %d]", who, res, EDT_MAX_RES);
    return false;
}

extern "C" int cphb_dt_create(float voxel_size, int resolution, const float origin[3], void *stream, cphb_dt **out) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!out) { cphb_set_error("cphb_dt_create: null argument"); return CPHB_ERR_INVALID; }
    if (!edt_res_ok(resolution, "cphb_dt_create")) return CPHB_ERR_INVALID;
    cphb_dt *g = new cphb_dt();
    memset(g, 0, sizeof(*g));
    g->voxel_size = voxel_size;
    g->res = resolution;
    for (int a = 0; a < 3; ++a) g->origin[a] = origin ? origin[a] : 0.f;
    g->cells = (size_t)resolution * resolution * resolution;
    int rc = edt_alloc_grid(g, resolution, &g->nearest, &g->dist, s);
    if (rc) { delete g; return rc; }
    CPHB_LAUNCH(edt_fill_kernel, edt_blocks(g->cells, 256, CPHB_SMS * 8), 256, 0, s, g->nearest, g->dist, (size_t)0, g->cells);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        cphb_set_error("cphb_dt_create: %s", cudaGetErrorString(e));
        cphb_dt_destroy(g);
        return CPHB_ERR_CUDA;
    }
    *out = g;
    return CPHB_OK;
}

extern "C" void cphb_dt_destroy(cphb_dt *g) {
    if (!g) return;
    cudaFreeAsync(g->nearest, 0);
    cudaFreeAsync(g->dist, 0);
    delete g;
}

// DenseGrid::Reconstruct (densegrid.inl:128-134): the linear prefix of the old cells is kept, the rest are defaults
extern "C" int cphb_dt_reconstruct(cphb_dt *g, float voxel_size, int resolution, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g) { cphb_set_error("cphb_dt_reconstruct: null handle"); return CPHB_ERR_INVALID; }
    if (!edt_res_ok(resolution, "cphb_dt_reconstruct")) return CPHB_ERR_INVALID;
    const size_t cells = (size_t)resolution * resolution * resolution;
    uint32_t *nearest;
    float *dist;
    int rc = edt_alloc_grid(g, resolution, &nearest, &dist, s);
    if (rc) return rc;
    const size_t keep = cells < g->cells ? cells : g->cells;
    cudaError_t e = cudaMemcpyAsync(nearest, g->nearest, sizeof(uint32_t) * keep, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dist, g->dist, sizeof(float) * keep, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess && keep < cells) {
        CPHB_LAUNCH(edt_fill_kernel, edt_blocks(cells - keep, 256, CPHB_SMS * 8), 256, 0, s, nearest, dist, keep, cells);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
        cphb_set_error("cphb_dt_reconstruct: %s", cudaGetErrorString(e));
        cphb_free_async(nearest, s);
        cphb_free_async(dist, s);
        return CPHB_ERR_CUDA;
    }
    cphb_free_async(g->nearest, s);
    cphb_free_async(g->dist, s);
    g->nearest = nearest;
    g->dist = dist;
    g->voxel_size = voxel_size;
    g->res = resolution;
    g->cells = cells;
    return CPHB_OK;
}

extern "C" int cphb_dt_set_geometry(cphb_dt *g, float voxel_size, const float origin[3]) {
    if (!g) { cphb_set_error("cphb_dt_set_geometry: null handle"); return CPHB_ERR_INVALID; }
    g->voxel_size = voxel_size;  // voxel_size_ / origin_ are public members of the reference
    if (origin) for (int a = 0; a < 3; ++a) g->origin[a] = origin[a];
    return CPHB_OK;
}

// the three sweeps after a stamp into g->dist (borrowed as the bitmap)
static int edt_sweeps(cphb_dt *g, int with_distance, cudaStream_t s) {
    const int r = g->res;
    const size_t lines = (size_t)r * r;
    cphb_scratch sc(s);
    uint32_t *stack = nullptr;
    int rc = sc.alloc(&stack, g->cells);
    if (rc) return rc;
    CPHB_LAUNCH(edt_sweep_z_kernel, (unsigned)((lines * 32 + 255) / 256), 256, 0, s, (const unsigned *)g->dist, r, g->nearest);
    CPHB_LAUNCH(edt_sweep_kernel<1>, (unsigned)((lines + 127) / 128), 128, 0, s, g->nearest, stack, g->dist, r, g->voxel_size, with_distance);
    CPHB_LAUNCH(edt_sweep_kernel<0>, (unsigned)((lines + 127) / 128), 128, 0, s, g->nearest, stack, g->dist, r, g->voxel_size, with_distance);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

static int edt_compute_cells(cphb_dt *g, const int32_t *cells, size_t n, int map, float vs, const float og[3], int with_distance,
                             cudaStream_t s) {
    const size_t words = (g->cells + 31) / 32;
    CPHB_CUDA(cudaMemsetAsync(g->dist, 0, sizeof(unsigned) * words, s));
    CPHB_LAUNCH(edt_stamp_kernel, edt_blocks(n, 256, CPHB_SMS * 8), 256, 0, s, cells, n, g->res, map, vs, og[0], og[1], og[2],
                g->origin[0], g->origin[1], g->origin[2], (unsigned *)g->dist);
    return edt_sweeps(g, with_distance, s);
}

extern "C" int cphb_dt_compute_sites(cphb_dt *g, const int32_t *cells, size_t n, int with_distance, void *stream) {
    if (!g || (n && !cells)) { cphb_set_error("cphb_dt_compute_sites: null argument"); return CPHB_ERR_INVALID; }
    const float zero[3] = {0.f, 0.f, 0.f};
    return edt_compute_cells(g, cells, n, 0, 0.f, zero, with_distance, (cudaStream_t)stream);
}

extern "C" int cphb_dt_compute_voxel_grid(cphb_dt *g, const int32_t *keys, size_t n, float vg_voxel_size, const float vg_origin[3],
                                          int with_distance, void *stream) {
    if (!g || !vg_origin || (n && !keys)) { cphb_set_error("cphb_dt_compute_voxel_grid: null argument"); return CPHB_ERR_INVALID; }
    if (fabsf(g->voxel_size - vg_voxel_size) > FLT_EPSILON) {  // distancetransform.cu:331-337: logged, grid unchanged
        cphb_set_error("Unsupport computing Voronoi diagrams from different voxel size.");
        return CPHB_ERR_INVALID;
    }
    return edt_compute_cells(g, keys, n, 1, g->voxel_size, vg_origin, with_distance, (cudaStream_t)stream);
}

// DistanceTransform::CreateFromOccupancyGrid (distancetransform_factory.cu:40-62), completed by the EDT: the sites are
// the occupied cells of the dense array
extern "C" int cphb_dt_from_occgrid(const cphb_occgrid *occ, void *stream, cphb_dt **out) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!occ || !out) { cphb_set_error("cphb_dt_from_occgrid: null argument"); return CPHB_ERR_INVALID; }
    float vs, origin[3];
    cphb_occgrid_params prm;
    cphb_occgrid_geometry(occ, &vs, origin);
    cphb_occgrid_get_params(occ, &prm);
    if (vs <= 0.f) { cphb_set_error("[CreateOccupancyGrid] occupancy grid  voxel_size <= 0."); return CPHB_ERR_INVALID; }
    const int r = cphb_occgrid_resolution(occ);
    cphb_dt *g = nullptr;
    int rc = cphb_dt_create(vs, r, origin, stream, &g);
    if (rc) return rc;
    const size_t words = (g->cells + 31) / 32;
    CPHB_LAUNCH(edt_stamp_occ_kernel, edt_blocks(words * 32, 256, CPHB_SMS * 8), 256, 0, s, cphb_occgrid_data(occ), g->cells,
                prm.occ_prob_thres_log, (unsigned *)g->dist);
    rc = edt_sweeps(g, 1, s);
    if (rc) { cphb_dt_destroy(g); return rc; }
    *out = g;
    return CPHB_OK;
}

extern "C" int cphb_dt_get_distances(const cphb_dt *g, const float *points, size_t n, float *out, void *stream) {
    if (!g || (n && (!points || !out))) { cphb_set_error("cphb_dt_get_distances: null argument"); return CPHB_ERR_INVALID; }
    if (n == 0) return CPHB_OK;
    CPHB_LAUNCH(edt_query_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, points, n, g->dist, g->res, g->voxel_size,
                g->origin[0], g->origin[1], g->origin[2], out);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}

// DenseGrid::GetVoxel (densegrid.inl:137-155): floor((point - origin) / vs) + res / 2 per axis; outside the grid (any
// axis) or NaN: *h_found = 0 and the default voxel
extern "C" int cphb_dt_get_voxel(const cphb_dt *g, const float point[3], int *h_found, int32_t h_nearest[3], int *h_state,
                                 float *h_distance, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!g || !point || !h_found) { cphb_set_error("cphb_dt_get_voxel: null argument"); return CPHB_ERR_INVALID; }
    const int half = g->res / 2;
    size_t idx = 0;
    bool in = true;
    for (int a = 0; a < 3; ++a) {
        const float f = floorf((point[a] - g->origin[a]) / g->voxel_size);
        in = in && f >= (float)-half && f < (float)(g->res - half);
        idx = idx * g->res + (in ? (size_t)((int)f + half) : 0);
    }
    uint32_t p = EDT_NOT_SITE;
    float d = 0.f;
    if (in) {
        CPHB_CUDA(cudaMemcpyAsync(&p, g->nearest + idx, 4, cudaMemcpyDeviceToHost, s));
        CPHB_CUDA(cudaMemcpyAsync(&d, g->dist + idx, 4, cudaMemcpyDeviceToHost, s));
        CPHB_CUDA(cudaStreamSynchronize(s));
    }
    *h_found = in ? 1 : 0;
    if (h_nearest) { h_nearest[0] = (p >> 20) & 1023u; h_nearest[1] = (p >> 10) & 1023u; h_nearest[2] = p & 1023u; }
    if (h_state) *h_state = (p & EDT_NOT_SITE) ? 2 : 0;
    if (h_distance) *h_distance = d;
    return CPHB_OK;
}

extern "C" const float *cphb_dt_distance_data(const cphb_dt *g) { return g ? g->dist : nullptr; }
extern "C" const uint32_t *cphb_dt_nearest_data(const cphb_dt *g) { return g ? g->nearest : nullptr; }
