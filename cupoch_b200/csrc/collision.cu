// collision.cu -- collision::ComputeIntersection (collision.h:36-160, collision.cu:1137-1231) between VoxelGrids,
// OccupancyGrids and Box / Sphere / Capsule primitives.  SURVEY 8f rank 11.
//
// The reference builds an LBVH over the target on every call and walks it with a 10000-entry candidate buffer on each
// thread's stack (40 KB of local memory, and candidates past the 10000th are never tested).  A grid target needs no
// tree: its elements are integer keys, so a query computes the key range its (margin-widened) box can touch and looks
// those keys up directly.
//   * VoxelGrid target: key - min key packed 21 bits per axis into a u64 and radix-sorted with the original index
//     (keys may be unsorted and repeated).  One (x, y) row of a range is one binary search for (x, y, z_lo) and a scan
//     along z, so a query costs its rows plus the keys present in them, not its volume.
//   * OccupancyGrid target: the dense log-odds grid is the lookup table; a cell is an element when it is inside the
//     grid's bound box and cphb_occ_keep(p, thres, 2) (ExtractOccupiedVoxels' predicate, shared with occgrid.cu) holds.
//   * Grid query: one thread per query element; a primitive query: one block per primitive, the rows (VoxelGrid) or
//     cells (OccupancyGrid) of its range strided over the block.
//   * Primitive target: each block of 256 query elements stages the primitives in tiles of 256, keeps (in index order)
//     those whose conservative box meets the block's box, and each thread tests its element against that short list
//     in ascending index order, so its first hit is the smallest colliding index.
// Every candidate gets the exact test and the smallest colliding target index is kept.  The per-query results are then
// compacted (cphb_compact_flags) and gathered into pairs.  A call makes a fixed number of launches for each operand
// pair whatever the sizes.
//
// Arithmetic (DESIGN.md arithmetic contract; oracle/collision.c restates it): every operation is rounded on its own
// (the library is built with -fmad=false), in the operand order written here; the reference's double constants act
// in float.  The exact tests restate intersection_test.inl:120-262 and distance_test.inl:47-110 as they are, including
// BoxBox's use of the first rotation as given, its A2 x B0 term with r(0, 1), CapsuleAABB's unconditional hit when
// the ray enters through a corner region, and Corner() picking all three coordinates from bit 0.
#include <float.h>
#include <math.h>
#include <string.h>

#include "voxelkey.cuh"

#define COLL_BLOCK 256

// A grid as the kernels see it.  Element key k covers [k * vs + o, (k + 1) * vs + o]; every element's key lies in
// [lo, hi].  VoxelGrid: element i is keys[i], its index i.  OccupancyGrid: cell = k + half, index = linear cell index.
struct CollGrid {
    float vs, o[3];
    int lo[3], hi[3];
    int occ;
    // VoxelGrid
    const int32_t *keys;
    const uint64_t *skeys;  // sorted packed keys (target only)
    const uint32_t *sidx;   // their original indices
    size_t n;
    // OccupancyGrid
    const float *prob;
    const int32_t *sel;     // query only: box positions of the occupied cells, ascending
    int res, half;
    float thres;
};

__device__ __forceinline__ int occ_linear(const CollGrid &g, int x, int y, int z) {
    return ((x + g.half) * g.res + (y + g.half)) * g.res + (z + g.half);
}
// query element j of a grid -> key and index
__device__ __forceinline__ void grid_elem(const CollGrid &g, size_t j, int k[3], int &id) {
    if (!g.occ) {
        k[0] = g.keys[3 * j]; k[1] = g.keys[3 * j + 1]; k[2] = g.keys[3 * j + 2];
        id = (int)j;
        return;
    }
    const size_t pos = (size_t)g.sel[j];
    const size_t dy = (size_t)(g.hi[1] - g.lo[1] + 1), dz = (size_t)(g.hi[2] - g.lo[2] + 1);
    k[0] = g.lo[0] + (int)(pos / (dy * dz));
    const size_t r = pos % (dy * dz);
    k[1] = g.lo[1] + (int)(r / dz);
    k[2] = g.lo[2] + (int)(r % dz);
    id = occ_linear(g, k[0], k[1], k[2]);
}
__device__ __forceinline__ void key_box(const CollGrid &g, const int k[3], float lo[3], float hi[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = (float)k[a] * g.vs + g.o[a];
        hi[a] = (float)(k[a] + 1) * g.vs + g.o[a];
    }
}
// the keys of g whose box can meet [blo, bhi]: floor with one guard key on each side, clamped to g's keys.  NaN
// bounds give the whole key range.  false: none.
__device__ __forceinline__ bool key_range(const CollGrid &g, const float blo[3], const float bhi[3], int lo[3], int hi[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        double l = (double)floorf((blo[a] - g.o[a]) / g.vs) - 1.0;
        double h = (double)floorf((bhi[a] - g.o[a]) / g.vs) + 1.0;
        l = fmax(l, (double)g.lo[a]);
        h = fmin(h, (double)g.hi[a]);
        if (!(l <= h)) return false;
        lo[a] = (int)l;
        hi[a] = (int)h;
    }
    return true;
}

// lookups: f(key, index) for every element of g in the row (x, y, z0..z1), or in a cell
template <class F>
__device__ __forceinline__ void vg_row(const CollGrid &g, int x, int y, int z0, int z1, F &f) {
    const uint64_t kl = cphb_key_pack(g.lo, x, y, z0), kh = cphb_key_pack(g.lo, x, y, z1);
    for (size_t a = cphb_key_lower_bound(g.skeys, g.n, kl); a < g.n; ++a) {
        const uint64_t k = g.skeys[a];
        if (k > kh) break;
        const int key[3] = {x, y, g.lo[2] + (int)(k & ((1ull << CPHB_KEY_AXIS_BITS) - 1))};
        f(key, (int)g.sidx[a]);
    }
}
template <class F>
__device__ __forceinline__ void occ_cell(const CollGrid &g, int x, int y, int z, F &f) {
    const int lin = occ_linear(g, x, y, z);
    if (cphb_occ_keep(__ldg(g.prob + lin), g.thres, 2)) {
        const int key[3] = {x, y, z};
        f(key, lin);
    }
}

// ------------------------------------------------------------------------------------------------ exact tests
__device__ __forceinline__ float dot3f(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// distance_test::PointAABBSquared (distance_test.inl:47-57)
__device__ __forceinline__ float point_aabb2(const float p[3], const float lo[3], const float hi[3]) {
    float d2 = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float v = p[i];
        if (v < lo[i]) d2 += (lo[i] - v) * (lo[i] - v);
        if (v > hi[i]) d2 += (v - hi[i]) * (v - hi[i]);
    }
    return d2;
}
__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }
// distance_test::LineSegmentLineSegmentSquared (distance_test.inl:59-110)
__device__ float seg_seg2(const float p0[3], const float q0[3], const float p1[3], const float q1[3]) {
    float d0[3], d1[3], r[3];
    for (int i = 0; i < 3; ++i) { d0[i] = q0[i] - p0[i]; d1[i] = q1[i] - p1[i]; r[i] = p0[i] - p1[i]; }
    const float a = dot3f(d0, d0), e = dot3f(d1, d1), f = dot3f(d1, r);
    float s, t;
    if (a <= FLT_EPSILON && e <= FLT_EPSILON) {
        s = 0.f;
        t = 0.f;
    } else if (a <= FLT_EPSILON) {
        s = 0.f;
        t = clamp01(f / e);
    } else {
        const float c = dot3f(d0, r);
        if (e <= FLT_EPSILON) {
            t = 0.f;
            s = clamp01(-c / a);
        } else {
            const float b = dot3f(d0, d1);
            const float denom = a * e - b * b;
            s = (denom != 0.f) ? clamp01((b * f - c * e) / denom) : 0.f;
            t = (b * s + f) / e;
            if (t < 0.f) {
                t = 0.f;
                s = clamp01(-c / a);
            } else if (t > 1.f) {
                t = 1.f;
                s = clamp01((b - c) / a);
            }
        }
    }
    float w[3];
    for (int i = 0; i < 3; ++i) w[i] = (p0[i] + s * d0[i]) - (p1[i] + t * d1[i]);
    return dot3f(w, w);
}
// intersection_test::RayAABB (:120-143) + CapsuleAABB (:211-262)
__device__ bool capsule_aabb(float radius, const float p[3], const float d[3], const float lo[3], const float hi[3]) {
    float elo[3], ehi[3];
    for (int i = 0; i < 3; ++i) { elo[i] = lo[i] - radius; ehi[i] = hi[i] + radius; }
    float tmin = 0.f, tmax = FLT_MAX;
    for (int i = 0; i < 3; ++i) {
        if (fabsf(d[i]) < FLT_EPSILON) {
            if (p[i] < elo[i] || p[i] > ehi[i]) return false;
        } else {
            const float ood = 1.0f / d[i];
            float t1 = (elo[i] - p[i]) * ood, t2 = (ehi[i] - p[i]) * ood;
            if (t1 > t2) { const float x = t1; t1 = t2; t2 = x; }
            if (t1 > tmin) tmin = t1;
            if (t2 < tmax) tmax = t2;
            if (tmin > tmax) return false;
        }
    }
    if (tmin > 1.0f) return false;
    int u = 0, v = 0;
    for (int i = 0; i < 3; ++i) {
        const float q = p[i] + d[i] * tmin;
        if (q < lo[i]) u |= 1 << i;
        if (q > hi[i]) v |= 1 << i;
    }
    const int m = u + v;
    if (m == 7) return true;
    if ((m & (m - 1)) == 0) return true;
    float pd[3], c0[3], c1[3];
    for (int i = 0; i < 3; ++i) {
        pd[i] = p[i] + d[i];
        c0[i] = ((u ^ 7) & 1) ? hi[i] : lo[i];  // Corner(min, max, n) reads bit 0 for every axis
        c1[i] = (v & 1) ? hi[i] : lo[i];
    }
    return seg_seg2(p, pd, c0, c1) <= radius * radius;
}
// intersection_test::BoxBox (:153-209) with rot2 = I
__device__ bool box_box(const float e1[3], const float R[9], const float c1[3], const float e2[3], const float c2[3]) {
    float r[9], ar[9], t[3], dc[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            r[3 * i + j] = (R[3 * i] * (j == 0 ? 1.f : 0.f) + R[3 * i + 1] * (j == 1 ? 1.f : 0.f)) + R[3 * i + 2] * (j == 2 ? 1.f : 0.f);
            ar[3 * i + j] = fabsf(r[3 * i + j]) + FLT_EPSILON;
        }
    for (int i = 0; i < 3; ++i) dc[i] = c2[i] - c1[i];
    for (int i = 0; i < 3; ++i) t[i] = (R[3 * i] * dc[0] + R[3 * i + 1] * dc[1]) + R[3 * i + 2] * dc[2];
#define RR(i, j) r[3 * (i) + (j)]
#define AR(i, j) ar[3 * (i) + (j)]
    for (int i = 0; i < 3; ++i)
        if (fabsf(t[i]) > e1[i] + ((AR(i, 0) * e2[0] + AR(i, 1) * e2[1]) + AR(i, 2) * e2[2])) return false;
    for (int i = 0; i < 3; ++i)
        if (fabsf((t[0] * RR(0, i) + t[1] * RR(1, i)) + t[2] * RR(2, i)) > ((AR(0, i) * e1[0] + AR(1, i) * e1[1]) + AR(2, i) * e1[2]) + e2[i])
            return false;
    float ra, rb;
    ra = e1[1] * AR(2, 0) + e1[2] * AR(1, 0); rb = e2[1] * AR(0, 2) + e2[2] * AR(0, 1);
    if (fabsf(t[2] * RR(1, 0) - t[1] * RR(2, 0)) > ra + rb) return false;
    ra = e1[1] * AR(2, 1) + e1[2] * AR(1, 1); rb = e2[0] * AR(0, 2) + e2[2] * AR(0, 0);
    if (fabsf(t[2] * RR(1, 1) - t[1] * RR(2, 1)) > ra + rb) return false;
    ra = e1[1] * AR(2, 2) + e1[2] * AR(1, 2); rb = e2[0] * AR(0, 1) + e2[1] * AR(0, 0);
    if (fabsf(t[2] * RR(1, 2) - t[1] * RR(2, 2)) > ra + rb) return false;
    ra = e1[0] * AR(2, 0) + e1[2] * AR(0, 0); rb = e2[1] * AR(1, 2) + e2[2] * AR(1, 1);
    if (fabsf(t[0] * RR(2, 0) - t[2] * RR(0, 0)) > ra + rb) return false;
    ra = e1[0] * AR(2, 1) + e1[2] * AR(0, 1); rb = e2[0] * AR(1, 2) + e2[2] * AR(1, 0);
    if (fabsf(t[0] * RR(2, 1) - t[2] * RR(0, 1)) > ra + rb) return false;
    ra = e1[0] * AR(2, 2) + e1[2] * AR(0, 2); rb = e2[0] * AR(1, 1) + e2[1] * AR(1, 0);
    if (fabsf(t[0] * RR(2, 2) - t[2] * RR(0, 2)) > ra + rb) return false;
    ra = e1[0] * AR(1, 0) + e1[1] * AR(0, 0); rb = e2[1] * AR(2, 2) + e2[2] * AR(2, 1);
    if (fabsf(t[1] * RR(0, 1) - t[0] * RR(1, 0)) > ra + rb) return false;  // r(0, 1), as the reference writes it
    ra = e1[0] * AR(1, 1) + e1[1] * AR(0, 1); rb = e2[0] * AR(2, 2) + e2[2] * AR(2, 0);
    if (fabsf(t[1] * RR(0, 1) - t[0] * RR(1, 1)) > ra + rb) return false;
    ra = e1[0] * AR(1, 2) + e1[1] * AR(0, 2); rb = e2[0] * AR(2, 1) + e2[1] * AR(2, 0);
    if (fabsf(t[1] * RR(0, 2) - t[0] * RR(1, 2)) > ra + rb) return false;
#undef RR
#undef AR
    return true;
}
// a primitive against grid element k (collision.cu:221-298): centre (k + 0.5) * vs + o, half size vs / 2
__device__ bool prim_elem(const cphb_primitive &p, const int k[3], const CollGrid &g, float margin) {
    const float half = g.vs / 2.f;
    float c[3], lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        c[a] = ((float)k[a] + 0.5f) * g.vs + g.o[a];
        lo[a] = c[a] - half;
        hi[a] = c[a] + half;
    }
    const float *T = p.transform;
    if (p.type == CPHB_PRIM_BOX) {
        const float e1[3] = {p.lengths[0] * 0.5f, p.lengths[1] * 0.5f, p.lengths[2] * 0.5f};
        const float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
        const float t1[3] = {T[3], T[7], T[11]};
        const float e2[3] = {half + margin, half + margin, half + margin};
        return box_box(e1, R, t1, e2, c);
    }
    if (p.type == CPHB_PRIM_SPHERE) {
        const float r = p.radius + margin;
        const float ctr[3] = {T[3], T[7], T[11]};
        return point_aabb2(ctr, lo, hi) <= r * r;
    }
    if (p.type == CPHB_PRIM_CAPSULE) {
        const float r = p.radius + margin;
        const float hh = 0.5f * p.height;
        const float s[3] = {T[3] - hh * T[2], T[7] - hh * T[6], T[11] - hh * T[10]};
        const float d[3] = {p.height * T[2], p.height * T[6], p.height * T[10]};
        return capsule_aabb(r, s, d, lo, hi);
    }
    return false;  // Cylinder and anything else: the reference's default branch
}

// ------------------------------------------------------------------------------------------------ kernels
// grid-stride min / max of the keys: warp and block reductions, then one global atomic per block and bound
__global__ void __launch_bounds__(COLL_BLOCK) coll_key_bounds_kernel(const int32_t *__restrict__ keys, size_t n, int *b) {
    __shared__ int s[6];
    if (threadIdx.x < 6) s[threadIdx.x] = threadIdx.x < 3 ? INT_MAX : INT_MIN;
    __syncthreads();
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        for (int a = 0; a < 3; ++a) {
            const int k = keys[3 * i + a];
            lo[a] = min(lo[a], k);
            hi[a] = max(hi[a], k);
        }
    for (int a = 0; a < 3; ++a) {
        const int l = __reduce_min_sync(CPHB_FULL, lo[a]), h = __reduce_max_sync(CPHB_FULL, hi[a]);
        if (lane_id() == 0) { atomicMin(&s[a], l); atomicMax(&s[3 + a], h); }
    }
    __syncthreads();
    if (threadIdx.x < 3) atomicMin(&b[threadIdx.x], s[threadIdx.x]);
    else if (threadIdx.x < 6) atomicMax(&b[threadIdx.x], s[threadIdx.x]);
}
__global__ void __launch_bounds__(COLL_BLOCK) coll_pack_kernel(const int32_t *__restrict__ keys, size_t n, int3 lo3, uint64_t *packed,
                                                                uint32_t *idx) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int lo[3] = {lo3.x, lo3.y, lo3.z};
    packed[i] = cphb_key_pack(lo, keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]);
    idx[i] = (uint32_t)i;
}
// the occupied cells of an OccupancyGrid query's bound box (box order = ascending linear index)
__global__ void __launch_bounds__(COLL_BLOCK) coll_occ_flag_kernel(const CollGrid g, size_t m, uint8_t *keep) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    const size_t dy = (size_t)(g.hi[1] - g.lo[1] + 1), dz = (size_t)(g.hi[2] - g.lo[2] + 1);
    const int x = g.lo[0] + (int)(i / (dy * dz)), yz = (int)(i % (dy * dz));
    const int lin = occ_linear(g, x, g.lo[1] + yz / (int)dz, g.lo[2] + yz % (int)dz);
    keep[i] = cphb_occ_keep(g.prob[lin], g.thres, 2) ? 1 : 0;
}

// conservative box of the grid elements (of a grid with voxel size vs) that a primitive can collide with, margin
// included: lo > hi when it collides with none, +-inf when it may collide with any (non-finite or singular input)
__device__ __forceinline__ bool all_finite(const float *v, int n) {
    for (int i = 0; i < n; ++i)
        if (!isfinite(v[i])) return false;
    return true;
}
__global__ void __launch_bounds__(COLL_BLOCK) coll_prim_box_kernel(const cphb_primitive *__restrict__ prims, size_t n, float vs, float margin,
                                                                  float4 *box) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const cphb_primitive p = prims[i];
    const float *T = p.transform;
    const float c[3] = {T[3], T[7], T[11]};
    double ext[3] = {-1.0, -1.0, -1.0};  // < 0: no element
    bool any = false;
    const float half = vs / 2.f;
    if (p.type == CPHB_PRIM_BOX) {
        // a hit passes the three tests on the first box's axes: |(R d)_j| <= B_j, d = centre - c; so
        // |d_i| <= sum_j |R^-1_ij| B_j
        const float e2 = half + margin;
        if (!all_finite(T, 12) || !all_finite(p.lengths, 3)) {
            any = true;
        } else {
            const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
            const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
            if (!(fabs(det) > 1e-12)) {
                any = true;
            } else {
                const double inv[9] = {(R[4] * R[8] - R[5] * R[7]) / det, (R[2] * R[7] - R[1] * R[8]) / det, (R[1] * R[5] - R[2] * R[4]) / det,
                                       (R[5] * R[6] - R[3] * R[8]) / det, (R[0] * R[8] - R[2] * R[6]) / det, (R[2] * R[3] - R[0] * R[5]) / det,
                                       (R[3] * R[7] - R[4] * R[6]) / det, (R[1] * R[6] - R[0] * R[7]) / det, (R[0] * R[4] - R[1] * R[3]) / det};
                double B[3];
                bool none = false;
                for (int j = 0; j < 3; ++j) {
                    B[j] = 0.5 * (double)p.lengths[j];
                    double mag = fabs(B[j]);
                    for (int k = 0; k < 3; ++k) {
                        B[j] += (fabs(R[3 * j + k]) + (double)FLT_EPSILON) * (double)e2;
                        mag += (fabs(R[3 * j + k]) + (double)FLT_EPSILON) * fabs((double)e2);
                    }
                    B[j] += 1e-5 * mag + 1e-30;  // the float test's rounding
                    if (B[j] < 0.0) none = true;
                }
                if (!none)
                    for (int a = 0; a < 3; ++a)
                        ext[a] = fabs(inv[3 * a]) * B[0] + fabs(inv[3 * a + 1]) * B[1] + fabs(inv[3 * a + 2]) * B[2];
            }
        }
    } else if (p.type == CPHB_PRIM_SPHERE || p.type == CPHB_PRIM_CAPSULE) {
        const float r = p.radius + margin;
        const float vals[2] = {r, p.height};
        if (!all_finite(T, 12) || !all_finite(vals, 2)) {
            any = true;
        } else {
            // a sphere hit is within |r| of the centre; a capsule hit is within |r| of its segment
            const double hz = p.type == CPHB_PRIM_CAPSULE ? 0.5 * fabs((double)p.height) : 0.0;
            for (int a = 0; a < 3; ++a) ext[a] = fabs((double)r) + hz * fabs((double)T[4 * a + 2]);
        }
    }
    float4 lo, hi;
    if (any) {
        lo = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
        hi = make_float4(INFINITY, INFINITY, INFINITY, 0.f);
    } else if (ext[0] < 0.0 || ext[1] < 0.0 || ext[2] < 0.0) {
        lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f);
        hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    } else {
        float l[3], h[3];
        for (int a = 0; a < 3; ++a) {
            // one element of slack plus a relative margin for the float rounding of the centres and the tests
            const double g = (double)vs + 1e-5 * (fabs((double)c[a]) + ext[a]) + 1e-30;
            l[a] = (float)((double)c[a] - ext[a] - g);
            h[a] = (float)((double)c[a] + ext[a] + g);
        }
        lo = make_float4(l[0], l[1], l[2], 0.f);
        hi = make_float4(h[0], h[1], h[2], 0.f);
    }
    box[2 * i] = lo;
    box[2 * i + 1] = hi;
}

struct GridHit {  // grid query element against grid target elements: inclusive box overlap (lbvh aabb.cuh:19-25)
    const CollGrid *t;
    float qlo[3], qhi[3];
    int best;
    __device__ __forceinline__ void operator()(const int k[3], int idx) {
        if (idx >= best) return;
        float lo[3], hi[3];
        key_box(*t, k, lo, hi);
        for (int a = 0; a < 3; ++a)
            if (!(qlo[a] <= hi[a] && qhi[a] >= lo[a])) return;
        best = idx;
    }
};
// one thread per query grid element, grid target
__global__ void __launch_bounds__(COLL_BLOCK) coll_grid_grid_kernel(const CollGrid t, const CollGrid q, size_t nq, float margin,
                                                                   int32_t *best, uint8_t *keep) {
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (j >= nq) return;
    int k[3], id;
    grid_elem(q, j, k, id);
    GridHit f;
    f.t = &t;
    f.best = INT_MAX;
    key_box(q, k, f.qlo, f.qhi);
    for (int a = 0; a < 3; ++a) { f.qlo[a] = f.qlo[a] - margin; f.qhi[a] = f.qhi[a] + margin; }
    int lo[3], hi[3];
    if (key_range(t, f.qlo, f.qhi, lo, hi)) {
        for (int x = lo[0]; x <= hi[0]; ++x)
            for (int y = lo[1]; y <= hi[1]; ++y) {
                if (!t.occ) vg_row(t, x, y, lo[2], hi[2], f);
                else
                    for (int z = lo[2]; z <= hi[2]; ++z) occ_cell(t, x, y, z, f);
            }
    }
    best[j] = f.best == INT_MAX ? -1 : f.best;
    keep[j] = f.best != INT_MAX;
}

struct PrimHit {  // a primitive query against grid target elements
    const CollGrid *t;
    const cphb_primitive *p;
    float margin;
    int best;
    __device__ __forceinline__ void operator()(const int k[3], int idx) {
        if (idx < best && prim_elem(*p, k, *t, margin)) best = idx;
    }
};
// one block per primitive, grid target: the rows (VoxelGrid) or cells (OccupancyGrid) of its range strided over the block
__global__ void __launch_bounds__(COLL_BLOCK) coll_prim_grid_kernel(const CollGrid t, const cphb_primitive *__restrict__ prims,
                                                                   const float4 *__restrict__ pbox, float margin, int32_t *best,
                                                                   uint8_t *keep) {
    __shared__ int s_best;
    const size_t j = blockIdx.x;
    if (threadIdx.x == 0) s_best = INT_MAX;
    __syncthreads();
    const cphb_primitive p = prims[j];
    const float4 bl = pbox[2 * j], bh = pbox[2 * j + 1];
    const float blo[3] = {bl.x, bl.y, bl.z}, bhi[3] = {bh.x, bh.y, bh.z};
    int lo[3], hi[3];
    if (bl.x <= bh.x && bl.y <= bh.y && bl.z <= bh.z && key_range(t, blo, bhi, lo, hi)) {
        PrimHit f;
        f.t = &t;
        f.p = &p;
        f.margin = margin;
        f.best = INT_MAX;
        const size_t ny = (size_t)(hi[1] - lo[1] + 1), nz = (size_t)(hi[2] - lo[2] + 1);
        const size_t rows = (size_t)(hi[0] - lo[0] + 1) * ny;
        if (!t.occ) {
            for (size_t r = threadIdx.x; r < rows; r += blockDim.x)
                vg_row(t, lo[0] + (int)(r / ny), lo[1] + (int)(r % ny), lo[2], hi[2], f);
        } else {
            const size_t cells = rows * nz;
            for (size_t c = threadIdx.x; c < cells; c += blockDim.x) {
                const size_t r = c / nz;
                occ_cell(t, lo[0] + (int)(r / ny), lo[1] + (int)(r % ny), lo[2] + (int)(c % nz), f);
            }
        }
        if (f.best != INT_MAX) atomicMin(&s_best, f.best);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        best[j] = s_best == INT_MAX ? -1 : s_best;
        keep[j] = s_best != INT_MAX;
    }
}

// primitive target, grid query: 256 query elements per block, primitives staged in index-ordered tiles of 256
__global__ void __launch_bounds__(COLL_BLOCK) coll_grid_prim_kernel(const CollGrid q, size_t nq, const cphb_primitive *__restrict__ prims,
                                                                   const float4 *__restrict__ pbox, size_t np, float margin,
                                                                   int32_t *best, uint8_t *keep) {
    __shared__ unsigned s_lo[3], s_hi[3];
    __shared__ int s_list[COLL_BLOCK];
    __shared__ int s_warp[COLL_BLOCK / 32 + 1];
    const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool valid = j < nq;
    int k[3] = {0, 0, 0}, id = 0;
    float lo[3] = {0.f, 0.f, 0.f}, hi[3] = {0.f, 0.f, 0.f};
    if (valid) {
        grid_elem(q, j, k, id);
        key_box(q, k, lo, hi);
    }
    if (threadIdx.x < 3) { s_lo[threadIdx.x] = 0xffffffffu; s_hi[threadIdx.x] = 0u; }
    __syncthreads();
    for (int a = 0; a < 3; ++a) {
        const unsigned l = __reduce_min_sync(CPHB_FULL, valid ? f2ord(lo[a]) : 0xffffffffu);
        const unsigned h = __reduce_max_sync(CPHB_FULL, valid ? f2ord(hi[a]) : 0u);
        if (lane_id() == 0) { atomicMin(&s_lo[a], l); atomicMax(&s_hi[a], h); }
    }
    __syncthreads();
    const float blo[3] = {ord2f(s_lo[0]), ord2f(s_lo[1]), ord2f(s_lo[2])}, bhi[3] = {ord2f(s_hi[0]), ord2f(s_hi[1]), ord2f(s_hi[2])};
    int found = -1;
    for (size_t base = 0; base < np; base += COLL_BLOCK) {
        const size_t pi = base + threadIdx.x;
        bool take = false;
        float4 pl, ph;
        if (pi < np) {
            pl = pbox[2 * pi];
            ph = pbox[2 * pi + 1];
            take = pl.x <= bhi[0] && ph.x >= blo[0] && pl.y <= bhi[1] && ph.y >= blo[1] && pl.z <= bhi[2] && ph.z >= blo[2];
        }
        const unsigned ball = __ballot_sync(CPHB_FULL, take);
        const int w = threadIdx.x >> 5;
        if (lane_id() == 0) s_warp[w] = __popc(ball);
        __syncthreads();
        if (threadIdx.x == 0) {
            int acc = 0;
            for (int i = 0; i < COLL_BLOCK / 32; ++i) { const int c = s_warp[i]; s_warp[i] = acc; acc += c; }
            s_warp[COLL_BLOCK / 32] = acc;
        }
        __syncthreads();
        if (take) s_list[s_warp[w] + __popc(ball & ((1u << lane_id()) - 1u))] = (int)pi;
        __syncthreads();
        const int cnt = s_warp[COLL_BLOCK / 32];
        if (valid && found < 0) {
            for (int e = 0; e < cnt; ++e) {
                const int pidx = s_list[e];
                const float4 el = pbox[2 * pidx], eh = pbox[2 * pidx + 1];
                if (!(el.x <= hi[0] && eh.x >= lo[0] && el.y <= hi[1] && eh.y >= lo[1] && el.z <= hi[2] && eh.z >= lo[2])) continue;
                if (prim_elem(prims[pidx], k, q, margin)) { found = pidx; break; }
            }
        }
        if (__syncthreads_and(!valid || found >= 0)) break;
    }
    if (valid) {
        best[j] = found;
        keep[j] = found >= 0;
    }
}

// pairs (target index, query index) of the colliding query elements
__global__ void __launch_bounds__(COLL_BLOCK) coll_gather_kernel(const int32_t *__restrict__ sel, size_t m, const int32_t *__restrict__ best,
                                                                const CollGrid q, int q_grid, int32_t *pairs) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    const size_t j = (size_t)sel[i];
    int id = (int)j;
    if (q_grid && q.occ) {
        int k[3];
        grid_elem(q, j, k, id);
    }
    pairs[2 * i] = best[j];
    pairs[2 * i + 1] = id;
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
int cphb_sort_voxel_keys(const int32_t *keys, size_t n, cphb_scratch &sc, cphb_sorted_keys *out, cudaStream_t s, const char *who) {
    int *d_b = nullptr;
    uint64_t *pk = nullptr, *pk2 = nullptr;
    uint32_t *ix = nullptr, *ix2 = nullptr;
    int rc = sc.alloc(&d_b, 6);
    if (!rc) rc = sc.alloc(&pk, n);
    if (!rc) rc = sc.alloc(&pk2, n);
    if (!rc) rc = sc.alloc(&ix, n);
    if (!rc) rc = sc.alloc(&ix2, n);
    if (rc) return rc;
    const int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    CPHB_CUDA(cudaMemcpyAsync(d_b, init, sizeof(init), cudaMemcpyHostToDevice, s));
    const unsigned grid = (unsigned)((n + COLL_BLOCK - 1) / COLL_BLOCK);
    CPHB_LAUNCH(coll_key_bounds_kernel, grid < CPHB_SMS * 8 ? grid : CPHB_SMS * 8, COLL_BLOCK, 0, s, keys, n, d_b);
    int hb[6];
    rc = cphb_read_back(hb, d_b, sizeof(hb), s, who);
    if (rc) return rc;
    for (int x = 0; x < 3; ++x) {
        if ((long long)hb[3 + x] - (long long)hb[x] >= (1ll << CPHB_KEY_AXIS_BITS)) {
            cphb_set_error("%s: VoxelGrid keys span %lld >= 2^21 on axis %d", who, (long long)hb[3 + x] - (long long)hb[x] + 1, x);
            return CPHB_ERR_INVALID;
        }
        out->lo[x] = hb[x];
        out->hi[x] = hb[3 + x];
    }
    CPHB_LAUNCH(coll_pack_kernel, grid, COLL_BLOCK, 0, s, keys, n, make_int3(hb[0], hb[1], hb[2]), pk, ix);
    rc = cphb_sort_pairs_u64(pk, pk2, ix, ix2, n, 3 * CPHB_KEY_AXIS_BITS, s);
    if (rc) return rc;
    out->skeys = pk2;
    out->sidx = ix2;
    return CPHB_OK;
}

static bool vs_ok(float vs) { return isfinite(vs) && vs > 0.f; }

// grid operand -> CollGrid with its element count (VoxelGrid: keys; OccupancyGrid: the bound box volume, enumerated later)
static int coll_grid_of(const cphb_coll_operand *op, CollGrid *g, cudaStream_t s) {
    memset(g, 0, sizeof(*g));
    if (op->kind == CPHB_COLL_VOXEL_GRID) {
        g->vs = op->voxel_size;
        for (int a = 0; a < 3; ++a) g->o[a] = op->origin[a];
        g->keys = op->keys;
        g->n = op->n;
        return CPHB_OK;
    }
    cphb_occgrid_view v;
    cphb_occgrid_view_of(op->occ, &v);
    cphb_occgrid_geometry(op->occ, &g->vs, g->o);
    g->occ = 1;
    g->prob = v.prob;
    g->res = v.res;
    g->half = v.res / 2;
    g->thres = v.thres;
    unsigned h[6];
    int rc = cphb_read_back(h, v.bounds, sizeof(h), s, "cphb_compute_intersection");
    if (rc) return rc;
    for (int a = 0; a < 3; ++a) {
        g->lo[a] = (int)h[a] - g->half;
        g->hi[a] = (int)h[3 + a] - g->half;
    }
    return CPHB_OK;
}

static int coll_invalid(const char *what) {
    cphb_set_error("cphb_compute_intersection: %s", what);
    return CPHB_ERR_INVALID;
}
static int coll_check_operand(const cphb_coll_operand *op) {
    if (op->kind == CPHB_COLL_VOXEL_GRID) {
        if (op->n && !op->keys) return coll_invalid("null VoxelGrid keys");
        if (op->n && !vs_ok(op->voxel_size)) return coll_invalid("VoxelGrid voxel size is not positive and finite");
        if (op->n > (size_t)INT32_MAX) return coll_invalid("more than 2^31-1 voxels");
        return CPHB_OK;
    }
    if (op->kind == CPHB_COLL_OCCUPANCY_GRID) {
        if (!op->occ) return coll_invalid("null OccupancyGrid");
        float vs, o[3];
        cphb_occgrid_geometry(op->occ, &vs, o);
        if (!vs_ok(vs)) return coll_invalid("OccupancyGrid voxel size is not positive and finite");
        return CPHB_OK;
    }
    if (op->kind == CPHB_COLL_PRIMITIVES) {
        if (op->n && !op->primitives) return coll_invalid("null primitives");
        if (op->n > (size_t)INT32_MAX) return coll_invalid("more than 2^31-1 primitives");
        return CPHB_OK;
    }
    return coll_invalid("unknown operand kind");
}

extern "C" int cphb_compute_intersection(const cphb_coll_operand *a, const cphb_coll_operand *b, float margin, int32_t *pairs_out,
                                         size_t capacity, size_t *h_count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!a || !b || !h_count || (capacity && !pairs_out)) {
        cphb_set_error("cphb_compute_intersection: null argument");
        return CPHB_ERR_INVALID;
    }
    *h_count = 0;
    int rc = coll_check_operand(a);
    if (!rc) rc = coll_check_operand(b);
    if (rc) return rc;
    const bool a_prim = a->kind == CPHB_COLL_PRIMITIVES, b_prim = b->kind == CPHB_COLL_PRIMITIVES;
    if ((a_prim && b_prim) || (a->kind == CPHB_COLL_OCCUPANCY_GRID && b->kind == CPHB_COLL_OCCUPANCY_GRID)) {
        cphb_set_error("cphb_compute_intersection: the pair (%d, %d) is not supported", a->kind, b->kind);
        return CPHB_ERR_INVALID;
    }
    if (!isfinite(margin)) {
        cphb_set_error("cphb_compute_intersection: margin %g is not finite", (double)margin);
        return CPHB_ERR_INVALID;
    }
    if ((a->kind != CPHB_COLL_OCCUPANCY_GRID && a->n == 0) || (b->kind != CPHB_COLL_OCCUPANCY_GRID && b->n == 0)) return CPHB_OK;

    cphb_scratch sc(s);
    CollGrid t, q;
    memset(&t, 0, sizeof(t));
    memset(&q, 0, sizeof(q));
    if (!a_prim) {
        rc = coll_grid_of(a, &t, s);
        if (rc) return rc;
        if (t.occ && (t.hi[0] < t.lo[0] || t.hi[1] < t.lo[1] || t.hi[2] < t.lo[2])) return CPHB_OK;
    }
    if (!b_prim) {
        rc = coll_grid_of(b, &q, s);
        if (rc) return rc;
        if (q.occ && (q.hi[0] < q.lo[0] || q.hi[1] < q.lo[1] || q.hi[2] < q.lo[2])) return CPHB_OK;
    }
    // VoxelGrid target: key bounds, then the packed keys sorted with their indices
    if (!a_prim && !t.occ) {
        cphb_sorted_keys sk;
        rc = cphb_sort_voxel_keys(t.keys, t.n, sc, &sk, s, "cphb_compute_intersection");
        if (rc) return rc;
        for (int x = 0; x < 3; ++x) {
            t.lo[x] = sk.lo[x];
            t.hi[x] = sk.hi[x];
        }
        t.skeys = sk.skeys;
        t.sidx = sk.sidx;
    }
    // the query's elements
    size_t nq = b_prim ? b->n : q.n;
    if (!b_prim && q.occ) {
        const size_t m = (size_t)(q.hi[0] - q.lo[0] + 1) * (size_t)(q.hi[1] - q.lo[1] + 1) * (size_t)(q.hi[2] - q.lo[2] + 1);
        uint8_t *box_keep = nullptr;
        int32_t *occ_sel = nullptr;
        rc = sc.alloc(&box_keep, m);
        if (!rc) rc = sc.alloc(&occ_sel, m);
        if (rc) return rc;
        CPHB_LAUNCH(coll_occ_flag_kernel, (unsigned)((m + COLL_BLOCK - 1) / COLL_BLOCK), COLL_BLOCK, 0, s, q, m, box_keep);
        rc = cphb_compact_flags(box_keep, m, occ_sel, &nq, s);
        if (rc) return rc;
        q.sel = occ_sel;
        if (nq == 0) return CPHB_OK;
    }
    int32_t *best = nullptr, *sel = nullptr;
    uint8_t *keep = nullptr;
    float4 *pbox = nullptr;
    rc = sc.alloc(&best, nq);
    if (!rc) rc = sc.alloc(&keep, nq);
    if (!rc) rc = sc.alloc(&sel, nq);
    if (!rc && (a_prim || b_prim)) rc = sc.alloc(&pbox, 2 * (a_prim ? a->n : b->n));
    if (rc) return rc;
    const unsigned gq = (unsigned)((nq + COLL_BLOCK - 1) / COLL_BLOCK);
    if (a_prim) {
        CPHB_LAUNCH(coll_prim_box_kernel, (unsigned)((a->n + COLL_BLOCK - 1) / COLL_BLOCK), COLL_BLOCK, 0, s, a->primitives, a->n, q.vs, margin, pbox);
        CPHB_LAUNCH(coll_grid_prim_kernel, gq, COLL_BLOCK, 0, s, q, nq, a->primitives, pbox, a->n, margin, best, keep);
    } else if (b_prim) {
        CPHB_LAUNCH(coll_prim_box_kernel, (unsigned)((b->n + COLL_BLOCK - 1) / COLL_BLOCK), COLL_BLOCK, 0, s, b->primitives, b->n, t.vs, margin, pbox);
        CPHB_LAUNCH(coll_prim_grid_kernel, (unsigned)nq, COLL_BLOCK, 0, s, t, b->primitives, pbox, margin, best, keep);
    } else {
        CPHB_LAUNCH(coll_grid_grid_kernel, gq, COLL_BLOCK, 0, s, t, q, nq, margin, best, keep);
    }
    size_t m = 0;
    rc = cphb_compact_flags(keep, nq, sel, &m, s);  // synchronises
    if (rc) return rc;
    *h_count = m;
    const size_t w = m < capacity ? m : capacity;
    if (w) {
        CPHB_LAUNCH(coll_gather_kernel, (unsigned)((w + COLL_BLOCK - 1) / COLL_BLOCK), COLL_BLOCK, 0, s, sel, w, best, q, b_prim ? 0 : 1, pairs_out);
    }
    return cphb_read_back(nullptr, nullptr, 0, s, "cphb_compute_intersection");
}
