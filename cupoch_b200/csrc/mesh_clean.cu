// mesh_clean.cu -- TriangleMesh cleanup (RemoveDuplicatedVertices / RemoveDuplicatedTriangles /
// RemoveUnreferencedVertices / RemoveDegenerateTriangles), the triangle part of operator+=, and
// GetSelfIntersectingTriangles (DESIGN section 4 item 26).  Reference: geometry/trianglemesh.cu (TM) 903-1141.
//
// Every entry first checks each vertex index against [0, n_vertices); a bad one is CPHB_ERR_INVALID and no output is
// meaningful (the caller keeps its mesh).  Outputs are separate buffers sized like the inputs.
//
// The Remove* operations are stable radix sorts, head-flag uniques, block compactions and remaps.  The self-
// intersection search is a uniform grid with an ownership rule: a pair whose boxes overlap is tested only in the cell
// that holds the componentwise maximum of the two boxes' minimum corners, and only once there.  Triangles covering more
// than SI_K cells are tested against every box by one warp each.  No float atomics; hits are sorted on i * n_t + j.
//
// Arithmetic: IEEE float32 with no contraction (build.py's -fmad=false), in the published operand order of Moller's
// NoDivTriTriIsect; |d| < EPSILON compares in double, as the published code's double EPSILON makes it.
#include <math.h>

#include <cub/device/device_scan.cuh>

#include "cphb_internal.cuh"
#include "sum_values.cuh"

#define MC_BLOCK 256
// a triangle whose box covers at most SI_K grid cells goes through the grid; a larger one is tested by one warp
// against every box
#define SI_K 64
// candidate pairs per thread in the grid tier's count and write passes
#define SI_CHUNK 32
#define SI_AXIS_CELLS (1u << 20)

static unsigned mc_blocks(size_t n) { return n ? (unsigned)((n + MC_BLOCK - 1) / MC_BLOCK) : 1u; }

static int mc_invalid(const char *who, const char *what) {
    cphb_set_error("%s: %s", who, what);
    return CPHB_ERR_INVALID;
}
static const char *MC_BAD_INDEX = "a triangle's vertex index is outside [0, n_vertices)";

static int mc_bits(size_t n) {  // bits holding every value < n
    int b = 1;
    while (b < 32 && (n >> b) != 0) ++b;
    return b;
}

// CUB's exclusive sum of n u64 values (2 launches)
static int mc_scan_u64(cphb_scratch &sc, const unsigned long long *in, unsigned long long *out, size_t n, cudaStream_t s) {
    size_t tmp_bytes = 0;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, in, out, (int64_t)n, s));
    char *tmp = nullptr;
    const int rc = sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 16);
    if (rc) return rc;
    CPHB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int64_t)n, s));
    g_cphb_launches += 2;
    return CPHB_OK;
}

__device__ __forceinline__ bool mc_index_ok(int32_t v, size_t nv) { return v >= 0 && (size_t)v < nv; }

// ================================================================================================== lexicographic sort
// rows [n][3] u32 -> perm: the row indices in lexicographic order, stable (three stable passes, column 2 first)
__global__ void __launch_bounds__(MC_BLOCK) mc_gather_col_kernel(const uint32_t *__restrict__ rows, const uint32_t *__restrict__ perm,
                                                                 size_t n, int col, uint32_t *__restrict__ keys) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    keys[p] = rows[3 * (size_t)(perm ? perm[p] : p) + col];
}
__global__ void __launch_bounds__(MC_BLOCK) mc_iota_kernel(uint32_t *__restrict__ a, size_t n) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p < n) a[p] = (uint32_t)p;
}

// perm and tmp hold n + 1 entries; keys and skeys n
static int mc_lex_sort3(const uint32_t *rows, size_t n, int bits, uint32_t *keys, uint32_t *skeys, uint32_t *perm, uint32_t *tmp,
                        cudaStream_t s) {
    CPHB_LAUNCH(mc_iota_kernel, mc_blocks(n), MC_BLOCK, 0, s, perm, n);
    for (int col = 2; col >= 0; --col) {
        CPHB_LAUNCH(mc_gather_col_kernel, mc_blocks(n), MC_BLOCK, 0, s, rows, perm, n, col, keys);
        const int rc = cphb_sort_pairs_u32(keys, skeys, perm, tmp, n, bits, s);
        if (rc) return rc;
        CPHB_CUDA(cudaMemcpyAsync(perm, tmp, sizeof(uint32_t) * n, cudaMemcpyDeviceToDevice, s));
    }
    return CPHB_OK;
}

__device__ __forceinline__ bool mc_row_eq(const uint32_t *r, uint32_t a, uint32_t b) {
    return r[3 * (size_t)a] == r[3 * (size_t)b] && r[3 * (size_t)a + 1] == r[3 * (size_t)b + 1] && r[3 * (size_t)a + 2] == r[3 * (size_t)b + 2];
}

// ================================================================================================== RemoveDuplicatedVertices
// vertex i -> its canonical key row: f2ord(x + 0.0f) per axis (so -0 and +0 are one key), or all ones for a vertex with
// a NaN coordinate, which sorts last and merges with nothing
__global__ void __launch_bounds__(MC_BLOCK) mc_vertex_keys_kernel(const float *__restrict__ v, size_t nv, uint32_t *__restrict__ rows,
                                                                  uint8_t *__restrict__ nan) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= nv) return;
    const float x = v[3 * i] + 0.0f, y = v[3 * i + 1] + 0.0f, z = v[3 * i + 2] + 0.0f;
    const bool bad = x != x || y != y || z != z;
    nan[i] = bad;
    rows[3 * i] = bad ? 0xffffffffu : f2ord(x);
    rows[3 * i + 1] = bad ? 0xffffffffu : f2ord(y);
    rows[3 * i + 2] = bad ? 0xffffffffu : f2ord(z);
}

// head[p] = 1 when sorted position p starts a run of equal positions
__global__ void __launch_bounds__(MC_BLOCK) mc_vertex_heads_kernel(const uint32_t *__restrict__ rows, const uint32_t *__restrict__ perm,
                                                                   const uint8_t *__restrict__ nan, size_t n, unsigned long long *__restrict__ head) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    head[p] = p == 0 || nan[perm[p]] || !mc_row_eq(rows, perm[p], perm[p - 1]);
}

// position p of the sorted order, run number u = incl[p] - 1: the first of the run writes its vertex's attributes to
// row u, and every position maps its old index to u
__global__ void __launch_bounds__(MC_BLOCK) mc_vertex_write_kernel(const uint32_t *__restrict__ perm, const unsigned long long *__restrict__ head,
                                                                   const unsigned long long *__restrict__ excl, size_t n, const float *__restrict__ v,
                                                                   const float *__restrict__ vn, const float *__restrict__ vc,
                                                                   float *__restrict__ ov, float *__restrict__ on, float *__restrict__ oc,
                                                                   int32_t *__restrict__ old_to_new) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    const size_t i = perm[p];
    const size_t u = (size_t)(excl[p] + head[p]) - 1;
    old_to_new[i] = (int32_t)u;
    if (!head[p]) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ov[3 * u + k] = v[3 * i + k];
        if (vn) on[3 * u + k] = vn[3 * i + k];
        if (vc) oc[3 * u + k] = vc[3 * i + k];
    }
}

// every corner through old_to_new (the indices were checked before)
__global__ void __launch_bounds__(MC_BLOCK) mc_remap_kernel(const int32_t *__restrict__ tri, size_t nc, const int32_t *__restrict__ old_to_new,
                                                            int32_t *__restrict__ out) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k < nc) out[k] = old_to_new[tri[k]];
}

__global__ void __launch_bounds__(MC_BLOCK) mc_check_kernel(const int32_t *__restrict__ tri, size_t nc, size_t nv, int *__restrict__ bad) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k < nc && !mc_index_ok(tri[k], nv)) *bad = 1;
}

static int mc_check_indices(const int32_t *tri, size_t nt, size_t nv, const char *who, cudaStream_t s) {
    if (nt == 0) return CPHB_OK;
    cphb_scratch sc(s);
    int *bad = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_LAUNCH(mc_check_kernel, mc_blocks(3 * nt), MC_BLOCK, 0, s, tri, 3 * nt, nv, bad);
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    return h_bad ? mc_invalid(who, MC_BAD_INDEX) : CPHB_OK;
}

static int mc_check_sizes(size_t nv, size_t nt, const char *who) {
    if (nv > (size_t)INT32_MAX || nt > (size_t)INT32_MAX) return mc_invalid(who, "more than 2^31 - 1 vertices or triangles");
    return CPHB_OK;
}

extern "C" int cphb_mesh_remove_duplicated_vertices(const float *vertices, const float *vertex_normals, const float *vertex_colors,
                                                    size_t n_vertices, const int32_t *triangles, size_t n_triangles, float *out_vertices,
                                                    float *out_normals, float *out_colors, int32_t *out_triangles, size_t *h_n_vertices,
                                                    void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_remove_duplicated_vertices";
    if (!h_n_vertices) return mc_invalid(who, "null argument");
    *h_n_vertices = 0;
    int rc = mc_check_sizes(n_vertices, n_triangles, who);
    if (rc) return rc;
    if ((n_vertices && (!vertices || !out_vertices)) || (n_triangles && (!triangles || !out_triangles)) || (vertex_normals && !out_normals) ||
        (vertex_colors && !out_colors))
        return mc_invalid(who, "null argument");
    rc = mc_check_indices(triangles, n_triangles, n_vertices, who, s);
    if (rc || n_vertices == 0) return rc;
    const size_t n = n_vertices;
    cphb_scratch sc(s);
    uint32_t *rows = nullptr, *keys = nullptr, *skeys = nullptr, *perm = nullptr, *tmp = nullptr;
    uint8_t *nan = nullptr;
    unsigned long long *head = nullptr, *excl = nullptr;
    int32_t *o2n = nullptr;
    rc = sc.alloc(&rows, 3 * n);
    if (!rc) rc = sc.alloc(&keys, n);
    if (!rc) rc = sc.alloc(&skeys, n);
    if (!rc) rc = sc.alloc(&perm, n + 1);
    if (!rc) rc = sc.alloc(&tmp, n + 1);
    if (!rc) rc = sc.alloc(&nan, n);
    if (!rc) rc = sc.alloc(&head, n + 1);
    if (!rc) rc = sc.alloc(&excl, n + 1);
    if (!rc) rc = sc.alloc(&o2n, n);
    if (rc) return rc;
    CPHB_LAUNCH(mc_vertex_keys_kernel, mc_blocks(n), MC_BLOCK, 0, s, vertices, n, rows, nan);
    rc = mc_lex_sort3(rows, n, 32, keys, skeys, perm, tmp, s);
    if (rc) return rc;
    CPHB_LAUNCH(mc_vertex_heads_kernel, mc_blocks(n), MC_BLOCK, 0, s, rows, perm, nan, n, head);
    CPHB_CUDA(cudaMemsetAsync(head + n, 0, sizeof(unsigned long long), s));
    rc = mc_scan_u64(sc, head, excl, n + 1, s);
    if (rc) return rc;
    CPHB_LAUNCH(mc_vertex_write_kernel, mc_blocks(n), MC_BLOCK, 0, s, perm, head, excl, n, vertices, vertex_normals, vertex_colors,
                out_vertices, out_normals, out_colors, o2n);
    if (n_triangles)
        CPHB_LAUNCH(mc_remap_kernel, mc_blocks(3 * n_triangles), MC_BLOCK, 0, s, triangles, 3 * n_triangles, o2n, out_triangles);
    unsigned long long k = 0;
    rc = cphb_read_back(&k, excl + n, sizeof(k), s, who);
    if (rc) return rc;
    *h_n_vertices = (size_t)k;
    return CPHB_OK;
}

// ================================================================================================== RemoveDuplicatedTriangles
// align_triangle_functor (TM:95-105): rotate so the smallest index comes first, orientation kept
__global__ void __launch_bounds__(MC_BLOCK) mc_align_kernel(const int32_t *__restrict__ tri, size_t nt, uint32_t *__restrict__ rows) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const int32_t a = tri[3 * t], b = tri[3 * t + 1], c = tri[3 * t + 2];
    int32_t r0, r1, r2;
    if (a <= b) {
        if (a <= c) r0 = a, r1 = b, r2 = c;
        else r0 = c, r1 = a, r2 = b;
    } else {
        if (b <= c) r0 = b, r1 = c, r2 = a;
        else r0 = c, r1 = a, r2 = b;
    }
    rows[3 * t] = (uint32_t)r0;
    rows[3 * t + 1] = (uint32_t)r1;
    rows[3 * t + 2] = (uint32_t)r2;
}

__device__ __forceinline__ bool mc_tri_first(const uint32_t *rows, const uint32_t *perm, size_t p, size_t n) {
    return p < n && (p == 0 || !mc_row_eq(rows, perm[p], perm[p - 1]));
}
__global__ void __launch_bounds__(MC_BLOCK) mc_tri_unique_count_kernel(const uint32_t *__restrict__ rows, const uint32_t *__restrict__ perm,
                                                                       size_t n, unsigned *__restrict__ counts) {
    const unsigned c = block_flag_count(mc_tri_first(rows, perm, blockIdx.x * (size_t)blockDim.x + threadIdx.x, n));
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}
__global__ void __launch_bounds__(MC_BLOCK) mc_tri_unique_write_kernel(const uint32_t *__restrict__ rows, const uint32_t *__restrict__ perm,
                                                                       size_t n, const unsigned *__restrict__ offsets, const float *__restrict__ tn,
                                                                       int32_t *__restrict__ out, float *__restrict__ out_tn) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool f = mc_tri_first(rows, perm, p, n);
    const unsigned r = block_flag_rank(f);
    if (!f) return;
    const size_t o = offsets[blockIdx.x] + (size_t)r, t = perm[p];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out[3 * o + k] = (int32_t)rows[3 * t + k];
        if (tn) out_tn[3 * o + k] = tn[3 * t + k];
    }
}

extern "C" int cphb_mesh_remove_duplicated_triangles(const int32_t *triangles, const float *triangle_normals, size_t n_triangles,
                                                     size_t n_vertices, int32_t *out_triangles, float *out_triangle_normals,
                                                     size_t *h_n_triangles, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_remove_duplicated_triangles";
    if (!h_n_triangles) return mc_invalid(who, "null argument");
    *h_n_triangles = 0;
    int rc = mc_check_sizes(n_vertices, n_triangles, who);
    if (rc) return rc;
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || !out_triangles || (triangle_normals && !out_triangle_normals)) return mc_invalid(who, "null argument");
    rc = mc_check_indices(triangles, n_triangles, n_vertices, who, s);
    if (rc) return rc;
    const size_t n = n_triangles;
    const unsigned nb = mc_blocks(n);
    cphb_scratch sc(s);
    uint32_t *rows = nullptr, *keys = nullptr, *skeys = nullptr, *perm = nullptr, *tmp = nullptr;
    unsigned *counts = nullptr, *total = nullptr;
    rc = sc.alloc(&rows, 3 * n);
    if (!rc) rc = sc.alloc(&keys, n);
    if (!rc) rc = sc.alloc(&skeys, n);
    if (!rc) rc = sc.alloc(&perm, n + 1);
    if (!rc) rc = sc.alloc(&tmp, n + 1);
    if (!rc) rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (rc) return rc;
    CPHB_LAUNCH(mc_align_kernel, nb, MC_BLOCK, 0, s, triangles, n, rows);
    rc = mc_lex_sort3(rows, n, mc_bits(n_vertices), keys, skeys, perm, tmp, s);
    if (rc) return rc;
    CPHB_LAUNCH(mc_tri_unique_count_kernel, nb, MC_BLOCK, 0, s, rows, perm, n, counts);
    cphb_scan_block_counts(counts, nb, total, s);
    CPHB_LAUNCH(mc_tri_unique_write_kernel, nb, MC_BLOCK, 0, s, rows, perm, n, counts, triangle_normals, out_triangles, out_triangle_normals);
    unsigned k = 0;
    rc = cphb_read_back(&k, total, sizeof(k), s, who);
    if (rc) return rc;
    *h_n_triangles = k;
    return CPHB_OK;
}

// ================================================================================================== RemoveUnreferencedVertices
__global__ void __launch_bounds__(MC_BLOCK) mc_mark_kernel(const int32_t *__restrict__ tri, size_t nc, size_t nv, uint8_t *__restrict__ ref,
                                                           int *__restrict__ bad) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k >= nc) return;
    const int32_t v = tri[k];
    if (mc_index_ok(v, nv))
        ref[v] = 1;
    else
        *bad = 1;
}
__global__ void __launch_bounds__(MC_BLOCK) mc_ref_count_kernel(const uint8_t *__restrict__ ref, size_t n, unsigned *__restrict__ counts) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const unsigned c = block_flag_count(i < n && ref[i]);
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}
__global__ void __launch_bounds__(MC_BLOCK) mc_ref_write_kernel(const uint8_t *__restrict__ ref, size_t n, const unsigned *__restrict__ offsets,
                                                                const float *__restrict__ v, const float *__restrict__ vn,
                                                                const float *__restrict__ vc, float *__restrict__ ov, float *__restrict__ on,
                                                                float *__restrict__ oc, int32_t *__restrict__ old_to_new) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool f = i < n && ref[i];
    const unsigned r = block_flag_rank(f);
    if (!f) return;
    const size_t o = offsets[blockIdx.x] + (size_t)r;
    old_to_new[i] = (int32_t)o;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ov[3 * o + k] = v[3 * i + k];
        if (vn) on[3 * o + k] = vn[3 * i + k];
        if (vc) oc[3 * o + k] = vc[3 * i + k];
    }
}

extern "C" int cphb_mesh_remove_unreferenced_vertices(const float *vertices, const float *vertex_normals, const float *vertex_colors,
                                                      size_t n_vertices, const int32_t *triangles, size_t n_triangles, float *out_vertices,
                                                      float *out_normals, float *out_colors, int32_t *out_triangles, size_t *h_n_vertices,
                                                      void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_remove_unreferenced_vertices";
    if (!h_n_vertices) return mc_invalid(who, "null argument");
    *h_n_vertices = 0;
    int rc = mc_check_sizes(n_vertices, n_triangles, who);
    if (rc) return rc;
    if ((n_vertices && (!vertices || !out_vertices)) || (n_triangles && (!triangles || !out_triangles)) || (vertex_normals && !out_normals) ||
        (vertex_colors && !out_colors))
        return mc_invalid(who, "null argument");
    if (n_vertices == 0) return n_triangles ? mc_invalid(who, MC_BAD_INDEX) : CPHB_OK;
    const size_t n = n_vertices, nc = 3 * n_triangles;
    const unsigned nb = mc_blocks(n);
    cphb_scratch sc(s);
    uint8_t *ref = nullptr;
    int32_t *o2n = nullptr;
    unsigned *counts = nullptr, *total = nullptr;
    int *bad = nullptr;
    rc = sc.alloc(&ref, n);
    if (!rc) rc = sc.alloc(&o2n, n);
    if (!rc) rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (!rc) rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_CUDA(cudaMemsetAsync(ref, 0, n, s));
    if (nc) CPHB_LAUNCH(mc_mark_kernel, mc_blocks(nc), MC_BLOCK, 0, s, triangles, nc, n, ref, bad);
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    if (h_bad) return mc_invalid(who, MC_BAD_INDEX);
    CPHB_LAUNCH(mc_ref_count_kernel, nb, MC_BLOCK, 0, s, ref, n, counts);
    cphb_scan_block_counts(counts, nb, total, s);
    CPHB_LAUNCH(mc_ref_write_kernel, nb, MC_BLOCK, 0, s, ref, n, counts, vertices, vertex_normals, vertex_colors, out_vertices, out_normals,
                out_colors, o2n);
    if (nc) CPHB_LAUNCH(mc_remap_kernel, mc_blocks(nc), MC_BLOCK, 0, s, triangles, nc, o2n, out_triangles);
    unsigned k = 0;
    rc = cphb_read_back(&k, total, sizeof(k), s, who);
    if (rc) return rc;
    *h_n_vertices = k;
    return CPHB_OK;
}

// ================================================================================================== RemoveDegenerateTriangles
__device__ __forceinline__ bool mc_nondegenerate(const int32_t *tri, size_t t, size_t n) {
    if (t >= n) return false;
    const int32_t a = tri[3 * t], b = tri[3 * t + 1], c = tri[3 * t + 2];
    return a != b && b != c && c != a;
}
__global__ void __launch_bounds__(MC_BLOCK) mc_degen_count_kernel(const int32_t *__restrict__ tri, size_t n, unsigned *__restrict__ counts) {
    const unsigned c = block_flag_count(mc_nondegenerate(tri, blockIdx.x * (size_t)blockDim.x + threadIdx.x, n));
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}
__global__ void __launch_bounds__(MC_BLOCK) mc_degen_write_kernel(const int32_t *__restrict__ tri, size_t n, const unsigned *__restrict__ offsets,
                                                                  const float *__restrict__ tn, int32_t *__restrict__ out,
                                                                  float *__restrict__ out_tn) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool f = mc_nondegenerate(tri, t, n);
    const unsigned r = block_flag_rank(f);
    if (!f) return;
    const size_t o = offsets[blockIdx.x] + (size_t)r;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out[3 * o + k] = tri[3 * t + k];
        if (tn) out_tn[3 * o + k] = tn[3 * t + k];
    }
}

extern "C" int cphb_mesh_remove_degenerate_triangles(const int32_t *triangles, const float *triangle_normals, size_t n_triangles,
                                                     size_t n_vertices, int32_t *out_triangles, float *out_triangle_normals,
                                                     size_t *h_n_triangles, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_remove_degenerate_triangles";
    if (!h_n_triangles) return mc_invalid(who, "null argument");
    *h_n_triangles = 0;
    int rc = mc_check_sizes(n_vertices, n_triangles, who);
    if (rc) return rc;
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || !out_triangles || (triangle_normals && !out_triangle_normals)) return mc_invalid(who, "null argument");
    rc = mc_check_indices(triangles, n_triangles, n_vertices, who, s);
    if (rc) return rc;
    const unsigned nb = mc_blocks(n_triangles);
    cphb_scratch sc(s);
    unsigned *counts = nullptr, *total = nullptr;
    rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (rc) return rc;
    CPHB_LAUNCH(mc_degen_count_kernel, nb, MC_BLOCK, 0, s, triangles, n_triangles, counts);
    cphb_scan_block_counts(counts, nb, total, s);
    CPHB_LAUNCH(mc_degen_write_kernel, nb, MC_BLOCK, 0, s, triangles, n_triangles, counts, triangle_normals, out_triangles, out_triangle_normals);
    unsigned k = 0;
    rc = cphb_read_back(&k, total, sizeof(k), s, who);
    if (rc) return rc;
    *h_n_triangles = k;
    return CPHB_OK;
}

// ================================================================================================== operator+= (triangles)
__global__ void __launch_bounds__(MC_BLOCK) mc_append_kernel(const int32_t *__restrict__ a, size_t nca, size_t nva, const int32_t *__restrict__ b,
                                                             size_t ncb, size_t nvb, int32_t *__restrict__ out, int *__restrict__ bad) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k < nca) {
        const int32_t v = a[k];
        if (!mc_index_ok(v, nva)) *bad = 1;
        out[k] = v;
    } else if (k < nca + ncb) {
        const int32_t v = b[k - nca];
        if (!mc_index_ok(v, nvb)) *bad = 1;
        out[k] = (int32_t)((size_t)v + nva);
    }
}

extern "C" int cphb_mesh_append_triangles(const int32_t *triangles_a, size_t n_triangles_a, size_t n_vertices_a, const int32_t *triangles_b,
                                          size_t n_triangles_b, size_t n_vertices_b, int32_t *out_triangles, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_append_triangles";
    if (n_vertices_a + n_vertices_b > (size_t)INT32_MAX || n_triangles_a + n_triangles_b > (size_t)INT32_MAX)
        return mc_invalid(who, "more than 2^31 - 1 vertices or triangles");
    const size_t nc = 3 * (n_triangles_a + n_triangles_b);
    if (nc == 0) return CPHB_OK;
    if ((n_triangles_a && !triangles_a) || (n_triangles_b && !triangles_b) || !out_triangles) return mc_invalid(who, "null argument");
    cphb_scratch sc(s);
    int *bad = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_LAUNCH(mc_append_kernel, mc_blocks(nc), MC_BLOCK, 0, s, triangles_a, 3 * n_triangles_a, n_vertices_a, triangles_b, 3 * n_triangles_b,
                n_vertices_b, out_triangles, bad);
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    return h_bad ? mc_invalid(who, MC_BAD_INDEX) : CPHB_OK;
}

// ================================================================================================== the predicate
// NoDivTriTriIsect (Moller 1997, June 1999 revision; the reference's third_party/tomasakeninemoeller/opttritri.h) with
// USE_EPSILON_TEST, restated: same operand order, same comparisons.
__device__ __forceinline__ bool tt_edge_edge(float Ax, float Ay, const float *V0, const float *U0, const float *U1, int i0, int i1) {
    const float Bx = U0[i0] - U1[i0], By = U0[i1] - U1[i1], Cx = V0[i0] - U0[i0], Cy = V0[i1] - U0[i1];
    const float f = Ay * Bx - Ax * By, d = By * Cx - Bx * Cy;
    if ((f > 0 && d >= 0 && d <= f) || (f < 0 && d <= 0 && d >= f)) {
        const float e = Ax * Cy - Ay * Cx;
        if (f > 0) {
            if (e >= 0 && e <= f) return true;
        } else {
            if (e <= 0 && e >= f) return true;
        }
    }
    return false;
}
__device__ __forceinline__ bool tt_edge_tri(const float *V0, const float *V1, const float *U0, const float *U1, const float *U2, int i0, int i1) {
    const float Ax = V1[i0] - V0[i0], Ay = V1[i1] - V0[i1];
    return tt_edge_edge(Ax, Ay, V0, U0, U1, i0, i1) || tt_edge_edge(Ax, Ay, V0, U1, U2, i0, i1) || tt_edge_edge(Ax, Ay, V0, U2, U0, i0, i1);
}
__device__ __forceinline__ bool tt_point_in_tri(const float *V0, const float *U0, const float *U1, const float *U2, int i0, int i1) {
    float a = U1[i1] - U0[i1], b = -(U1[i0] - U0[i0]), c = -a * U0[i0] - b * U0[i1];
    const float d0 = a * V0[i0] + b * V0[i1] + c;
    a = U2[i1] - U1[i1];
    b = -(U2[i0] - U1[i0]);
    c = -a * U1[i0] - b * U1[i1];
    const float d1 = a * V0[i0] + b * V0[i1] + c;
    a = U0[i1] - U2[i1];
    b = -(U0[i0] - U2[i0]);
    c = -a * U2[i0] - b * U2[i1];
    const float d2 = a * V0[i0] + b * V0[i1] + c;
    return d0 * d1 > 0.0f && d0 * d2 > 0.0f;
}
__device__ __noinline__ bool tt_coplanar(const float *N, const float *V0, const float *V1, const float *V2, const float *U0, const float *U1,
                                         const float *U2) {
    const float A0 = fabsf(N[0]), A1 = fabsf(N[1]), A2 = fabsf(N[2]);
    int i0, i1;
    if (A0 > A1) {
        if (A0 > A2) i0 = 1, i1 = 2;
        else i0 = 0, i1 = 1;
    } else {
        if (A2 > A1) i0 = 0, i1 = 1;
        else i0 = 0, i1 = 2;
    }
    if (tt_edge_tri(V0, V1, U0, U1, U2, i0, i1) || tt_edge_tri(V1, V2, U0, U1, U2, i0, i1) || tt_edge_tri(V2, V0, U0, U1, U2, i0, i1))
        return true;
    return tt_point_in_tri(V0, U0, U1, U2, i0, i1) || tt_point_in_tri(U0, V0, V1, V2, i0, i1);
}

// NEWCOMPUTE_INTERVALS: false when the triangles are coplanar (the caller then runs the coplanar test)
__device__ __forceinline__ bool tt_intervals(float VV0, float VV1, float VV2, float D0, float D1, float D2, float D0D1, float D0D2, float &A,
                                             float &B, float &C, float &X0, float &X1) {
    if (D0D1 > 0.0f) {
        A = VV2; B = (VV0 - VV2) * D2; C = (VV1 - VV2) * D2; X0 = D2 - D0; X1 = D2 - D1;
    } else if (D0D2 > 0.0f) {
        A = VV1; B = (VV0 - VV1) * D1; C = (VV2 - VV1) * D1; X0 = D1 - D0; X1 = D1 - D2;
    } else if (D1 * D2 > 0.0f || D0 != 0.0f) {
        A = VV0; B = (VV1 - VV0) * D0; C = (VV2 - VV0) * D0; X0 = D0 - D1; X1 = D0 - D2;
    } else if (D1 != 0.0f) {
        A = VV1; B = (VV0 - VV1) * D1; C = (VV2 - VV1) * D1; X0 = D1 - D0; X1 = D1 - D2;
    } else if (D2 != 0.0f) {
        A = VV2; B = (VV0 - VV2) * D2; C = (VV1 - VV2) * D2; X0 = D2 - D0; X1 = D2 - D1;
    } else {
        return false;
    }
    return true;
}

__device__ __forceinline__ float tt_dot(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ void tt_cross(float *d, const float *a, const float *b) {
    d[0] = a[1] * b[2] - a[2] * b[1];
    d[1] = a[2] * b[0] - a[0] * b[2];
    d[2] = a[0] * b[1] - a[1] * b[0];
}
// FABS(x) < EPSILON with the published double EPSILON: the comparison is in double
__device__ __forceinline__ float tt_eps(float x) { return (double)fabsf(x) < 0.000001 ? 0.0f : x; }

__device__ bool tt_no_div_isect(const float *V0, const float *V1, const float *V2, const float *U0, const float *U1, const float *U2) {
    float E1[3], E2[3], N1[3], N2[3], D[3];
    E1[0] = V1[0] - V0[0]; E1[1] = V1[1] - V0[1]; E1[2] = V1[2] - V0[2];
    E2[0] = V2[0] - V0[0]; E2[1] = V2[1] - V0[1]; E2[2] = V2[2] - V0[2];
    tt_cross(N1, E1, E2);
    const float d1 = -tt_dot(N1, V0);
    const float du0 = tt_eps(tt_dot(N1, U0) + d1), du1 = tt_eps(tt_dot(N1, U1) + d1), du2 = tt_eps(tt_dot(N1, U2) + d1);
    const float du0du1 = du0 * du1, du0du2 = du0 * du2;
    if (du0du1 > 0.0f && du0du2 > 0.0f) return false;
    E1[0] = U1[0] - U0[0]; E1[1] = U1[1] - U0[1]; E1[2] = U1[2] - U0[2];
    E2[0] = U2[0] - U0[0]; E2[1] = U2[1] - U0[1]; E2[2] = U2[2] - U0[2];
    tt_cross(N2, E1, E2);
    const float d2 = -tt_dot(N2, U0);
    const float dv0 = tt_eps(tt_dot(N2, V0) + d2), dv1 = tt_eps(tt_dot(N2, V1) + d2), dv2 = tt_eps(tt_dot(N2, V2) + d2);
    const float dv0dv1 = dv0 * dv1, dv0dv2 = dv0 * dv2;
    if (dv0dv1 > 0.0f && dv0dv2 > 0.0f) return false;
    tt_cross(D, N1, N2);
    float mx = fabsf(D[0]);
    int index = 0;
    const float bb = fabsf(D[1]), cc = fabsf(D[2]);
    if (bb > mx) mx = bb, index = 1;
    if (cc > mx) mx = cc, index = 2;
    const float vp0 = V0[index], vp1 = V1[index], vp2 = V2[index];
    const float up0 = U0[index], up1 = U1[index], up2 = U2[index];
    float a, b, c, x0, x1;
    if (!tt_intervals(vp0, vp1, vp2, dv0, dv1, dv2, dv0dv1, dv0dv2, a, b, c, x0, x1)) return tt_coplanar(N1, V0, V1, V2, U0, U1, U2);
    float d, e, f, y0, y1;
    if (!tt_intervals(up0, up1, up2, du0, du1, du2, du0du1, du0du2, d, e, f, y0, y1)) return tt_coplanar(N1, V0, V1, V2, U0, U1, U2);
    const float xx = x0 * x1, yy = y0 * y1, xxyy = xx * yy;
    float tmp = a * xxyy;
    float i10 = tmp + b * x1 * yy, i11 = tmp + c * x0 * yy;
    tmp = d * xxyy;
    float i20 = tmp + e * xx * y1, i21 = tmp + f * xx * y0;
    if (i10 > i11) { const float t = i10; i10 = i11; i11 = t; }
    if (i20 > i21) { const float t = i20; i20 = i21; i21 = t; }
    return !(i11 < i20 || i21 < i10);
}

// intersection_test::TriangleTriangle3d (intersection_test.inl:47-69): the six vertices centred on their mean and
// divided by their per-axis deviation (sum of squares / 5, square root, + 1e-12), then NoDivTriTriIsect
__device__ bool tt_triangle_triangle(const float (&P)[3][3], const float (&Q)[3][3]) {
    float mu[3], sg[3], pm[3][3], qm[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        mu[k] = (P[0][k] + P[1][k] + P[2][k] + Q[0][k] + Q[1][k] + Q[2][k]) / 6.0f;
        float sq = 0.f;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const float dd = (j < 3 ? P[j][k] : Q[j - 3][k]) - mu[k];
            sq = j == 0 ? dd * dd : sq + dd * dd;
        }
        sg[k] = sqrtf(sq / 5.0f) + 1e-12f;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            pm[j][k] = (P[j][k] - mu[k]) / sg[k];
            qm[j][k] = (Q[j][k] - mu[k]) / sg[k];
        }
    }
    return tt_no_div_isect(pm[0], pm[1], pm[2], qm[0], qm[1], qm[2]);
}

// ================================================================================================== GetSelfIntersectingTriangles
struct SiGrid {
    float o[3];    // origin: the smallest minimum corner of the finite triangles' boxes
    float inv[3];  // 1 / cell size per axis
};

__device__ __forceinline__ uint32_t si_cell(float x, const SiGrid &g, int a) {
    const float c = fminf(floorf((x - g.o[a]) * g.inv[a]), (float)(SI_AXIS_CELLS - 1));
    return (uint32_t)fmaxf(c, 0.f);
}
__device__ __forceinline__ uint64_t si_key(uint32_t x, uint32_t y, uint32_t z) { return (uint64_t)x << 40 | (uint64_t)y << 20 | z; }

// per triangle: the box (lo xyz, hi xyz) and whether all nine coordinates are finite
struct SiBoxTerms {
    const float *vtx;
    size_t nv;
    const int32_t *tri;
    float *box;        // [nt][6]
    uint8_t *fin;      // [nt]
    unsigned *bounds;  // ordered-uint min xyz, max xyz over the finite boxes
    int *bad;
    // v[0]: the box's largest extent, v[1]: 1 for a finite triangle (both 0 otherwise)
    __device__ void operator()(size_t t, float (&v)[2]) const {
        v[0] = v[1] = 0.f;
        int32_t f[3];
        bool ok = true;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            f[j] = tri[3 * t + j];
            ok = ok && mc_index_ok(f[j], nv);
        }
        if (!ok) {
            *bad = 1;
            fin[t] = 0;
            return;
        }
        float lo[3], hi[3];
        bool finite = true;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float a = vtx[3 * (size_t)f[0] + k], b = vtx[3 * (size_t)f[1] + k], c = vtx[3 * (size_t)f[2] + k];
            finite = finite && isfinite(a) && isfinite(b) && isfinite(c);
            lo[k] = fminf(fminf(a, b), c);
            hi[k] = fmaxf(fmaxf(a, b), c);
        }
        fin[t] = finite;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            box[6 * t + k] = lo[k];
            box[6 * t + 3 + k] = hi[k];
        }
        if (!finite) return;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(bounds + k, f2ord(lo[k]));
            atomicMax(bounds + 3 + k, f2ord(hi[k]));
        }
        v[0] = fmaxf(fmaxf(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2]);
        v[1] = 1.f;
    }
};

__device__ __forceinline__ void si_range(const float *bx, const SiGrid &g, uint32_t (&c0)[3], uint32_t (&c1)[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        c0[a] = si_cell(bx[a], g, a);
        c1[a] = si_cell(bx[3 + a], g, a);
    }
}

// per triangle: the number of grid entries (its cells when it covers at most SI_K, else 0) and whether it is large;
// the block's count of large triangles to lcounts
__global__ void __launch_bounds__(MC_BLOCK) si_cells_kernel(const float *__restrict__ box, const uint8_t *__restrict__ fin, size_t nt, SiGrid g,
                                                            unsigned long long *__restrict__ ecount, uint8_t *__restrict__ large,
                                                            unsigned *__restrict__ lcounts) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    bool big = false;
    if (t < nt) {
        unsigned long long c = 0;
        if (fin[t]) {
            uint32_t c0[3], c1[3];
            si_range(box + 6 * t, g, c0, c1);
            const unsigned long long cells = (unsigned long long)(c1[0] - c0[0] + 1) * (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
            big = cells > SI_K;
            c = big ? 0ull : cells;
        }
        ecount[t] = c;
        large[t] = big;
    } else if (t == nt) {
        ecount[t] = 0ull;
    }
    const unsigned n = block_flag_count(big);
    if (threadIdx.x == 0) lcounts[blockIdx.x] = n;
}

// per triangle: its (cell key, triangle) entries from eoff[t], cells in (x, y, z) order; a large triangle's index to
// lids at its rank
__global__ void __launch_bounds__(MC_BLOCK) si_entries_kernel(const float *__restrict__ box, const uint8_t *__restrict__ large, size_t nt,
                                                              SiGrid g, const unsigned long long *__restrict__ eoff, const unsigned *__restrict__ loff,
                                                              uint64_t *__restrict__ keys, uint32_t *__restrict__ vals, uint32_t *__restrict__ lids) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool big = t < nt && large[t];
    const unsigned r = block_flag_rank(big);
    if (t >= nt) return;
    if (big) {
        lids[loff[blockIdx.x] + r] = (uint32_t)t;
        return;
    }
    unsigned long long o = eoff[t];
    if (eoff[t + 1] == o) return;
    uint32_t c0[3], c1[3];
    si_range(box + 6 * t, g, c0, c1);
    for (uint32_t x = c0[0]; x <= c1[0]; ++x)
        for (uint32_t y = c0[1]; y <= c1[1]; ++y)
            for (uint32_t z = c0[2]; z <= c1[2]; ++z) {
                keys[o] = si_key(x, y, z);
                vals[o] = (uint32_t)t;
                ++o;
            }
}

// sorted entry p: the number of later entries in its cell (each pair of a cell is enumerated from its first entry)
__global__ void __launch_bounds__(MC_BLOCK) si_run_kernel(const uint64_t *__restrict__ k, size_t ne, unsigned long long *__restrict__ pc) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p > ne) return;
    if (p == ne) {
        pc[p] = 0ull;
        return;
    }
    const uint64_t key = k[p];
    size_t lo = p + 1, hi = ne;  // first entry after p with a larger key
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (k[mid] <= key)
            lo = mid + 1;
        else
            hi = mid;
    }
    pc[p] = lo - p - 1;
}

struct SiView {
    const float *vtx;
    const int32_t *tri;
    const float *box;
    const uint8_t *fin, *large;
    size_t nt;
};

__device__ __forceinline__ bool si_overlap(const float *a, const float *b) {
    return a[0] <= b[3] && b[0] <= a[3] && a[1] <= b[4] && b[1] <= a[4] && a[2] <= b[5] && b[2] <= a[5];
}
__device__ __forceinline__ bool si_share(const int32_t *a, const int32_t *b) {
    return a[0] == b[0] || a[0] == b[1] || a[0] == b[2] || a[1] == b[0] || a[1] == b[1] || a[1] == b[2] || a[2] == b[0] || a[2] == b[1] ||
           a[2] == b[2];
}
// i < j, both finite, boxes overlapping, no shared index: the predicate
__device__ __forceinline__ bool si_test(const SiView &v, size_t i, size_t j) {
    float P[3][3], Q[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            P[c][k] = v.vtx[3 * (size_t)v.tri[3 * i + c] + k];
            Q[c][k] = v.vtx[3 * (size_t)v.tri[3 * j + c] + k];
        }
    return tt_triangle_triangle(P, Q);
}

// grid candidate (entry p, its partner q = p + 1 + r in the same cell): 0 not a candidate, 1 a miss, 2 a hit; the pair
// to (i, j)
__device__ __forceinline__ int si_grid_pair(const SiView &v, const SiGrid &g, const uint64_t *keys, const uint32_t *vals, size_t p, size_t q,
                                            size_t &i, size_t &j) {
    const size_t a = vals[p], b = vals[q];
    i = a < b ? a : b;
    j = a < b ? b : a;
    const float *bi = v.box + 6 * i, *bj = v.box + 6 * j;
    if (!si_overlap(bi, bj) || si_share(v.tri + 3 * i, v.tri + 3 * j)) return 0;
    // ownership: only the cell holding the maximum of the two minimum corners tests the pair
    const uint64_t own = si_key(si_cell(fmaxf(bi[0], bj[0]), g, 0), si_cell(fmaxf(bi[1], bj[1]), g, 1), si_cell(fmaxf(bi[2], bj[2]), g, 2));
    if (own != keys[p]) return 0;
    return si_test(v, i, j) ? 2 : 1;
}

// thread w of the grid tier: candidates [w SI_CHUNK, (w + 1) SI_CHUNK) of the T enumerated in (entry, partner) order.
// WRITE 0 counts hits to hc[w] and adds the tested pairs to *cand; WRITE 1 writes the hit keys i n_t + j from hoff[w].
template <int WRITE>
__global__ void __launch_bounds__(MC_BLOCK) si_grid_kernel(SiView v, SiGrid g, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                           const unsigned long long *__restrict__ poff, size_t ne, unsigned long long T, size_t nw,
                                                           unsigned long long *__restrict__ hc, unsigned long long *__restrict__ cand,
                                                           uint64_t *__restrict__ out) {
    const size_t w = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    unsigned long long tested = 0, hits = 0;
    if (w < nw) {
        unsigned long long c = (unsigned long long)w * SI_CHUNK;
        const unsigned long long end = min(c + SI_CHUNK, T);
        size_t lo = 0, hi = ne;  // the entry whose range [poff[p], poff[p + 1]) holds c
        while (lo < hi) {
            const size_t mid = (lo + hi + 1) / 2;
            if (poff[mid] <= c)
                lo = mid;
            else
                hi = mid - 1;
        }
        size_t p = lo;
        unsigned long long o = WRITE ? hc[w] : 0ull;
        for (; c < end; ++c) {
            while (poff[p + 1] <= c) ++p;
            size_t i, j;
            const int r = si_grid_pair(v, g, keys, vals, p, p + 1 + (size_t)(c - poff[p]), i, j);
            tested += r != 0;
            if (r == 2) {
                if (WRITE) out[o] = (uint64_t)i * v.nt + j;
                ++o;
                ++hits;
            }
        }
        if (!WRITE) hc[w] = hits;
    }
    if (!WRITE) {
        tested = __reduce_add_sync(CPHB_FULL, (unsigned)tested);
        if (lane_id() == 0 && tested) atomicAdd(cand, tested);
    }
}

// warp l of the large tier: large triangle L = lids[l] against every triangle m.  The pair belongs here when m is small,
// or when m is large and L < m.  WRITE as si_grid_kernel, counts to hc[l], keys from hoff[l], in ascending m.
template <int WRITE>
__global__ void __launch_bounds__(MC_BLOCK) si_large_kernel(SiView v, const uint32_t *__restrict__ lids, size_t nl,
                                                            unsigned long long *__restrict__ hc, unsigned long long *__restrict__ cand,
                                                            uint64_t *__restrict__ out) {
    const size_t l = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    if (l >= nl) return;
    const size_t L = lids[l];
    const float *bl = v.box + 6 * L;
    unsigned long long o = WRITE ? hc[l] : 0ull, tested = 0;
    for (size_t base = 0; base < v.nt; base += 32) {
        const size_t m = base + lane_id();
        bool hit = false;
        if (m < v.nt && m != L && v.fin[m] && (!v.large[m] || L < m) && si_overlap(bl, v.box + 6 * m) &&
            !si_share(v.tri + 3 * L, v.tri + 3 * m)) {
            ++tested;
            hit = L < m ? si_test(v, L, m) : si_test(v, m, L);
        }
        const unsigned bal = __ballot_sync(CPHB_FULL, hit);
        if (WRITE && hit) {
            const size_t i = L < m ? L : m, j = L < m ? m : L;
            out[o + __popc(bal & ((1u << lane_id()) - 1u))] = (uint64_t)i * v.nt + j;
        }
        o += __popc(bal);
    }
    if (!WRITE) {
        tested = __reduce_add_sync(CPHB_FULL, (unsigned)tested);
        if (lane_id() == 0) {
            hc[l] = o;
            if (tested) atomicAdd(cand, tested);
        }
    }
}

__global__ void __launch_bounds__(MC_BLOCK) si_pairs_kernel(const uint64_t *__restrict__ k, size_t n, size_t nt, int32_t *__restrict__ pairs) {
    const size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    pairs[2 * p] = (int32_t)(k[p] / nt);
    pairs[2 * p + 1] = (int32_t)(k[p] % nt);
}

extern "C" int cphb_mesh_self_intersecting_triangles(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                                     int32_t *pairs, size_t capacity, size_t *h_n_pairs, size_t *h_n_candidates,
                                                     void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_self_intersecting_triangles";
    if (!h_n_pairs) return mc_invalid(who, "null argument");
    *h_n_pairs = 0;
    if (h_n_candidates) *h_n_candidates = 0;
    int rc = mc_check_sizes(n_vertices, n_triangles, who);
    if (rc) return rc;
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || (n_vertices && !vertices) || (capacity && !pairs)) return mc_invalid(who, "null argument");
    const size_t nt = n_triangles;

    // 1. boxes, finiteness, the mesh box and the mean largest extent (float64, fixed order)
    cphb_scratch sa(s);
    float *box = nullptr;
    uint8_t *fin = nullptr, *large = nullptr;
    unsigned *bounds = nullptr;
    int *bad = nullptr;
    unsigned long long *meta = nullptr;  // E, T, H, candidates
    rc = sa.alloc(&box, 6 * nt);
    if (!rc) rc = sa.alloc(&fin, nt);
    if (!rc) rc = sa.alloc(&large, nt);
    if (!rc) rc = sa.alloc(&bounds, 6);
    if (!rc) rc = sa.alloc(&bad, 1);
    if (!rc) rc = sa.alloc(&meta, 4);
    if (rc) return rc;
    const unsigned init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
    CPHB_CUDA(cudaMemcpyAsync(bounds, init, sizeof(init), cudaMemcpyHostToDevice, s));
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_CUDA(cudaMemsetAsync(meta, 0, 4 * sizeof(unsigned long long), s));
    double sums[2] = {0.0, 0.0};
    rc = sum_values<2>(SiBoxTerms{vertices, n_vertices, triangles, box, fin, bounds, bad}, nt, sums, s);
    if (rc) return rc;
    int h_bad = 0;
    unsigned h_bounds[6];
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (!rc) rc = cphb_read_back(h_bounds, bounds, sizeof(h_bounds), s, who);
    if (rc) return rc;
    if (h_bad) return mc_invalid(who, MC_BAD_INDEX);
    // cell size per axis: the mean largest box extent, raised to the mesh box's extent / 2^20 (at most 2^20 cells per
    // axis, so a key fits 60 bits) and to 1e-30 (a finite 1 / h); cell(x) = clamp(floor((x - o) * inv), 0, 2^20 - 1)
    SiGrid g;
    const double mean = sums[1] > 0.0 ? sums[0] / sums[1] : 1.0;
    for (int a = 0; a < 3; ++a) {
        const bool any = sums[1] > 0.0;
        const float lo = any ? ord2f(h_bounds[a]) : 0.f, hi = any ? ord2f(h_bounds[3 + a]) : 0.f;
        double h = mean;
        const double ext = ((double)hi - (double)lo) / (double)SI_AXIS_CELLS;
        if (ext > h) h = ext;
        if (!(h >= 1e-30)) h = h > 0.0 ? 1e-30 : 1.0;
        g.o[a] = lo;
        g.inv[a] = (float)(1.0 / h);
    }

    // 2. grid entries of the small triangles, and the list of the large ones
    const unsigned nbt = mc_blocks(nt + 1);
    cphb_scratch sb(s);
    unsigned long long *ecount = nullptr, *eoff = nullptr;
    unsigned *lcounts = nullptr, *ltotal = nullptr;
    uint32_t *lids = nullptr;
    rc = sb.alloc(&ecount, nt + 1);
    if (!rc) rc = sb.alloc(&eoff, nt + 1);
    if (!rc) rc = sb.alloc(&lcounts, (size_t)nbt + 4);
    if (!rc) rc = sb.alloc(&ltotal, 1);
    if (!rc) rc = sb.alloc(&lids, nt);
    if (rc) return rc;
    CPHB_LAUNCH(si_cells_kernel, nbt, MC_BLOCK, 0, s, box, fin, nt, g, ecount, large, lcounts);
    rc = mc_scan_u64(sb, ecount, eoff, nt + 1, s);
    if (rc) return rc;
    cphb_scan_block_counts(lcounts, nbt, ltotal, s);
    unsigned long long h_E = 0;
    unsigned h_L = 0;
    rc = cphb_read_back(&h_E, eoff + nt, sizeof(h_E), s, who);
    if (!rc) rc = cphb_read_back(&h_L, ltotal, sizeof(h_L), s, who);
    if (rc) return rc;
    if (h_E > (unsigned long long)INT32_MAX - 1) return mc_invalid(who, "2^31 - 1 or more grid entries");
    const size_t ne = (size_t)h_E, nl = h_L;
    cphb_scratch sc(s);
    uint64_t *keys = nullptr, *skeys = nullptr;
    uint32_t *vals = nullptr, *svals = nullptr;
    unsigned long long *pc = nullptr, *poff = nullptr;
    rc = sc.alloc(&keys, ne + 1);
    if (!rc) rc = sc.alloc(&skeys, ne + 1);
    if (!rc) rc = sc.alloc(&vals, ne + 1);
    if (!rc) rc = sc.alloc(&svals, ne + 1);
    if (!rc) rc = sc.alloc(&pc, ne + 1);
    if (!rc) rc = sc.alloc(&poff, ne + 1);
    if (rc) return rc;
    if (ne == 0) CPHB_CUDA(cudaMemsetAsync(keys, 0, sizeof(uint64_t), s));
    CPHB_LAUNCH(si_entries_kernel, nbt, MC_BLOCK, 0, s, box, large, nt, g, eoff, lcounts, keys, vals, lids);
    rc = cphb_sort_pairs_u64(keys, skeys, vals, svals, ne ? ne : 1, 60, s);  // one dummy entry keeps the launch count fixed
    if (rc) return rc;
    CPHB_LAUNCH(si_run_kernel, mc_blocks(ne + 1), MC_BLOCK, 0, s, skeys, ne, pc);
    rc = mc_scan_u64(sc, pc, poff, ne + 1, s);
    if (rc) return rc;
    unsigned long long h_T = 0;
    rc = cphb_read_back(&h_T, poff + ne, sizeof(h_T), s, who);
    if (rc) return rc;

    // 3. count the hits of both tiers, scan, and write them when they fit
    const size_t nw = (size_t)((h_T + SI_CHUNK - 1) / SI_CHUNK);
    if (nw >= (size_t)INT32_MAX * MC_BLOCK) return mc_invalid(who, "2^44 or more candidate pairs in the grid");
    cphb_scratch sd(s);
    unsigned long long *hc = nullptr, *hoff = nullptr;
    rc = sd.alloc(&hc, nw + nl + 1);
    if (!rc) rc = sd.alloc(&hoff, nw + nl + 1);
    if (rc) return rc;
    const SiView v = {vertices, triangles, box, fin, large, nt};
    CPHB_CUDA(cudaMemsetAsync(hc + nw + nl, 0, sizeof(unsigned long long), s));
    CPHB_LAUNCH(si_grid_kernel<0>, mc_blocks(nw), MC_BLOCK, 0, s, v, g, skeys, svals, poff, ne, h_T, nw, hc, meta + 3, nullptr);
    CPHB_LAUNCH(si_large_kernel<0>, mc_blocks(32 * nl), MC_BLOCK, 0, s, v, lids, nl, hc + nw, meta + 3, nullptr);
    rc = mc_scan_u64(sd, hc, hoff, nw + nl + 1, s);
    if (rc) return rc;
    unsigned long long h_H = 0, h_C = 0;
    rc = cphb_read_back(&h_H, hoff + nw + nl, sizeof(h_H), s, who);
    if (!rc) rc = cphb_read_back(&h_C, meta + 3, sizeof(h_C), s, who);
    if (rc) return rc;
    if (h_H > (unsigned long long)INT32_MAX - 1) return mc_invalid(who, "2^31 - 1 or more intersecting pairs");
    *h_n_pairs = (size_t)h_H;
    if (h_n_candidates) *h_n_candidates = (size_t)h_C;
    if (!pairs || capacity < h_H) return CPHB_OK;
    const size_t nh = (size_t)h_H;
    uint64_t *hk = nullptr, *shk = nullptr;
    rc = sd.alloc(&hk, nh + 1);
    if (!rc) rc = sd.alloc(&shk, nh + 1);
    if (rc) return rc;
    if (nh == 0) CPHB_CUDA(cudaMemsetAsync(hk, 0, sizeof(uint64_t), s));
    CPHB_LAUNCH(si_grid_kernel<1>, mc_blocks(nw), MC_BLOCK, 0, s, v, g, skeys, svals, poff, ne, h_T, nw, hoff, nullptr, hk);
    CPHB_LAUNCH(si_large_kernel<1>, mc_blocks(32 * nl), MC_BLOCK, 0, s, v, lids, nl, hoff + nw, nullptr, hk);
    rc = cphb_sort_keys_u64(hk, shk, nh ? nh : 1, 62, s);  // i n_t + j < 2^62
    if (rc) return rc;
    CPHB_LAUNCH(si_pairs_kernel, mc_blocks(nh), MC_BLOCK, 0, s, shk, nh, nt, pairs);
    return cphb_read_back(nullptr, nullptr, 0, s, who);
}
