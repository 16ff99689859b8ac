// mesh.cu -- TriangleMesh::ComputeTriangleNormals and ComputeVertexNormals (DESIGN section 4 item 19), ComputeEdgeList,
// the four vertex filters, GetSurfaceArea and SamplePointsUniformly (item 24).  Reference: geometry/trianglemesh.cu (TM).
//
// Triangle normals are one thread per triangle.  Vertex normals sort the 3 m triangle corners by vertex (CUB's stable
// radix sort, so each vertex's corners stay in ascending (triangle, corner) order, the order of the reference's
// stable sort_by_key + reduce_by_key), then one thread per vertex finds its run by binary search and adds its
// triangles' normals left to right: deterministic, no float atomics.  A vertex in no triangle gets a zero normal,
// so vertex_normals stays aligned with vertices.
//
// Arithmetic: IEEE, no contraction (build.py's -fmad=false); the cross product is a1 b2 - a2 b1 ..., the normalisation
// is NormalizeNormals' rule, cphb_normalize3 (cphb_internal.cuh), which cphb_normalize_normals uses too.  oracle/tsdf_mesh.c
// states the same.
#include <math.h>

#include "cphb_internal.cuh"
#include "minstd.cuh"
#include "sum_values.cuh"

static unsigned mesh_blocks(size_t n, unsigned b) { return n ? (unsigned)((n + b - 1) / b) : 1u; }

static int mesh_invalid(const char *who, const char *what) {
    cphb_set_error("%s: %s", who, what);
    return CPHB_ERR_INVALID;
}

// compute_triangle_normals_functor (TM:466-477): (v1 - v0) x (v2 - v0); an index outside [0, nv) sets *bad
__global__ void __launch_bounds__(256) mesh_triangle_normals_kernel(const float *__restrict__ vtx, size_t nv, const int32_t *__restrict__ tri,
                                                                    size_t nt, int normalized, float *__restrict__ out, int *__restrict__ bad) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= nt) return;
    int32_t f[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        f[j] = tri[3 * t + j];
        if (f[j] < 0 || (size_t)f[j] >= nv) {
            *bad = 1;
            return;
        }
    }
    float a[3], b[3], n[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        a[k] = vtx[3 * (size_t)f[1] + k] - vtx[3 * (size_t)f[0] + k];
        b[k] = vtx[3 * (size_t)f[2] + k] - vtx[3 * (size_t)f[0] + k];
    }
    n[0] = a[1] * b[2] - a[2] * b[1];
    n[1] = a[2] * b[0] - a[0] * b[2];
    n[2] = a[0] * b[1] - a[1] * b[0];
    if (normalized) cphb_normalize3(n);
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * t + k] = n[k];
}

extern "C" int cphb_mesh_triangle_normals(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                          int normalized, float *triangle_normals, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_triangle_normals";
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || !triangle_normals || (n_vertices && !vertices)) return mesh_invalid(who, "null argument");
    cphb_scratch sc(s);
    int *bad = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_LAUNCH(mesh_triangle_normals_kernel, mesh_blocks(n_triangles, 256), 256, 0, s, vertices, n_vertices, triangles, n_triangles,
                normalized ? 1 : 0, triangle_normals, bad);
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    return h_bad ? mesh_invalid(who, "a triangle's vertex index is outside [0, n_vertices)") : CPHB_OK;
}

// corner k of the flattened triangle array: key = its vertex (n_vertices for an index out of range, which sorts last
// and sets *bad), value = k
__global__ void __launch_bounds__(256) mesh_corner_keys_kernel(const int32_t *__restrict__ tri, size_t nc, size_t nv,
                                                               uint32_t *__restrict__ keys, uint32_t *__restrict__ vals, int *__restrict__ bad) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k >= nc) return;
    const int32_t v = tri[k];
    const bool ok = v >= 0 && (size_t)v < nv;
    if (!ok) *bad = 1;
    keys[k] = ok ? (uint32_t)v : (uint32_t)nv;
    vals[k] = (uint32_t)k;
}

// vertex v: the sum of the normals of its corners' triangles, in the sorted (ascending corner) order, starting from the
// first term; 0 for a vertex in no triangle
__global__ void __launch_bounds__(256) mesh_vertex_normals_kernel(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                                  size_t nc, const float *__restrict__ tn, size_t nv, int normalized,
                                                                  float *__restrict__ out) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v >= nv) return;
    size_t lo = 0, hi = nc;  // first sorted corner with key >= v
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (keys[mid] < (uint32_t)v)
            lo = mid + 1;
        else
            hi = mid;
    }
    float n[3] = {0.f, 0.f, 0.f};
    for (size_t k = lo; k < nc && keys[k] == (uint32_t)v; ++k) {
        const size_t t = vals[k] / 3;
#pragma unroll
        for (int a = 0; a < 3; ++a) n[a] = k == lo ? tn[3 * t + a] : n[a] + tn[3 * t + a];
    }
    if (normalized) cphb_normalize3(n);
#pragma unroll
    for (int a = 0; a < 3; ++a) out[3 * v + a] = n[a];
}

extern "C" int cphb_mesh_vertex_normals(const int32_t *triangles, size_t n_triangles, const float *triangle_normals, size_t n_vertices,
                                        int normalized, float *vertex_normals, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_vertex_normals";
    if (n_vertices == 0 && n_triangles == 0) return CPHB_OK;
    if ((n_vertices && !vertex_normals) || (n_triangles && (!triangles || !triangle_normals))) return mesh_invalid(who, "null argument");
    const size_t nc = 3 * n_triangles;
    // the sort takes int32 counts and uint32 keys up to n_vertices
    if (nc > (size_t)INT32_MAX || n_vertices > (size_t)INT32_MAX) return mesh_invalid(who, "more than 2^31 - 1 corners or vertices");
    cphb_scratch sc(s);
    int *bad = nullptr;
    uint32_t *keys = nullptr, *vals = nullptr, *skeys = nullptr, *svals = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (!rc) rc = sc.alloc(&keys, nc + 1);
    if (!rc) rc = sc.alloc(&vals, nc + 1);
    if (!rc) rc = sc.alloc(&skeys, nc + 1);
    if (!rc) rc = sc.alloc(&svals, nc + 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_LAUNCH(mesh_corner_keys_kernel, mesh_blocks(nc, 256), 256, 0, s, triangles, nc, n_vertices, keys, vals, bad);
    int bits = 1;
    while (bits < 32 && (n_vertices >> bits) != 0) ++bits;  // keys are <= n_vertices
    rc = cphb_sort_pairs_u32(keys, skeys, vals, svals, nc, bits, s);
    if (rc) return rc;
    CPHB_LAUNCH(mesh_vertex_normals_kernel, mesh_blocks(n_vertices, 256), 256, 0, s, skeys, svals, nc, triangle_normals, n_vertices,
                normalized ? 1 : 0, vertex_normals);
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    return h_bad ? mesh_invalid(who, "a triangle's vertex index is outside [0, n_vertices)") : CPHB_OK;
}

// ================================================================================================== ComputeEdgeList
// compute_edge_list_functor (TM:54-74): the 6 directed edges of triangle t, as (u64)a << 32 | b, at 6 t .. 6 t + 5.  An
// index outside [0, nv) sets *bad (its edges are then made of vertex 0).
__global__ void __launch_bounds__(256) mesh_edge_keys_kernel(const int32_t *__restrict__ tri, size_t nt, size_t nv, uint64_t *__restrict__ keys,
                                                             uint32_t *__restrict__ vals, int *__restrict__ bad) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= nt) return;
    int32_t f[3];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        f[j] = tri[3 * t + j];
        ok = ok && f[j] >= 0 && (size_t)f[j] < nv;
    }
    if (!ok) {
        *bad = 1;
        f[0] = f[1] = f[2] = 0;
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const uint64_t lo = (uint32_t)min(f[j], f[(j + 1) % 3]), hi = (uint32_t)max(f[j], f[(j + 1) % 3]);
        keys[6 * t + 2 * j] = lo << 32 | hi;
        keys[6 * t + 2 * j + 1] = hi << 32 | lo;
        vals[6 * t + 2 * j] = vals[6 * t + 2 * j + 1] = 0u;
    }
}

// thrust::unique of the sorted keys as a block compaction: a key is kept when it differs from its predecessor
__device__ __forceinline__ bool mesh_edge_first(const uint64_t *k, size_t i, size_t n) { return i < n && (i == 0 || k[i] != k[i - 1]); }
__global__ void __launch_bounds__(256) mesh_edge_count_kernel(const uint64_t *__restrict__ k, size_t n, unsigned *__restrict__ counts) {
    const unsigned c = block_flag_count(mesh_edge_first(k, blockIdx.x * (size_t)blockDim.x + threadIdx.x, n));
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}
// rows are written only when the total fits the capacity
__global__ void __launch_bounds__(256) mesh_edge_write_kernel(const uint64_t *__restrict__ k, size_t n, const unsigned *__restrict__ offsets,
                                                              const unsigned *__restrict__ total, size_t capacity, int32_t *__restrict__ edges) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const bool v = mesh_edge_first(k, i, n);
    const unsigned r = block_flag_rank(v);
    if (v && edges && *total <= capacity) {
        const size_t o = offsets[blockIdx.x] + (size_t)r;
        edges[2 * o] = (int32_t)(k[i] >> 32);
        edges[2 * o + 1] = (int32_t)(uint32_t)k[i];
    }
}

extern "C" int cphb_mesh_edge_list(const int32_t *triangles, size_t n_triangles, size_t n_vertices, int32_t *edges, size_t capacity,
                                   size_t *h_n_edges, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_edge_list";
    if (!h_n_edges) return mesh_invalid(who, "null argument");
    *h_n_edges = 0;
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || (capacity && !edges)) return mesh_invalid(who, "null argument");
    const size_t ne = 6 * n_triangles;
    if (ne > (size_t)INT32_MAX || n_vertices > (size_t)INT32_MAX) return mesh_invalid(who, "more than 2^31 - 1 directed edges or vertices");
    const unsigned nb = (unsigned)((ne + 255) / 256);
    cphb_scratch sc(s);
    int *bad = nullptr;
    uint64_t *keys = nullptr, *skeys = nullptr;
    uint32_t *vals = nullptr, *svals = nullptr;
    unsigned *counts = nullptr, *total = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (!rc) rc = sc.alloc(&keys, ne);
    if (!rc) rc = sc.alloc(&skeys, ne);
    if (!rc) rc = sc.alloc(&vals, ne);
    if (!rc) rc = sc.alloc(&svals, ne);
    if (!rc) rc = sc.alloc(&counts, (size_t)nb + 4);
    if (!rc) rc = sc.alloc(&total, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    CPHB_LAUNCH(mesh_edge_keys_kernel, mesh_blocks(n_triangles, 256), 256, 0, s, triangles, n_triangles, n_vertices, keys, vals, bad);
    int bits = 1;
    while (bits < 32 && (n_vertices >> bits) != 0) ++bits;  // both halves are < n_vertices
    rc = cphb_sort_pairs_u64(keys, skeys, vals, svals, ne, 32 + bits, s);
    if (rc) return rc;
    CPHB_LAUNCH(mesh_edge_count_kernel, nb, 256, 0, s, skeys, ne, counts);
    cphb_scan_block_counts(counts, nb, total, s);
    CPHB_LAUNCH(mesh_edge_write_kernel, nb, 256, 0, s, skeys, ne, counts, total, edges ? capacity : 0, edges);
    int h_bad = 0;
    unsigned h_total = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (!rc) rc = cphb_read_back(&h_total, total, sizeof(unsigned), s, who);
    if (rc) return rc;
    if (h_bad) return mesh_invalid(who, "a triangle's vertex index is outside [0, n_vertices)");
    *h_n_edges = h_total;
    return CPHB_OK;
}

// ================================================================================================== the filters
// Per call: the edge list is checked (every index in [0, nv), pairs in non-decreasing (v, nb) order), vertex v's row
// [rows[v], rows[v + 1]) is found by binary search, and for Laplacian / Taubin the edge weights
// (float)(1.0 / ((double)|v_a - v_b| + 1e-12)) and each row's float sum of them are computed once from the input
// vertices (compute_weights_from_edges_functor, TM:121-129).  Then one launch per pass: thread v reads its row once per
// filtered attribute and sums the neighbours' values (weighted for Laplacian) left to right from the first term.  A
// vertex with an empty row keeps its value.  Every kernel after the check returns at once when the check failed, so
// bad edges are never followed; the host reads the flag once, at the end.
struct MeshPass {
    const float *in[3];  // vertices, normals, colours being filtered; NULL: not filtered
    float *out[3];
};

__global__ void __launch_bounds__(256) mesh_edges_check_kernel(const int32_t *__restrict__ e, size_t ne, size_t nv, int *__restrict__ bad) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= ne) return;
    const int32_t a = e[2 * i], b = e[2 * i + 1];
    bool ok = a >= 0 && (size_t)a < nv && b >= 0 && (size_t)b < nv;
    if (ok && i > 0) {
        const int32_t pa = e[2 * i - 2], pb = e[2 * i - 1];
        ok = pa < a || (pa == a && pb <= b);
    }
    if (!ok) *bad = 1;
}

// rows[v] = the first edge whose first index is >= v, v in [0, nv]
__global__ void __launch_bounds__(256) mesh_rows_kernel(const int32_t *__restrict__ e, size_t ne, size_t nv, uint32_t *__restrict__ rows,
                                                        const int *__restrict__ bad) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v > nv || *bad) return;
    size_t lo = 0, hi = ne;
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if ((size_t)e[2 * mid] < v)
            lo = mid + 1;
        else
            hi = mid;
    }
    rows[v] = (uint32_t)lo;
}

__global__ void __launch_bounds__(256) mesh_weights_kernel(const float *__restrict__ vtx, const int32_t *__restrict__ e, const uint32_t *__restrict__ rows,
                                                           size_t nv, float *__restrict__ w, float *__restrict__ tw, const int *__restrict__ bad) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v >= nv || *bad) return;
    const float px = vtx[3 * v], py = vtx[3 * v + 1], pz = vtx[3 * v + 2];
    float t = 0.f;
    for (uint32_t k = rows[v]; k < rows[v + 1]; ++k) {
        const size_t b = (size_t)e[2 * (size_t)k + 1];
        const float dx = px - vtx[3 * b], dy = py - vtx[3 * b + 1], dz = pz - vtx[3 * b + 2];
        const float dist = __fsqrt_rn(dx * dx + dy * dy + dz * dz);
        const float wk = (float)__ddiv_rn(1.0, __dadd_rn((double)dist, 1e-12));
        w[k] = wk;
        t = k == rows[v] ? wk : t + wk;
    }
    tw[v] = t;
}

// KIND 0 Sharpen:   prv + strength * (prv * (float)N - sum)              (TM:552-559)
// KIND 1 Simple:    (prv + sum) / (float)(1.0 + N), 1.0 + N in double   (TM:632-639)
// KIND 2 Laplacian: prv + lambda * (wsum / total_weight - prv)          (TM:146-153)
template <int KIND>
__global__ void __launch_bounds__(256) mesh_filter_pass_kernel(MeshPass p, const int32_t *__restrict__ e, const uint32_t *__restrict__ rows,
                                                               const float *__restrict__ w, const float *__restrict__ tw, size_t nv, float c,
                                                               const int *__restrict__ bad) {
    const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (v >= nv || *bad) return;
    const uint32_t lo = rows[v], hi = rows[v + 1];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float *in = p.in[a];
        if (!in) continue;
        float prv[3], sum[3], r[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) prv[k] = in[3 * v + k];
        if (lo == hi) {
#pragma unroll
            for (int k = 0; k < 3; ++k) p.out[a][3 * v + k] = prv[k];
            continue;
        }
        for (uint32_t j = lo; j < hi; ++j) {
            const size_t b = (size_t)e[2 * (size_t)j + 1];
            const float wj = KIND == 2 ? w[j] : 1.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float x = KIND == 2 ? wj * in[3 * b + k] : in[3 * b + k];
                sum[k] = j == lo ? x : sum[k] + x;
            }
        }
        if (KIND == 0) {
            const float cnt = (float)(hi - lo);
#pragma unroll
            for (int k = 0; k < 3; ++k) r[k] = prv[k] + c * (prv[k] * cnt - sum[k]);
        } else if (KIND == 1) {
            const float d = (float)(1.0 + (double)(hi - lo));
#pragma unroll
            for (int k = 0; k < 3; ++k) r[k] = __fdiv_rn(prv[k] + sum[k], d);
        } else {
            const float t = tw[v];
#pragma unroll
            for (int k = 0; k < 3; ++k) r[k] = prv[k] + c * (__fdiv_rn(sum[k], t) - prv[k]);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) p.out[a][3 * v + k] = r[k];
    }
}

extern "C" int cphb_mesh_filter(int kind, int number_of_iterations, float strength_or_lambda, float mu, const int32_t *edges, size_t n_edges,
                                size_t n_vertices, const float *vertices, const float *normals, const float *colors, int filter_mask,
                                float *out_vertices, float *out_normals, float *out_colors, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_filter";
    if (kind < CPHB_MESH_SHARPEN || kind > CPHB_MESH_TAUBIN) return mesh_invalid(who, "unknown filter kind");
    const float *in[3] = {vertices, normals, colors};
    float *out[3] = {out_vertices, out_normals, out_colors};
    for (int a = 0; a < 3; ++a)
        if (n_vertices && in[a] && !out[a]) return mesh_invalid(who, "an attribute without an output");
    if (n_edges && !edges) return mesh_invalid(who, "null argument");
    if (n_edges > (size_t)INT32_MAX || n_vertices > (size_t)INT32_MAX) return mesh_invalid(who, "more than 2^31 - 1 edges or vertices");
    if (n_vertices == 0) {
        if (n_edges) return mesh_invalid(who, "an edge's vertex index is outside [0, n_vertices)");
        return CPHB_OK;
    }
    const bool weighted = kind == CPHB_MESH_LAPLACIAN || kind == CPHB_MESH_TAUBIN;
    const size_t passes = number_of_iterations > 0 ? (size_t)number_of_iterations * (kind == CPHB_MESH_TAUBIN ? 2 : 1) : 0;
    bool filt[3];
    for (int a = 0; a < 3; ++a) filt[a] = in[a] && passes && ((filter_mask >> a) & 1);
    cphb_scratch sc(s);
    int *bad = nullptr;
    uint32_t *rows = nullptr;
    float *w = nullptr, *tw = nullptr, *tmp[3] = {nullptr, nullptr, nullptr};
    int rc = sc.alloc(&bad, 1);
    if (!rc) rc = sc.alloc(&rows, n_vertices + 1);
    if (!rc && weighted) rc = sc.alloc(&w, n_edges + 1);
    if (!rc && weighted) rc = sc.alloc(&tw, n_vertices);
    for (int a = 0; a < 3 && !rc; ++a)
        if (filt[a] && passes > 1) rc = sc.alloc(&tmp[a], 3 * n_vertices);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    if (n_edges) CPHB_LAUNCH(mesh_edges_check_kernel, mesh_blocks(n_edges, 256), 256, 0, s, edges, n_edges, n_vertices, bad);
    for (int a = 0; a < 3; ++a)
        if (in[a] && !filt[a]) CPHB_CUDA(cudaMemcpyAsync(out[a], in[a], 12 * n_vertices, cudaMemcpyDeviceToDevice, s));
    if (passes) {
        CPHB_LAUNCH(mesh_rows_kernel, mesh_blocks(n_vertices + 1, 256), 256, 0, s, edges, n_edges, n_vertices, rows, bad);
        if (weighted) CPHB_LAUNCH(mesh_weights_kernel, mesh_blocks(n_vertices, 256), 256, 0, s, vertices, edges, rows, n_vertices, w, tw, bad);
        // pass q writes the output when an even number of passes follow it, so the last pass always does
        MeshPass prev = {{nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr}};
        for (size_t q = 0; q < passes; ++q) {
            MeshPass p = {{nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr}};
            for (int a = 0; a < 3; ++a) {
                if (!filt[a]) continue;
                p.in[a] = q == 0 ? in[a] : prev.out[a];
                p.out[a] = (passes - 1 - q) % 2 == 0 ? out[a] : tmp[a];
            }
            const float c = kind == CPHB_MESH_TAUBIN && q % 2 == 1 ? mu : strength_or_lambda;
            const unsigned g = mesh_blocks(n_vertices, 256);
            if (kind == CPHB_MESH_SHARPEN)
                CPHB_LAUNCH(mesh_filter_pass_kernel<0>, g, 256, 0, s, p, edges, rows, w, tw, n_vertices, c, bad);
            else if (kind == CPHB_MESH_SIMPLE)
                CPHB_LAUNCH(mesh_filter_pass_kernel<1>, g, 256, 0, s, p, edges, rows, w, tw, n_vertices, c, bad);
            else
                CPHB_LAUNCH(mesh_filter_pass_kernel<2>, g, 256, 0, s, p, edges, rows, w, tw, n_vertices, c, bad);
            prev = p;
        }
    }
    int h_bad = 0;
    rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    return h_bad ? mesh_invalid(who, "the edge list has an index outside [0, n_vertices) or is not sorted") : CPHB_OK;
}

// ================================================================================================== GetSurfaceArea
// ComputeTriangleArea (trianglemesh.h:340-348): 0.5 * |(p0 - p1) x (p0 - p2)| in float32 (the reference's 0.5 * norm in
// double rounds to the same float: halving is exact).  An index outside [0, nv) sets *bad and gives 0.
__device__ __forceinline__ float mesh_triangle_area(const float *__restrict__ vtx, size_t nv, const int32_t *__restrict__ tri, size_t t,
                                                    int *__restrict__ bad) {
    int32_t f[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        f[j] = tri[3 * t + j];
        if (f[j] < 0 || (size_t)f[j] >= nv) {
            *bad = 1;
            return 0.f;
        }
    }
    const float *p0 = vtx + 3 * (size_t)f[0], *p1 = vtx + 3 * (size_t)f[1], *p2 = vtx + 3 * (size_t)f[2];
    const float x0 = p0[0] - p1[0], x1 = p0[1] - p1[1], x2 = p0[2] - p1[2];
    const float y0 = p0[0] - p2[0], y1 = p0[1] - p2[1], y2 = p0[2] - p2[2];
    const float c0 = x1 * y2 - x2 * y1, c1 = x2 * y0 - x0 * y2, c2 = x0 * y1 - x1 * y0;
    return 0.5f * __fsqrt_rn(c0 * c0 + c1 * c1 + c2 * c2);
}

struct MeshAreaTerms {
    const float *vtx;
    size_t nv;
    const int32_t *tri;
    float *areas;  // or NULL
    int *bad;
    __device__ void operator()(size_t t, float (&v)[1]) const {
        v[0] = mesh_triangle_area(vtx, nv, tri, t, bad);
        if (areas) areas[t] = v[0];
    }
};

extern "C" int cphb_mesh_surface_area(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                      float *triangle_areas, float *h_area, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_surface_area";
    if (!h_area) return mesh_invalid(who, "null argument");
    *h_area = 0.f;
    if (n_triangles == 0) return CPHB_OK;
    if (!triangles || !vertices) return mesh_invalid(who, "null argument");
    cphb_scratch sc(s);
    int *bad = nullptr;
    int rc = sc.alloc(&bad, 1);
    if (rc) return rc;
    CPHB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
    double total = 0.0;
    rc = sum_values<1>(MeshAreaTerms{vertices, n_vertices, triangles, triangle_areas, bad}, n_triangles, &total, s);
    int h_bad = 0;
    if (!rc) rc = cphb_read_back(&h_bad, bad, sizeof(int), s, who);
    if (rc) return rc;
    if (h_bad) return mesh_invalid(who, "a triangle's vertex index is outside [0, n_vertices)");
    *h_area = (float)total;
    return CPHB_OK;
}

// ================================================================================================== SamplePointsUniformly
// Areas -> a float64 scan in a fixed order: block b owns triangles [2048 b, 2048 b + 2048), thread t of it the 8
// consecutive triangles from 2048 b + 8 t and adds their areas in order from 0.0 (L_i); thread 0 forms the exclusive sums
// of the 256 thread totals in order from 0.0 (T_t), and one thread the exclusive sums of the block totals (B_b), so
// S_i = B_b + (T_t + L_i) and the total is the last S.  Triangle i owns the points [bnd[i], bnd[i + 1]) with
// bnd[i + 1] = clamp(llrint((S_i / S) * n), 0, n), bnd[0] = 0 and bnd[nt] = n (S is non-decreasing, so the clamp against
// bnd[i] a serial loop would apply changes nothing).  Point p: the triangle with bnd[i] <= p < bnd[i + 1] by binary
// search; r1, r2 = draws 2 p + 1 and 2 p + 2 of thrust::default_random_engine (seed 1), each mapped by thrust's
// uniform_real_distribution<float>(0, 1).
#define SAMP_PER_THREAD 8
#define SAMP_TILE (256 * SAMP_PER_THREAD)

__global__ void __launch_bounds__(256) mesh_area_scan_kernel(const float *__restrict__ vtx, size_t nv, const int32_t *__restrict__ tri, size_t nt,
                                                             double *__restrict__ pre, double *__restrict__ blk, int *__restrict__ bad) {
    __shared__ double s_tot[256];
    const size_t base = blockIdx.x * (size_t)SAMP_TILE + threadIdx.x * (size_t)SAMP_PER_THREAD;
    double loc[SAMP_PER_THREAD];
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < SAMP_PER_THREAD; ++j) {
        if (base + j < nt) acc = acc + (double)mesh_triangle_area(vtx, nv, tri, base + j, bad);
        loc[j] = acc;
    }
    s_tot[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 0.0;
        for (int t = 0; t < 256; ++t) {
            const double x = s_tot[t];
            s_tot[t] = r;
            r = r + x;
        }
        blk[blockIdx.x] = r;
    }
    __syncthreads();
    const double T = s_tot[threadIdx.x];
#pragma unroll
    for (int j = 0; j < SAMP_PER_THREAD; ++j)
        if (base + j < nt) pre[base + j] = T + loc[j];
}

// exclusive sums of the block totals in place, the total, and the status: 1 bad index, 2 total not positive and finite
__global__ void mesh_area_blocks_kernel(double *__restrict__ blk, unsigned nb, double *__restrict__ total, int *__restrict__ status) {
    double r = 0.0;
    for (unsigned b = 0; b < nb; ++b) {
        const double x = blk[b];
        blk[b] = r;
        r = r + x;
    }
    *total = r;
    if (*status == 0 && !(r > 0.0 && r <= 1.7976931348623157e308)) *status = 2;
}

__global__ void __launch_bounds__(256) mesh_sample_bounds_kernel(const double *__restrict__ pre, const double *__restrict__ blk,
                                                                 const double *__restrict__ total, size_t nt, uint32_t n, uint32_t *__restrict__ bnd,
                                                                 const int *__restrict__ status) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= nt || *status) return;
    if (i == 0) bnd[0] = 0u;
    if (i == nt - 1) {
        bnd[nt] = n;
        return;
    }
    const double S = __dadd_rn(blk[i / SAMP_TILE], pre[i]);
    const long long x = llrint(__dmul_rn(__ddiv_rn(S, *total), (double)n));
    bnd[i + 1] = (uint32_t)(x < 0 ? 0 : (x > (long long)n ? (long long)n : x));
}

// uniform_real_distribution<float>(0, 1) of a minstd draw x (thrust/random/detail/uniform_real_distribution.inl)
__device__ __forceinline__ float mesh_uniform01(uint32_t x) {
    float r = (float)(x - 1u);
    r = __fdiv_rn(r, 1.0f + (float)(CPHB_MINSTD_M - 1u - 1u));
    return r * (1.0f - 0.0f) + 0.0f;
}

struct MeshSampleArgs {
    const float *vtx, *vn, *tn, *vc;  // vertex normals / triangle normals / colours: NULL when absent
    const int32_t *tri;
    const uint32_t *bnd;
    size_t nt;
    uint32_t n;
    float *pts, *nrm, *col;
};

__global__ void __launch_bounds__(256) mesh_sample_points_kernel(MeshSampleArgs g, cphb_minstd_pow pw, const int *__restrict__ status) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.n || *status) return;
    size_t lo = 0, hi = g.nt;  // the number of bnd[1 ..] entries <= p
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (g.bnd[mid + 1] <= p)
            lo = mid + 1;
        else
            hi = mid;
    }
    const size_t t = lo;
    const uint32_t x1 = cphb_minstd_jump(1u, 2ull * p + 1ull, pw);
    const uint32_t x2 = cphb_minstd_mulmod(x1, CPHB_MINSTD_A);
    const float r1 = mesh_uniform01(x1), r2 = mesh_uniform01(x2);
    const float sr = __fsqrt_rn(r1);
    const float a = 1.f - sr, b = sr * (1.f - r2), c = sr * r2;
    const size_t f0 = (size_t)g.tri[3 * t], f1 = (size_t)g.tri[3 * t + 1], f2 = (size_t)g.tri[3 * t + 2];
#pragma unroll
    for (int k = 0; k < 3; ++k) g.pts[3 * (size_t)p + k] = a * g.vtx[3 * f0 + k] + b * g.vtx[3 * f1 + k] + c * g.vtx[3 * f2 + k];
    if (g.nrm) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
            g.nrm[3 * (size_t)p + k] = g.tn ? g.tn[3 * t + k] : a * g.vn[3 * f0 + k] + b * g.vn[3 * f1 + k] + c * g.vn[3 * f2 + k];
    }
    if (g.col) {
#pragma unroll
        for (int k = 0; k < 3; ++k) g.col[3 * (size_t)p + k] = a * g.vc[3 * f0 + k] + b * g.vc[3 * f1 + k] + c * g.vc[3 * f2 + k];
    }
}

extern "C" int cphb_mesh_sample_points_uniformly(const float *vertices, size_t n_vertices, const int32_t *triangles, size_t n_triangles,
                                                 const float *vertex_normals, const float *triangle_normals, const float *vertex_colors,
                                                 size_t number_of_points, float *points, float *normals, float *colors, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const char *who = "cphb_mesh_sample_points_uniformly";
    if (number_of_points == 0) return mesh_invalid(who, "number_of_points is 0");
    if (number_of_points > CPHB_MESH_MAX_SAMPLES) return mesh_invalid(who, "number_of_points exceeds 2^30 - 1 (two draws per point)");
    if (n_triangles == 0) return mesh_invalid(who, "the mesh has no triangles");
    if (n_triangles > (size_t)INT32_MAX) return mesh_invalid(who, "more than 2^31 - 1 triangles");
    if (!vertices || !triangles || !points || (normals && !triangle_normals && !vertex_normals) || (colors && !vertex_colors))
        return mesh_invalid(who, "null argument");
    const unsigned nb = (unsigned)((n_triangles + SAMP_TILE - 1) / SAMP_TILE);
    cphb_scratch sc(s);
    int *status = nullptr;
    double *pre = nullptr, *blk = nullptr, *total = nullptr;
    uint32_t *bnd = nullptr;
    int rc = sc.alloc(&status, 1);
    if (!rc) rc = sc.alloc(&pre, n_triangles);
    if (!rc) rc = sc.alloc(&blk, nb);
    if (!rc) rc = sc.alloc(&total, 1);
    if (!rc) rc = sc.alloc(&bnd, n_triangles + 1);
    if (rc) return rc;
    cphb_minstd_pow pw;
    cphb_minstd_table(&pw);
    CPHB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), s));
    CPHB_LAUNCH(mesh_area_scan_kernel, nb, 256, 0, s, vertices, n_vertices, triangles, n_triangles, pre, blk, status);
    CPHB_LAUNCH(mesh_area_blocks_kernel, 1, 1, 0, s, blk, nb, total, status);
    CPHB_LAUNCH(mesh_sample_bounds_kernel, mesh_blocks(n_triangles, 256), 256, 0, s, pre, blk, total, n_triangles, (uint32_t)number_of_points,
                bnd, status);
    MeshSampleArgs g = {vertices, normals ? vertex_normals : nullptr, normals ? triangle_normals : nullptr, colors ? vertex_colors : nullptr,
                        triangles, bnd, n_triangles, (uint32_t)number_of_points, points, normals, colors};
    CPHB_LAUNCH(mesh_sample_points_kernel, mesh_blocks(number_of_points, 256), 256, 0, s, g, pw, status);
    int h_status = 0;
    rc = cphb_read_back(&h_status, status, sizeof(int), s, who);
    if (rc) return rc;
    if (h_status == 1) return mesh_invalid(who, "a triangle's vertex index is outside [0, n_vertices)");
    if (h_status == 2) return mesh_invalid(who, "the surface area is not positive and finite");
    return CPHB_OK;
}
