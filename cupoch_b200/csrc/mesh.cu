// mesh.cu -- TriangleMesh::ComputeTriangleNormals and ComputeVertexNormals (DESIGN section 4 item 19).  Reference:
// geometry/trianglemesh.cu (TM).
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
#include "cphb_internal.cuh"

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
