// search.cu -- batched exact kNN / radius search on the Hilbert-AABB index.
// Replaces KDTreeFlann::SearchKNN / SearchRadius (kdtree_flann.cu:35-80,
// kdtree_flann.inl:70-122) and flann's nearestKernel
// (kdtree_cuda_3d_index.cu:52-154) with its result sets (result_set.h).
//
// Queries are ordered along the target's Hilbert curve first (one radix sort)
// so that each warp's 32 queries form a compact cluster; a warp then walks the
// 32-ary AABB hierarchy cooperatively (cphb_internal.cuh).  Results are written
// back at the queries' original positions.
#include <float.h>

#include "cphb_internal.cuh"
#include "cphb_searchk.cuh"
#include "fused_neighbourhood.cuh"

template <int TOP>
__global__ void __launch_bounds__(256) search1_kernel(IndexView ix, const float *__restrict__ qxyz,
                                                      const uint32_t *__restrict__ perm, size_t nq, float r2,
                                                      int32_t *__restrict__ out_idx, float *__restrict__ out_d2,
                                                      unsigned long long *count) {
    __shared__ __align__(16) float4 s_tile[8][2 * CPHB_LEAF];
    __shared__ uint64_t s_bar[8][2];
    const int warp = threadIdx.x >> 5;
    WarpSearch w;
    warp_search_setup(w, s_tile[warp], s_bar[warp]);
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    w.valid = i < nq;
    size_t pos = 0;
    w.qx = w.qy = w.qz = 0.f;
    if (w.valid) {
        pos = perm ? perm[i] : i;
        w.qx = qxyz[3 * pos];
        w.qy = qxyz[3 * pos + 1];
        w.qz = qxyz[3 * pos + 2];
    }
    const unsigned long long init = (r2 > 0.f) ? init_key(r2) : 0ull;  // r2==0: d2 < 0 never holds
    w.best = init;
    w.bound = (unsigned)(init >> 32);
    warp_query_box(w);
    if (__any_sync(CPHB_FULL, w.valid)) warp_nn_search<TOP>(ix, w);
    bool found = w.valid && w.best != init;
    if (w.valid) {
        out_idx[pos] = found ? (int32_t)(unsigned)(w.best & 0xffffffffull) : -1;
        out_d2[pos] = found ? __uint_as_float((unsigned)(w.best >> 32)) : INFINITY;
    }
    unsigned f = __ballot_sync(CPHB_FULL, found);
    if (count && lane_id() == 0 && f) atomicAdd(count, (unsigned long long)__popc(f));
}

template <int TOP>
__global__ void searchk_kernel(IndexView ix, const float *__restrict__ qxyz, const uint32_t *__restrict__ perm,
                               size_t nq, float r2, int k, int32_t *__restrict__ out_idx,
                               float *__restrict__ out_d2, unsigned long long *count) {
    extern __shared__ __align__(16) unsigned char smem[];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, qxyz, 0, nq, perm, 0, r2, k, pos);
    fused_query_search<TOP>(ix, w);
    int filled = 0;
    if (w.valid) {
        for (int j = 0; j < k; ++j) {
            unsigned long long key = w.list[j * 32];
            bool ok = key < init;
            out_idx[pos * k + j] = ok ? (int32_t)(unsigned)(key & 0xffffffffull) : -1;
            out_d2[pos * k + j] = ok ? __uint_as_float((unsigned)(key >> 32)) : INFINITY;
            filled += ok;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) filled += __shfl_xor_sync(CPHB_FULL, filled, o);
    if (count && lane_id() == 0 && filled) atomicAdd(count, (unsigned long long)filled);
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
// k_limit: SearchKNN rejects knn > NUM_MAX_NN (kdtree_flann.cu:52-54); SearchRadius has no such check (:70-72) -- DBSCAN's
// default asks for max_nn = 101 -- so there the limit is what one warp's lists can hold in shared memory
#define CPHB_RADIUS_MAX_NN 256

// the search kernel's launch, and the read-back of the found count into *h_count when it is given
static int search_launch(const cphb_index *index, const float *query, const uint32_t *perm, size_t nq, float r2, int k,
                         int32_t *idx, float *d2, unsigned long long *count, int64_t *h_count, cudaStream_t s) {
    if (count) CPHB_CUDA(cudaMemsetAsync(count, 0, 8, s));
    if (k == 1) {
        const unsigned grid = (unsigned)((nq + 255) / 256);
        if (index->v.top <= 3)
            CPHB_LAUNCH(search1_kernel<3>, grid, 256, 0, s, index->v, query, perm, nq, r2, idx, d2, count);
        else
            CPHB_LAUNCH(search1_kernel<5>, grid, 256, 0, s, index->v, query, perm, nq, r2, idx, d2, count);
        CPHB_CHECK_LAUNCH();
    } else {
        const int rc = launch_fused(index, searchk_kernel<3>, searchk_kernel<5>, nq, k, s, query, perm, nq, r2, k, idx, d2, count);
        if (rc) return rc;
    }
    if (h_count) {
        unsigned long long h = 0;
        const int rc = cphb_read_back(&h, count, 8, s, "search");
        if (rc) return rc;
        *h_count = (int64_t)h;
    }
    return CPHB_OK;
}

static int search_impl(const cphb_index *index, const float *query, size_t nq, float r2, int k, int k_limit, int32_t *idx,
                       float *d2, int64_t *h_count, cudaStream_t s) {
    if (!index || !query || !idx || !d2) {
        cphb_set_error("search: null argument");
        return CPHB_ERR_INVALID;
    }
    // kdtree_flann.cu:46-48,70-72: empty data / query -> -1
    if (index->v.n == 0 || nq == 0) {
        cphb_set_error("search: empty index or query (reference returns -1)");
        return CPHB_ERR_INVALID;
    }
    if (k < 0 || k > k_limit) {  // NUM_MAX_NN, kdtree_search_param.h:26
        cphb_set_error("search: k=%d outside [0,%d]", k, k_limit);
        return CPHB_ERR_INVALID;
    }
    if (h_count) *h_count = 0;
    if (k == 0) return CPHB_OK;
    cphb_scratch sc(s);
    uint32_t *perm = nullptr;
    unsigned long long *count = nullptr;
    int rc = CPHB_OK;
    if (nq > 32) {
        rc = sc.alloc(&perm, nq);
        if (!rc) rc = cphb_hilbert_order_n(query, nq, perm, index->bounds, 1, nq < index->v.n ? nq : (size_t)index->v.n, s);
    }
    if (!rc && h_count) rc = sc.alloc(&count, 2);
    if (!rc) rc = search_launch(index, query, perm, nq, r2, k, idx, d2, count, h_count, s);
    return rc;
}

extern "C" int cphb_search_radius(const cphb_index *index, const float *query, size_t n_query, float radius,
                                  int max_nn, int32_t *idx, float *d2, int64_t *h_count, void *stream) {
    float r2 = radius * radius;  // kdtree_flann.inl:120 float(radius * radius); r2 == 0 matches nothing
    return search_impl(index, query, n_query, r2, max_nn, CPHB_RADIUS_MAX_NN, idx, d2, h_count, (cudaStream_t)stream);
}
extern "C" int cphb_search_hybrid(const cphb_index *index, const float *query, size_t n_query, float radius,
                                  int max_nn, int32_t *idx, float *d2, int64_t *h_count, void *stream) {
    return cphb_search_radius(index, query, n_query, radius, max_nn, idx, d2, h_count, stream);
}
extern "C" int cphb_search_knn(const cphb_index *index, const float *query, size_t n_query, int knn, int32_t *idx,
                               float *d2, int64_t *h_count, void *stream) {
    return search_impl(index, query, n_query, INFINITY, knn, 100, idx, d2, h_count, (cudaStream_t)stream);
}

int cphb_nbr_table_create(const float *points, size_t n, size_t first, size_t count, int knn, float radius, int max_nn,
                          cphb_nbr_table *t, cudaStream_t s) {
    const int k = (knn > 0) ? knn : max_nn;
    int rc = cphb_index_create(points, n, s, &t->ix);
    if (!rc) rc = cphb_alloc_async((void **)&t->idx, sizeof(int32_t) * count * k, s);
    if (!rc) rc = cphb_alloc_async((void **)&t->d2, sizeof(float) * count * k, s);
    if (!rc) {
        const float *q = points + 3 * first;
        if (knn > 0) rc = cphb_search_knn(t->ix, q, count, k, t->idx, t->d2, nullptr, s);
        else rc = cphb_search_radius(t->ix, q, count, radius, k, t->idx, t->d2, nullptr, s);
    }
    return rc;
}

int cphb_nbr_table_release(cphb_nbr_table *t, int rc, cudaStream_t s) {
    cphb_free_async(t->idx, s);
    cphb_free_async(t->d2, s);
    const cudaError_t e = cudaStreamSynchronize(s);
    cphb_index_destroy(t->ix);
    if (!rc && e != cudaSuccess) {
        cphb_set_error("neighbour-table client: %s", cudaGetErrorString(e));
        return CPHB_ERR_CUDA;
    }
    return rc;
}
