// cluster.cu -- PointCloud::ClusterDBSCAN (pointcloud_cluster.cu:30-179): an index client (SURVEY 8f rank 4).
//
// The reference: radius search with max_nn = max_edges + 1 -> directed graph (a point with >= min_points listed neighbours
// other than itself is a core point and keeps its edges, every other point has none) -> for i = 0 .. n-1: if i has not
// been reached yet, breadth-first search from i over the edges; the reached set is labelled with the next cluster id, or
// -1 when it has fewer than min_points members.  Its BFS does NOT stop at points reached by an earlier search, so a later
// search relabels whatever it reaches (border points end up in the LAST cluster that reaches them) -- reproduced here.
// Only core points matter as seeds: a non-core seed reaches itself alone (label -1, which it has from the start), and
// whether it counts as "visited" never influences another search.
//
// Here: the library's own radius search, one kernel for the degrees, then ONE persistent block that walks the seeds in
// index order and expands each search's frontier with all its threads (work ~ edges traversed, instead of the reference's
// full-cloud pass per BFS level).  Labels do not depend on the order in which a level's points are discovered.
#include "cphb_internal.cuh"

__global__ void __launch_bounds__(256) dbscan_degree_kernel(const int32_t *__restrict__ idx, size_t n, int K, int min_points,
                                                            int *degree) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = 0;
    for (int k = 0; k < K; ++k) {
        const int32_t j = idx[i * K + k];
        c += (j >= 0 && (size_t)j != i);
    }
    degree[i] = (c >= min_points) ? c : 0;  // compute_vertex_degree_functor (:34-55)
}

#define DB_THREADS 1024
__global__ void __launch_bounds__(DB_THREADS) dbscan_bfs_kernel(const int32_t *__restrict__ idx, const int *__restrict__ degree,
                                                                unsigned n, int K, int min_points, int32_t *labels,
                                                                unsigned *stamp, int *visited, int32_t *queue,
                                                                int *n_clusters) {
    __shared__ unsigned s_tail, s_seed;
    const unsigned tid = threadIdx.x;
    for (unsigned i = tid; i < n; i += DB_THREADS) { labels[i] = -1; stamp[i] = 0u; visited[i] = 0; }
    __syncthreads();
    int cluster = 0;
    unsigned epoch = 0;
    unsigned cur = 0;
    while (true) {
        // next seed: smallest index >= cur that is a core point and has not been reached
        unsigned seed = 0xffffffffu;
        for (; cur < n; cur += DB_THREADS) {
            const unsigned i = cur + tid;
            const bool cand = i < n && degree[i] > 0 && visited[i] == 0;
            if (tid == 0) s_seed = 0xffffffffu;
            __syncthreads();
            if (cand) atomicMin(&s_seed, i);
            __syncthreads();
            seed = s_seed;
            __syncthreads();
            if (seed != 0xffffffffu) break;
        }
        if (seed == 0xffffffffu) break;
        ++epoch;
        if (tid == 0) { queue[0] = (int32_t)seed; stamp[seed] = epoch; s_tail = 1u; }
        __syncthreads();
        unsigned head = 0, tail = 1;
        while (head < tail) {  // one BFS level: every (point of the level, neighbour slot) pair
            const unsigned long long pairs = (unsigned long long)(tail - head) * (unsigned)K;
            for (unsigned long long p = tid; p < pairs; p += DB_THREADS) {
                const unsigned u = (unsigned)queue[head + (unsigned)(p / (unsigned)K)];
                if (degree[u] == 0) continue;  // not a core point: no edges
                const int32_t v = idx[(size_t)u * K + (unsigned)(p % (unsigned)K)];
                if (v < 0 || (unsigned)v == u) continue;
                if (atomicExch(&stamp[v], epoch) != epoch) queue[atomicAdd(&s_tail, 1u)] = v;
            }
            __syncthreads();
            head = tail;
            tail = s_tail;
            __syncthreads();
        }
        const bool noise = (int)tail < min_points;  // (never true for a core seed; kept for fidelity, :155-156)
        for (unsigned q = tid; q < tail; q += DB_THREADS) {
            const unsigned v = (unsigned)queue[q];
            labels[v] = noise ? -1 : cluster;
            visited[v] = 1;
        }
        if (!noise) ++cluster;
        __syncthreads();
        // (the scan resumes at the chunk that held this seed: later candidates of the chunk may have been reached)
    }
    if (tid == 0) *n_clusters = cluster;
}

// labels_out: device, n int32 (-1 = noise).  *h_n_clusters (optional) = number of cluster ids handed out.
extern "C" int cphb_cluster_dbscan(const float *points, size_t n, float eps, int min_points, int max_edges, int32_t *labels_out,
                                   int *h_n_clusters, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (h_n_clusters) *h_n_clusters = 0;
    if (n == 0) return CPHB_OK;
    if (!points || !labels_out || max_edges < 1 || max_edges > 255 || n > 0x7fffffffull) {
        cphb_set_error("cphb_cluster_dbscan: invalid argument (max_edges must be in [1, 255])");
        return CPHB_ERR_INVALID;
    }
    const int K = max_edges + 1;
    cphb_nbr_table t;
    cphb_scratch sc(s);
    int32_t *queue = nullptr;
    int *degree = nullptr, *visited = nullptr, *ncl = nullptr;
    unsigned *stamp = nullptr;
    int rc = cphb_nbr_table_create(points, n, 0, n, 0, eps, K, &t, s);
    if (!rc) rc = sc.alloc(&degree, n);
    if (!rc) rc = sc.alloc(&visited, n);
    if (!rc) rc = sc.alloc(&stamp, n);
    if (!rc) rc = sc.alloc(&queue, n);
    if (!rc) rc = sc.alloc(&ncl, 1);
    int h = 0;
    if (!rc) {
        CPHB_LAUNCH(dbscan_degree_kernel, (unsigned)((n + 255) / 256), 256, 0, s, t.idx, n, K, min_points, degree);
        CPHB_LAUNCH(dbscan_bfs_kernel, 1, DB_THREADS, 0, s, t.idx, degree, (unsigned)n, K, min_points, labels_out, stamp, visited,
                    queue, ncl);
        rc = cphb_read_back(&h, ncl, sizeof(int), s, "cphb_cluster_dbscan");
    }
    if (h_n_clusters) *h_n_clusters = h;
    sc.release();
    return cphb_nbr_table_release(&t, rc, s);
}
