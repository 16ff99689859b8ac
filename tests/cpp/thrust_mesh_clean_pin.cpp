// TriangleMesh::RemoveDuplicatedVertices and RemoveDuplicatedTriangles run by thrust itself: the toolkit's thrust headers
// compiled for the CPP backend with g++.  The key types, helper.h's lexicographic operator< (utility/helper.h:111-121),
// align_triangle_functor (trianglemesh.cu:95-105), compute_old_to_new_index_functor (:76-92) and the call sequences
// (RemoveDuplicatedVertices :903-969 with vertex normals, RemoveDuplicatedTriangles :971-1009 with triangle normals) are
// written as the reference writes them, minus __device__ and Eigen.
//   thrust_mesh_clean_pin IN OUT   IN = int32 n, n vertices [3] f32, n normals [3] f32, int32 m, m triangles [3] i32,
//   m triangle normals [3] f32; OUT = int32 k, k vertices, k normals, m remapped triangles; then int32 k2, k2 triangles,
//   k2 triangle normals
#include <thrust/iterator/discard_iterator.h>
#include <thrust/sequence.h>
#include <thrust/host_vector.h>
#include <thrust/iterator/constant_iterator.h>
#include <thrust/iterator/zip_iterator.h>
#include <thrust/reduce.h>
#include <thrust/scan.h>
#include <thrust/sort.h>
#include <thrust/transform.h>
#include <thrust/unique.h>

#include <cstdio>
#include <vector>

template <class T>
struct Vec3 {
    T v[3];
    bool operator==(const Vec3 &o) const { return v[0] == o.v[0] && v[1] == o.v[1] && v[2] == o.v[2]; }
};
template <class T>
bool operator<(const Vec3<T> &l, const Vec3<T> &r) {
    for (int i = 0; i < 3; ++i)
        if (l.v[i] != r.v[i]) return l.v[i] < r.v[i];
    return false;
}
typedef Vec3<float> Vector3f;
typedef Vec3<int> Vector3i;

struct align_triangle_functor {
    Vector3i operator()(const Vector3i &t) const {
        if (t.v[0] <= t.v[1]) {
            return (t.v[0] <= t.v[2]) ? Vector3i{{t.v[0], t.v[1], t.v[2]}} : Vector3i{{t.v[2], t.v[0], t.v[1]}};
        } else {
            return (t.v[1] <= t.v[2]) ? Vector3i{{t.v[1], t.v[2], t.v[0]}} : Vector3i{{t.v[2], t.v[0], t.v[1]}};
        }
    }
};

template <class T>
static bool rd(std::FILE *f, std::vector<T> &v, size_t n) {
    v.resize(n);
    return std::fread(v.data(), sizeof(T), n, f) == n;
}

int main(int argc, char **argv) {
    if (argc != 3) return 2;
    std::FILE *in = std::fopen(argv[1], "rb");
    if (!in) return 1;
    int n = 0, m = 0;
    std::vector<Vector3f> hv, hn, htn;
    std::vector<Vector3i> ht;
    if (std::fread(&n, 4, 1, in) != 1 || !rd(in, hv, n) || !rd(in, hn, n) || std::fread(&m, 4, 1, in) != 1 || !rd(in, ht, m) || !rd(in, htn, m))
        return 1;
    std::fclose(in);
    std::FILE *out = std::fopen(argv[2], "wb");
    {  // RemoveDuplicatedVertices with vertex normals (runs(vertex_normals_, dummy))
        thrust::host_vector<Vector3f> vertices(hv.begin(), hv.end()), normals(hn.begin(), hn.end());
        thrust::host_vector<int> index_new_to_old(n), idx_offsets(n, 0);
        thrust::sequence(index_new_to_old.begin(), index_new_to_old.end());
        thrust::sort_by_key(vertices.begin(), vertices.end(), thrust::make_zip_iterator(thrust::make_tuple(index_new_to_old.begin(), normals.begin())));
        auto end0 = thrust::reduce_by_key(vertices.begin(), vertices.end(), thrust::make_constant_iterator<int>(1), thrust::make_discard_iterator(),
                                          idx_offsets.begin());
        idx_offsets.resize(thrust::distance(idx_offsets.begin(), end0.second) + 1);
        thrust::exclusive_scan(idx_offsets.begin(), idx_offsets.end(), idx_offsets.begin());
        auto end1 = thrust::unique_by_key(vertices.begin(), vertices.end(), normals.begin());
        const int k = (int)thrust::distance(vertices.begin(), end1.first);
        std::vector<int> old_to_new(n);
        for (int idx = 0; idx < k; ++idx)
            for (int i = idx_offsets[idx]; i < idx_offsets[idx + 1]; ++i) old_to_new[index_new_to_old[i]] = idx;
        std::fwrite(&k, 4, 1, out);
        for (int i = 0; i < k; ++i) std::fwrite(vertices[i].v, 4, 3, out);
        for (int i = 0; i < k; ++i) std::fwrite(normals[i].v, 4, 3, out);
        for (int t = 0; t < m; ++t)
            for (int c = 0; c < 3; ++c) std::fwrite(&old_to_new[ht[t].v[c]], 4, 1, out);
    }
    {  // RemoveDuplicatedTriangles with triangle normals
        thrust::host_vector<Vector3i> tri(m);
        thrust::host_vector<Vector3f> tn(htn.begin(), htn.end());
        thrust::transform(ht.begin(), ht.end(), tri.begin(), align_triangle_functor());
        thrust::sort_by_key(tri.begin(), tri.end(), tn.begin());
        auto end = thrust::unique_by_key(tri.begin(), tri.end(), tn.begin());
        const int k = (int)thrust::distance(tri.begin(), end.first);
        std::fwrite(&k, 4, 1, out);
        for (int i = 0; i < k; ++i) std::fwrite(tri[i].v, 4, 3, out);
        for (int i = 0; i < k; ++i) std::fwrite(tn[i].v, 4, 3, out);
    }
    std::fclose(out);
    return 0;
}
