// VoxelGrid's += and AddVoxels run by thrust itself: the toolkit's thrust headers compiled for the CPP backend with g++.
// The key type, its lexicographic operator< (utility/helper.h:111-121), the Voxel record and the sort_by_key /
// unique_by_key (AddVoxels, voxelgrid.cu:299-319) and sort_by_key / reduce_by_key with add_voxel_color_functor and
// divide_voxel_color_functor (operator+=, voxelgrid.cu:235-281; voxelgrid.h:64-82) are written as the reference writes
// them, minus __device__ and Eigen.
//   thrust_voxel_merge_pin IN OUT   IN = int32 n, then n keys [3] int32, then n colours [3] float32 (this grid's voxels
//   followed by the other's); OUT = the AddVoxels result then the += result, each int32 m, m keys, m colours
#include <thrust/host_vector.h>
#include <thrust/iterator/constant_iterator.h>
#include <thrust/iterator/zip_iterator.h>
#include <thrust/reduce.h>
#include <thrust/sort.h>
#include <thrust/tuple.h>
#include <thrust/unique.h>

#include <cstdio>
#include <vector>

struct Vector3i {
    int v[3];
    bool operator==(const Vector3i &o) const { return v[0] == o.v[0] && v[1] == o.v[1] && v[2] == o.v[2]; }
};
bool operator<(const Vector3i &l, const Vector3i &r) {
    for (int i = 0; i < 3; ++i)
        if (l.v[i] != r.v[i]) return l.v[i] < r.v[i];
    return false;
}
struct Voxel {
    Vector3i grid_index_;
    float color_[3];
};
struct add_voxel_color_functor {
    thrust::tuple<Voxel, int> operator()(const thrust::tuple<Voxel, int> &x, const thrust::tuple<Voxel, int> &y) const {
        Voxel ans;
        ans.grid_index_ = thrust::get<0>(x).grid_index_;
        for (int a = 0; a < 3; ++a) ans.color_[a] = thrust::get<0>(x).color_[a] + thrust::get<0>(y).color_[a];
        return thrust::make_tuple(ans, thrust::get<1>(x) + thrust::get<1>(y));
    }
};

static void emit(std::FILE *f, const thrust::host_vector<Vector3i> &k, const thrust::host_vector<Voxel> &v, size_t m) {
    const int mi = (int)m;
    std::fwrite(&mi, sizeof(int), 1, f);
    for (size_t i = 0; i < m; ++i) std::fwrite(k[i].v, sizeof(int), 3, f);
    for (size_t i = 0; i < m; ++i) std::fwrite(v[i].color_, sizeof(float), 3, f);
}

int main(int argc, char **argv) {
    if (argc != 3) return 2;
    std::FILE *in = std::fopen(argv[1], "rb");
    if (!in) return 1;
    int n = 0;
    if (std::fread(&n, sizeof(int), 1, in) != 1) return 1;
    std::vector<int> kk(3 * (size_t)n);
    std::vector<float> cc(3 * (size_t)n);
    if (std::fread(kk.data(), sizeof(int), kk.size(), in) != kk.size() || std::fread(cc.data(), sizeof(float), cc.size(), in) != cc.size())
        return 1;
    std::fclose(in);
    thrust::host_vector<Vector3i> keys(n);
    thrust::host_vector<Voxel> values(n);
    for (int i = 0; i < n; ++i) {
        for (int a = 0; a < 3; ++a) {
            keys[i].v[a] = kk[3 * i + a];
            values[i].color_[a] = cc[3 * i + a];
        }
        values[i].grid_index_ = keys[i];
    }
    std::FILE *out = std::fopen(argv[2], "wb");
    if (!out) return 1;
    {  // AddVoxels
        thrust::host_vector<Vector3i> k = keys;
        thrust::host_vector<Voxel> v = values;
        thrust::sort_by_key(k.begin(), k.end(), v.begin());
        auto end = thrust::unique_by_key(k.begin(), k.end(), v.begin());
        emit(out, k, v, end.first - k.begin());
    }
    {  // operator+=
        thrust::host_vector<Vector3i> k = keys;
        thrust::host_vector<Voxel> v = values;
        thrust::sort_by_key(k.begin(), k.end(), v.begin());
        thrust::host_vector<int> counts(n);
        thrust::host_vector<Vector3i> new_keys(n);
        auto end = thrust::reduce_by_key(k.begin(), k.end(),
                                         thrust::make_zip_iterator(thrust::make_tuple(v.begin(), thrust::make_constant_iterator(1))),
                                         new_keys.begin(), thrust::make_zip_iterator(thrust::make_tuple(v.begin(), counts.begin())),
                                         thrust::equal_to<Vector3i>(), add_voxel_color_functor());
        const size_t m = end.first - new_keys.begin();
        for (size_t i = 0; i < m; ++i)
            for (int a = 0; a < 3; ++a) v[i].color_[a] = v[i].color_[a] / counts[i];
        emit(out, new_keys, v, m);
    }
    std::fclose(out);
    return 0;
}
