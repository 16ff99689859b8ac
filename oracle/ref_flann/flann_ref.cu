// flann_ref.cu -- C wrapper around the REFERENCE's own nearest-neighbour engine, the FLANN CUDA kd-tree that
// cupoch vendors (third_party/flann/algorithms/kdtree_cuda_3d_index.{h,cu}).
//
// TEST INFRASTRUCTURE ONLY (oracle/): this file is the few lines of glue a test needs to call the reference's
// index exactly the way cupoch::knn::KDTreeFlann does; it contains no reference code.  The reference sources are
// compiled WHERE THEY LIE in a cupoch checkout (oracle/ref_flann/Makefile) into oracle/_ref/libflann_ref.so,
// which is git-ignored and only ever loaded by tools/make_flann_golden.py (never by cupoch_b200/).
//
// Call sequence mirrored (reference file:line):
//   SetRawData    src/cupoch/knn/kdtree_flann.inl:125-144  float3 -> float4 (w = 0), Matrix with 16-B stride,
//                                                           KDTreeCuda3dIndexParams() (leaf_max_size 64), buildIndex()
//   SearchKNN     kdtree_flann.inl:70-95                     queries -> float4, matrices_in_gpu_ram, knnSearch
//   SearchRadius  kdtree_flann.inl:97-122                    SearchParams(-1, 0.0), max_neighbors = max_nn,
//                                                           radiusSearch(radius * radius)
// cupoch remaps nothing afterwards: FLANN's indices are positions in the data set as given.
#include <cuda_runtime.h>
#include <thrust/device_vector.h>

#include <memory>
#include <vector>

#define FLANN_USE_CUDA
#include "flann/flann.hpp"
#include "flann/algorithms/kdtree_cuda_3d_index.h"

namespace {
struct Ref {
    thrust::device_vector<float4> data;
    std::unique_ptr<flann::Matrix<float>> dataset;
    std::unique_ptr<flann::KDTreeCuda3dIndex<flann::L2<float>>> index;
};
thrust::device_vector<float4> to_float4(const float *h_xyz, int n) {
    std::vector<float4> h((size_t)n);
    for (int i = 0; i < n; ++i) h[i] = make_float4(h_xyz[3 * i], h_xyz[3 * i + 1], h_xyz[3 * i + 2], 0.f);
    return thrust::device_vector<float4>(h.begin(), h.end());
}
}  // namespace

extern "C" void *fref_build(const float *h_xyz, int n) {
    try {
        Ref *r = new Ref();
        r->data = to_float4(h_xyz, n);
        r->dataset.reset(new flann::Matrix<float>((float *)thrust::raw_pointer_cast(r->data.data()), (size_t)n, 3,
                                                  sizeof(float) * 4));
        flann::KDTreeCuda3dIndexParams index_params;
        r->index.reset(new flann::KDTreeCuda3dIndex<flann::L2<float>>(*r->dataset, index_params));
        r->index->buildIndex();
        return r;
    } catch (...) {
        return nullptr;
    }
}

extern "C" void fref_free(void *h) { delete (Ref *)h; }

// h_idx / h_d2: [nq][k] host arrays.  returns 0 on success
extern "C" int fref_knn(void *h, const float *h_q, int nq, int k, int *h_idx, float *h_d2) {
    try {
        Ref *r = (Ref *)h;
        thrust::device_vector<float4> q = to_float4(h_q, nq);
        thrust::device_vector<int> idx((size_t)nq * k);
        thrust::device_vector<float> d2((size_t)nq * k);
        flann::Matrix<float> qm((float *)thrust::raw_pointer_cast(q.data()), (size_t)nq, 3, sizeof(float) * 4);
        flann::Matrix<int> im(thrust::raw_pointer_cast(idx.data()), (size_t)nq, (size_t)k);
        flann::Matrix<float> dm(thrust::raw_pointer_cast(d2.data()), (size_t)nq, (size_t)k);
        flann::SearchParams param;
        param.matrices_in_gpu_ram = true;
        r->index->knnSearch(qm, im, dm, (size_t)k, param);
        cudaDeviceSynchronize();
        thrust::copy(idx.begin(), idx.end(), h_idx);
        thrust::copy(d2.begin(), d2.end(), h_d2);
        return 0;
    } catch (...) {
        return -1;
    }
}

extern "C" int fref_radius(void *h, const float *h_q, int nq, float radius, int max_nn, int *h_idx, float *h_d2) {
    try {
        Ref *r = (Ref *)h;
        thrust::device_vector<float4> q = to_float4(h_q, nq);
        thrust::device_vector<int> idx((size_t)nq * max_nn);
        thrust::device_vector<float> d2((size_t)nq * max_nn);
        flann::Matrix<float> qm((float *)thrust::raw_pointer_cast(q.data()), (size_t)nq, 3, sizeof(float) * 4);
        flann::Matrix<int> im(thrust::raw_pointer_cast(idx.data()), (size_t)nq, (size_t)max_nn);
        flann::Matrix<float> dm(thrust::raw_pointer_cast(d2.data()), (size_t)nq, (size_t)max_nn);
        flann::SearchParams param(-1, 0.0);
        param.max_neighbors = max_nn;
        param.matrices_in_gpu_ram = true;
        r->index->radiusSearch(qm, im, dm, float(radius * radius), param);
        cudaDeviceSynchronize();
        thrust::copy(idx.begin(), idx.end(), h_idx);
        thrust::copy(d2.begin(), d2.end(), h_d2);
        return 0;
    } catch (...) {
        return -1;
    }
}
