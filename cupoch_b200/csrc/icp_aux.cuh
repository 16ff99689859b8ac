// icp_aux.cuh -- working-copy kernels of the loop: source gather, correspondence compaction, PointCloud::Transform
// Part of the icp.cu translation unit (included there); split out for readability only.
#pragma once

// ---------------------------------------------------------------------------
// source preparation + correspondence compaction kernels
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gather_source_kernel(const float *__restrict__ xyz, const float *__restrict__ nrm,
                                                            const float *__restrict__ col, const float *__restrict__ cov,
                                                            int cov_col_major, const uint32_t *__restrict__ perm_all,
                                                            unsigned lo, unsigned n, unsigned n_pad, float4 *o_xyz,
                                                            float4 *o_nrm, float4 *o_col, float4 *o_cov) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    const uint32_t *perm = perm_all + lo;  // this rank's block of the Hilbert order
    if (i < n) {
        size_t j = perm[i];
        o_xyz[i] = make_float4(xyz[3 * j], xyz[3 * j + 1], xyz[3 * j + 2], __uint_as_float((unsigned)j));
        if (o_nrm) o_nrm[i] = make_float4(nrm[3 * j], nrm[3 * j + 1], nrm[3 * j + 2], 0.f);
        if (o_col) o_col[i] = make_float4(col[3 * j], col[3 * j + 1], col[3 * j + 2], 0.f);
        if (o_cov) {
            const float *c = cov + 9 * j;
            for (int r = 0; r < 3; ++r)
                o_cov[(size_t)r * n_pad + i] = cov_col_major ? make_float4(c[r], c[3 + r], c[6 + r], 0.f)
                                                             : make_float4(c[3 * r], c[3 * r + 1], c[3 * r + 2], 0.f);
        }
    } else {
        // padding lanes: a copy of the last real point keeps loads in bounds; w = -1, never "valid"
        size_t j = n ? perm[n - 1] : 0;
        float4 p = n ? make_float4(xyz[3 * j], xyz[3 * j + 1], xyz[3 * j + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        p.w = __uint_as_float(0xffffffffu);
        o_xyz[i] = p;
        if (o_nrm) o_nrm[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (o_col) o_col[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (o_cov)
            for (int r = 0; r < 3; ++r) o_cov[(size_t)r * n_pad + i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// Private copies of the target attributes in INDEX order (icp_types.cuh): row p belongs to the point ix.pts[p].
// Padding rows (w == -1) are zero.  intensity(): colored_icp.cu:176-181, evaluated once here instead of once per row.
__global__ void __launch_bounds__(256) gather_target_kernel(const float4 *__restrict__ pts, size_t n_pad,
                                                            const float *__restrict__ nrm, const float *__restrict__ col,
                                                            const float *__restrict__ grad, const float *__restrict__ cov,
                                                            int cov_col_major, float4 *o_nrm, float4 *o_grad, float4 *o_cov) {
    size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (p >= n_pad) return;
    const unsigned j = __float_as_uint(pts[p].w);
    const bool real = j != 0xffffffffu;
    const size_t j3 = 3 * (size_t)j;
    if (o_nrm) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (real) {
            v.x = nrm[j3]; v.y = nrm[j3 + 1]; v.z = nrm[j3 + 2];
            if (col) v.w = intensity(col[j3], col[j3 + 1], col[j3 + 2]);
        }
        o_nrm[p] = v;
    }
    if (o_grad) o_grad[p] = real ? make_float4(grad[j3], grad[j3 + 1], grad[j3 + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (o_cov) {
        const float *c = cov + 9 * (size_t)j;
#pragma unroll
        for (int r = 0; r < 3; ++r)
            o_cov[3 * p + r] = !real ? make_float4(0.f, 0.f, 0.f, 0.f)
                                     : cov_col_major ? make_float4(c[r], c[3 + r], c[6 + r], 0.f)
                                                     : make_float4(c[3 * r], c[3 * r + 1], c[3 * r + 2], 0.f);
    }
}

// stable compaction of (i, corr_index[i]) with corr_index[i] >= 0 (registration.cu:54-69)
#define CMP_BLOCK 1024
__global__ void __launch_bounds__(CMP_BLOCK) compact_count_kernel(const int32_t *__restrict__ ci, unsigned n,
                                                                  unsigned *block_counts) {
    unsigned i = blockIdx.x * CMP_BLOCK + threadIdx.x;
    unsigned c = block_flag_count(i < n && ci[i] >= 0);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}
__global__ void __launch_bounds__(CMP_BLOCK) compact_write_kernel(const int32_t *__restrict__ ci, unsigned n,
                                                                  const unsigned *__restrict__ block_offsets,
                                                                  int32_t *out_pairs) {
    unsigned i = blockIdx.x * CMP_BLOCK + threadIdx.x;
    int32_t j = i < n ? ci[i] : -1;
    bool v = j >= 0;
    unsigned r = block_flag_rank(v);
    if (v) {
        unsigned pos = block_offsets[blockIdx.x] + r;
        out_pairs[2 * (size_t)pos] = (int32_t)i;
        out_pairs[2 * (size_t)pos + 1] = j;
    }
}

// PointCloud::Transform as a standalone op (pointcloud.cu:293-299)
__global__ void __launch_bounds__(256) transform_kernel(float *p, float *nrm, float *cov, int cov_col_major, size_t n,
                                                        const float *__restrict__ Tdev) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float U[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) U[k] = Tdev[k];
    if (p) {
        float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
        p[3 * i] = __fadd_rn(dot3(U[0], U[1], U[2], x, y, z), U[3]);
        p[3 * i + 1] = __fadd_rn(dot3(U[4], U[5], U[6], x, y, z), U[7]);
        p[3 * i + 2] = __fadd_rn(dot3(U[8], U[9], U[10], x, y, z), U[11]);
    }
    if (nrm) {
        float x = nrm[3 * i], y = nrm[3 * i + 1], z = nrm[3 * i + 2];
        nrm[3 * i] = dot3(U[0], U[1], U[2], x, y, z);
        nrm[3 * i + 1] = dot3(U[4], U[5], U[6], x, y, z);
        nrm[3 * i + 2] = dot3(U[8], U[9], U[10], x, y, z);
    }
    if (cov) {
        float C[9], tmp[9], O[9];
        float *c = cov + 9 * i;
        for (int r = 0; r < 3; ++r)
            for (int q = 0; q < 3; ++q) C[3 * r + q] = c[cov_col_major ? 3 * q + r : 3 * r + q];
        const float R[9] = {U[0], U[1], U[2], U[4], U[5], U[6], U[8], U[9], U[10]};
        for (int r = 0; r < 3; ++r)
            for (int q = 0; q < 3; ++q)
                tmp[3 * r + q] = dot3(R[3 * r], R[3 * r + 1], R[3 * r + 2], C[q], C[3 + q], C[6 + q]);
        for (int r = 0; r < 3; ++r)
            for (int q = 0; q < 3; ++q)
                O[3 * r + q] = dot3(tmp[3 * r], tmp[3 * r + 1], tmp[3 * r + 2], R[3 * q], R[3 * q + 1], R[3 * q + 2]);
        for (int r = 0; r < 3; ++r)
            for (int q = 0; q < 3; ++q) c[cov_col_major ? 3 * q + r : 3 * r + q] = O[3 * r + q];
    }
}

