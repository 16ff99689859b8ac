// icp_solve.cuh -- the device-side epilogue of one iteration: 6x6 determinant / LDLT / solve, Kabsch, convergence test, pose composition
// Part of the icp.cu translation unit (included there, in this order: icp_types, icp_solve, icp_rows); split out
// for readability only -- the arithmetic contract and the reference citations are stated in icp.cu.
#pragma once

// ===========================================================================
// finalize: 6x6 solve / Kabsch / convergence (one thread)
// ===========================================================================
// Both routines are written with compile-time indices only (pivot rows are brought in by predicated swaps over every
// candidate row), so the 6x6 matrix lives in registers: no shared / local memory round trip on the dependent chain.
// The arithmetic -- every operation and its order -- is that of Eigen's PartialPivLU determinant and LDLT
// (eigen.cu:92,103); the CPU oracle restates the same sequence independently.
__device__ __forceinline__ void swapf(float &a, float &b, bool doit) {
    const float t = a;
    a = doit ? b : a;
    b = doit ? t : b;
}
__device__ __forceinline__ float det6_partial_piv(const float *A_in) {
    float A[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) A[i][j] = A_in[6 * i + j];
    float det = 1.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        int p = k;
        float best = fabsf(A[k][k]);
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
            if (fabsf(A[i][k]) > best) { best = fabsf(A[i][k]); p = i; }
        if (best == 0.f) return 0.f;
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
#pragma unroll
            for (int j = 0; j < 6; ++j) swapf(A[k][j], A[i][j], p == i);
        if (p != k) det = -det;
        const float piv = A[k][k];
        det = det * piv;
#pragma unroll
        for (int i = k + 1; i < 6; ++i) {
            const float f = A[i][k] / piv;
#pragma unroll
            for (int j = k + 1; j < 6; ++j) A[i][j] = A[i][j] - f * A[k][j];
        }
    }
    return det;
}
// Eigen LDLT (diagonal pivoting, lower) + solve; eigen.cu:103 A.ldlt().solve(b)
__device__ __forceinline__ void ldlt6_solve(const float *A_in, const float *b, float *x) {
    float A[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) A[i][j] = A_in[6 * i + j];
    int tr[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        int ib = k;
        float big = fabsf(A[k][k]);
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
            if (fabsf(A[i][i]) > big) { big = fabsf(A[i][i]); ib = i; }
        tr[k] = ib;
        // symmetric swap of rows / columns k and ib in the lower triangle, for whichever candidate c == ib
#pragma unroll
        for (int c = k + 1; c < 6; ++c) {
            const bool doit = (ib == c);
#pragma unroll
            for (int j = 0; j < k; ++j) swapf(A[k][j], A[c][j], doit);
#pragma unroll
            for (int i = c + 1; i < 6; ++i) swapf(A[i][k], A[i][c], doit);
            swapf(A[k][k], A[c][c], doit);
#pragma unroll
            for (int i = k + 1; i < c; ++i) swapf(A[i][k], A[c][i], doit);
        }
        float temp[6];
        if (k > 0) {
#pragma unroll
            for (int j = 0; j < k; ++j) temp[j] = A[j][j] * A[k][j];
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < k; ++j) s = s + A[k][j] * temp[j];
            A[k][k] = A[k][k] - s;
#pragma unroll
            for (int i = k + 1; i < 6; ++i) {
                float s2 = 0.f;
#pragma unroll
                for (int j = 0; j < k; ++j) s2 = s2 + A[i][j] * temp[j];
                A[i][k] = A[i][k] - s2;
            }
        }
        const float akk = A[k][k];
        if (fabsf(akk) > 0.f)
#pragma unroll
            for (int i = k + 1; i < 6; ++i) A[i][k] = A[i][k] / akk;
    }
    float y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] = b[i];
#pragma unroll
    for (int k = 0; k < 6; ++k)
#pragma unroll
        for (int c = k + 1; c < 6; ++c) swapf(y[k], y[c], tr[k] == c);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        float s = y[i];
#pragma unroll
        for (int j = 0; j < i; ++j) s = s - A[i][j] * y[j];
        y[i] = s;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] = (fabsf(A[i][i]) > FLT_MIN) ? y[i] / A[i][i] : 0.f;
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        float s = y[i];
#pragma unroll
        for (int j = i + 1; j < 6; ++j) s = s - A[j][i] * y[j];
        y[i] = s;
    }
#pragma unroll
    for (int k = 5; k >= 0; --k)
#pragma unroll
        for (int c = k + 1; c < 6; ++c) swapf(y[k], y[c], tr[k] == c);
#pragma unroll
    for (int i = 0; i < 6; ++i) x[i] = y[i];
}
__device__ void identity4(float *T) {
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.f : 0.f;
}
__device__ void se3_exp(const float *x, float *T) {  // eigen.cu:28-50
    identity4(T);
    T[3] = x[3]; T[7] = x[4]; T[11] = x[5];
    float th = sqrtf((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
    if (th == 0) return;
    float w0 = x[0] / th, w1 = x[1] / th, w2 = x[2] / th;
    float c = (float)cos((double)th), s = (float)sin((double)th);
    float oc = 1 - c;
    T[0] = c + w0 * w0 * oc;
    T[1] = w0 * w1 * oc - w2 * s;
    T[2] = w1 * s + w0 * w2 * oc;
    T[4] = w2 * s + w0 * w1 * oc;
    T[5] = c + w1 * w1 * oc;
    T[6] = -w0 * s + w1 * w2 * oc;
    T[8] = -w1 * s + w0 * w2 * oc;
    T[9] = w0 * s + w1 * w2 * oc;
    T[10] = c + w2 * w2 * oc;
}
// the normal equations of the 32 sums: A (symmetric 6x6) and b = -JTr
__device__ __forceinline__ void jtj_system(const double *S, float (&A)[36], float (&b)[6]) {
    int p = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int c = a; c < 6; ++c) { float v = (float)S[p++]; A[6 * a + c] = v; A[6 * c + a] = v; }
#pragma unroll
    for (int a = 0; a < 6; ++a) b[a] = -(float)S[21 + a];
}
// eigen.cu:88-100: the update is rejected (identity) when |det| < det_thresh or det is not finite
__device__ __forceinline__ bool det_accepts(float det, float det_thresh) {
    return !(fabsf(det) < det_thresh || isnan(det) || isinf(det));
}
__device__ bool solve_jtj(const double *S, float det_thresh, float *T) {
    float A[36], b[6], x[6];
    jtj_system(S, A, b);
    identity4(T);
    if (det_thresh > 0 && !det_accepts(det6_partial_piv(A), det_thresh)) return false;
    ldlt6_solve(A, b, x);
    se3_exp(x, T);
    return true;
}
__device__ __noinline__ float det_core(const double *S) {
    float A[36], b[6];
    jtj_system(S, A, b);
    return det6_partial_piv(A);
}
__device__ __noinline__ void solve_core(const double *S, float *T) {
    float A[36], b[6], x[6];
    jtj_system(S, A, b);
    ldlt6_solve(A, b, x);
    se3_exp(x, T);
}
struct SolveSmem {
    float T[16];
    double S[32];  // the iteration's 32 sums, staged for the solving lane
    float det;     // icp_finalize<KIND, true>: the determinant, computed by a second warp while the first one solves
};
// Called by every warp of a block that is NOT the last to arrive, after a __syncthreads that made m.S (this block's own
// partial sums) visible: lane 0 of warp 0 runs the solve and lane 0 of warp 1 the determinant, the very functions
// icp_finalize<KIND, true> calls, and the results are dropped.  Only their instructions matter: the iteration's working
// set evicts the kernel's code from L2 between launches, so the last block's single-lane solve would otherwise fetch its
// unrolled code line by line from HBM (config 2 on the H100, launch 20: 9.1 us cold, 2.6 us warm; DESIGN section 5).
template <int KIND>
__device__ void warm_solve(const IcpArgs &a, SolveSmem &m) {
    if (KIND == CPHB_EST_POINT_TO_POINT || lane_id() != 0) return;  // (Kabsch: a different, shorter epilogue)
    constexpr bool uses_det = (KIND != CPHB_EST_GENERALIZED_ICP);
    const int warp = threadIdx.x >> 5;
    if (warp == 0) solve_core(m.S, m.T);
    else if (warp == 1 && uses_det && a.det_thresh > 0) m.det = det_core(m.S);
}

__device__ void matmul4(const float *A, const float *B, float *C) {  // registration.cu:159
    float R[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            R[4 * i + j] = ((A[4 * i] * B[j] + A[4 * i + 1] * B[4 + j]) + A[4 * i + 2] * B[8 + j]) + A[4 * i + 3] * B[12 + j];
    for (int i = 0; i < 16; ++i) C[i] = R[i];
}
// one-sided Jacobi SVD (double) -- stands in for Eigen::JacobiSVD<Matrix3f> (kabsch.cu:108-109);
// R = V diag(1,1,det(UV)) U^T is unique whatever the SVD's sign/ordering conventions.
__device__ void svd3(const double *A, double *U, double *s, double *V) {
    double B[9];
    for (int i = 0; i < 9; ++i) { B[i] = A[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < 3; ++i) {
                    al += B[3 * i + p] * B[3 * i + p];
                    be += B[3 * i + q] * B[3 * i + q];
                    ga += B[3 * i + p] * B[3 * i + q];
                }
                if (fabs(ga) <= 1e-300 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
                off += fabs(ga);
                double zeta = (be - al) / (2.0 * ga);
                double t = ((zeta >= 0) ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < 3; ++i) {
                    double bp = B[3 * i + p], bq = B[3 * i + q];
                    B[3 * i + p] = c * bp - sn * bq;
                    B[3 * i + q] = sn * bp + c * bq;
                    double vp = V[3 * i + p], vq = V[3 * i + q];
                    V[3 * i + p] = c * vp - sn * vq;
                    V[3 * i + q] = sn * vp + c * vq;
                }
            }
        if (off == 0) break;
    }
    for (int j = 0; j < 3; ++j) {
        double nn = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
        s[j] = nn;
        for (int i = 0; i < 3; ++i) U[3 * i + j] = (nn > 0) ? B[3 * i + j] / nn : 0.0;
    }
    for (int j = 0; j < 3; ++j)
        if (s[j] == 0) {
            int a = (j + 1) % 3, b = (j + 2) % 3;
            if (s[a] > 0 && s[b] > 0) {
                U[j] = U[3 + a] * U[6 + b] - U[6 + a] * U[3 + b];
                U[3 + j] = U[6 + a] * U[b] - U[a] * U[6 + b];
                U[6 + j] = U[a] * U[3 + b] - U[3 + a] * U[b];
            }
        }
    // A = 0 (one correspondence, or every model point at its centre): Eigen's JacobiSVD returns U = V = I, so Kabsch
    // gives the identity rotation; a zero U here would make R = 0 and collapse the cloud onto one point
    if (s[0] == 0 && s[1] == 0 && s[2] == 0)
        for (int i = 0; i < 9; ++i) U[i] = (i % 4 == 0) ? 1.0 : 0.0;
}
// kabsch.cu:42-120 incl. the divide-by-model.size() quirk (:76-78,107)
__device__ void kabsch_from_sums(const double *S, unsigned long long n_model, float *T) {
    identity4(T);
    double C = S[29];
    float div = 1.0f / (float)n_model;
    float mc[3], tc[3];
    for (int a = 0; a < 3; ++a) { mc[a] = (float)S[a] * div; tc[a] = (float)S[3 + a] * div; }
    double H[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            double h = S[6 + 3 * a + b] - (double)mc[a] * S[3 + b] - S[a] * (double)tc[b] + C * (double)mc[a] * (double)tc[b];
            H[3 * a + b] = (double)((float)h / (float)n_model);
        }
    double U[9], sv[3], V[9], UV[9];
    svd3(H, U, sv, V);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) UV[3 * i + j] = U[3 * i] * V[j] + U[3 * i + 1] * V[3 + j] + U[3 * i + 2] * V[6 + j];
    double dd = UV[0] * (UV[4] * UV[8] - UV[5] * UV[7]) - UV[1] * (UV[3] * UV[8] - UV[5] * UV[6]) +
                UV[2] * (UV[3] * UV[7] - UV[4] * UV[6]);
    double ss[3] = {1.0, 1.0, dd};
    float R[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double r = 0;
            for (int k = 0; k < 3; ++k) r += V[3 * i + k] * ss[k] * U[3 * j + k];
            R[3 * i + j] = (float)r;
        }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[4 * i + j] = R[3 * i + j];
        T[4 * i + 3] = tc[i] - dot3(R[3 * i], R[3 * i + 1], R[3 * i + 2], mc[0], mc[1], mc[2]);
    }
}

// registration.cu:71-78,154-172 -- after the grid-wide sum.
// S = m.S: the 32 sums of this iteration, staged in shared memory by the caller (also in st->total for the host).
// PAR = false: runs in ONE WARP (all 32 lanes call it).
// PAR = true : called by EVERY warp of a block of >= 2 warps, after a __syncthreads that made m.S visible.  The 6x6
//              determinant (partial-pivot LU) and the LDLT solve are independent chains of equal length on one lane:
//              warp 1 computes the determinant while warp 0 solves; one __syncthreads joins them.  Same operations,
//              same results.
template <int KIND, bool PAR = false>
__device__ void icp_finalize(const IcpArgs &a, IcpState *st, SolveSmem &m) {
    const int lane = lane_id();
    const double *S = m.S;
    if (PAR) {
        const int warp = threadIdx.x >> 5;
        constexpr bool uses_det = (KIND != CPHB_EST_POINT_TO_POINT && KIND != CPHB_EST_GENERALIZED_ICP);
        if (warp == 1 && lane == 0 && uses_det && a.det_thresh > 0) m.det = det_core(S);
        if (warp != 0) {
            __syncthreads();
            return;
        }
    }
    int action = 0;  // 0 = nothing more, 1 = compute an update
    double cnt = 0.0;
    if (lane == 0) {
        cnt = S[29];
        float fit = 0.f, rmse = 0.f;
        if (cnt > 0) {
            fit = (float)cnt / (float)a.n_total;
            rmse = sqrtf((float)S[28] / (float)cnt);
        }
        const float pf = st->fitness, pr = st->rmse;
        st->fitness = fit;
        st->rmse = rmse;
        st->n_corr = (long long)cnt;
        if (a.step_mode) {
            action = 0;
        } else if (a.launch_idx > 0 && fabsf(pf - fit) < a.rel_fitness && fabsf(pr - rmse) < a.rel_rmse) {
            st->converged = 1;
            st->done = (a.corr_index && a.launch_idx < a.max_iter) ? 1 : 2;
        } else if (a.launch_idx >= a.max_iter) {
            st->done = 2;
        } else {
            action = 1;
        }
    }
    action = __shfl_sync(CPHB_FULL, action, 0);
    if (lane == 0) dbg_time(a, 5, false);
    bool joined = false;  // PAR: warp 0 meets the other warps at exactly one __syncthreads on every (warp-uniform) path
    if (!action) {
        if (PAR) __syncthreads();
        return;
    }
    const bool have_corr = __shfl_sync(CPHB_FULL, (int)(cnt > 0), 0) != 0;
    if (lane == 0) identity4(m.T);
    __syncwarp();
    if (have_corr) {
        if (KIND == CPHB_EST_POINT_TO_POINT) {
            if (lane == 0) kabsch_from_sums(S, a.n_total, m.T);
            __syncwarp();
        } else {
            bool have = true;
            if ((KIND == CPHB_EST_POINT_TO_PLANE || KIND == CPHB_EST_COLORED_ICP) && !a.tgt_nrm) have = false;
            if (KIND == CPHB_EST_SYMMETRIC && (!a.tgt_nrm || !a.src_nrm)) have = false;
            if (KIND == CPHB_EST_COLORED_ICP && (!a.has_tgt_col || !a.src_col)) have = false;
            if (KIND == CPHB_EST_GENERALIZED_ICP && (!a.tgt_cov || !a.src_cov)) have = false;
            if (have) {
                const float dt = (KIND == CPHB_EST_GENERALIZED_ICP) ? -1.f : a.det_thresh;
                // one lane, everything in registers (a warp-parallel shared-memory version spends most of its time in
                // __syncwarp-separated steps)
                bool ok = true;
                if (PAR) {
                    if (lane == 0) solve_core(S, m.T);  // solve first, learn the determinant afterwards (it only decides accept / reject)
                    __syncthreads();
                    joined = true;
                    if (lane == 0) {
                        if (dt > 0 && !det_accepts(m.det, dt)) ok = false;
                        dbg_time(a, 6, false);
                    }
                } else if (lane == 0) {
                    ok = solve_jtj(S, dt, m.T);
                    dbg_time(a, 6, false);
                }
                ok = __shfl_sync(CPHB_FULL, (int)ok, 0) != 0;
                if (!ok && lane == 0) identity4(m.T);
                if (ok && KIND == CPHB_EST_SYMMETRIC && lane == 0) {  // transformation_estimation.cu:319-339
                    double R[9], R2[9];
                    for (int i = 0; i < 3; ++i)
                        for (int j = 0; j < 3; ++j) R[3 * i + j] = (double)m.T[4 * i + j];
                    for (int i = 0; i < 3; ++i)
                        for (int j = 0; j < 3; ++j)
                            R2[3 * i + j] = R[3 * i] * R[j] + R[3 * i + 1] * R[3 + j] + R[3 * i + 2] * R[6 + j];
                    for (int i = 0; i < 3; ++i)
                        for (int j = 0; j < 3; ++j) m.T[4 * i + j] = (float)R2[3 * i + j];
                }
                __syncwarp();
            }
        }
    }
    if (PAR && !joined) __syncthreads();
    // transformation = update * transformation (registration.cu:159): one output element per lane
    float tn = 0.f;
    if (lane < 16) {
        const int i = lane >> 2, j = lane & 3;
        const float *A = m.T, *B = st->T;
        tn = ((A[4 * i] * B[j] + A[4 * i + 1] * B[4 + j]) + A[4 * i + 2] * B[8 + j]) + A[4 * i + 3] * B[12 + j];
    }
    __syncwarp();
    if (lane == 0) dbg_time(a, 7, false);
    if (lane < 16) {
        st->T[lane] = tn;
        st->U[lane] = m.T[lane];
    }
    if (lane == 0) {
        st->apply_u = 1;
        st->iterations += 1;
    }
    __syncwarp();
}

