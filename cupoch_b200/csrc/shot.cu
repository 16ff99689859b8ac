// shot.cu -- registration::ComputeSHOTFeature (shot.cu:222-255): SHOT descriptors (352 bins) of every point.
//
// The reference writes an [n][k] index table and an [n][k] distance table, then runs one thread per point that carries
// its 352-float histogram in local memory and evaluates an acos and an atan2 for each neighbour in turn.  Here one index
// serves one fused kernel (fused_neighbourhood.cuh): shot_kernel searches each point's list into shared memory and
// consumes it there, so no [n][k] table exists.
//   frame      each lane builds its own query's local reference frame (compute_shot_lrf, :63-98) sequentially over its
//              own list, in list order;
//   histogram  the warp then takes its 32 queries in turn.  Lane l evaluates neighbours l, l + 32, ... of the query
//              (the float64 det_acosf / det_atan2f run in parallel) and stages their <= 5 (bin, weight) contributions;
//              the contributions are then added to the warp's 352-float shared-memory histogram one neighbour after
//              the other, in list order -- a neighbour's bins are distinct, so each bin's float32 sum is the
//              reference's sequence.  No atomics.  The norm is one lane's sequential sum of squares in bin order, and
//              the normalised row is stored coalesced.
// Queries are taken in index order (self_order of fused_query_setup).
//
// Arithmetic (DESIGN.md arithmetic contract; oracle/shot.c restates it).  compute_shot_functor (:100-218) operation by
// operation with C++ promotion as written: the clamps of cos_desc, of the inclination cosine and of the azimuth distance
// are float64 fmin / fmax (NaN loses) rounded to float; bindist = ((1.0 + cos_desc) * 10) / 2.0 and radius * 3.0 / 4.0
// are float64 rounded to float; step_index rounds (float)(bindist +- 0.5); the PST_RAD_* constants are float.  Eigen's
// dot and cross are the library's dot3 / cross3; cov += (w q) q^T and every other float operation is IEEE and unfused
// (-fmad=false); acos / atan2 are det_acosf / det_atan2f.  z / x are the columns of FastEigen3x3's smallest / largest
// eigenvalue as minCoeff / maxCoeff pick them (first strict improvement).  The norm is Eigen's non-vectorised linear
// redux: bins 0..351 squared and summed in float32 in order.
#include <math.h>

#include "cphb_eigen3.cuh"
#include "cphb_internal.cuh"
#include "fused_neighbourhood.cuh"

#define SHOT_DIM 352
#define SHOT_BINS 10        // n_bins_: 11 cosine columns per volume (step_index reaches 10)
#define SHOT_MIN_NB 5       // min_neighbors_
#define SHOT_SECTORS 32     // max_angular_sectors_
#define SHOT_KNN_MAX 100    // KDTreeFlann's NUM_MAX_NN
#define SHOT_RADIUS_MAX 256 // the radius search's own limit (search.cu CPHB_RADIUS_MAX_NN)
// per warp, after the lists: the histogram and 32 neighbours x 5 staged (bin, weight) contributions
#define SHOT_STAGE (32 * 5)
#define SHOT_EXTRA (SHOT_DIM * sizeof(float) + SHOT_STAGE * (sizeof(int) + sizeof(float)))

#define PST_RAD_45 0.78539816339744830961566084581988f
#define PST_RAD_90 1.5707963267948966192313216916398f
#define PST_RAD_135 2.3561944901923449288469825374596f
#define PST_RAD_PI_7_8 2.7488935718910690836548129603691f

// min(max(v, lo), hi) of the reference with a float v and double bounds: float64 fmax / fmin, rounded to float
__device__ __forceinline__ float clamp_d(float v, double lo, double hi) { return (float)fmin(fmax((double)v, lo), hi); }

// one neighbour's contributions (compute_shot_functor :111-211): bin[c] < 0 marks an absent one
__device__ __forceinline__ void shot_neighbour(float qx, float qy, float qz, float dist, const float (&X)[3],
                                               const float (&Y)[3], const float (&Z)[3], float r12, float r14, float r34,
                                               int step, int cos_col, float cos_w, float init_w, int (&bin)[5],
                                               float (&wt)[5]) {
    float x = dot3(qx, qy, qz, X[0], X[1], X[2]);
    float y = dot3(qx, qy, qz, Y[0], Y[1], Y[2]);
    float z = dot3(qx, qy, qz, Z[0], Z[1], Z[2]);
    if ((double)fabsf(x) < 1.0e-30) x = 0.f;
    if ((double)fabsf(y) < 1.0e-30) y = 0.f;
    if ((double)fabsf(z) < 1.0e-30) z = 0.f;
    const int bit4 = (y > 0.f || (y == 0.f && x < 0.f)) ? 1 : 0;
    const int bit3 = (x > 0.f || (x == 0.f && y > 0.f)) ? !bit4 : bit4;
    int desc = ((bit4 << 3) + (bit3 << 2)) << 1;
    if (x * y > 0.f || x == 0.f) desc += (fabsf(x) >= fabsf(y)) ? 0 : 4;
    else desc += (fabsf(x) > fabsf(y)) ? 4 : 0;
    desc += z > 0.f ? 1 : 0;
    desc += (dist > r12) ? 2 : 0;
    const int vol = desc * (SHOT_BINS + 1);
    bin[0] = vol + cos_col;  // interpolation on the cosine: the same column for every neighbour of the point
    wt[0] = cos_w;
    bin[1] = bin[2] = bin[3] = -1;
    wt[1] = wt[2] = wt[3] = 0.f;
    float iw = init_w;
    if (dist > r12) {  // interpolation on the distance (adjacent husks)
        const float rd = (dist - r34) / r12;
        if (dist > r34) {
            iw += 1.f - rd;
        } else {
            iw += 1.f + rd;
            bin[1] = (desc - 2) * (SHOT_BINS + 1) + step;
            wt[1] = -rd;
        }
    } else {
        const float rd = (dist - r14) / r12;
        if (dist < r14) {
            iw += 1.f + rd;
        } else {
            iw += 1.f - rd;
            bin[1] = (desc + 2) * (SHOT_BINS + 1) + step;
            wt[1] = rd;
        }
    }
    const float inc = det_acosf(clamp_d(z / dist, -1.0, 1.0));  // interpolation on the inclination
    if (inc > PST_RAD_90 || ((double)fabsf(inc - PST_RAD_90) < 1e-30 && z <= 0.f)) {
        const float d = (inc - PST_RAD_135) / PST_RAD_90;
        if (inc > PST_RAD_135) {
            iw += 1.f - d;
        } else {
            iw += 1.f + d;
            bin[2] = (desc + 1) * (SHOT_BINS + 1) + step;
            wt[2] = -d;
        }
    } else {
        const float d = (inc - PST_RAD_45) / PST_RAD_90;
        if (inc < PST_RAD_45) {
            iw += 1.f + d;
        } else {
            iw += 1.f - d;
            bin[2] = (desc - 1) * (SHOT_BINS + 1) + step;
            wt[2] = d;
        }
    }
    if (y != 0.f || x != 0.f) {  // interpolation on the azimuth (adjacent horizontal volumes)
        const float az = det_atan2f(y, x);
        const int sel = desc >> 2;
        const float start = -PST_RAD_PI_7_8;
        const float ad = clamp_d((az - (start + PST_RAD_45 * (float)sel)) / PST_RAD_45, -0.5, 0.5);
        if (ad > 0.f) {
            iw += 1.f - ad;
            bin[3] = ((desc + 4) % SHOT_SECTORS) * (SHOT_BINS + 1) + step;
            wt[3] = ad;
        } else {
            iw += 1.f + ad;
            bin[3] = ((desc - 4 + SHOT_SECTORS) % SHOT_SECTORS) * (SHOT_BINS + 1) + step;
            wt[3] = -ad;
        }
    }
    bin[4] = vol + step;
    wt[4] = iw;
}

template <int TOP>
__global__ void shot_kernel(IndexView ix, const float *__restrict__ pts, const float *__restrict__ nrm, float r2, int k,
                            float radius, float *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem[];
    WarpSearchK w;
    size_t pos;
    const unsigned long long init = fused_query_setup(w, smem, ix, pts, 0, 0, nullptr, 1, r2, k, pos);
    fused_query_search<TOP>(ix, w);
    const int lane = lane_id();
    float *hist = (float *)fused_warp_extra(smem, k, SHOT_EXTRA);
    int *st_bin = (int *)(hist + SHOT_DIM);
    float *st_w = (float *)(st_bin + SHOT_STAGE);
    const unsigned long long *lists = w.list - lane;  // slot j of lane l: lists[j * 32 + l]

    // ---- this lane's frame (compute_shot_lrf, :63-98) and the point's cosine column (:115-117, :142-151)
    float X[3] = {0.f, 0.f, 0.f}, Y[3] = {0.f, 0.f, 0.f}, Z[3] = {0.f, 0.f, 0.f};
    int cnt = 0, n_nb = 0, step = 0, cos_col = 0;
    float cos_w = 0.f, init_w = 0.f;
    if (w.valid) {
        float cov[9];
#pragma unroll
        for (int a = 0; a < 9; ++a) cov[a] = 0.f;
        float w_total = 0.f;
        for (int j = 0; j < k; ++j) {
            const unsigned long long key = w.list[j * 32];
            if (!(key < init)) break;  // ascending: the unfilled slots are at the end
            ++cnt;
            const unsigned id = (unsigned)(key & 0xffffffffull);
            if (id == (unsigned)pos) continue;  // self, by index only
            const float q[3] = {pts[3 * (size_t)id] - w.qx, pts[3 * (size_t)id + 1] - w.qy, pts[3 * (size_t)id + 2] - w.qz};
            const float wgt = radius - sqrtf(__uint_as_float((unsigned)(key >> 32)));
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float wq = wgt * q[a];
#pragma unroll
                for (int b = 0; b < 3; ++b) cov[3 * a + b] = cov[3 * a + b] + wq * q[b];
            }
            w_total = w_total + wgt;
            ++n_nb;
        }
#pragma unroll
        for (int a = 0; a < 9; ++a) cov[a] = cov[a] / w_total;  // w_total == 0: NaN coefficients, as the reference
        float e[3], V[9];
        fast_eigen3x3(cov, e, V);
        int mn = 0, mx = 0;
        if (e[1] < e[mn]) mn = 1;
        if (e[2] < e[mn]) mn = 2;
        if (e[1] > e[mx]) mx = 1;
        if (e[2] > e[mx]) mx = 2;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            Z[r] = mn == 0 ? V[3 * r] : (mn == 1 ? V[3 * r + 1] : V[3 * r + 2]);
            X[r] = mx == 0 ? V[3 * r] : (mx == 1 ? V[3 * r + 1] : V[3 * r + 2]);
        }
        int n_px = 0, n_pz = 0;
        for (int j = 0; j < cnt; ++j) {
            const unsigned long long key = w.list[j * 32];
            const unsigned id = (unsigned)(key & 0xffffffffull);
            if (id == (unsigned)pos) continue;
            const float q0 = pts[3 * (size_t)id] - w.qx, q1 = pts[3 * (size_t)id + 1] - w.qy, q2 = pts[3 * (size_t)id + 2] - w.qz;
            n_px += dot3(q0, q1, q2, X[0], X[1], X[2]) >= 0.f;
            n_pz += dot3(q0, q1, q2, Z[0], Z[1], Z[2]) >= 0.f;
        }
        if (n_px < n_nb - n_px) { X[0] = -X[0]; X[1] = -X[1]; X[2] = -X[2]; }
        if (n_pz < n_nb - n_pz) { Z[0] = -Z[0]; Z[1] = -Z[1]; Z[2] = -Z[2]; }
        cross3(Z, X, Y);
        const float cos_desc = clamp_d(dot3(Z[0], Z[1], Z[2], nrm[3 * pos], nrm[3 * pos + 1], nrm[3 * pos + 2]), -1.0, 1.0);
        float bindist = (float)(((1.0 + (double)cos_desc) * SHOT_BINS) / 2.0);
        step = (bindist < 0.f) ? (int)ceilf((float)((double)bindist - 0.5)) : (int)floorf((float)((double)bindist + 0.5));
        bindist = bindist - (float)step;
        init_w = 1.f - fabsf(bindist);
        if (bindist > 0.f) { cos_col = (step + 1) % SHOT_BINS; cos_w = bindist; }
        else { cos_col = (step - 1 + SHOT_BINS) % SHOT_BINS; cos_w = -bindist; }
    }
    const float r12 = (float)((double)radius * 0.5);
    const float r34 = (float)((double)radius * 3.0 / 4.0);
    const float r14 = (float)((double)radius * 0.25);

    // ---- the warp's 32 histograms, one query after the other
    for (int t = 0; t < 32; ++t) {
        if (!__shfl_sync(CPHB_FULL, (int)w.valid, t)) continue;  // uniform: the padded tail of the index
        const unsigned pos_t = __shfl_sync(CPHB_FULL, (unsigned)pos, t);
        const int cnt_t = __shfl_sync(CPHB_FULL, cnt, t);
        const int nb_t = __shfl_sync(CPHB_FULL, n_nb, t);
        const float px = __shfl_sync(CPHB_FULL, w.qx, t), py = __shfl_sync(CPHB_FULL, w.qy, t),
                    pz = __shfl_sync(CPHB_FULL, w.qz, t);
        float Xt[3], Yt[3], Zt[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            Xt[a] = __shfl_sync(CPHB_FULL, X[a], t);
            Yt[a] = __shfl_sync(CPHB_FULL, Y[a], t);
            Zt[a] = __shfl_sync(CPHB_FULL, Z[a], t);
        }
        const int step_t = __shfl_sync(CPHB_FULL, step, t), col_t = __shfl_sync(CPHB_FULL, cos_col, t);
        const float cw_t = __shfl_sync(CPHB_FULL, cos_w, t), iw_t = __shfl_sync(CPHB_FULL, init_w, t);
        for (int b = lane; b < SHOT_DIM; b += 32) hist[b] = 0.f;
        __syncwarp();
        if (nb_t >= SHOT_MIN_NB) {  // fewer frame neighbours: an all-zero row (:106-108)
            for (int base = 0; base < cnt_t; base += 32) {
                const int j = base + lane;
                int bin[5] = {-1, -1, -1, -1, -1};
                float wt[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
                if (j < cnt_t) {
                    const unsigned long long key = lists[j * 32 + t];
                    const unsigned id = (unsigned)(key & 0xffffffffull);
                    const float dist = sqrtf(__uint_as_float((unsigned)(key >> 32)));
                    if (id != pos_t && dist != 0.f)  // self by index; a coincident duplicate adds nothing (:114)
                        shot_neighbour(pts[3 * (size_t)id] - px, pts[3 * (size_t)id + 1] - py, pts[3 * (size_t)id + 2] - pz,
                                       dist, Xt, Yt, Zt, r12, r14, r34, step_t, col_t, cw_t, iw_t, bin, wt);
                }
#pragma unroll
                for (int c = 0; c < 5; ++c) {
                    st_bin[lane * 5 + c] = bin[c];
                    st_w[lane * 5 + c] = wt[c];
                }
                __syncwarp();
                const int m = min(32, cnt_t - base);
                for (int s = 0; s < m; ++s) {  // neighbour order; lane c < 5 adds contribution c (distinct bins)
                    if (lane < 5) {
                        const int b = st_bin[s * 5 + lane];
                        if (b >= 0) hist[b] = hist[b] + st_w[s * 5 + lane];
                    }
                    __syncwarp();
                }
            }
        }
        float norm = 0.f;
        if (lane == 0) {
            float sq = hist[0] * hist[0];
            for (int b = 1; b < SHOT_DIM; ++b) sq = sq + hist[b] * hist[b];
            norm = sqrtf(sq);
        }
        norm = __shfl_sync(CPHB_FULL, norm, 0);
        float *row = out + (size_t)pos_t * SHOT_DIM;
        for (int b = lane; b < SHOT_DIM; b += 32) row[b] = norm > 0.f ? hist[b] / norm : hist[b];
        __syncwarp();
    }
}

extern "C" int cphb_compute_shot_feature(const float *points, const float *normals, size_t n, float radius, int knn,
                                         float search_radius, int max_nn, float *out_features, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const int k = (knn > 0) ? knn : max_nn;
    if ((knn > 0 && knn > SHOT_KNN_MAX) || (knn <= 0 && (max_nn < 0 || max_nn > SHOT_RADIUS_MAX)) || n > (size_t)INT32_MAX) {
        cphb_set_error("cphb_compute_shot_feature: knn = %d, max_nn = %d, n = %zu (need knn <= %d, 0 <= max_nn <= %d, "
                       "n <= 2^31-1)", knn, max_nn, n, SHOT_KNN_MAX, SHOT_RADIUS_MAX);
        return CPHB_ERR_INVALID;
    }
    if (n == 0) return CPHB_OK;
    if (!points || !normals || !out_features) {
        cphb_set_error("cphb_compute_shot_feature: null argument (the reference requires normals)");
        return CPHB_ERR_INVALID;
    }
    if (k == 0) {  // nothing is listed: every point has fewer than 5 frame neighbours
        CPHB_CUDA(cudaMemsetAsync(out_features, 0, n * SHOT_DIM * sizeof(float), s));
        return CPHB_OK;
    }
    const float r2 = (knn > 0) ? INFINITY : search_radius * search_radius;  // kdtree_flann.inl:120
    cphb_index *ix = nullptr;
    int rc = cphb_index_create(points, n, s, &ix);
    if (!rc) {
        const size_t lanes = (size_t)ix->v.n_leaves * CPHB_LEAF;  // the indexed points in index order
        rc = launch_fused_extra(ix, shot_kernel<3>, shot_kernel<5>, lanes, k, SHOT_EXTRA, s, points, normals, r2, k, radius,
                                out_features);
    }
    const cudaError_t e = cudaStreamSynchronize(s);
    if (ix) cphb_index_destroy(ix);
    if (!rc && e != cudaSuccess) {
        cphb_set_error("shot_kernel: %s", cudaGetErrorString(e));
        rc = CPHB_ERR_CUDA;
    }
    return rc;
}
