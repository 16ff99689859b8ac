// icp_kernels.cuh -- the kernels of one ICP iteration.  Part of the icp.cu translation unit (included there).
//
//   icp_iteration_kernel<KIND, TOP, ROLE>   transform -> certificate / exact 1-NN search -> estimator rows -> sums -> solve.
//       Two regimes, chosen on the DEVICE from the previous launch's statistics (no host round trip inside the loop), and
//       two separately compiled instances launched back to back every iteration; the instance the current regime does not
//       concern returns at its first instructions:
//        ROLE 0, searching regime  (tiles need searches, cost varies 10x): persistent warps claim tiles from an atomic counter,
//                          rows are staged in shared memory and every tile writes its 32 column sums to tile_sums[tile]
//                          (schedule-independent).  Compiled for 96 registers = 20 warps / SM.
//        ROLE 1, certified regime  (>= 90 % of the previous launch's tiles were skipped by their certificates): static round-
//                          robin tile schedule, cp.async pipeline, the normal-equation sums of every tile on the FP64 tensor
//                          cores (one 8 x 8 Gram fragment per warp), block rows -> last-arriving block adds them in block
//                          order, exchanges them with the other ranks and runs the solve IN THE SAME LAUNCH.  The per-
//                          point stream is marked evict-first in L2, and the blocks that are not last run the grid sum
//                          and the solve once on their own sums, so that the last block's serial tail runs warm code
//                          (the working set evicts the kernel's instructions from L2 every launch).
//        ROLE 1 after a searching launch: fixed-order sum of the tile sums + (exchange +) solve (icp_reduce_body).
//   icp_finalize_kernel    the solve alone, after an NCCL all-reduce of the sums (multi-GPU, --comm nccl).
//
// Target attributes are read from the context's private copies in INDEX order (icp_types.cuh): the match of a source point
// is remembered as a POSITION in the index, so the warm start, the certificate test and the rows read ix.pts[p] / tgt_nrm[p]
// with one aligned 16-byte load each.
#pragma once

__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// cp.async (LDGSTS): global -> shared without a register in between
__device__ __forceinline__ void cp_async_16(void *smem, const void *gmem) {  // .cg: straight from L2, no L1 allocation
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_8(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
// Certified regime: the per-point stream (the working copy and the (match, slack) pairs, read and rewritten once per
// launch) is marked evict-first in L2, so that it does not push out what is reused across launches -- the gathered target
// rows and the kernel's own code (config 2 on the H100: 1.5 % on the launch loop, DESIGN section 5)
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void cp_async_16(void *smem, const void *gmem, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_8(void *smem, const void *gmem, uint64_t pol) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 8, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(float4 *p, float4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(int2 *p, int2 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.s32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// certified regime: software pipeline depth.  Tile T's target rows are requested ICP_GD tiles ahead (that needs tile T's
// match position, i.e. its stage), the (point, match, slack) stages ICP_NS = 2 * ICP_GD tiles ahead.
#define ICP_GD 2
#define ICP_NS (2 * ICP_GD)
// Certified regime: the normal-equation sums of a tile on the FP64 tensor cores.  The 30 products a tile contributes per
// row are entries of the Gram matrix of the 32 x 8 matrix V = (J0..J5, r, one): eight DMMA.8x8x4 (A = V^T, B = V, four
// points per step; for a Gram matrix both fragments hold the SAME value per lane) accumulate it in a 2-register
// fragment per lane -- instead of 30 float64 accumulators (60 registers) per lane and a 30-column warp reduction at
// the end.  Products of two floats are exact in float64 and every accumulation step rounds once, exactly as DFMA does;
// only the (fixed) order of the additions differs.
// float -> double: the hardware conversion (F2F.F64.F32 on the XU pipe).  An exact integer-pipe form measured inside the
// +-2 % run-to-run spread (config 2 on the H100, profiles/h100_tuning_sweep.txt: 7216 it/s vs 7069).
__device__ __forceinline__ double f2d(float f) { return (double)f; }
__device__ __forceinline__ void dmma_8x8x4(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// pull the rows of target position p that a tile reads first into L1 (no register is tied up, nothing waits)
template <int KIND>
__device__ __forceinline__ void prefetch_target(const IcpArgs &a, size_t p) {
    prefetch_l1(a.ix.pts + p);
    if ((KIND == CPHB_EST_POINT_TO_PLANE || KIND == CPHB_EST_SYMMETRIC || KIND == CPHB_EST_COLORED_ICP) && a.tgt_nrm)
        prefetch_l1(a.tgt_nrm + p);
    if (KIND == CPHB_EST_COLORED_ICP && a.tgt_grad) prefetch_l1(a.tgt_grad + p);
    if (KIND == CPHB_EST_GENERALIZED_ICP && a.tgt_cov) prefetch_l1(a.tgt_cov + 3 * p);  // 48 B: one or two sectors
}

#define ICP_SEARCH_WARPS 4
// Two instances of the kernel, launched back to back every iteration (the regime is decided on the DEVICE, so each
// instance checks the state and the one whose regime is not current leaves at once):
//   ROLE 0  searching regime.  The traversal is bound by instruction issue at low occupancy, so it is compiled for MORE
//           resident warps (96 registers: 5 blocks = 20 warps / SM).
//   ROLE 1  certified regime (the normal-equation sums of its tiles go into one 8 x 8 DMMA Gram fragment per warp, see
//           dmma_8x8x4) -- and, when the launch before it searched, the fixed-order sum of its tile sums + solve (what
//           used to be a third kernel, icp_reduce_kernel).
// ROLE 1: 4 blocks = 16 warps / SM.  The Gram fragment is two registers per lane, so the registers would allow 24-32
// warps (80-64 registers), but more resident blocks buy nothing (config 2 on the H100, profiles/h100_tuning_sweep.txt:
// compiled for 6 blocks 7188 it/s vs 7069 for the same build at 4, a grid of 2 / 3 blocks per SM 7166 / 7395, all inside
// the +-2 % spread): the certified launch's SM throughput saturates near 16 warps and every extra block adds launch,
// pipeline-fill and grid-sum work.
#define ICP_MIN_BLOCKS 4
// ROLE 0: 96 registers = 20 warps / SM.  Config 2 on the H100 (profiles/h100_tuning_sweep.txt): a grid of 3 / 4 blocks per SM 6576 / 7047
// it/s; compiled for 4 / 6 blocks 7058 / 7214 it/s against 7069 for the same build at 5.
#define ICP_MIN_BLOCKS_SEARCH 5
// Programmatic dependent launch: the kernels of the loop are launched with stream serialisation relaxed, so the next
// kernel's blocks are already resident (waiting in griddepcontrol.wait) while the last block of the current one sums and
// solves: the launch latency of every kernel boundary is hidden (+3.5 % on config 2)
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// the columns of the 32-double sums layout (icp_types.cuh) that an estimator fills
__host__ __device__ constexpr bool pair_live(bool p2p, int p) { return p2p ? (p < 15 || p == 28 || p == 29) : p < 30; }

// the target-side values of index position p (tp = ix.pts[p] is already in registers)
template <int KIND>
__device__ __forceinline__ void load_tgt_ix(const IcpArgs &a, unsigned p, const float4 &tp, TgtVals &t) {
    t.vt[0] = tp.x; t.vt[1] = tp.y; t.vt[2] = tp.z;
    t.ok = true;
    if (KIND == CPHB_EST_POINT_TO_PLANE) t.ok = a.tgt_nrm != nullptr;
    if (KIND == CPHB_EST_SYMMETRIC) t.ok = a.tgt_nrm && a.src_nrm;
    if (KIND == CPHB_EST_COLORED_ICP) t.ok = a.tgt_nrm && a.has_tgt_col && a.src_col && a.tgt_grad;
    if (KIND == CPHB_EST_GENERALIZED_ICP) t.ok = a.tgt_cov && a.src_cov;
    if (!t.ok) return;
    if (KIND == CPHB_EST_POINT_TO_PLANE || KIND == CPHB_EST_SYMMETRIC || KIND == CPHB_EST_COLORED_ICP) {
        const float4 n4 = a.tgt_nrm[p];
        t.nt[0] = n4.x; t.nt[1] = n4.y; t.nt[2] = n4.z;
        t.it = n4.w;
    }
    if (KIND == CPHB_EST_COLORED_ICP) {
        const float4 g4 = a.tgt_grad[p];
        t.gt[0] = g4.x; t.gt[1] = g4.y; t.gt[2] = g4.z;
    }
    if (KIND == CPHB_EST_GENERALIZED_ICP) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float4 c4 = a.tgt_cov[3 * (size_t)p + r];
            t.ct[3 * r] = c4.x; t.ct[3 * r + 1] = c4.y; t.ct[3 * r + 2] = c4.z;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// per-tile building blocks shared by the two regimes (identical arithmetic: the regime never changes a result bit)
// ---------------------------------------------------------------------------------------------------------------------
struct LaunchCtx {
    float U[12];  // update to apply (identity rows when !apply)
    unsigned long long init;
    bool apply, materialize, write_corr, use_cert;
};

// PointCloud::Transform(update) on the working copy (pointcloud.cu:293-299) for lane i: lane_transform computes the
// updated point / normal / covariance, lane_writeback stores them (the reference transforms in place every iteration,
// registration.cu:160, so rounding accumulates exactly like this)
template <int KIND>
__device__ __forceinline__ void lane_transform(const IcpArgs &a, const LaunchCtx &c, unsigned i, float4 &s, float (&sn)[3],
                                               float (&Cs)[9]) {
    const float *U = c.U;
    if (c.apply) {
        const float x = s.x, y = s.y, z = s.z;
        s.x = __fadd_rn(dot3(U[0], U[1], U[2], x, y, z), U[3]);
        s.y = __fadd_rn(dot3(U[4], U[5], U[6], x, y, z), U[7]);
        s.z = __fadd_rn(dot3(U[8], U[9], U[10], x, y, z), U[11]);
    }
    if (KIND == CPHB_EST_SYMMETRIC && a.src_nrm) {
        const float4 n4 = a.src_nrm[i];
        if (c.apply) {
            sn[0] = dot3(U[0], U[1], U[2], n4.x, n4.y, n4.z);
            sn[1] = dot3(U[4], U[5], U[6], n4.x, n4.y, n4.z);
            sn[2] = dot3(U[8], U[9], U[10], n4.x, n4.y, n4.z);
        } else {
            sn[0] = n4.x; sn[1] = n4.y; sn[2] = n4.z;
        }
    }
    if (KIND == CPHB_EST_GENERALIZED_ICP && a.src_cov) {
        float C[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float4 c4 = a.src_cov[(size_t)r * a.n_pad + i];
            C[3 * r] = c4.x; C[3 * r + 1] = c4.y; C[3 * r + 2] = c4.z;
        }
        if (c.apply) {  // RotateCovariances (geometry_utils.cu:257-265): (R*C)*R^T
            float tmp[9];
            const float R[9] = {U[0], U[1], U[2], U[4], U[5], U[6], U[8], U[9], U[10]};
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int q = 0; q < 3; ++q)
                    tmp[3 * r + q] = dot3(R[3 * r], R[3 * r + 1], R[3 * r + 2], C[q], C[3 + q], C[6 + q]);
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int q = 0; q < 3; ++q)
                    Cs[3 * r + q] = dot3(tmp[3 * r], tmp[3 * r + 1], tmp[3 * r + 2], R[3 * q], R[3 * q + 1], R[3 * q + 2]);
        } else {
#pragma unroll
            for (int r = 0; r < 9; ++r) Cs[r] = C[r];
        }
    }
}

template <int KIND>
__device__ __forceinline__ void lane_writeback(const IcpArgs &a, const LaunchCtx &c, unsigned i, const float4 &s,
                                               const float (&sn)[3], const float (&Cs)[9]) {
    if (!c.apply || a.step_mode) return;
    a.src[i] = s;
    if (KIND == CPHB_EST_SYMMETRIC && a.src_nrm) a.src_nrm[i] = make_float4(sn[0], sn[1], sn[2], 0.f);
    if (KIND == CPHB_EST_GENERALIZED_ICP && a.src_cov)
#pragma unroll
        for (int r = 0; r < 3; ++r) a.src_cov[(size_t)r * a.n_pad + i] = make_float4(Cs[3 * r], Cs[3 * r + 1], Cs[3 * r + 2], 0.f);
}
// the same stores with an L2 cache policy (certified regime)
template <int KIND>
__device__ __forceinline__ void lane_writeback(const IcpArgs &a, const LaunchCtx &c, unsigned i, const float4 &s,
                                               const float (&sn)[3], const float (&Cs)[9], uint64_t pol) {
    if (!c.apply || a.step_mode) return;
    st_hint(&a.src[i], s, pol);
    if (KIND == CPHB_EST_SYMMETRIC && a.src_nrm) st_hint(&a.src_nrm[i], make_float4(sn[0], sn[1], sn[2], 0.f), pol);
    if (KIND == CPHB_EST_GENERALIZED_ICP && a.src_cov)
#pragma unroll
        for (int r = 0; r < 3; ++r)
            st_hint(&a.src_cov[(size_t)r * a.n_pad + i], make_float4(Cs[3 * r], Cs[3 * r + 1], Cs[3 * r + 2], 0.f), pol);
}

// Warm start + certificate (DESIGN.md 3.1.8).  prev[i].y is a lower bound (rounded down) on the distance from this point's
// position at the time it was last searched (minus the displacements since) to every target point other than its match.
// If, after this iteration's displacement, the old match is still strictly closer than that bound, no other point can
// have a smaller (d2, index) key: the search would return the same match, so the lane skips it.  All roundings go
// against the certificate (slack down, distances up, 1e-5 relative guard against the <= 3e-7 relative error of the
// float d2 arithmetic the keys are made of).
// in: s (transformed), (ox, oy, oz) the position the slack refers to, pv.  out: best key, cert, slack, margin; tp = ix.pts[pv.x]
// (PRE: tp already holds ix.pts[pv.x])
template <bool PRE = false>
__device__ __forceinline__ void lane_warm_start(const IcpArgs &a, const LaunchCtx &c, bool in_range, const float4 &s, float ox,
                                                float oy, float oz, const int2 pv, float4 &tp, unsigned long long &best,
                                                bool &cert, float &slk, float &margin) {
    best = c.init;
    cert = false;
    slk = 0.f;
    margin = 0.f;
    if (!(a.prev && in_range)) return;
    const int pp = pv.x;
    float disp = 0.f;
    if (c.use_cert) {
        disp = __fmul_ru(sqrt_approx(dist2(s.x, s.y, s.z, ox, oy, oz)), 1.00001f);
        slk = __fsub_rd(__int_as_float(pv.y), disp);  // NaN (never searched) stays NaN: no certificate
        margin = __fmul_ru(a.cert_gain, disp);
    }
    if (pp >= 0) {
        // warm start: last iteration's match is a candidate like any other (same key arithmetic), so the result is
        // unchanged; it only tightens the bounds early
        if (!PRE) tp = a.ix.pts[pp];
        const float d2p = dist2(s.x, s.y, s.z, tp.x, tp.y, tp.z);
        const unsigned long long kp = ((unsigned long long)__float_as_uint(d2p) << 32) | __float_as_uint(tp.w);
        if (kp < c.init) {
            best = kp;
            if (c.use_cert) cert = __fmul_ru(sqrt_approx(d2p), 1.00001f) < slk;
        }
        if (!cert && margin > 0.f) {
            // local scale: a leaf holds 32 neighbouring points, so sqrt(largest face area / 32) is about the point
            // spacing around the match (surface or volume sampling alike, within 2x)
            const Box bx = a.ix.boxes[0][(unsigned)pp >> 5];
            const float ex = bx.hi.x - bx.lo.x, ey = bx.hi.y - bx.lo.y, ez = bx.hi.z - bx.lo.z;
            const float area = fmaxf(ex * ey, fmaxf(ex * ez, ey * ez));
            if (margin > a.cert_cap * sqrtf(area * (1.f / 32.f))) margin = 0.f;
        }
    } else if (c.use_cert) {
        cert = slk > a.r_up;  // every target point is still outside the radius
        if (margin > a.cert_cap_r) margin = 0.f;
    }
    if (cert) margin = 0.f;
}

// what a lane remembers for the next iteration (its match position + certificate slack) and the correspondence output
__device__ __forceinline__ void lane_store_match(const IcpArgs &a, const LaunchCtx &c, unsigned i, unsigned orig, bool in_range,
                                                 bool found, int pos, unsigned j, bool cert, float slk, unsigned best_hi,
                                                 unsigned m1, unsigned m2, unsigned rb) {
    if (a.prev && !a.step_mode) {
        // searched lanes: everything not evaluated lies outside the final relaxed bound, everything evaluated except the
        // winner is at least sqrt(m2) away.  m1 is the winner's own d2 (its leaf is always scanned); if it is not -- no
        // match, or a tie -- m1 itself belongs to another point
        const unsigned other = (found && m1 == best_hi) ? m2 : m1;
        const float l2 = __uint_as_float(min(other, rb));
        const float fresh = __fmul_rd(sqrt_approx(l2), 0.99999f);
        a.prev[i] = make_int2(found ? pos : -1, __float_as_int(cert ? slk : fresh));
    }
    if (c.write_corr && in_range) a.corr_index[orig] = found ? (int32_t)j : -1;
}
// lane_store_match of a certified tile (every in-range lane keeps its match and its decremented slack), with an L2
// cache policy on the (match, slack) store
__device__ __forceinline__ void lane_store_certified(const IcpArgs &a, const LaunchCtx &c, unsigned i, unsigned orig, bool in_range,
                                                     bool found, int pos, unsigned j, float slk, uint64_t pol) {
    if (a.prev && !a.step_mode) st_hint(&a.prev[i], make_int2(found ? pos : -1, __float_as_int(slk)), pol);
    if (c.write_corr && in_range) a.corr_index[orig] = found ? (int32_t)j : -1;
}

// the same values from the certified regime's shared-memory copy of the next tile's target rows ([NG][32] float4,
// filled by cp.async one tile ahead: slot 0 the point, then normal(+intensity) [, gradient] or the 3 covariance rows)
template <int KIND>
__device__ __forceinline__ void load_tgt_smem(const IcpArgs &a, const float4 *gat, int lane, const float4 &tp, TgtVals &t) {
    t.vt[0] = tp.x; t.vt[1] = tp.y; t.vt[2] = tp.z;
    t.ok = true;
    if (KIND == CPHB_EST_POINT_TO_PLANE) t.ok = a.tgt_nrm != nullptr;
    if (KIND == CPHB_EST_SYMMETRIC) t.ok = a.tgt_nrm && a.src_nrm;
    if (KIND == CPHB_EST_COLORED_ICP) t.ok = a.tgt_nrm && a.has_tgt_col && a.src_col && a.tgt_grad;
    if (KIND == CPHB_EST_GENERALIZED_ICP) t.ok = a.tgt_cov && a.src_cov;
    if (!t.ok) return;
    if (KIND == CPHB_EST_POINT_TO_PLANE || KIND == CPHB_EST_SYMMETRIC || KIND == CPHB_EST_COLORED_ICP) {
        const float4 n4 = gat[32 + lane];
        t.nt[0] = n4.x; t.nt[1] = n4.y; t.nt[2] = n4.z;
        t.it = n4.w;
    }
    if (KIND == CPHB_EST_COLORED_ICP) {
        const float4 g4 = gat[64 + lane];
        t.gt[0] = g4.x; t.gt[1] = g4.y; t.gt[2] = g4.z;
    }
    if (KIND == CPHB_EST_GENERALIZED_ICP) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float4 c4 = gat[32 * (1 + r) + lane];
            t.ct[3 * r] = c4.x; t.ct[3 * r + 1] = c4.y; t.ct[3 * r + 2] = c4.z;
        }
    }
}
// issue the copies for target position p (this lane's slots)
template <int KIND>
__device__ __forceinline__ void gather_issue(const IcpArgs &a, float4 *gat, int lane, int p) {
    if (p < 0) return;
    cp_async_16(&gat[lane], &a.ix.pts[p]);
    if ((KIND == CPHB_EST_POINT_TO_PLANE || KIND == CPHB_EST_SYMMETRIC || KIND == CPHB_EST_COLORED_ICP) && a.tgt_nrm)
        cp_async_16(&gat[32 + lane], &a.tgt_nrm[p]);
    if (KIND == CPHB_EST_COLORED_ICP && a.tgt_grad) cp_async_16(&gat[64 + lane], &a.tgt_grad[p]);
    if (KIND == CPHB_EST_GENERALIZED_ICP && a.tgt_cov)
#pragma unroll
        for (int r = 0; r < 3; ++r) cp_async_16(&gat[32 * (1 + r) + lane], &a.tgt_cov[3 * (size_t)p + r]);
}

template <int KIND, int NROWS>
__device__ __forceinline__ void lane_rows_vals(const IcpArgs &a, bool found, const TgtVals &t, const float4 &s,
                                               const float (&sn)[3], const float (&Cs)[9], unsigned i, float (&J)[NROWS][6],
                                               float (&r)[NROWS]) {
#pragma unroll
    for (int q = 0; q < NROWS; ++q) {
        r[q] = 0.f;
#pragma unroll
        for (int c = 0; c < 6; ++c) J[q][c] = 0.f;
    }
    if (found) {
        const float4 cs4 = (KIND == CPHB_EST_COLORED_ICP && a.src_col) ? a.src_col[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        build_rows_vals<KIND, NROWS>(a.sg, a.sp, s.x, s.y, s.z, sn, cs4, Cs, t, J, r);
        drop_nonfinite_rows<NROWS>(J, r);
    }
}
template <int KIND, int NROWS>
__device__ __forceinline__ void lane_rows(const IcpArgs &a, bool found, unsigned pos, const float4 &tp, const float4 &s,
                                          const float (&sn)[3], const float (&Cs)[9], unsigned i, float (&J)[NROWS][6],
                                          float (&r)[NROWS]) {
#pragma unroll
    for (int q = 0; q < NROWS; ++q) {
        r[q] = 0.f;
#pragma unroll
        for (int c = 0; c < 6; ++c) J[q][c] = 0.f;
    }
    if (found) {
        TgtVals t;
        load_tgt_ix<KIND>(a, pos, tp, t);
        const float4 cs4 = (KIND == CPHB_EST_COLORED_ICP && a.src_col) ? a.src_col[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        build_rows_vals<KIND, NROWS>(a.sg, a.sp, s.x, s.y, s.z, sn, cs4, Cs, t, J, r);
        drop_nonfinite_rows<NROWS>(J, r);
    }
}

// ===========================================================================
// the fused per-iteration kernel
// ===========================================================================
// One tile of the searching regime: transform -> warm start / certificate -> exact search -> match bookkeeping -> rows ->
// the tile's 32 column sums (lane p: column p) in `acc`.  Returns true when the tile was skipped by its certificates.
template <int KIND, int TOP>
__device__ __forceinline__ bool search_tile(const IcpArgs &a, const LaunchCtx &c, WarpSearchC &w, double *rows, unsigned tile,
                                            float4 s, const int2 pv, double &acc) {
    constexpr int NROWS = (KIND == CPHB_EST_COLORED_ICP) ? 2 : (KIND == CPHB_EST_GENERALIZED_ICP) ? 3 : 1;
    constexpr bool P2P = (KIND == CPHB_EST_POINT_TO_POINT);
    const int lane = lane_id();
    const unsigned i = tile * 32 + lane;  // position in the working copy (< n_pad)
    const unsigned orig = __float_as_uint(s.w);
    const bool in_range = i < a.n_src;
    const float ox = s.x, oy = s.y, oz = s.z;  // position the certificate slack refers to
    float sn[3] = {0.f, 0.f, 0.f};
    float Cs[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    lane_transform<KIND>(a, c, i, s, sn, Cs);
    lane_writeback<KIND>(a, c, i, s, sn, Cs);

    // ---- SearchRadius(.., max_nn = 1) (registration.cu:47) ---------------------------
    float4 tp = make_float4(0.f, 0.f, 0.f, 0.f);
    bool cert;
    float slk;
    lane_warm_start(a, c, in_range, s, ox, oy, oz, pv, tp, w.best, cert, slk, w.margin);
    const unsigned long long before = w.best;
    w.qx = s.x; w.qy = s.y; w.qz = s.z;
    w.m1 = 0x7f800000u;
    w.m2 = 0x7f800000u;
    w.valid = in_range && !cert;
    w.track = __any_sync(CPHB_FULL, w.valid && w.margin > 0.f);
    w.refresh();
    warp_update_bound(w);
    w.warm = __all_sync(CPHB_FULL, !w.valid || w.best < c.init);  // every searching lane starts from a real candidate
    int pos = pv.x;
    const bool searched = __any_sync(CPHB_FULL, w.valid);
    if (searched) {
        warp_query_box(w);
        warp_nn_search<TOP>(a.ix, w);
        if (w.best != before) {
            pos = (int)a.ix.inv[(unsigned)(w.best & 0xffffffffull)];
            tp = a.ix.pts[pos];
        }
    }
    if (a.dbg) {
        const unsigned nc = __popc(__ballot_sync(CPHB_FULL, cert));
        if (lane == 0) {
            atomicAdd(&a.dbg[min(a.launch_idx, 63)], nc);
            if (!searched) atomicAdd(&a.dbg[64 + min(a.launch_idx, 63)], 1u);
        }
    }
    const bool found = in_range && (w.best != c.init);
    const unsigned j = (unsigned)(w.best & 0xffffffffull);
    const float d2 = __uint_as_float((unsigned)(w.best >> 32));
    lane_store_match(a, c, i, orig, in_range, found, pos, j, cert, slk, (unsigned)(w.best >> 32), w.m1, w.m2, w.rb);
    acc = 0.0;
    if (c.materialize) return !searched;  // fitness / rmse / T of this pose are already in the state

    // ---- rows: J (6), r; staged as doubles, one row of 9 per lane ---------------------
    float J[NROWS][6], r[NROWS];
    lane_rows<KIND, NROWS>(a, found, (unsigned)pos, tp, s, sn, Cs, i, J, r);
    // stage + accumulate: lane L adds column pair (ca, cb) over the 32 staged rows, in row order
    const unsigned char(*pair)[2] = P2P ? c_pair_p2p : c_pair_jtj;
    const int ca = pair[lane][0], cb = pair[lane][1];
    const unsigned live = P2P ? c_live_p2p : c_live_jtj;
#pragma unroll
    for (int q = 0; q < NROWS; ++q) {
        double *my = rows + lane * ROW_STRIDE;
#pragma unroll
        for (int k = 0; k < 6; ++k) my[k] = f2d(J[q][k]);
        my[6] = f2d(r[q]);
        my[7] = (q == 0 && found) ? f2d(d2) : 0.0;
        my[8] = (q == 0 && found) ? 1.0 : 0.0;
        __syncwarp();
#pragma unroll 8
        for (int t = 0; t < 32; ++t) acc = fma(rows[t * ROW_STRIDE + ca], rows[t * ROW_STRIDE + cb], acc);
        __syncwarp();
    }
    if (!((live >> lane) & 1u)) acc = 0.0;
    return !searched;
}

template <int KIND>
__device__ void icp_static_tail(const IcpArgs &a, IcpState *st, double (*s_rowbuf)[32], SolveSmem &s_solve, unsigned *s_flag,
                                const double row, bool materialize, unsigned n_skipped_block);

template <int KIND, int BLOCK>
__device__ void icp_reduce_body(const IcpArgs &a, double (*s_acc)[32], unsigned *s_last, SolveSmem &s_solve);

template <int KIND, int TOP, int ROLE>
__global__ void __launch_bounds__(ICP_SEARCH_WARPS * 32, ROLE == 0 ? ICP_MIN_BLOCKS_SEARCH : ICP_MIN_BLOCKS)
icp_iteration_kernel(const __grid_constant__ IcpArgs a) {
    __shared__ __align__(16) float4 s_tile[ICP_SEARCH_WARPS][2 * CPHB_LEAF];
    __shared__ uint64_t s_bar[ICP_SEARCH_WARPS][2];
    __shared__ double s_rows[ICP_SEARCH_WARPS][32 * ROW_STRIDE];
    __shared__ SolveSmem s_solve;
    __shared__ unsigned s_flag;
    __shared__ __align__(16) unsigned char s_pipe[ICP_SEARCH_WARPS][ICP_NS * 32 * 24];  // certified regime: cp.async stages
    constexpr int NG = (KIND == CPHB_EST_POINT_TO_POINT) ? 1 : (KIND == CPHB_EST_GENERALIZED_ICP) ? 4 : (KIND == CPHB_EST_COLORED_ICP) ? 3 : 2;
    __shared__ __align__(16) float4 s_gat[ICP_SEARCH_WARPS][ICP_GD * NG * 32];  // certified regime: target rows of the next tiles

    IcpState *st = a.st;
    const int warp = threadIdx.x >> 5, lane = lane_id();
    grid_dependency_wait();  // everything below reads state the previous launch wrote
    // the per-launch state: ONE warp instruction per block fetches the 15 words (a few thousand warps reading the same
    // line one word at a time serialise in its L2 slice: ~20 % of a certified launch's warp time before this)
    __shared__ unsigned s_hdr[16];
    if (threadIdx.x < 16) {
        const unsigned k = threadIdx.x;
        const unsigned *src = (k < 12) ? reinterpret_cast<const unsigned *>(&st->U[k])
                              : (k == 12) ? reinterpret_cast<const unsigned *>(&st->done)
                              : (k == 13) ? reinterpret_cast<const unsigned *>(&st->apply_u)
                              : (k == 14) ? reinterpret_cast<const unsigned *>(&st->static_sched)
                                          : reinterpret_cast<const unsigned *>(&st->flag_parity);
        s_hdr[k] = *(volatile const unsigned *)src;
    }
    __syncthreads();
    const int done = (int)s_hdr[12];
    const int apply_u = (int)s_hdr[13];
    const int static_word = (int)s_hdr[14];
    const unsigned flag_parity = s_hdr[15] & 1u;
    if (done == 2) return;
    LaunchCtx c;
    c.materialize = (done == 1);
    c.apply = a.step_mode ? true : (!c.materialize && apply_u != 0);
#pragma unroll
    for (int k = 0; k < 12; ++k) c.U[k] = c.apply ? __uint_as_float(s_hdr[k]) : ((k % 5 == 0) ? 1.f : 0.f);
    c.init = (a.r2 > 0.f) ? init_key(a.r2) : 0ull;
    c.write_corr = a.corr_index && (c.materialize || a.step_mode || a.launch_idx == a.max_iter);
    c.use_cert = a.prev && !a.step_mode && a.cert_gain > 0.f;

    const unsigned n_tiles = a.n_pad / 32;
    const unsigned total_warps = gridDim.x * ICP_SEARCH_WARPS;
    const unsigned gw = blockIdx.x * ICP_SEARCH_WARPS + warp;
    constexpr int NROWS = (KIND == CPHB_EST_COLORED_ICP) ? 2 : (KIND == CPHB_EST_GENERALIZED_ICP) ? 3 : 1;
    constexpr bool P2P = (KIND == CPHB_EST_POINT_TO_POINT);
    // once (nearly) every tile is skipped by its certificates the tiles cost the same: static round-robin schedule, no
    // atomics.  Sums never depend on which regime ran: the searching regime's are per tile, the certified regime's per
    // warp of a FIXED schedule (+ per tile for the few tiles that still need a search).
    const bool static_regime = a.static_sched && !a.step_mode && static_word != 0;

    if (lane == 0) {
        mbar_init(&s_bar[warp][0], 1);
        mbar_init(&s_bar[warp][1], 1);
        fence_mbar_init();
    }
    __syncwarp();
    WarpSearchC w;
    w.tile = s_tile[warp];
    w.bar = s_bar[warp];
    w.phase = 0;
    w.warm = false;
    w.tmax = a.tmax;

    if constexpr (ROLE == 1) {
        if (!static_regime) {
            // the ROLE 0 launch before this one searched: fixed-order sum of its tile sums + solve
            static_assert(sizeof(s_pipe) >= sizeof(double) * 8 * 32, "reduce scratch");
            icp_reduce_body<KIND, ICP_SEARCH_WARPS * 32>(a, (double(*)[32])s_pipe, &s_flag, s_solve);
            return;
        }
        if (a.dbg && threadIdx.x == 0 && blockIdx.x == 0) a.dbg[192 + min(a.launch_idx, 63)] = 1u;
        if (lane == 0) { dbg_time(a, 0, true); dbg_time(a, 11, false); }
        // ======================= certified regime ==================================================================
        // Every tile whose 32 lanes are certified (99.7 % of them on config 2): transform, certificate test, rows, products
        // into the warp's 8 x 8 Gram fragment on the FP64 tensor cores.  A tile with an uncertified lane goes through the
        // searching regime's per-tile routine instead and its sums are added to the warp's running row; the fragment
        // (three registers with the d2 sum) stays live across the search -- which tiles take that path depends on the data
        // only, so the sums stay reproducible.
        // Software pipeline, two tiles deep, without tying up registers: the point and the (match, slack) pair of the tile
        // AFTER NEXT travel global -> shared memory by cp.async while the current tile is processed; at the top of a tile
        // the next tile's match positions are read back from shared memory and the target rows they point to are pulled
        // into L1, so those have a whole tile to arrive.
        // Tiles that needed a search in the LAST certified launch (a stable set: the same near-equidistant points every
        // iteration) are flagged in a bitmap.  The last `helper_blocks` blocks of the grid run exactly those tiles, bitmap
        // word by bitmap word (a fixed assignment), from the first microsecond of the launch; the other warps skip them,
        // so no warp of the static schedule is held up by a search -- unless a NEW tile needs one, which is handled in line
        // and flagged for the next launch.  Every tile is processed exactly once either way.
        const unsigned *flag_cur = a.flag_bits + flag_parity * a.flag_words;
        unsigned *flag_next = a.flag_bits + (flag_parity ^ 1u) * a.flag_words;
        const unsigned helper_blocks = (a.helper_blocks < gridDim.x) ? a.helper_blocks : 0u;
        const unsigned main_blocks = gridDim.x - helper_blocks;
        const unsigned main_warps = main_blocks * ICP_SEARCH_WARPS;
        if (blockIdx.x >= main_blocks) {
            // ---- helper role ----
            double hrow = 0.0;
            unsigned n_skip = 0;
            const unsigned hw = (blockIdx.x - main_blocks) * ICP_SEARCH_WARPS + warp, H = helper_blocks * ICP_SEARCH_WARPS;
            const unsigned n_words = (n_tiles + 31) / 32;
            for (unsigned wd = hw; wd < n_words; wd += H) {
                unsigned bits = __ldg(&flag_cur[wd]);
                while (bits) {
                    const unsigned t = wd * 32 + (unsigned)(__ffs(bits) - 1);
                    bits &= bits - 1;
                    if (t >= n_tiles) break;
                    const float4 s = a.src[t * 32 + lane];
                    const int2 pv = a.prev[t * 32 + lane];
                    double acc;
                    const bool skipped = search_tile<KIND, TOP>(a, c, w, s_rows[warp], t, s, pv, acc);
                    hrow += acc;
                    if (skipped) ++n_skip;
                    else if (lane == 0) atomicOr(&flag_next[wd], 1u << (t & 31));  // still needs its search next time
                }
            }
            if (lane == 0) { dbg_time(a, 1, false); dbg_time(a, 10, false); }
            icp_static_tail<KIND>(a, st, (double(*)[32])s_pipe, s_solve, &s_flag, hrow, c.materialize, n_skip);
            return;
        }
        // ---- main role ----
        double gc0 = 0.0, gc1 = 0.0;  // this lane's two elements of the warp's 8 x 8 Gram fragment: G[lane/4][2 (lane%4) + {0,1}]
        double d2acc = 0.0;           // this lane's sum of d2 (not an entry of the Gram matrix of V)
        float *stage = reinterpret_cast<float *>(s_rows[warp]);  // [32 points][8] floats (the searching code's row buffer, idle here)
        double wrow = 0.0;  // lane p: column p of what this warp has folded so far
        unsigned n_skipped = 0;
        bool searched_inline = false;
        unsigned tile = gw;
        float4 *pipe_s = reinterpret_cast<float4 *>(s_pipe[warp]);                // [NS][32] float4, then [NS][32] int2
        int2 *pipe_pv = reinterpret_cast<int2 *>(s_pipe[warp] + ICP_NS * 32 * 16);
        const uint64_t pol_stream = l2_evict_first();
        auto stage_load = [&](unsigned t, int slot) {  // tile t -> stage slot (this lane's entries only)
            if (t < n_tiles) {
                cp_async_16(&pipe_s[slot * 32 + lane], &a.src[t * 32 + lane], pol_stream);
                cp_async_8(&pipe_pv[slot * 32 + lane], &a.prev[t * 32 + lane], pol_stream);
            }
        };
        // Pipeline (all copies are cp.async, one commit group per tile iteration, so the group arithmetic is uniform):
        //   iteration i commits G_i = { stage(i + NS), target rows of tile i + GD }   (the latter needs stage(i + GD))
        //   at its top it needs stage(i), the rows of tile i (G_{i-GD}) and stage(i + GD) (G_{i+GD-NS} = G_{i-GD}):
        //   everything but the GD - 1 most recent groups -> cp.async.wait_group GD - 1.
        // A lane only ever reads and refills its own entries, so a buffer may be refilled right after the lane read it.
#pragma unroll
        for (int j = 0; j < ICP_NS; ++j) {
            stage_load(tile + (unsigned)j * main_warps, j);
            cp_async_commit();
        }
        cp_async_wait<ICP_NS - ICP_GD>();  // stages 0 .. GD-1 have landed
#pragma unroll
        for (int j = 0; j < ICP_GD; ++j) {
            if (tile + (unsigned)j * main_warps < n_tiles) gather_issue<KIND>(a, s_gat[warp] + j * NG * 32, lane, pipe_pv[j * 32 + lane].x);
            cp_async_commit();
        }
        unsigned fw = (tile < n_tiles) ? __ldg(&flag_cur[tile >> 5]) : 0u;  // flag word of the next tile, one tile ahead
        int slot = 0, gslot = 0;
        // The hot loop holds no search code: a tile that needs a search breaks out of it, is handled below (cold) and the
        // loop is re-entered -- the instructions a certified tile executes stay one compact run.
        float4 cold_s = make_float4(0.f, 0.f, 0.f, 0.f);
        int2 cold_pv = make_int2(-1, 0);
        for (;;) {
        bool cold = false;
        for (; tile < n_tiles; tile += main_warps) {
            cp_async_wait<ICP_GD - 1>();
            const unsigned t1 = tile + main_warps, tg = tile + ICP_GD * main_warps, tn = tile + ICP_NS * main_warps;
            float4 *gat = s_gat[warp] + gslot * NG * 32;
            const float4 s0 = pipe_s[slot * 32 + lane];  // (untransformed point)
            float4 s = s0;
            const int2 pv = pipe_pv[slot * 32 + lane];
            const bool flagged = (fw >> (tile & 31)) & 1u;  // a helper warp runs this tile
            if (t1 < n_tiles) fw = __ldg(&flag_cur[t1 >> 5]);
            float4 tp = gat[lane];
            TgtVals tv;
            load_tgt_smem<KIND>(a, gat, lane, tp, tv);
            // (reads above first, same lane: now the entries may be refilled) this iteration's group
            stage_load(tn, slot);
            if (tg < n_tiles) gather_issue<KIND>(a, gat, lane, pipe_pv[((slot + ICP_GD) % ICP_NS) * 32 + lane].x);
            cp_async_commit();
            slot = (slot + 1) % ICP_NS;
            gslot = (gslot + 1) % ICP_GD;
            const unsigned i = tile * 32 + lane;
            const unsigned orig = __float_as_uint(s.w);
            const bool in_range = i < a.n_src;
            const float ox = s.x, oy = s.y, oz = s.z;
            float sn[3] = {0.f, 0.f, 0.f};
            float Cs[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            lane_transform<KIND>(a, c, i, s, sn, Cs);
            unsigned long long best;
            bool cert;
            float slk, margin;
            lane_warm_start<true>(a, c, in_range, s, ox, oy, oz, pv, tp, best, cert, slk, margin);
            if (flagged) continue;
            const bool need_search = __any_sync(CPHB_FULL, in_range && !cert);
            if (need_search) {  // not predicted by the flags (the first certified launch, or a point that drifted)
                cold = true;
                cold_s = s0;
                cold_pv = pv;
                break;
            }
            ++n_skipped;
            lane_writeback<KIND>(a, c, i, s, sn, Cs, pol_stream);
            if (a.dbg) {
                const unsigned nc = __popc(__ballot_sync(CPHB_FULL, cert));
                if (lane == 0) {
                    atomicAdd(&a.dbg[min(a.launch_idx, 63)], nc);
                    atomicAdd(&a.dbg[64 + min(a.launch_idx, 63)], 1u);
                }
            }
            const bool found = in_range && (best != c.init);
            const unsigned j = (unsigned)(best & 0xffffffffull);
            const float d2 = __uint_as_float((unsigned)(best >> 32));
            // (every in-range lane is certified: it keeps its decremented slack, the match is unchanged)
            lane_store_certified(a, c, i, orig, in_range, found, pv.x, j, slk, pol_stream);
            if (c.materialize) continue;  // fitness / rmse / T of this pose are already in the state
            float J[NROWS][6], r[NROWS];
            lane_rows_vals<KIND, NROWS>(a, found, tv, s, sn, Cs, i, J, r);
            // the warp's rows into its Gram fragment (exact products, one rounding per addition); the fragment is read
            // out once, after the last tile
#pragma unroll
            for (int q = 0; q < NROWS; ++q) {
                __syncwarp();  // every lane has read the previous row's stage
                *reinterpret_cast<float4 *>(stage + lane * 8) = make_float4(J[q][0], J[q][1], J[q][2], J[q][3]);
                *reinterpret_cast<float4 *>(stage + lane * 8 + 4) = make_float4(J[q][4], J[q][5], r[q], (q == 0 && found) ? 1.f : 0.f);
                __syncwarp();
#pragma unroll
                for (int m4 = 0; m4 < 8; ++m4) {  // points 4 m4 .. 4 m4 + 3; lane: V[point 4 m4 + lane % 4][column lane / 4] (conflict-free)
                    const double x = f2d(stage[(4 * m4 + (lane & 3)) * 8 + (lane >> 2)]);
                    dmma_8x8x4(gc0, gc1, x, x);
                }
            }
            if (found) d2acc += f2d(d2);
        }
        if (!cold) break;
        // ---- cold: tile `tile` needs its search, its sums go into the warp's running row; then the hot loop resumes
        // with the next tile.
        if (lane == 0) atomicOr(&flag_next[tile >> 5], 1u << (tile & 31));
        {   // (the Gram fragment is three registers: it simply stays live across the search)
            double acc;
            __syncwarp();
            search_tile<KIND, TOP>(a, c, w, s_rows[warp], tile, cold_s, cold_pv, acc);
            searched_inline = true;
            wrow += acc;
            __syncwarp();
        }
        if (a.dbg && lane == 0) atomicAdd(&a.dbg[128 + min(a.launch_idx, 63)], 1u);
        tile += main_warps;
        }
        cp_async_wait_0();
        if (lane == 0) { dbg_time(a, 1, false); dbg_time(a, searched_inline ? 9 : 8, false); }
        // lane p keeps column p
        double row = wrow;
        if (!c.materialize) {
            // the fragment IS the warp's sum: lay the 8 x 8 matrix out in shared memory and let lane p pick the entry
            // of its column pair (JTJ kinds: columns 0..6 = J0..J5, r; 7 = one.  P2P: 0..5 = s, t; 7 = one)
            double *gm = s_rows[warp];  // [8][8]
            __syncwarp();
            gm[(lane >> 2) * 8 + 2 * (lane & 3)] = gc0;
            gm[(lane >> 2) * 8 + 2 * (lane & 3) + 1] = gc1;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d2acc += __shfl_xor_sync(CPHB_FULL, d2acc, o);
            __syncwarp();
            const unsigned char(*pair)[2] = P2P ? c_pair_p2p : c_pair_jtj;
            int ga = pair[lane][0], gb = pair[lane][1];
            // the tables name 9 values (.., d2 = 7, one = 8); here 'one' is column 7 and sum d2 is carried separately
            double g = 0.0;
            if (ga == 7 && gb == 8) g = d2acc;  // (d2, one)
            else {
                ga = (ga == 8) ? 7 : ga;
                gb = (gb == 8) ? 7 : gb;
                g = gm[ga * 8 + gb];
            }
            if (pair_live(P2P, lane)) row += g;
        }
        icp_static_tail<KIND>(a, st, (double(*)[32])s_pipe, s_solve, &s_flag, row, c.materialize, n_skipped);
        return;
    } else {
    if (static_regime) return;  // the ROLE 1 launch right behind this one runs the certified regime
    // ======================= searching regime ======================================================================
    // Each warp starts on a static tile (its global warp id) and then claims RANGES of consecutive tiles from an atomic
    // counter: one tile at a time while tiles need a search (cost varies 10x between tiles, fine-grained claims keep
    // every warp busy), up to claim_max at a time once its tiles are skipped by their certificates.
    // Software pipeline: the claim after next and the loads of the NEXT tile's point and certificate are issued at the top
    // of the current tile, and the target rows the next tile reads first are pulled into L1 at the end of the current one.
    unsigned tile = gw;
    unsigned range_end = tile + 1;   // current range [tile, range_end)
    unsigned pend = 0, pend_sz = 1;  // claim in flight (result in lane 0) and its size
    unsigned csize = 1;              // size of the next claim
    unsigned n_skipped = 0;
    if (lane == 0) pend = atomicAdd(&st->tile_counter, 1u);
    float4 s_pf = make_float4(0.f, 0.f, 0.f, 0.f);
    int2 pv_pf = make_int2(-1, 0);
    if (tile < n_tiles) {
        s_pf = a.src[tile * 32 + lane];
        if (a.prev) pv_pf = a.prev[tile * 32 + lane];
    }
    unsigned tn = 0;
    for (; tile < n_tiles; tile = tn) {
        const float4 s = s_pf;
        const int2 pv = pv_pf;
        tn = tile + 1;
        if (tn >= range_end) {  // last tile of the range: the next one comes from the claim in flight
            tn = __shfl_sync(CPHB_FULL, pend, 0) + total_warps;
            range_end = min(tn + pend_sz, n_tiles);
            pend_sz = csize;
            if (lane == 0) pend = atomicAdd(&st->tile_counter, csize);
        }
        if (tn < n_tiles) {
            s_pf = a.src[tn * 32 + lane];
            if (a.prev) pv_pf = a.prev[tn * 32 + lane];
        }
        double acc;
        const bool skipped = search_tile<KIND, TOP>(a, c, w, s_rows[warp], tile, s, pv, acc);
        if (!c.materialize) a.tile_sums[(size_t)tile * 32 + lane] = acc;
        if (skipped) {
            csize = min(csize * 2, a.claim_max);
            ++n_skipped;
        } else {
            csize = 1;
        }
        if (tn < n_tiles && pv_pf.x >= 0) prefetch_target<KIND>(a, (size_t)pv_pf.x);
    }
    if (a.static_sched && lane == 0 && n_skipped) atomicAdd(&st->cert_tiles, n_skipped);
    }
}

// Warp g of the last block adds the block rows g, g+W, ... (W warps per block) in that order, with 32 loads in flight.
// Not inlined: the blocks that are not last run it once on a single row (icp_static_tail), so that its code is warm.
__device__ __noinline__ double grid_row_sum(const double *partials, unsigned nb) {
    const int warp = threadIdx.x >> 5, lane = lane_id();
    double t = 0.0;
    for (unsigned b = warp; b < nb; b += 32 * ICP_SEARCH_WARPS) {
        double v[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) {
            const unsigned bb = b + u * ICP_SEARCH_WARPS;
            v[u] = (bb < nb) ? __ldcg(&partials[(size_t)bb * 32 + lane]) : 0.0;  // x + 0.0 is exact
        }
#pragma unroll
        for (int u = 0; u < 32; ++u) t += v[u];
    }
    return t;
}

// Tail of a certified-regime launch: block rows -> last-arriving block adds them in block order -> (multi-GPU exchange) ->
// solve.  `row`: lane p of every warp holds column p of the warp's
// sums.
template <int KIND>
__device__ void icp_static_tail(const IcpArgs &a, IcpState *st, double (*s_rowbuf)[32], SolveSmem &s_solve, unsigned *s_flag,
                                const double row, bool materialize, unsigned n_skipped) {
    const int warp = threadIdx.x >> 5, lane = lane_id();
    __syncthreads();  // (s_rowbuf aliases the cp.async stages of the block's warps)
    s_rowbuf[warp][lane] = row;
    if (lane == 0 && n_skipped) {
        atomicAdd(&st->cert_tiles, n_skipped);
        __threadfence();  // performed before this block's ticket below
    }
    __syncthreads();
    if (warp == 0) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < ICP_SEARCH_WARPS; ++k) t += s_rowbuf[k][lane];  // fixed order: warps of the block
        a.partials[(size_t)blockIdx.x * 32 + lane] = t;
        s_solve.S[lane] = t;  // (input of the warm-up below)
        __threadfence();
        __syncwarp();
        if (lane == 0) {
            const unsigned tk = atomicAdd(&st->block_ticket, 1u);
            *s_flag = (tk == gridDim.x - 1) ? 1u : 0u;
        }
    }
    __syncthreads();
    if (!*s_flag) {
        // not the last block: run the grid sum (on this block's own row) and the solve once and drop the results, so that
        // the last block finds their instructions warm (warm_solve, icp_solve.cuh)
        if (!materialize) {
            if (warp == 0) s_solve.S[lane] += 0.0 * grid_row_sum(a.partials + (size_t)blockIdx.x * 32, 1);
            __syncthreads();
            warm_solve<KIND>(a, s_solve);
        }
        return;
    }
    __threadfence();
    if (threadIdx.x == 0) {
        dbg_time(a, 2, false);
        // the state the epilogue reads after the grid sum (previous fitness / rmse, pose): have it in L1 by then
        prefetch_l1(&st->T[0]);
        prefetch_l1(&st->fitness);
    }
    const unsigned n_tiles = a.n_pad / 32;
    {   // every block has finished reading this launch's flag bitmap: clear it (it collects the flags of the launch after
        // next) and make the one written during this launch current
        const unsigned par = *(volatile unsigned *)&st->flag_parity & 1u;
        unsigned *cur = a.flag_bits + par * a.flag_words;
        for (unsigned k = threadIdx.x; k < a.flag_words; k += blockDim.x) cur[k] = 0u;
        __syncthreads();
        if (threadIdx.x == 0) st->flag_parity = par ^ 1u;
    }
    if (materialize) {  // this launch only wrote the correspondences of an already evaluated pose
        if (threadIdx.x == 0) {
            st->block_ticket = 0; st->tile_counter = 0; st->cert_tiles = 0; st->static_sched = 0; st->done = 2;
            st->tail_done = a.launch_idx + 1;
        }
        return;
    }
    // all warps of the block share the grid sum (the accumulators of the tile loop are dead here, so the registers are free)
    const double t = grid_row_sum(a.partials, gridDim.x);
    __syncthreads();
    s_rowbuf[warp][lane] = t;
    __syncthreads();
    if (warp == 0) {
        double tt = 0.0;
#pragma unroll
        for (int k = 0; k < ICP_SEARCH_WARPS; ++k) tt += s_rowbuf[k][lane];
        if (a.use_p2p) tt = p2p_exchange_sum(a.p2p, tt, &st->comm_timeout);  // the collective, fused: NVLink stores + flags
        if (a.defer_finalize) st->local[lane] = tt;
        else st->total[lane] = tt;
        s_solve.S[lane] = tt;
        __syncwarp();
        if (lane == 0) dbg_time(a, 3, false);
        if (lane == 0) {
            st->block_ticket = 0;
            st->tile_counter = 0;
            st->static_sched = ((unsigned long long)st->cert_tiles * 10ull >= (unsigned long long)n_tiles * 9ull) ? 1 : 0;
            st->cert_tiles = 0;
            st->tail_done = a.launch_idx + 1;
        }
    }
    __syncthreads();  // the sums are staged: warp 1 takes the determinant while warp 0 solves (icp_finalize<KIND, true>)
    if (!a.defer_finalize) icp_finalize<KIND, true>(a, st, s_solve);
    if (warp == 0) {
        __threadfence();
        if (lane == 0) dbg_time(a, 4, false);
    }
}

// Fixed-order grid sum of the tile sums of a searching-regime launch, then (last block) the host-side part of the loop.
// Runs on the first a.reduce_grid blocks of the ROLE 1 launch; block b owns a contiguous chunk of tiles.  The summation
// order is defined for 8 row groups per block and does not depend on BLOCK (a block of fewer than 8 warps takes several
// groups per warp): group g adds the tiles t0 + g, t0 + g + 8, ... in increasing order, the 8 group sums are added in
// group order, the block sums in the same two-level order over blocks.
template <int KIND, int BLOCK>
__device__ void icp_reduce_body(const IcpArgs &a, double (*s_acc)[32], unsigned *s_last, SolveSmem &s_solve) {
    constexpr int GROUPS = 8, WARPS = BLOCK / 32;
    IcpState *st = a.st;
    if (blockIdx.x >= a.reduce_grid) return;
    if (*(volatile int *)&st->tail_done == a.launch_idx + 1) return;  // (the search launch reduced and solved by itself)
    const int done = *(volatile int *)&st->done;
    if (done == 2) return;
    if (done == 1) {  // the search launch before this one only materialised correspondences
        if (blockIdx.x == 0 && threadIdx.x == 0) { st->tile_counter = 0; st->cert_tiles = 0; st->static_sched = 0; st->done = 2; }
        return;
    }
    const unsigned n_tiles = a.n_pad / 32;
    const unsigned chunk = (n_tiles + a.reduce_grid - 1) / a.reduce_grid;
    const unsigned t0 = blockIdx.x * chunk, t1 = min(n_tiles, t0 + chunk);
    const int c = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int g = warp; g < GROUPS; g += WARPS) {
        // 8 loads in flight per thread, added in tile order (x + 0.0 is exact, so the padding loads of the
        // last batch do not change the sum): the naive loop serialises one L2 round trip per tile
        double t = 0.0;
        for (unsigned k = t0 + g; k < t1; k += 8 * GROUPS) {
            double v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const unsigned kk = k + u * GROUPS;
                v[u] = (kk < t1) ? __ldcg(&a.tile_sums[(size_t)kk * 32 + c]) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) t += v[u];
        }
        s_acc[g][c] = t;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < GROUPS; ++k) t += s_acc[k][threadIdx.x];
        a.partials[(size_t)blockIdx.x * 32 + threadIdx.x] = t;
        s_solve.S[threadIdx.x] = t;  // (input of the warm-up below)
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = atomicAdd(&st->ticket, 1u);
        *s_last = (t == a.reduce_grid - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (!*s_last) {
        warm_solve<KIND>(a, s_solve);  // (see icp_static_tail)
        return;
    }
    __threadfence();
    if (threadIdx.x == 0) {
        prefetch_l1(&st->T[0]);
        prefetch_l1(&st->fitness);
    }
    for (int g = warp; g < GROUPS; g += WARPS) {  // the grid sum (fixed order: row groups of 8, then the 8 group sums)
        double t = 0.0;
        for (unsigned b = g; b < a.reduce_grid; b += 8 * GROUPS) {
            double v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const unsigned bb = b + u * GROUPS;
                v[u] = (bb < a.reduce_grid) ? __ldcg(&a.partials[(size_t)bb * 32 + c]) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) t += v[u];
        }
        s_acc[g][c] = t;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < GROUPS; ++k) t += s_acc[k][threadIdx.x];
        if (a.use_p2p) t = p2p_exchange_sum(a.p2p, t, &st->comm_timeout);  // the collective, fused: NVLink stores + flags
        if (a.defer_finalize) st->local[threadIdx.x] = t;
        else st->total[threadIdx.x] = t;
        s_solve.S[threadIdx.x] = t;
        __syncwarp();
        if (threadIdx.x == 0) {
            st->ticket = 0;
            st->tile_counter = 0;
            st->static_sched = ((unsigned long long)st->cert_tiles * 10ull >= (unsigned long long)n_tiles * 9ull) ? 1 : 0;
            st->cert_tiles = 0;
        }
    }
    static_assert(WARPS >= 2, "icp_finalize<KIND, true> needs a second warp");
    __syncthreads();
    if (!a.defer_finalize) icp_finalize<KIND, true>(a, st, s_solve);
    if (threadIdx.x < 32) __threadfence();
}

// multi-GPU: runs after the all-reduce of st->local into st->total
template <int KIND>
__global__ void icp_finalize_kernel(const __grid_constant__ IcpArgs a) {
    __shared__ SolveSmem s_solve;
    if (threadIdx.x < 32 && a.st->done != 2) {
        s_solve.S[threadIdx.x] = a.st->total[threadIdx.x];
        __syncwarp();
        icp_finalize<KIND>(a, a.st, s_solve);
    }
}
