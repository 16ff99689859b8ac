// icp_types.cuh -- per-registration device state, kernel arguments and the column-pair tables of the staged reducer
// Part of the icp.cu translation unit (included there, in this order: icp_types, icp_solve, icp_rows); split out
// for readability only -- the arithmetic contract and the reference citations are stated in icp.cu.
#pragma once

#define ICP_BLOCK 256
#define ICP_WARPS (ICP_BLOCK / 32)
#define ROW_STRIDE 9 /* doubles per staged row: J0..J5, r, d2, one */

struct IcpState {
    double total[32];
    double local[32];
    float T[16];
    float U[16];
    float fitness, rmse;
    int done;        // 0 running, 1 converged (materialise correspondences next), 2 finished
    int iterations;  // updates applied
    int converged;
    int apply_u;
    unsigned ticket;
    unsigned tile_counter;
    unsigned cert_tiles;  // tiles skipped by their certificates in the launch just finished
    int static_sched;     // next search launch may use the static tile schedule (see icp_iteration_kernel)
    int tail_done;        // launch_idx + 1 of the last search launch that reduced and solved in its own tail
    unsigned block_ticket;  // arrival counter of that tail
    unsigned flag_parity;   // which of the two tile bitmaps holds the last certified launch's "needed a search" flags
    long long n_corr;
    unsigned comm_timeout;  // the peer-memory exchange gave up waiting for a rank (cphb_internal.cuh)
    unsigned pad_local;  // host-side staging only (count of locally written correspondence pairs)
    unsigned pad_;
};

struct IcpArgs {
    IndexView ix;
    float4 *src;            // working copy, Hilbert order, w = original index
    float4 *src_nrm;        // working normals (Symmetric) or null
    float4 *src_cov;        // working covariances: 3 float4 rows per point, [3][n_pad] (GICP) or null
    const float4 *src_col;  // colors in Hilbert order (Colored) or null
    // target attributes, private copies in INDEX order (position p of ix.pts <-> row p here), built once per context:
    //   tgt_nrm[p]  = (nx, ny, nz, intensity(colour))   P2Plane / Symmetric / Colored, else null
    //   tgt_grad[p] = (gx, gy, gz, 0)                    Colored, else null
    //   tgt_cov[3 p + r] = row r of the covariance       GICP (row-major whatever the caller's layout), else null
    // the matched point itself is ix.pts[p] (xyz, w = original index)
    const float4 *tgt_nrm, *tgt_grad, *tgt_cov;
    int has_tgt_col;
    IcpState *st;
    double *partials;     // [max(reduce grid, ROLE 1 grid)][32]
    double *tile_sums;    // [n_pad/32][32]
    unsigned *flag_bits;  // [2][flag_words] certified regime: bit t = tile t needed a search in the last certified launch
    unsigned flag_words;  // words per bitmap
    unsigned helper_blocks;  // certified regime: the last blocks of the grid run the flagged tiles (0 = none)
    unsigned reduce_grid;    // blocks of the ROLE 1 launch that sum the tile sums of a searching launch
    int2 *prev;           // [n_pad] per source position: .x INDEX POSITION of last iteration's match (-1 none), .y float bits
                          // of the certificate slack (lower bound on the distance to every OTHER target point); or null
    float cert_gain;      // margin = cert_gain * displacement (0 disables the certificates)
    float cert_cap;       // matched lanes: margins above cert_cap * (point spacing in the match's leaf) are not worth
                          // the wider search (-> plain search)
    float cert_cap_r;     // unmatched lanes: same, as a distance (a fraction of max_correspondence_distance)
    float r_up;           // max_correspondence_distance rounded up (certified 'still unmatched' test)
    unsigned *dbg;        // [2][64] certified lanes / skipped tiles per launch (CPHB_DEBUG_CERT) or null
    unsigned claim_max;   // largest range of tiles one claim may take (certified regime)
    int static_sched;     // allow the atomics-free static schedule once >= 90 % of the tiles are skipped
    int32_t *corr_index;  // [n_src] matched target index per ORIGINAL source index, or null
    unsigned long long n_total;
    unsigned n_src, n_pad;
    float r2;
    float rel_fitness, rel_rmse, det_thresh, sg, sp;
    int launch_idx, max_iter;
    int defer_finalize;  // multi-GPU over NCCL: stop after writing st->local
    int use_p2p;         // multi-GPU over the fused peer-memory exchange
    P2pView p2p;
    int step_mode;       // debug hook: one search + sums, no solve
    int tmax;            // transposed-scan threshold (CPHB_TRANSPOSE_MAX)
};

// sums layout (32 doubles): JTJ kinds: 0..20 JTJ upper | 21..26 JTr | 27 r^2 | 28 sum d2 | 29 count
//                           P2P      : 0..2 sum s | 3..5 sum t | 6..14 sum s t^T | 28 sum d2 | 29 count
__constant__ unsigned char c_pair_jtj[32][2] = {
    {0, 0}, {0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {1, 1}, {1, 2}, {1, 3}, {1, 4}, {1, 5},
    {2, 2}, {2, 3}, {2, 4}, {2, 5}, {3, 3}, {3, 4}, {3, 5}, {4, 4}, {4, 5}, {5, 5},
    {0, 6}, {1, 6}, {2, 6}, {3, 6}, {4, 6}, {5, 6}, {6, 6}, {7, 8}, {8, 8}, {8, 8}, {8, 8}};
__constant__ unsigned char c_pair_p2p[32][2] = {
    {0, 8}, {1, 8}, {2, 8}, {3, 8}, {4, 8}, {5, 8}, {0, 3}, {0, 4}, {0, 5}, {1, 3}, {1, 4},
    {1, 5}, {2, 3}, {2, 4}, {2, 5}, {8, 8}, {8, 8}, {8, 8}, {8, 8}, {8, 8}, {8, 8},
    {8, 8}, {8, 8}, {8, 8}, {8, 8}, {8, 8}, {8, 8}, {8, 8}, {7, 8}, {8, 8}, {8, 8}, {8, 8}};
__constant__ unsigned c_live_jtj = 0x3fffffffu;                          // lanes 0..29
__constant__ unsigned c_live_p2p = 0x00007fffu | (1u << 28) | (1u << 29);  // 0..14, 28, 29

#ifdef __CUDACC__
// CPHB_DEBUG_CERT timeline (globaltimer ns) of launch 20: dbg[256 + 2k .. ] as u64: 0 first block start (min), 1 last warp out
// of the tile loop (max), 2 last-arriving block enters the grid sum, 3 grid sum done, 4 solve done, 5.. inside the solve
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void dbg_time(const IcpArgs &a, int slot, bool take_min) {
    if (!a.dbg || a.launch_idx != 20) return;
    unsigned long long *p = reinterpret_cast<unsigned long long *>(a.dbg + 256) + slot;
    if (take_min) atomicMin(p, gtime());
    else atomicMax(p, gtime());
}
#endif
