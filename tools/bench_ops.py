#!/usr/bin/env python3
"""Config 3 of BASELINE.json: VoxelDownSample(voxel=0.02) + SearchRadius(k=1, r=0.05) on 10M points, 1 GPU.
Prints one JSON object (not the headline bench line; see bench.py).  Also runs the size-independent
property checks used as full-size parity evidence (sortedness, conservation, containment)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--voxel", type=float, default=0.02)
    ap.add_argument("--radius", type=float, default=0.05)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--attrs", default="p", help="p | pn | pnc")
    ap.add_argument("--normals", type=int, default=0, help="also time EstimateNormals(KNN k) of the 10 M cloud (fused kernel, and the two-pass form)")
    ap.add_argument("--filters", action="store_true",
                    help="also time the SURVEY 8f rows: RemoveRadiusOutliers / RemoveStatisticalOutliers / VoxelGrid")
    ap.add_argument("--segment-plane", action="store_true",
                    help="instead: time PointCloud::SegmentPlane per phase at N = 1 M, 10 M and T = 100, 1000")
    args = ap.parse_args()
    if args.segment_plane:
        return segment_plane(args.reps)
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    L = _lib.lib()
    n = args.points
    pts = datagen.uniform_cube(n, 21, hi=(4, 4, 1))
    pc = cph.geometry.PointCloud(pts)
    if "n" in args.attrs:
        pc.normals = datagen.unit_normals(n, 22)
    if "c" in args.attrs:
        pc.colors = datagen.uniform_cube(n, 23)
    A = len(args.attrs)
    flush = DeviceArray((256 << 20,), np.uint8)
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn, reps):
        ts, out = [], None
        for _ in range(reps):
            L.cphb_memset(flush.ptr, 0, flush.nbytes, None)
            L.cphb_stream_synchronize(None)
            L.cphb_event_record(ev[0], None)
            out = fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms))
            ts.append(ms.value)
        return float(np.median(ts)), float(np.min(ts)), out

    for _ in range(2):
        down = pc.voxel_down_sample(args.voxel)
    v_med, v_min, down = timed(lambda: pc.voxel_down_sample(args.voxel), args.reps)
    n_out = len(down)
    # ---- properties (full size) -------------------------------------------------------------
    dp = down.points.cpu()
    mn = pts.min(0) - np.float32(args.voxel) * np.float32(0.5)
    key = np.floor((dp - mn) / np.float32(args.voxel)).astype(np.int64)
    packed = (key[:, 0] << 42) | (key[:, 1] << 21) | key[:, 2]
    props = {"lexicographic_order": bool((np.diff(packed) > 0).all()),
             "n_out": int(n_out),
             "distinct_voxels_of_input": int(len(np.unique((np.floor((pts - mn) / np.float32(args.voxel)).astype(np.int64)
                                                            * np.array([1 << 42, 1 << 21, 1])).sum(1))))}
    props["count_matches"] = props["n_out"] == props["distinct_voxels_of_input"]
    props["centroid_conserved"] = None
    # ---- kNN leg -----------------------------------------------------------------------------
    tree = cph.geometry.KDTreeFlann(down)
    for _ in range(2):
        tree.search_radius(pc.points, args.radius, 1)
    k_med, k_min, (cnt, idx, d2) = timed(lambda: tree.search_radius(pc.points, args.radius, 1), args.reps)
    idx_h, d2_h = idx.cpu()[:, 0], d2.cpu()[:, 0]
    sample = np.random.default_rng(0).choice(n, 2000, replace=False)
    bf = ((pts[sample, None, :].astype(np.float32) - dp[None, :, :]) ** 2).sum(-1) if n_out <= 200000 else None
    props["knn_found_all"] = bool(cnt == n)
    if bf is not None:
        props["knn_sample_matches_bruteforce"] = bool((bf.argmin(1) == idx_h[sample]).mean() > 0.999)
    self_tree = cph.geometry.KDTreeFlann(pc)
    self_tree.search_radius(pc.points, args.radius, 1)  # warm-up: the first call grows the allocation pool
    s_med, s_min, (cnt2, idx2, _) = timed(lambda: self_tree.search_radius(pc.points, args.radius, 1), max(2, args.reps // 2))
    props["self_query_identity"] = bool((idx2.cpu()[:, 0] == np.arange(n)).mean() > 0.9999)
    extra = {}
    if args.normals:
        # SURVEY 8f rank 1: EstimateNormals in one kernel (search + cumulants + eigen-solve) vs search -> [n][k] table -> kernel
        param = cph.geometry.KDTreeSearchParamKNN(args.normals)
        pc.estimate_normals(param)
        f_med, f_min, _ = timed(lambda: pc.estimate_normals(param), max(2, args.reps // 2))
        fused = pc.normals.cpu()
        os.environ["CPHB_NORMALS_UNFUSED"] = "1"
        pc.estimate_normals(param)
        u_med, u_min, _ = timed(lambda: pc.estimate_normals(param), max(2, args.reps // 2))
        two = pc.normals.cpu()
        del os.environ["CPHB_NORMALS_UNFUSED"]
        extra["estimate_normals"] = {"knn": args.normals, "fused_ms_median": f_med, "two_pass_ms_median": u_med,
                                     "table_bytes_not_written_and_reread": int(2 * 8 * args.normals * n),
                                     "fused_equals_two_pass_bit_for_bit": bool(np.array_equal(fused, two))}
    if args.filters:
        # SURVEY 8f rows on the same 10 M cloud: size-independent properties instead of an oracle run
        VG = cph.geometry.VoxelGrid
        for _ in range(2):
            vg = VG.create_from_point_cloud(pc, args.voxel)
        g_med, g_min, vg = timed(lambda: VG.create_from_point_cloud(pc, args.voxel), args.reps)
        gk = vg.get_voxels()[0].astype(np.int64)
        gp = (gk[:, 0] << 42) | (gk[:, 1] << 21) | gk[:, 2]
        extra["voxel_grid"] = {"ms_median": g_med, "ms_min": g_min, "n_voxels": int(len(vg)),
                               "lexicographic_order": bool((np.diff(gp) > 0).all()),
                               "count_matches_voxel_down_sample": bool(len(vg) == n_out)}
        nb, rr = 16, 2.0 * args.voxel
        for _ in range(1):
            pc.remove_radius_outlier(nb, rr)
        r_med, r_min, (rout, ridx) = timed(lambda: pc.remove_radius_outlier(nb, rr), max(2, args.reps // 2))
        kept = ridx.cpu()
        extra["remove_radius_outlier"] = {"nb_points": nb, "radius": rr, "ms_median": r_med, "ms_min": r_min,
                                          "kept": int(len(kept)), "ascending": bool((np.diff(kept) > 0).all()),
                                          "idempotent_on_kept_count": None}
        k_nb = 20
        pc.remove_statistical_outlier(k_nb, 2.0)
        t_med, t_min, (sout, sidx) = timed(lambda: pc.remove_statistical_outlier(k_nb, 2.0), max(2, args.reps // 2))
        skept = sidx.cpu()
        extra["remove_statistical_outlier"] = {"nb_neighbors": k_nb, "std_ratio": 2.0, "ms_median": t_med, "ms_min": t_min,
                                               "kept": int(len(skept)), "ascending": bool((np.diff(skept) > 0).all()),
                                               "stats_mean_std_threshold": list(pc.last_outlier_stats)}
    peak = 6585.1
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    vox_bytes = 12 * A * n + 12 * A * n_out
    knn_bytes = 32 * n
    print(json.dumps({
        "config": "config3: VoxelDownSample(%.3g) + SearchRadius(k=1, r=%.3g) on %d uniform points in [0,4)x[0,4)x[0,1), attrs=%s"
                  % (args.voxel, args.radius, n, args.attrs),
        "voxel": {"ms_median": v_med, "ms_min": v_min, "mpoints_per_sec": n / v_med * 1e-3, "n_out": n_out,
                  "roofline": {"algorithmic_bytes": vox_bytes, "achieved_gbs": vox_bytes / v_med * 1e-6,
                               "frac": vox_bytes / v_med * 1e-6 / peak}},
        "knn_vs_downsampled": {"ms_median": k_med, "ms_min": k_min, "mqueries_per_sec": n / k_med * 1e-3,
                               "roofline": {"algorithmic_bytes": knn_bytes, "achieved_gbs": knn_bytes / k_med * 1e-6,
                                            "frac": knn_bytes / k_med * 1e-6 / peak}},
        "knn_self": {"ms_median": s_med, "mqueries_per_sec": n / s_med * 1e-3},
        "properties": props, "launches": int(L.cphb_launch_count()), **extra,
    }))


def segment_plane(reps):
    """SegmentPlane(0.01, 3, T) on datagen.plane_scene(N): CUDA-event time of the whole call and of its three phases
    (sampling = T key kernels + T stable radix sorts; scoring = planes + one pass over the cloud for all T hypotheses +
    selection; final = flags, compaction, refit), the single-threaded oracle port on the same input (run once), and
    whether the two agree.  Seeds: rand() after srand(1), as a fresh cupoch process draws them."""
    import subprocess
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    from oracle import segment_plane_py as seg_oracle
    L = _lib.lib()
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    libc = C.CDLL(None)
    libc.rand.restype = C.c_int
    ev = [L.cphb_event_create() for _ in range(2)]
    rows = []
    for n in (1_000_000, 10_000_000):
        pts = datagen.plane_scene(n, 11)
        pc = cph.geometry.PointCloud(pts)
        d_idx = DeviceArray((n,), np.int32)
        for T in (100, 1000):
            libc.srand(1)
            seeds = (C.c_int32 * T)(*[libc.rand() for _ in range(T)])
            plane, fr, ph = (C.c_float * 4)(), (C.c_float * 2)(), (C.c_float * 3)()
            m, best = C.c_size_t(0), C.c_int32(0)
            calls, phases = [], []
            for r in range(reps + 1):  # the first call warms the allocation pool and the modules
                L.cphb_event_record(ev[0], None)
                _lib.check(L.cphb_segment_plane(pc.points.ptr, n, 0.01, 3, T, seeds, plane, d_idx.ptr, C.byref(m),
                                                C.byref(best), fr, ph, None))
                L.cphb_event_record(ev[1], None)
                ms = C.c_float(0)
                L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms))
                if r:
                    calls.append(ms.value)
                    phases.append(list(ph))
            med = float(np.median(calls))
            ph_med = [float(np.median([p[k] for p in phases])) for k in range(3)]
            row = {"n": n, "iterations": T}
            if n * T > 1e9:  # the sequential oracle needs minutes here (about 3 s per 1e8 point-iterations)
                rows.append(dict(row, cpu_baseline=None, note="oracle not run at n * T > 1e9"))
            else:
                t0 = time.perf_counter()
                o_plane, o_idx, o_best, _, _ = seg_oracle.segment_plane(pts, 0.01, 3, np.array(seeds, np.int32))
                cpu_s = time.perf_counter() - t0
                rows.append(dict(row, cpu_baseline={"seconds": cpu_s, "cores": 1, "kind": "port"},
                                 speedup_vs_cpu_baseline=cpu_s * 1e3 / med,
                                 parity_vs_cpu_baseline=bool(o_best == best.value
                                                             and np.array_equal(o_plane, np.array(plane, np.float32))
                                                             and np.array_equal(o_idx, d_idx.cpu()[:m.value]))))
            rows[-1].update({
                "call_ms_median": med, "call_ms_min": float(np.min(calls)),
                "phase_ms_median": dict(zip(("sampling", "scoring", "final"), ph_med)),
                "phase_share": dict(zip(("sampling", "scoring", "final"), [p / sum(ph_med) for p in ph_med])),
                "sampling_us_per_iteration": ph_med[0] * 1e3 / T,
                "scoring_point_hypotheses_per_s": n * T / (ph_med[1] * 1e-3),
                "inliers": int(m.value), "best_iteration": int(best.value),
            })
    print(json.dumps({"op": "PointCloud::SegmentPlane(0.01, 3, T) on datagen.plane_scene(N, 11)", "gpu": gpu, "reps": reps,
                      "launches": int(L.cphb_launch_count()), "rows": rows}))


if __name__ == "__main__":
    main()
