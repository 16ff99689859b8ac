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
    ap.add_argument("--fps", action="store_true",
                    help="instead: time PointCloud::FarthestPointDownSample at N = 100 k, 1 M, 10 M and 1024, 8192 samples")
    ap.add_argument("--iss", action="store_true",
                    help="instead: time geometry::keypoint::ComputeISSKeypoints (defaults, automatic radii) at N = 1 M, 10 M")
    ap.add_argument("--shot", action="store_true",
                    help="instead: time registration::ComputeSHOTFeature (Radius(r, 100), r = 5 spacings) at N = 100 k, 1 M")
    ap.add_argument("--crop", action="store_true",
                    help="instead: time crop / pass_through_filter / remove_none_finite_points / uniform_down_sample / "
                         "get_oriented_bounding_box on the 10 M config-3 cloud with normals and colours")
    ap.add_argument("--out", default=None, help="--shot, --crop: also write the JSON object to this file")
    ap.add_argument("--edt", action="store_true",
                    help="instead: time geometry::DistanceTransform::ComputeEDT at 256^3 and 512^3 and GetDistances of 10 M points")
    ap.add_argument("--voxelgrid", action="store_true",
                    help="instead: time the VoxelGrid operations (CreateDense, carving, CheckIfIncluded, +=, "
                         "CreateFromOccupancyGrid) on the config-3 VoxelGrid and 512^3 grids")
    ap.add_argument("--collision", action="store_true",
                    help="instead: time collision::ComputeIntersection on the config-3 VoxelGrid, a 512^3 OccupancyGrid and "
                         "1 / 1e4 primitives")
    ap.add_argument("--tsdf", action="store_true",
                    help="instead: time UniformTSDFVolume Integrate of a 640x480 frame at 256^3 and 512^3 per colour type, "
                         "both extractions and a 640x480 Raycast")
    ap.add_argument("--tsdf-mesh", action="store_true",
                    help="instead: time UniformTSDFVolume.extract_triangle_mesh and compute_vertex_normals at 256^3 and 512^3 "
                         "after 8 ring-camera sphere views")
    ap.add_argument("--depth-cloud", action="store_true",
                    help="instead: time PointCloud.create_from_rgbd_image and create_from_depth_image at 640x480 and 1280x720")
    ap.add_argument("--mesh-ops", action="store_true",
                    help="instead: time TriangleMesh.compute_edge_list, the four filters at 1 and 100 iterations, "
                         "get_surface_area and sample_points_uniformly (1 M, 10 M points) on the --tsdf-mesh sphere meshes")
    ap.add_argument("--mesh-clean", action="store_true",
                    help="time the TriangleMesh Remove* operations and GetSelfIntersectingTriangles on the --mesh-ops sphere meshes")
    ap.add_argument("--mesh-voxel", action="store_true",
                    help="instead: time VoxelGrid.create_from_triangle_mesh_within_bounds (sizing and writing call apart) on "
                         "the --mesh-ops sphere meshes at 1x and 2x their voxel size, a two-triangle 512^2 plane and a coarse "
                         "20-triangle solid in a 512^3 grid, with per-kernel times from torch.profiler")
    args = ap.parse_args()
    if args.mesh_voxel:
        return mesh_voxel(args.reps, args.out)
    if args.mesh_clean:
        return mesh_clean(args.reps, args.out)
    if args.mesh_ops:
        return mesh_ops(args.reps, args.out)
    if args.depth_cloud:
        return depth_cloud(args.reps, args.out)
    if args.tsdf_mesh:
        return tsdf_mesh(args.reps, args.out)
    if args.tsdf:
        return tsdf(args.reps, args.out)
    if args.collision:
        return collision(args.reps, args.out)
    if args.voxelgrid:
        return voxelgrid(args.reps, args.out)
    if args.edt:
        return edt(args.reps)
    if args.segment_plane:
        return segment_plane(args.reps)
    if args.fps:
        return fps(args.reps)
    if args.iss:
        return iss(args.reps)
    if args.shot:
        return shot(args.reps, args.out)
    if args.crop:
        return crop(args.reps, args.points, args.out)
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


def fps(reps):
    """cphb_farthest_point_down_sample on datagen.surface(N, 11): CUDA-event time of the call (one persistent launch),
    against a reference-shaped loop in torch on the same GPU (one step per sample: torch.minimum of the distances,
    argmax, .item() -- launches and a host round trip per sample, as thrust::transform_reduce has in the reference),
    timed by the host clock, which the .item() of every step synchronises.  torch rounds the squared distance
    differently (no FMA), so its picks are counted against the product's, not asserted.  N = 100 k and 1 M keep the
    points in shared memory, 10 M streams them (the switch is at SMs * 14336 points).  The CPU oracle runs where
    N * samples <= 2e9 (single-threaded, a few seconds) and must agree bit for bit."""
    import subprocess
    import torch
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    from oracle import fps_py as orc
    L = _lib.lib()
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ev = [L.cphb_event_create() for _ in range(2)]
    rows = []
    for n in (100_000, 1_000_000, 10_000_000):
        pts = datagen.surface(n, 11)[0]
        pc = cph.geometry.PointCloud(pts)
        P = torch.from_numpy(pts).cuda()
        for S in (1024, 8192):
            d_idx = DeviceArray((S,), np.int32)
            calls = []
            for r in range(reps + 1):  # the first call warms the allocation pool and the module
                L.cphb_event_record(ev[0], None)
                _lib.check(L.cphb_farthest_point_down_sample(pc.points.ptr, n, S, d_idx.ptr, None, None))
                L.cphb_event_record(ev[1], None)
                ms = C.c_float(0)
                _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
                if r:
                    calls.append(ms.value)
            idx = d_idx.cpu()
            med = float(np.median(calls))

            def torch_loop():
                dist = torch.full((n,), float("inf"), device="cuda")
                far, sel = 0, []
                for _ in range(S):
                    sel.append(far)
                    dist = torch.minimum(dist, ((P - P[far]) ** 2).sum(1))
                    far = int(torch.argmax(dist).item())
                return np.array(sel, np.int32)

            torch_loop()
            t_calls = []
            for _ in range(max(2, reps // 2)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                t_idx = torch_loop()
                t_calls.append((time.perf_counter() - t0) * 1e3)
            t_med = float(np.median(t_calls))
            agree = t_idx == idx
            row = {"n": n, "num_samples": S, "points_in_shared_memory": bool(n <= sms * 14336),
                   "call_ms_median": med, "call_ms_min": float(np.min(calls)), "us_per_sample": med * 1e3 / S,
                   "torch_loop": {"ms_median": t_med, "ms_min": float(np.min(t_calls)), "us_per_sample": t_med * 1e3 / S,
                                  "index_agreement": float(agree.mean()),
                                  "first_disagreement": None if agree.all() else int(np.argmin(agree))},
                   "speedup_vs_torch_loop": t_med / med}
            if n * S <= 2e9:
                t0 = time.perf_counter()
                o_idx, _ = orc.farthest_point_down_sample(pts, S)
                row["cpu_oracle"] = {"seconds": time.perf_counter() - t0, "threads": 1,
                                     "parity": bool(np.array_equal(o_idx, idx))}
            else:
                row["cpu_oracle"] = None
            rows.append(row)
        del P
        torch.cuda.empty_cache()
    print(json.dumps({"op": "PointCloud::FarthestPointDownSample(S) on datagen.surface(N, 11)", "gpu": gpu, "reps": reps,
                      "sms": sms, "launches": int(L.cphb_launch_count()), "rows": rows}))


ISS_PHASES = (("radii", ("iss_knn2", "iss_tile_sum", "iss_radii")), ("saliency", ("iss_saliency",)),
              ("suppression", ("iss_suppress",)), ("compaction_gather", ("keep_", "select_rows")))


def eigvals3(A):
    """ascending eigenvalues of a batch of symmetric 3x3 float32 matrices, closed form (trigonometric), in torch.
    torch.linalg.eigvalsh raised CUSOLVER_STATUS_INVALID_VALUE on these batches on the H100 (torch 2.11, CUDA 12.8)."""
    import torch
    q = A.diagonal(dim1=1, dim2=2).sum(1) / 3
    B = A - q[:, None, None] * torch.eye(3, device=A.device)
    p = torch.sqrt((B * B).sum((1, 2)) / 6).clamp(min=1e-30)
    r = (torch.linalg.det(B / p[:, None, None]) / 2).clamp(-1, 1)
    phi = torch.acos(r) / 3
    e3 = q + 2 * p * torch.cos(phi)
    e1 = q + 2 * p * torch.cos(phi + 2 * np.pi / 3)
    return torch.stack([e1, 3 * q - e1 - e3, e3], 1)


def iss(reps):
    """compute_iss_keypoints(pc) with the defaults (automatic radii, max_neighbors 100) on datagen.surface(N, 11) over a
    sqrt(N / 1e5)-wide square:
    CUDA-event time of the whole Python call (index build, the fused kernels, compaction, gather), and per-phase kernel
    times from torch.profiler in a separate profiled call (radii = kNN-2 + tiled sum; saliency; suppression; compaction
    + gather; the rest is the index build).  Comparison arm shaped like the reference (iss_keypoints.cu:108-172) on the
    same GPU, timed by the host clock around a synchronised run: cphb_search_knn(k = 2) + a torch sum for the radii,
    cphb_search_radius into [n][100] tables twice, torch for the cumulants (float32 sums over the table rows),
    closed-form 3x3 eigenvalues in torch (eigvals3, float32) and the suppression gather.  Its eigen-solver is not FastEigen3x3, so its keypoints
    are compared as a set (Jaccard overlap), not asserted."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    L = _lib.lib()
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]
    kp_fn = cph.geometry.keypoint.compute_iss_keypoints
    rows = []
    for n in (1_000_000, 10_000_000):
        # extent sqrt(N / 1e5): 1e5 points per unit square.  On the unit square at 1 M every neighbourhood covariance is
        # within 1e-5 of zero, and the reference's absolute isZero test leaves no salient point at all
        pts = datagen.surface(n, 11, extent=float(np.sqrt(n / 1e5)))[0]
        pc = cph.geometry.PointCloud(pts)
        calls = []
        for r in range(reps + 1):  # the first call warms the allocation pool and the modules
            L.cphb_event_record(ev[0], None)
            out, mask = kp_fn(pc)
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                calls.append(ms.value)
        radii = pc.last_iss_radii
        keep = mask.cpu()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            kp_fn(pc)
            torch.cuda.synchronize()
        phase_ms = {name: 0.0 for name, _ in ISS_PHASES}
        phase_ms["index_build"] = 0.0
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t <= 0 or "Memset" in e.key or "Memcpy" in e.key:
                continue
            name = next((p for p, keys in ISS_PHASES if any(k in e.key for k in keys)), "index_build")
            phase_ms[name] += t

        def reference_shaped():
            P = torch.as_tensor(pc.points, device="cuda")
            tree = cph.geometry.KDTreeFlann(pc)
            _, i2, d2 = tree.search_knn(pc.points, 2)
            res = torch.sqrt(torch.as_tensor(d2, device="cuda")[:, 1].sum() / n)
            rs, rn = float(6 * res), float(4 * res)
            _, idx, _ = tree.search_radius(pc.points, rs, 100)
            I = torch.as_tensor(idx, device="cuda")
            sal = torch.empty(n, device="cuda")
            for lo in range(0, n, 1 << 20):  # the cumulants per table row, chunked only to bound torch's temporaries
                J = I[lo:lo + (1 << 20)]
                ok = (J >= 0).unsqueeze(-1)
                X = P[J.clamp(min=0).long()] * ok
                cnt = ok.sum(1).float()
                mu = X.sum(1) / cnt
                cov = torch.einsum("nki,nkj->nij", X, X) / cnt.unsqueeze(-1) - mu.unsqueeze(-1) * mu.unsqueeze(-2)
                e = eigvals3(cov / cov.flatten(1).amax(1).clamp(min=1e-30)[:, None, None])
                nonzero = (cov.flatten(1).abs() > 1e-5).any(1)
                s = torch.where((cnt[:, 0] >= 5) & nonzero & (e[:, 2] > 0) & (e[:, 1] / e[:, 2] < 0.975) & (e[:, 0] / e[:, 1] < 0.975),
                                e[:, 0], torch.full_like(e[:, 0], -1.0))
                sal[lo:lo + len(J)] = s
            del I, X
            _, idx, _ = tree.search_radius(pc.points, rn, 100)
            I = torch.as_tensor(idx, device="cuda")
            nb = torch.where(I >= 0, sal[I.clamp(min=0).long()], torch.full_like(sal[:1], -2.0).expand_as(I))
            m = (sal >= 0) & ~(nb > sal[:, None]).any(1)
            return m.cpu().numpy()

        reference_shaped()
        t_calls = []
        for _ in range(max(2, reps // 2)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t_mask = reference_shaped()
            torch.cuda.synchronize()
            t_calls.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.empty_cache()
        t_med = float(np.median(t_calls))
        med = float(np.median(calls))
        inter, union = int((keep & t_mask).sum()), int((keep | t_mask).sum())
        rows.append({"n": n, "radii": list(radii), "keypoints": int(keep.sum()), "call_ms_median": med,
                     "call_ms_min": float(np.min(calls)), "phase_ms_profiled": phase_ms,
                     "tables_not_written_bytes": int(2 * 100 * 8 * n + 2 * 8 * n),
                     "reference_shaped": {"ms_median": t_med, "ms_min": float(np.min(t_calls)), "keypoints": int(t_mask.sum()),
                                          "jaccard_overlap": inter / union if union else 1.0},
                     "speedup_vs_reference_shaped": t_med / med})
    print(json.dumps({"op": "geometry::keypoint::ComputeISSKeypoints(defaults) on datagen.surface(N, 11)", "gpu": gpu,
                      "reps": reps, "launches": int(L.cphb_launch_count()), "rows": rows}))


SHOT_PHASES = (("shot_kernel", ("shot_kernel",)),)


def shot(reps, out=None):
    """compute_shot_feature(pc, r, KDTreeSearchParamRadius(r, 100)) with r = 5 x the point spacing on datagen.surface(N,
    11) over a sqrt(N / 1e5)-wide square (1e5 points per unit square); normals from EstimateNormals(KNN 30), not timed.
    CUDA-event time of the whole Python call after a warm-up call, and per-kernel times from torch.profiler in a separate
    profiled call (shot_kernel; the rest is the index build).  Comparison arm: the library's own search_radius writing
    the [n][100] index and distance tables the reference materialises before its descriptor pass (shot.cu:229-245),
    index build included, timed by CUDA events -- a lower bound on the reference's first stage only.  The reference
    binary itself is not run here."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    L = _lib.lib()
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times = []
        for r in range(reps + 1):  # the first call warms the allocation pool and the modules
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    rows = []
    for n in (100_000, 1_000_000):
        pts = datagen.surface(n, 11, extent=float(np.sqrt(n / 1e5)))[0]
        pc = cph.geometry.PointCloud(pts)
        pc.estimate_normals(cph.geometry.KDTreeSearchParamKNN(30))
        r = float(np.float32(5.0 / np.sqrt(1e5)))
        param = cph.geometry.KDTreeSearchParamRadius(r, 100)
        calls = timed(lambda: cph.registration.compute_shot_feature(pc, r, param))
        f = cph.registration.compute_shot_feature(pc, r, param).cpu()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cph.registration.compute_shot_feature(pc, r, param)
            torch.cuda.synchronize()
        phase_ms = {"shot_kernel": 0.0, "index_build": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t <= 0 or "Memset" in e.key or "Memcpy" in e.key:
                continue
            phase_ms["shot_kernel" if "shot_kernel" in e.key else "index_build"] += t

        def tables():
            tree = cph.geometry.KDTreeFlann(pc)
            return tree.search_radius(pc.points, r, 100)

        table_calls = timed(tables)
        listed = int(tables()[0])  # the number of (point, neighbour) slots filled
        med = float(np.median(calls))
        rows.append({"n": n, "radius": r, "mean_listed_neighbours": listed / n,
                     "nonzero_rows": int((np.abs(f).sum(1) > 0).sum()),
                     "call_ms_median": med, "call_ms_min": float(np.min(calls)), "phase_ms_profiled": phase_ms,
                     "descriptor_bytes_written": int(n * 352 * 4),
                     "tables_not_written_bytes": int(n * 100 * (4 + 4)),
                     "reference_first_stage_tables": {"ms_median": float(np.median(table_calls)),
                                                      "ms_min": float(np.min(table_calls))},
                     "speedup_vs_cupoch": "not measured"})
        torch.cuda.empty_cache()
    res = {"op": "registration::ComputeSHOTFeature(pc, r, KDTreeSearchParamRadius(r, 100)), r = 5 spacings, on "
                 "datagen.surface(N, 11) at 1e5 points per unit square", "gpu": gpu, "reps": reps, "rows": rows}
    print(json.dumps(res))
    if out:
        with open(out, "w") as fh:
            json.dump(res, fh)


HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def edt_bytes_model(r):
    """HBM bytes of one ComputeEDT at res r (a model, not a measurement).  Per cell: the bitmap clear, stamp and read
    (3 / 8 B); sweep z writes nearest (4 B); sweeps y and x each read nearest, write and read back their stack and write
    nearest (16 B), and sweep x also writes the distance (4 B).  A stack entry is written only for a candidate that is
    not dominated when it arrives and read back only where the envelope moves, so the stack terms lie between 0 and 8 B
    per sweep: 24.4 B per cell at least, 40.4 B at most."""
    cells = r ** 3
    return {"min": int(cells * (3 / 8 + 4 + 8 + 12)), "max": int(cells * (3 / 8 + 4 + 16 + 20))}


def edt(reps):
    """DistanceTransform(1 / r, r).compute_edt(voxel grid) at r = 256 and 512: CUDA-event time of the whole call (clear,
    stamp, three sweeps), median of `reps` calls after one warm-up call, and the same for compute_voronoi_diagram.  The
    sites are datagen.surface sheets (z = 0.1 sin(4 pi x) cos(4 pi y)) stacked along z and voxelised at the grid's own
    voxel size, about 1 % of the cells.  The device result is checked against the CPU oracle at 256^3.  Then
    get_distances of 10 M uniform points in the grid's box.  CPU arm: scipy.ndimage.distance_transform_edt of the same
    site mask on the host (single-threaded: scipy's EDT has no thread option), one call."""
    import subprocess
    from scipy import ndimage
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    from oracle import edt_py
    L = _lib.lib()
    G = cph.geometry
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        calls = []
        for k in range(reps + 1):
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if k:
                calls.append(ms.value)
        return float(np.median(calls)), float(np.min(calls))

    rows = []
    for r in (256, 512):
        vs = 1.0 / r
        layers = r // 100 + 1
        sheets = []
        for i in range(layers):
            p = datagen.surface(4 * r * r, 70 + i)[0]
            p[:, 2] += np.float32(-0.35 + 0.7 * (i + 0.5) / layers)
            sheets.append(p)
        pts = np.concatenate(sheets)
        vg = G.VoxelGrid.create_from_point_cloud_within_bounds(G.PointCloud(pts), vs, (0, 0, -0.5), (1, 1, 0.5))
        dt = G.DistanceTransform(vs, r, (0.5, 0.5, 0.0))
        edt_ms, edt_min = timed(lambda: dt.compute_edt(vg))
        vor_ms, vor_min = timed(lambda: dt.compute_voronoi_diagram(vg))
        dt.compute_edt(vg)
        dist = dt.to_torch().cpu().numpy()
        near = DeviceArray((r, r, r), np.uint32, ptr=L.cphb_dt_nearest_data(dt._h), base=dt).cpu()
        sites = (near & ((1 << 30) - 1)) == edt_cell_codes(r)
        occupancy = float(sites.mean())
        row = {"res": r, "voxel_grid_keys": len(vg), "site_occupancy": occupancy, "compute_edt_ms_median": edt_ms,
               "compute_edt_ms_min": edt_min, "compute_voronoi_ms_median": vor_ms, "compute_voronoi_ms_min": vor_min}
        model = edt_bytes_model(r)
        row["bytes_model"] = model
        row["bytes_model_share_of_hbm_peak"] = {k: v / HBM_BYTES_PER_S / (edt_ms * 1e-3) for k, v in model.items()}
        if r == 256:
            o = edt_py.compute_voxel_grid(r, vs, (0.5, 0.5, 0.0), vg.voxels_keys.cpu(), vg.voxel_size, vg.origin)
            row["oracle_parity"] = bool(np.array_equal(o[2].view(np.uint32), dist.view(np.uint32)) and
                                        np.array_equal(o[1] == 2, (near >> 30) & 1 == 1))
        t0 = time.perf_counter()
        ref = ndimage.distance_transform_edt(~sites)
        row["scipy_edt_cpu"] = {"seconds": time.perf_counter() - t0, "threads": 1,
                                "max_abs_diff_in_voxels": float(np.abs(ref * vs - dist).max() / vs)}
        rows.append(row)
        if r == 512:
            n = 10_000_000
            q = DeviceArray.from_numpy(datagen.uniform_cube(n, 5, lo=(0, 0, -0.5), hi=(1, 1, 0.5)))
            q_ms, q_min = timed(lambda: dt.get_distances(q))
            query = {"res": r, "queries": n, "ms_median": q_ms, "ms_min": q_min,
                     "bytes_model": n * (12 + 4 + 4), "note": "12 B point + 4 B result + one 4 B distance gather per query"}
        del dt
    print(json.dumps({"op": "geometry::DistanceTransform::ComputeEDT(VoxelGrid) and GetDistances", "gpu": gpu, "reps": reps,
                      "hbm_peak_bytes_per_s": HBM_BYTES_PER_S, "launches": int(L.cphb_launch_count()), "rows": rows,
                      "get_distances": query}))


def edt_cell_codes(r):
    """x << 20 | y << 10 | z of every cell of an r^3 grid (a site is its own nearest site)"""
    g = np.arange(r, dtype=np.uint32)
    return (g[:, None, None] << 20) | (g[None, :, None] << 10) | g[None, None, :]


H100_HBM_BYTES_PER_S = 3.35e12  # NVIDIA's H100 SXM data sheet (700 W); a share of it is not a claim that it was reached


def crop_bytes_model(op, n, m):
    """least HBM traffic of each call on a cloud of n points with normals and colours (three float32[3] arrays), m rows
    out: a selection reads 12 B of xyz and writes 1 B of flag per point, then reads and writes the m gathered rows
    (3 x 12 B each way); the uniform stride is the gather alone; the OBB reads the points for the mean, the moments and
    the transform copy, writes and rereads the copy, and reads the transformed copy for the bounds."""
    if op == "uniform_down_sample(5)":
        return 72 * m
    if op == "get_oriented_bounding_box":
        return 12 * n * 6
    return 13 * n + 72 * m


def crop(reps, n, out=None):
    """The region-selection and cleanup calls on the config-3 cloud (datagen.uniform_cube(N, 21) in [0,4)x[0,4)x[0,1),
    unit normals, colours): CUDA-event time of the whole Python call, which ends in a host synchronise, after a cache
    flush; each kernel's device time from torch.profiler in a separate profiled call; the bytes model above over the
    summed kernel time as a share of the data-sheet bandwidth.  remove_none_finite_points works in place, so every rep
    runs on a fresh copy (made outside the timed window) with 1 % of the rows NaN."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.utility import DeviceArray
    L = _lib.lib()
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    G = cph.geometry
    pts = datagen.uniform_cube(n, 21, hi=(4, 4, 1))
    pc = G.PointCloud(pts)
    pc.normals = datagen.unit_normals(n, 22)
    pc.colors = datagen.uniform_cube(n, 23)
    bad = pts.copy()
    bad[np.random.default_rng(24).choice(n, n // 100, replace=False), 1] = np.nan
    pc_bad = G.PointCloud(bad)
    pc_bad.normals, pc_bad.colors = pc.normals, pc.colors
    c, s_ = np.cos(np.pi / 6), np.sin(np.pi / 6)
    obb = G.OrientedBoundingBox((2, 2, 0.5), [[c, -s_, 0], [s_, c, 0], [0, 0, 1]], (2.6, 2.6, 1.2))
    fresh = {}

    def nonfinite():
        return fresh.pop("pc").remove_none_finite_points()

    def prep_nonfinite():
        fresh["pc"] = pc_bad.clone()

    calls = [("crop(AABB [0,2]x[0,4]x[0,1])", lambda: pc.crop(G.AxisAlignedBoundingBox((0, 0, 0), (2, 4, 1))), None),
             ("crop(OBB 30 deg about z)", lambda: pc.crop(obb), None),
             ("pass_through_filter(2, 0.0, 0.5)", lambda: pc.pass_through_filter(2, 0.0, 0.5), None),
             ("remove_none_finite_points(1 % NaN)", nonfinite, prep_nonfinite),
             ("uniform_down_sample(5)", lambda: pc.uniform_down_sample(5), None),
             ("get_oriented_bounding_box", lambda: pc.get_oriented_bounding_box(), None)]
    flush = DeviceArray((256 << 20,), np.uint8)
    ev = [L.cphb_event_create() for _ in range(2)]
    rows = []
    for name, fn, prep in calls:
        ts = []
        for r in range(reps + 1):  # the first call warms the allocation pool and the modules
            if prep:
                prep()
            L.cphb_memset(flush.ptr, 0, flush.nbytes, None)
            L.cphb_stream_synchronize(None)
            L.cphb_event_record(ev[0], None)
            res = fn()
            L.cphb_event_record(ev[1], None)
            L.cphb_stream_synchronize(None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                ts.append(ms.value)
        m = len(res) if isinstance(res, G.PointCloud) else 0
        if prep:
            prep()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0:
                kernels[e.key] = kernels.get(e.key, 0.0) + t
        kern_ms = sum(t for k, t in kernels.items() if "Memset" not in k and "Memcpy" not in k)
        nbytes = crop_bytes_model(name, n, m)
        rows.append({"op": name, "n": n, "rows_out": m, "call_ms_median": float(np.median(ts)),
                     "call_ms_min": float(np.min(ts)), "kernel_ms_profiled": kernels, "kernel_ms_sum": kern_ms,
                     "bytes_model": nbytes,
                     "share_of_3.35TBps_over_kernel_time": nbytes / (kern_ms * 1e-3) / H100_HBM_BYTES_PER_S if kern_ms else None,
                     "share_of_3.35TBps_over_call_time": nbytes / (float(np.median(ts)) * 1e-3) / H100_HBM_BYTES_PER_S})
    obj = {"op": "bounding-box selection and cleanup on the config-3 cloud (uniform_cube(N, 21) in [0,4)x[0,4)x[0,1), "
                 "normals and colours)", "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def collision_bytes_model(kind_t, n_t, kind_q, n_q, m, box_cells=0):
    """HBM bytes one compute_intersection call must move at least (a model, not a measurement): a VoxelGrid target's
    keys read twice (bounds, pack) and sorted (12-byte key + index pairs, read and written by each of 8 radix passes);
    the query's elements read once (keys, 88-byte primitives, or the bound box of an OccupancyGrid query flagged and
    compacted); per query element its best index, flag and compaction slot (9 B); 8 B per pair.  Lookups into the
    target are not counted: they mostly hit L2."""
    b = 0
    if kind_t == "vg":
        b += 24 * n_t + 2 * 12 * n_t * 9
    b += {"vg": 12, "prim": 88 + 32, "occ": 0}[kind_q] * n_q
    b += 5 * box_cells + 4 * n_q if kind_q == "occ" else 0
    return b + 9 * n_q + 8 * m


def collision(reps, out=None):
    """compute_intersection on the config-3 cloud (uniform_cube(10 M, 21) in [0,4)x[0,4)x[0,1)) voxelised at 0.02
    (about 2 M voxels): against itself moved by (0.3, 0.2, 0.1) voxels at margins 0 and 2 voxels; a 512^3
    OccupancyGrid (voxel 0.02) after inserting a 1 M-point scan, in both orders against that grid; 1 and 1e4 mixed
    primitives in both orders; one box whose region covers about 1e6 cells.  CUDA-event median and minimum of `reps`
    calls after a warm-up call, the kernel time of one further call from torch.profiler, the bytes model beside it."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    L = _lib.lib()
    K = cph.collision
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times = []
        for r in range(reps + 1):
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    vs = 0.02
    pc = cph.geometry.PointCloud(datagen.uniform_cube(10_000_000, 21, hi=(4, 4, 1)))
    tgt = cph.geometry.VoxelGrid.create_from_point_cloud(pc, vs)
    del pc
    qry = cph.geometry.VoxelGrid()
    qry.voxel_size, qry.voxels_keys = tgt.voxel_size, tgt.voxels_keys
    qry.origin = tgt.origin + np.float32(vs) * np.array([0.3, 0.2, 0.1], np.float32)
    scan = datagen.surface(1_000_000, 11, extent=4.0)[0] + np.array([0, 0, 0.5], np.float32)
    occ = cph.geometry.OccupancyGrid(vs, 512, (2.0, 2.0, 0.5))
    occ.insert(cph.geometry.PointCloud(scan.astype(np.float32)), (2.0, 2.0, 3.0))
    lo, hi = occ._bounds()
    box_cells = int(np.prod((hi - lo + 1).astype(np.int64)))
    rng = np.random.default_rng(3)
    prims = K.PrimitiveArray()
    for i in range(10_000):
        c = rng.uniform((0, 0, 0), (4, 4, 1))
        T = np.eye(4, dtype=np.float32)
        T[:3, 3] = c
        a = rng.uniform(0, np.pi)
        T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        s = rng.uniform(1, 5) * vs
        prims.append([K.Box([s, s, s], T), K.Sphere(s, c), K.Capsule(s / 2, 2 * s, T)][i % 3])
    one = K.PrimitiveArray([prims[0]])
    big = K.PrimitiveArray([K.Box([2.0, 2.0, 2.0], np.array([[1, 0, 0, 2], [0, 1, 0, 2], [0, 0, 1, 0.5], [0, 0, 0, 1]], np.float32))])
    n_vg = len(tgt)
    work = [("vg x vg, margin 0", tgt, qry, 0.0, ("vg", n_vg, "vg", n_vg)),
            ("vg x vg, margin 2 vs", tgt, qry, 2 * vs, ("vg", n_vg, "vg", n_vg)),
            ("occ x vg", occ, qry, 0.0, ("occ", 0, "vg", n_vg)),
            ("vg x occ", tgt, occ, 0.0, ("vg", n_vg, "occ", None)),
            ("vg x 1 primitive", tgt, one, 0.0, ("vg", n_vg, "prim", 1)),
            ("1 primitive x vg", one, tgt, 0.0, ("prim", 1, "vg", n_vg)),
            ("vg x 1e4 primitives", tgt, prims, 0.0, ("vg", n_vg, "prim", 10_000)),
            ("1e4 primitives x vg", prims, tgt, 0.0, ("prim", 10_000, "vg", n_vg)),
            ("vg x one box over ~1e6 cells", tgt, big, 0.0, ("vg", n_vg, "prim", 1))]
    rows = []
    for name, a, b, margin, shape in work:
        ts = timed(lambda: K.compute_intersection(a, b, margin))
        res = K.compute_intersection(a, b, margin)
        m = len(res.collision_index_pairs)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            K.compute_intersection(a, b, margin)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
                kernels[e.key[:60]] = kernels.get(e.key[:60], 0.0) + t
        kern_ms = float(sum(kernels.values()))
        kt, nt, kq, nq = shape
        nq = m if nq is None else nq  # an OccupancyGrid query: its occupied cells are not known up front
        nbytes = collision_bytes_model(kt, nt, kq, nq, m, box_cells if kq == "occ" else 0)
        rows.append({"workload": name, "pairs": m, "call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)),
                     "kernel_ms_profiled": kernels, "kernel_ms_sum": kern_ms, "bytes_model": nbytes,
                     "share_of_3.35TBps_over_kernel_time": nbytes / (kern_ms * 1e-3) / HBM_BYTES_PER_S if kern_ms else None})
    obj = {"op": "collision::ComputeIntersection on the config-3 cloud voxelised at 0.02 (%d voxels), a 512^3 "
                 "OccupancyGrid after a 1 M-point scan (%d cells in its bound box) and 1 / 1e4 mixed primitives" % (n_vg, box_cells),
           "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def voxelgrid_bytes_model(op, n, m=0):
    """least HBM traffic of one call: keys and colours are 12 bytes each a voxel; a sort pass reads and writes 8-byte
    packed keys and 4-byte indices (counted once), a query reads 12 bytes and writes 1"""
    if op == "dense":
        return 24 * n
    if op == "carve":
        return 12 * n + 24 * m
    if op == "included":
        return 12 * n + 24 * n + 13 * m
    if op == "merge":
        return 48 * n + 24 * n + 24 * m
    if op in ("vg_from_occ", "pc_from_occ"):
        return 4 * n + 24 * m  # the log-odds of the grid's bound box (n cells) read once, the rows written
    raise ValueError(op)


def voxelgrid(reps, out=None):
    """CreateDense at 256^3 and 512^3; one carve of a dense 512^3 grid by a sphere's depth map; CheckIfIncluded of 10 M
    queries against the config-3 cloud voxelised at 0.02 (about 2 M voxels); += of that grid and a shifted one; both
    CreateFromOccupancyGrid calls on a 512^3 grid after a 1 M-point scan.  CUDA-event median and minimum of `reps` calls
    after a warm-up call (host upload of queries and images included where the call takes host data), the kernel time
    of one further call from torch.profiler, and the bytes model beside it."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G = cph.geometry
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn, prep=None):
        times = []
        for r in range(reps + 1):
            arg = prep() if prep else None
            L.cphb_event_record(ev[0], None)
            fn(arg)
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    vs = 0.02
    pts = datagen.uniform_cube(10_000_000, 21, hi=(4, 4, 1))
    a = G.VoxelGrid.create_from_point_cloud_within_bounds(G.PointCloud(pts), vs, (0, 0, 0), (6, 4, 1))
    b = G.VoxelGrid.create_from_point_cloud_within_bounds(G.PointCloud((pts + np.float32([2, 0, 0])).astype(np.float32)), vs,
                                                          (0, 0, 0), (6, 4, 1))
    del pts
    q = np.random.default_rng(1).uniform((0, 0, 0), (4, 4, 1), (10_000_000, 3)).astype(np.float32)
    scan = datagen.surface(1_000_000, 11, extent=4.0)[0] + np.array([0, 0, 0.5], np.float32)
    occ = G.OccupancyGrid(vs, 512, (2.0, 2.0, 0.5))
    occ.insert(G.PointCloud(scan.astype(np.float32)), (2.0, 2.0, 3.0))
    K, E = ring_cameras(1, 640, 480)[0]
    img = G.Image(sphere_depth(K, E, 640, 480, 0.8))
    cam = cph.camera.PinholeCameraParameters(cph.camera.PinholeCameraIntrinsic(640, 480, K[0, 0], K[1, 1], K[0, 2], K[1, 2]), E)
    n_occ = len(occ.extract_occupied_voxels()[0])
    lo, hi = occ._bounds()
    box_cells = int(np.prod((hi - lo + 1).astype(np.int64)))

    def dense(r):
        return lambda _: G.VoxelGrid.create_dense((-1, -1, -1), 2.0 / r, 2, 2, 2)

    def fresh512():
        return G.VoxelGrid.create_dense((-1, -1, -1), 2.0 / 512, 2, 2, 2)

    carved = len(fresh512().carve_depth_map(img, cam))
    work = [("CreateDense 256^3", dense(256), None, ("dense", 256 ** 3, 0)),
            ("CreateDense 512^3", dense(512), None, ("dense", 512 ** 3, 0)),
            ("CarveDepthMap of a dense 512^3 grid, 640x480 depth map", lambda g: g.carve_depth_map(img, cam), fresh512,
             ("carve", 512 ** 3, carved)),
            ("CheckIfIncluded, 10 M queries, %d voxels" % len(a), lambda _: a.check_if_included(q), None,
             ("included", len(a), len(q))),
            ("+= of %d and %d voxels" % (len(a), len(b)), lambda _: a + b, None, ("merge", len(a) + len(b), len(a + b))),
            ("VoxelGrid.create_from_occupancy_grid 512^3", lambda _: G.VoxelGrid.create_from_occupancy_grid(occ), None,
             ("vg_from_occ", box_cells, n_occ)),
            ("PointCloud.create_from_occupancy_grid 512^3", lambda _: G.PointCloud.create_from_occupancy_grid(occ), None,
             ("pc_from_occ", box_cells, n_occ))]
    rows = []
    for name, fn, prep, (op, n, m) in work:
        ts = timed(fn, prep)
        arg = prep() if prep else None
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(arg)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
                kernels[e.key[:60]] = kernels.get(e.key[:60], 0.0) + t
        kern_ms = float(sum(kernels.values()))
        nbytes = voxelgrid_bytes_model(op, n, m)
        rows.append({"workload": name, "n": n, "m": m, "call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)),
                     "kernel_ms_profiled": kernels, "kernel_ms_sum": kern_ms, "bytes_model": nbytes,
                     "share_of_3.35TBps_over_kernel_time": nbytes / (kern_ms * 1e-3) / HBM_BYTES_PER_S if kern_ms else None})
        del arg
    obj = {"op": "VoxelGrid operations: dense grids, carving, CheckIfIncluded and += on the config-3 cloud voxelised at "
                 "0.02, CreateFromOccupancyGrid on a 512^3 grid after a 1 M-point scan (%d occupied cells)" % n_occ,
           "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def tsdf_integrate_bytes(updated, planes, w, h, color_bytes):
    """least HBM traffic of one Integrate: each updated voxel reads and writes its 8-byte {tsdf, weight} pair and 8 bytes
    per colour plane; the depth image (4 bytes a pixel) and the colour image are read once.  A voxel that projects
    outside the image or behind the truncation touches no voxel memory, so it is not counted."""
    return updated * (16 + 8 * planes) + 4 * w * h + color_bytes * w * h


def tsdf(reps, out=None):
    """UniformTSDFVolume(2.0, res, 0.04) with res = 256 and 512 and each colour type: Integrate of one 640 x 480 frame of a
    sphere of radius 0.6 seen from 2.5 (repeated into the same volume), then ExtractPointCloud, ExtractVoxelPointCloud and
    a 640 x 480 Raycast after 8 views.  CUDA-event median and minimum of `reps` calls after a warm-up call (the Python
    call, with its synchronise), the kernel times of one further call from torch.profiler, and the Integrate bytes model
    over the kernel time against 3.35 TB/s."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G, I = cph.geometry, cph.integration
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times = []
        for r in range(reps + 1):
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
                k[e.key[:60]] = k.get(e.key[:60], 0.0) + t
        return k

    w, h = 640, 480
    cams = ring_cameras(8, w, h)
    rng = np.random.default_rng(2)
    frames = []
    for K, E in cams:
        d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
        frames.append((K, E, d16, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)))
    CT = I.TSDFVolumeColorType
    rows = []
    for res in (256, 512):
        for ct in (CT.NoColor, CT.RGB8, CT.Gray32):
            K, E, d16, col = frames[0]
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            im = G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, ct == CT.Gray32)
            vol = I.UniformTSDFVolume(2.0, res, 0.04, ct)
            vol.integrate(im, intr, E)
            updated = int(np.count_nonzero(vol.planes()[0].cpu()[:, 1]))
            ts = timed(lambda: vol.integrate(im, intr, E))
            k = kernels(lambda: vol.integrate(im, intr, E))
            kern = sum(v for n, v in k.items() if "integrate" in n)
            planes = {CT.NoColor: 0, CT.RGB8: 3, CT.Gray32: 1}[ct]
            nbytes = tsdf_integrate_bytes(updated, planes, w, h, {CT.NoColor: 0, CT.RGB8: 3, CT.Gray32: 4}[ct])
            rows.append({"op": "Integrate 640x480", "res": res, "color_type": ct.name, "updated_voxels": updated,
                         "call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)), "kernel_ms_profiled": k,
                         "integrate_kernel_ms": kern, "bytes_model": nbytes,
                         "share_of_3.35TBps_over_kernel_time": nbytes / (kern * 1e-3) / HBM_BYTES_PER_S if kern else None})
            del vol
        vol = I.UniformTSDFVolume(2.0, res, 0.04, CT.RGB8)
        for K, E, d16, col in frames:
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False), intr, E)
        K, E = frames[0][:2]
        intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        for name, fn, count in (("ExtractPointCloud", vol.extract_point_cloud, lambda r: len(r)),
                                ("ExtractVoxelPointCloud", vol.extract_voxel_point_cloud, lambda r: len(r)),
                                ("Raycast 640x480", lambda: vol.raycast(intr, E, 0.04), lambda r: len(r))):
            n_out = count(fn())
            ts = timed(fn)
            k = kernels(fn)
            rows.append({"op": name, "res": res, "color_type": "RGB8", "rows": n_out, "call_ms_median": float(np.median(ts)),
                         "call_ms_min": float(np.min(ts)), "kernel_ms_profiled": k, "kernel_ms_sum": float(sum(k.values()))})
        del vol
    obj = {"op": "UniformTSDFVolume(2.0, res, 0.04): 640x480 sphere frames (radius 0.6, cameras at 2.5); extractions and "
                 "Raycast after 8 views", "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def depth_cloud_bytes(w, h, stride, depth_bytes, color_bytes, rows, attrs):
    """least HBM traffic of one CreateFrom*Image call: each sampled pixel's depth (and colour) read once, `attrs` float3
    attributes written per output row.  The structured normal's neighbour reads are not counted (they hit cache
    lines the row above and below already bring in)."""
    samples = (w // stride) * (h // stride)
    return samples * (depth_bytes + color_bytes) + 12 * attrs * rows


def depth_cloud(reps, out=None):
    """PointCloud.create_from_rgbd_image (RGB8 colour, without and with structured normals, valid rows only and every row)
    and create_from_depth_image (uint16, strides 1 and 4) at 640 x 480 and 1280 x 720: a sphere of radius 0.6 seen from
    2.5 over a wall, 10 % of the pixels holes.  CUDA-event median and minimum of `reps` Python calls after a warm-up
    call, the kernel times of one further call from torch.profiler, and the bytes model over the kernel time against
    3.35 TB/s."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G = cph.geometry
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times = []
        for r in range(reps + 1):
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
                k[e.key[:60]] = k.get(e.key[:60], 0.0) + t
        return k

    rows = []
    rng = np.random.default_rng(4)
    for w, h in ((640, 480), (1280, 720)):
        K, E = ring_cameras(8, w, h)[0]
        d = sphere_depth(K, E, w, h, 0.6)
        d = np.where(d > 0, d, 3.5).astype(np.float32)  # the wall behind the sphere
        d[rng.random(d.shape) < 0.1] = 0
        d16 = np.round(d * 1000).astype(np.uint16)
        col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
        im = G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 4.0, False)
        cases = [("CreateFromRGBDImage", 1, valid, normals, lambda v=valid, n=normals: G.PointCloud.create_from_rgbd_image(im, intr, E, v, -1.0, n))
                 for valid, normals in ((True, False), (True, True), (False, False))]
        depth_img = G.Image(d16)
        cases += [("CreateFromDepthImage uint16", s, True, False,
                   lambda s=s: G.PointCloud.create_from_depth_image(depth_img, intr, E, 1000.0, 4.0, s)) for s in (1, 4)]
        for name, stride, valid, normals, fn in cases:
            n_out = len(fn())
            ts = timed(fn)
            k = kernels(fn)
            kern = sum(v for kn, v in k.items() if "dc_" in kn)
            rgbd = name == "CreateFromRGBDImage"
            nbytes = depth_cloud_bytes(w, h, stride, 4 if rgbd else 2, 3 if rgbd else 0, n_out, 1 + rgbd + normals)
            rows.append({"op": name, "width": w, "height": h, "stride": stride, "project_valid_depth_only": valid,
                         "compute_normals": normals, "rows": n_out, "call_ms_median": float(np.median(ts)),
                         "call_ms_min": float(np.min(ts)), "kernel_ms_profiled": k, "depth_cloud_kernel_ms": kern,
                         "bytes_model": nbytes,
                         "share_of_3.35TBps_over_kernel_time": nbytes / (kern * 1e-3) / HBM_BYTES_PER_S if kern else None})
    obj = {"op": "PointCloud from depth / RGB-D frames: a sphere (radius 0.6, camera at 2.5) over a wall at 3.5 m, 10 % holes",
           "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def tsdf_mesh_bytes(n_voxels, nv, nt, colour_planes):
    """least HBM traffic of one ExtractTriangleMesh: the {tsdf, weight} plane read once (8 bytes a voxel), plus the
    outputs written once: 12 bytes a vertex, 12 a vertex colour when the volume has colour, 12 a triangle.  The colour
    planes are read only at the vertices' voxels, which is not counted; nor is the scratch (cube bytes, edge masks,
    positions)."""
    return 8 * n_voxels + 12 * nv * (2 if colour_planes else 1) + 12 * nt


def tsdf_mesh(reps, out=None):
    """UniformTSDFVolume(2.0, res, 0.04, RGB8) with res = 256 and 512 after the 8 ring-camera 640 x 480 views of a sphere
    of radius 0.6 (tests/test_gpu_tsdf.py's scene): extract_triangle_mesh (the sizing call and the writing call, as the
    Python front end makes them) and compute_vertex_normals of its mesh.  CUDA-event median and minimum of `reps` calls
    after a warm-up call, the kernel times of one further call from torch.profiler, and the bytes model of
    tsdf_mesh_bytes over the extraction's kernel time against 3.35 TB/s."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G, I = cph.geometry, cph.integration
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times = []
        for r in range(reps + 1):
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            if r:
                times.append(ms.value)
        return times

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) * 1e-3
            if t > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
                k[e.key[:60]] = k.get(e.key[:60], 0.0) + t
        return k

    w, h = 640, 480
    rng = np.random.default_rng(2)
    rows = []
    for res in (256, 512):
        vol = I.UniformTSDFVolume(2.0, res, 0.04, I.TSDFVolumeColorType.RGB8)
        for K, E in ring_cameras(8, w, h):
            d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False), intr, E)
        mesh = vol.extract_triangle_mesh()
        nv, nt = len(mesh.vertices), len(mesh.triangles)
        ts = timed(vol.extract_triangle_mesh)
        k = kernels(vol.extract_triangle_mesh)
        kern = float(sum(k.values()))
        nbytes = tsdf_mesh_bytes(res ** 3, nv, nt, 3)
        rows.append({"op": "ExtractTriangleMesh (sizing + writing call)", "res": res, "color_type": "RGB8", "vertices": nv,
                     "triangles": nt, "call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)),
                     "kernel_ms_profiled": k, "kernel_ms_sum": kern, "bytes_model": nbytes,
                     "share_of_3.35TBps_over_kernel_time": nbytes / (kern * 1e-3) / HBM_BYTES_PER_S if kern else None})

        def normals():
            mesh.triangle_normals = None
            mesh.compute_vertex_normals()
        ts = timed(normals)
        k = kernels(normals)
        rows.append({"op": "ComputeVertexNormals (triangle normals first)", "res": res, "vertices": nv, "triangles": nt,
                     "call_ms_median": float(np.median(ts)), "call_ms_min": float(np.min(ts)), "kernel_ms_profiled": k,
                     "kernel_ms_sum": float(sum(k.values()))})
        del mesh, vol
    obj = {"op": "UniformTSDFVolume(2.0, res, 0.04, RGB8) after 8 640x480 ring-camera views of a sphere (radius 0.6, cameras "
                 "at 2.5): ExtractTriangleMesh and ComputeVertexNormals", "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")



def mesh_pass_bytes(nv, ne, n_attrs, weighted):
    """least HBM traffic of one filter pass: the row starts (4 bytes a vertex) and the edge list's neighbour column
    (4 bytes an edge, the pairs' 8 bytes as the edges are read whole) once, the weights (4 an edge) and the weight totals
    (4 a vertex) when weighted, and per filtered attribute the previous values read once and the new ones written once
    (12 + 12 bytes a vertex).  Neighbour values are counted once: each vertex is everybody's neighbour a few times, which
    the caches absorb."""
    return 4 * (nv + 1) + 8 * ne + (4 * ne + 4 * nv if weighted else 0) + 24 * nv * n_attrs


def mesh_ops(reps, out=None):
    """TriangleMesh operations on the --tsdf-mesh scene's meshes (UniformTSDFVolume(2.0, res, 0.04, RGB8), res = 256 and
    512, 8 ring-camera 640 x 480 sphere views) with vertex normals and colours: compute_edge_list; each filter at 1 and
    100 iterations over all three attributes; get_surface_area; sample_points_uniformly at 1 M and 10 M points.
    CUDA-event median and minimum of `reps` calls after a warm-up call, the engine launches of one call, and for the
    100-iteration filters the per-pass time ((t100 - t1) / 99 passes, / 198 for Taubin) against the bytes bound of
    mesh_pass_bytes at 3.35 TB/s."""
    import subprocess
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G, I = cph.geometry, cph.integration
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times, launches = [], 0
        for r in range(reps + 1):
            n0 = L.cphb_launch_count()
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            launches = L.cphb_launch_count() - n0
            if r:
                times.append(ms.value)
        return {"call_ms_median": float(np.median(times)), "call_ms_min": float(np.min(times)), "launches": int(launches)}

    w, h = 640, 480
    rng = np.random.default_rng(2)
    rows = []
    for res in (256, 512):
        vol = I.UniformTSDFVolume(2.0, res, 0.04, I.TSDFVolumeColorType.RGB8)
        for K, E in ring_cameras(8, w, h):
            d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False), intr, E)
        mesh = vol.extract_triangle_mesh()
        del vol
        mesh.compute_vertex_normals()
        nv, nt = len(mesh.vertices), len(mesh.triangles)
        base = {"res": res, "vertices": nv, "triangles": nt}
        rows.append(dict(base, op="compute_edge_list", **timed(mesh.compute_edge_list)))
        ne = len(mesh.edge_list)
        rows[-1]["edges"] = ne
        for name, fn, per_it, weighted in (
                ("filter_sharpen", lambda it: mesh.filter_sharpen(it, 0.01), 1, False),
                ("filter_smooth_simple", lambda it: mesh.filter_smooth_simple(it), 1, False),
                ("filter_smooth_laplacian", lambda it: mesh.filter_smooth_laplacian(it, 0.5), 1, True),
                ("filter_smooth_taubin", lambda it: mesh.filter_smooth_taubin(it, 0.5, -0.53), 2, True)):
            t1 = timed(lambda: fn(1))
            t100 = timed(lambda: fn(100))
            rows.append(dict(base, op=name, iterations=1, **t1))
            per_pass = (t100["call_ms_median"] - t1["call_ms_median"]) / (99 * per_it)
            nbytes = mesh_pass_bytes(nv, ne, 3, weighted)
            rows.append(dict(base, op=name, iterations=100, **t100, pass_ms=per_pass, pass_bytes_bound=nbytes,
                             pass_share_of_3_35TBps_bytes_bound=nbytes / (per_pass * 1e-3) / HBM_BYTES_PER_S if per_pass > 0 else None))
        rows.append(dict(base, op="get_surface_area", **timed(mesh.get_surface_area)))
        for n in (1_000_000, 10_000_000):
            rows.append(dict(base, op="sample_points_uniformly", points=n, **timed(lambda: mesh.sample_points_uniformly(n))))
        del mesh
    obj = {"op": "TriangleMesh edge list, filters, surface area and uniform sampling on the ExtractTriangleMesh meshes of "
                 "UniformTSDFVolume(2.0, res, 0.04, RGB8) after 8 640x480 ring-camera sphere views, with vertex normals and "
                 "colours", "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def mesh_voxel_bytes(nv, nt, voxels):
    """the compulsory bytes of one cphb_voxel_grid_from_triangle_mesh call, from shapes: the mesh read once (12 B a vertex,
    12 B a triangle) and the keys and colours written (24 B a voxel).  The walk is bound by the exact test's arithmetic
    and the sort, not by these bytes, so their share of 3.35 TB/s says how far the call is from a pure copy."""
    return 12 * nv + 12 * nt + 24 * voxels


def mesh_voxel(reps, out=None):
    """VoxelGrid.create_from_triangle_mesh_within_bounds on: the --mesh-ops sphere meshes (UniformTSDFVolume(2.0, res,
    0.04, RGB8), res 256 and 512, 8 ring-camera 640 x 480 views) at 1x and 2x their voxel size 2 / res over their
    bounds widened by half a voxel; a tilted two-triangle plane over a 512^2 x 10 grid; an icosahedron of radius 200
    in a 512^3 grid.  The sizing call (capacity 0) and the writing call are timed apart with CUDA events (median and
    minimum of `reps` after a warm-up), with the engine launches of each; then one profiled pair per workload gives each
    kernel's device time (torch.profiler).  mesh_voxel_bytes has the bytes model."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G, I = cph.geometry, cph.integration
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times, launches = [], 0
        for r in range(reps + 1):
            n0 = L.cphb_launch_count()
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            launches = L.cphb_launch_count() - n0
            if r:
                times.append(ms.value)
        return {"ms_median": float(np.median(times)), "ms_min": float(np.min(times)), "launches": int(launches)}

    workloads = []
    w, h = 640, 480
    rng = np.random.default_rng(2)
    for res in (256, 512):
        vol = I.UniformTSDFVolume(2.0, res, 0.04, I.TSDFVolumeColorType.RGB8)
        for K, E in ring_cameras(8, w, h):
            d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False), intr, E)
        mesh = vol.extract_triangle_mesh()
        del vol
        mn, mx = mesh.get_min_bound(), mesh.get_max_bound()
        for f in (1, 2):
            vs = np.float32(2.0 * f / res)
            hv = vs * np.float32(0.5)
            workloads.append(("sphere_res%d_x%d" % (res, f), mesh, float(vs), mn - hv, mx + hv))
    plane = G.TriangleMesh(np.array([[0.1, 0.1, 3.2], [511.9, 0.1, 4.9], [0.1, 511.9, 3.7], [511.9, 511.9, 5.3]], np.float32),
                           np.array([[0, 1, 2], [1, 3, 2]], np.int32))
    workloads.append(("plane_512x512", plane, 1.0, np.zeros(3, np.float32), np.float32([512, 512, 10])))
    p = (1 + 5 ** 0.5) / 2
    iv = np.array([[-1, p, 0], [1, p, 0], [-1, -p, 0], [1, -p, 0], [0, -1, p], [0, 1, p], [0, -1, -p], [0, 1, -p], [p, 0, -1],
                   [p, 0, 1], [-p, 0, -1], [-p, 0, 1]])
    iv = (iv / np.linalg.norm(iv[0]) * 200.0 + [256.3, 255.7, 256.1]).astype(np.float32)
    it = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
                   [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7],
                   [9, 8, 1]], np.int32)
    workloads.append(("icosahedron_r200_in_512", G.TriangleMesh(iv, it), 1.0, np.zeros(3, np.float32), np.float32([512] * 3)))

    rows = []
    for name, mesh, vs, lo, hi in workloads:
        nv, nt = len(mesh.vertices), len(mesh.triangles)
        f3 = lambda a: (C.c_float * 3)(*[float(x) for x in a])
        args = (mesh.vertices.ptr, nv, mesh.triangles.ptr, nt, vs, f3(lo), f3(hi))
        n = C.c_size_t(0)
        _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, None, None, 0, C.byref(n), None))
        m = n.value
        keys, cols = cph.utility.DeviceArray((max(m, 1), 3), np.int32), cph.utility.DeviceArray((max(m, 1), 3), np.float32)
        sizing = timed(lambda: _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, None, None, 0, C.byref(n), None)))
        writing = timed(lambda: _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, keys.ptr, cols.ptr, m, C.byref(n), None)))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, None, None, 0, C.byref(n), None))
            _lib.check(L.cphb_voxel_grid_from_triangle_mesh(*args, keys.ptr, cols.ptr, m, C.byref(n), None))
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                kernels[e.key[:80]] = {"calls": int(e.count), "us_total": float(t)}
        cnt = [int(round((float(hi[a]) - float(lo[a])) / vs)) for a in range(3)]
        bits = sum(max(1, int(np.ceil(np.log2(max(c, 2))))) for c in cnt)
        nbytes = mesh_voxel_bytes(nv, nt, m)
        row = {"workload": name, "vertices": nv, "triangles": nt, "voxel_size": vs, "grid": cnt, "voxels": m, "sizing_call": sizing,
               "writing_call": writing, "both_calls_ms_median": sizing["ms_median"] + writing["ms_median"],
               "compulsory_bytes": nbytes, "writing_call_share_of_3_35TBps": nbytes / (writing["ms_median"] * 1e-3) / HBM_BYTES_PER_S,
               "kernels_us_both_calls": kernels, "sort_passes": (bits + 7) // 8}
        rows.append(row)
        print(json.dumps({k: row[k] for k in ("workload", "triangles", "voxels", "both_calls_ms_median")}), flush=True)
    obj = {"op": "VoxelGrid.create_from_triangle_mesh_within_bounds (C entry point, sizing call then writing call)",
           "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def mesh_clean(reps, out=None):
    """TriangleMesh cleanup and GetSelfIntersectingTriangles (C entry points) on the --mesh-ops sphere meshes
    (UniformTSDFVolume(2.0, res, 0.04, RGB8), res 256 and 512, 8 ring-camera 640 x 480 views): each Remove* on the welded
    mesh and on its un-welded soup (every triangle its own three vertices), and the self-intersection search on the
    welded mesh, on the += union with a copy shifted by (0.3, 0.1, 0) and on the soup.  CUDA-event median and minimum of
    `reps` after a warm-up, with the engine launches; the search's sizing and writing calls apart, with its candidate
    pairs and hits; then one profiled call of each for per-kernel device times (torch.profiler)."""
    import subprocess
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing.datagen import ring_cameras, sphere_depth
    L = _lib.lib()
    G, I = cph.geometry, cph.integration
    DA = cph.utility.DeviceArray
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ev = [L.cphb_event_create() for _ in range(2)]

    def timed(fn):
        times, launches = [], 0
        for r in range(reps + 1):
            n0 = L.cphb_launch_count()
            L.cphb_event_record(ev[0], None)
            fn()
            L.cphb_event_record(ev[1], None)
            ms = C.c_float(0)
            _lib.check(L.cphb_event_elapsed_ms(ev[0], ev[1], C.byref(ms)))
            launches = L.cphb_launch_count() - n0
            if r:
                times.append(ms.value)
        return {"ms_median": float(np.median(times)), "ms_min": float(np.min(times)), "launches": int(launches)}

    def kernels(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                k[e.key[:80]] = {"calls": int(e.count), "us_total": float(t)}
        return k

    meshes = []
    w, h = 640, 480
    rng = np.random.default_rng(2)
    for res in (256, 512):
        vol = I.UniformTSDFVolume(2.0, res, 0.04, I.TSDFVolumeColorType.RGB8)
        for K, E in ring_cameras(8, w, h):
            d16 = np.round(sphere_depth(K, E, w, h, 0.6) * 1000).astype(np.uint16)
            intr = cph.camera.PinholeCameraIntrinsic(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            vol.integrate(G.RGBDImage.create_from_color_and_depth(G.Image(col), G.Image(d16), 1000.0, 100.0, False), intr, E)
        mesh = vol.extract_triangle_mesh()
        del vol
        v, t = mesh.vertices.cpu(), mesh.triangles.cpu()
        soup = G.TriangleMesh(v[t.reshape(-1)], np.arange(3 * len(t), dtype=np.int32).reshape(-1, 3))
        union = mesh + G.TriangleMesh(v + np.float32([0.3, 0.1, 0.0]), t)
        meshes.append((res, mesh, soup, union))

    rows = []
    for res, mesh, soup, union in meshes:
        for kind, m in (("welded", mesh), ("soup", soup)):
            nv, nt = len(m.vertices), len(m.triangles)
            ov, ot, otn = DA((nv, 3), np.float32), DA((nt, 3), np.int32), DA((nt, 3), np.float32)
            k = C.c_size_t(0)
            vargs = (m.vertices.ptr, None, None, nv, m.triangles.ptr, nt, ov.ptr, None, None, ot.ptr, C.byref(k), None)
            targs = (m.triangles.ptr, None, nt, nv, ot.ptr, None, C.byref(k), None)
            for op, fn, a in (("remove_duplicated_vertices", L.cphb_mesh_remove_duplicated_vertices, vargs),
                              ("remove_unreferenced_vertices", L.cphb_mesh_remove_unreferenced_vertices, vargs),
                              ("remove_duplicated_triangles", L.cphb_mesh_remove_duplicated_triangles, targs),
                              ("remove_degenerate_triangles", L.cphb_mesh_remove_degenerate_triangles, targs)):
                call = lambda fn=fn, a=a: _lib.check(fn(*a))
                row = {"workload": "sphere_res%d_%s" % (res, kind), "op": op, "vertices": nv, "triangles": nt, "call": timed(call)}
                row["kept"] = int(k.value)
                row["kernels_us"] = kernels(call)
                rows.append(row)
                print(json.dumps({x: row[x] for x in ("workload", "op", "kept")} | {"ms": row["call"]["ms_median"]}), flush=True)
        for kind, m in (("welded", mesh), ("union", union), ("soup", soup)):
            nv, nt = len(m.vertices), len(m.triangles)
            n, cand = C.c_size_t(0), C.c_size_t(0)
            args = (m.vertices.ptr, nv, m.triangles.ptr, nt)
            _lib.check(L.cphb_mesh_self_intersecting_triangles(*args, None, 0, C.byref(n), C.byref(cand), None))
            hits = n.value
            pairs = DA((max(hits, 1), 2), np.int32)
            sizing = lambda: _lib.check(L.cphb_mesh_self_intersecting_triangles(*args, None, 0, C.byref(n), C.byref(cand), None))
            writing = lambda: _lib.check(L.cphb_mesh_self_intersecting_triangles(*args, pairs.ptr, hits, C.byref(n), C.byref(cand), None))
            row = {"workload": "sphere_res%d_%s" % (res, kind), "op": "get_self_intersecting_triangles", "vertices": nv, "triangles": nt,
                   "hits": hits, "n_candidates": int(cand.value), "sizing_call": timed(sizing), "writing_call": timed(writing),
                   "kernels_us_writing_call": kernels(writing)}
            row["both_calls_ms_median"] = row["sizing_call"]["ms_median"] + row["writing_call"]["ms_median"]
            rows.append(row)
            print(json.dumps({x: row[x] for x in ("workload", "triangles", "hits", "n_candidates", "both_calls_ms_median")}), flush=True)
    obj = {"op": "TriangleMesh Remove* and GetSelfIntersectingTriangles (C entry points)", "gpu": gpu, "reps": reps, "rows": rows}
    line = json.dumps(obj)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")

if __name__ == "__main__":
    main()
