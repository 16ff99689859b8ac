#!/usr/bin/env python3
"""Per-launch profile of one config-2 registration (point-to-plane ICP, 1 M -> 1 M, 30 forced iterations).

    python tools/icp_launch_profile.py --out FILE [--label TEXT] [--points N] [--runs R]

Three child processes, each warmed up with one registration before the one it reports:
  events   CPHB_DEBUG_EVENTS=1: CUDA events before, between and after the two kernel instances of every launch
           (plain stream-ordered launches: programmatic dependent launch is off in this run)
  cert     CPHB_DEBUG_CERT=1: certified lanes, skipped tiles and tiles searched in line per launch, and the globaltimer
           timeline of launch 20 (tile loops, last block, grid sum, state read, solve, compose, finalize)
  plain    no hook: loop_ms of R registrations with programmatic dependent launch on, as bench.py times them
The card's name, power limit and maximum SM clock are read in the same run.  The section is APPENDED to FILE, so a
before / after pair lives in one file.
"""
import argparse
import os
import re
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(points, runs):
    sys.path.insert(0, ROOT)
    import numpy as np
    import cupoch_b200 as cph
    from cupoch_b200 import _lib
    from cupoch_b200.testing import datagen
    _lib.require_gpu()
    R = cph.registration
    tgt, tn = datagen.surface(points, 11)  # bench.py's make_workload
    src = datagen.make_source(tgt, datagen.gt_transform(), 13, 14, 5e-4)
    s, t = cph.geometry.PointCloud(src), cph.geometry.PointCloud(tgt)
    t.normals = tn
    est, crit = R.TransformationEstimationPointToPlane(), R.ICPConvergenceCriteria(0, 0, 30)
    init = np.eye(4, dtype=np.float32)
    R.registration_icp(s, t, 0.02, init, est, crit)  # warm-up (module load, pool)
    for _ in range(runs):
        r = R.registration_icp(s, t, 0.02, init, est, crit)
        print("loop_ms %.4f launches %d fitness %.6f" % (r.loop_ms, r.loop_launches, r.fitness), flush=True)


def run_child(env_extra, points, runs):
    env = dict(os.environ, **env_extra)
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--points", str(points), "--runs", str(runs)],
                       env=env, capture_output=True, text=True, cwd=ROOT)
    if p.returncode != 0:
        raise SystemExit("child failed (%s):\n%s\n%s" % (env_extra, p.stdout, p.stderr))
    return p.stdout, p.stderr


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader",
                            "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or q.stderr.strip()
    except Exception as e:  # the figures below are still device times; the card is then unknown
        return "unknown (%s)" % e


def med(v):
    return statistics.median(v) if v else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--label", default="")
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        child(a.points, a.runs)
        return
    if not a.out:
        ap.error("--out is required")

    _, ev_err = run_child({"CPHB_DEBUG_EVENTS": "1"}, a.points, 1)
    _, cert_err = run_child({"CPHB_DEBUG_CERT": "1"}, a.points, 1)
    plain_out, _ = run_child({}, a.points, a.runs)

    # the reported registration is the last one each child printed
    ev_line = [l for l in ev_err.splitlines() if re.match(r"^\s*\d+:[\d.]+/", l)][-1]
    launches = [tuple(float(x) for x in m.groups()) for m in re.finditer(r"(\d+):([\d.]+)/([\d.]+)/([\d.]+)", ev_line)]
    cert_line = [l for l in cert_err.splitlines() if re.match(r"^\s*\d+\*?:\d+/\d+", l)][-1]
    certified = {int(m.group(1)) for m in re.finditer(r"(\d+)\*:", cert_line)}
    timeline = [l.strip() for l in cert_err.splitlines() if "launch 20" in l][-2:]
    loops = [float(m.group(1)) for m in re.finditer(r"loop_ms ([\d.]+)", plain_out)]

    cert_r0 = [r0 for i, r0, r1, g in launches if int(i) in certified]
    cert_r1 = [r1 for i, r0, r1, g in launches if int(i) in certified]
    cert_gap = [g for i, r0, r1, g in launches if int(i) in certified and int(i) < len(launches) - 1]
    srch_r0 = [r0 for i, r0, r1, g in launches if int(i) not in certified]
    srch_r1 = [r1 for i, r0, r1, g in launches if int(i) not in certified]

    L = []
    L.append("=" * 100)
    L.append("icp_launch_profile %s  (%s)" % (a.label, time.strftime("%Y-%m-%d %H:%M:%S")))
    L.append("card (name, power limit, max SM clock, driver): %s" % card())
    L.append("workload: config 2, point-to-plane ICP %d -> %d points, r = 0.02, 30 forced iterations = 31 launches" % (a.points, a.points))
    L.append("")
    L.append("[plain] loop_ms of %d registrations (programmatic dependent launch on, as bench.py): %s" % (len(loops), " ".join("%.3f" % x for x in loops)))
    L.append("        median %.3f ms = %.1f us per launch (both instances)" % (med(loops), 1e3 * med(loops) / 31))
    L.append("")
    L.append("[events] per launch, us: ROLE 0 instance / ROLE 1 instance / gap to the next launch (plain launches, no PDL)")
    L.append("        " + " ".join("%d%s:%.1f/%.1f/%.1f" % (int(i), "*" if int(i) in certified else "", r0, r1, g) for i, r0, r1, g in launches))
    L.append("        certified launches (%d): ROLE 0 median %.1f us, ROLE 1 median %.1f us (min %.1f, max %.1f), gap median %.1f us"
             % (len(cert_r1), med(cert_r0), med(cert_r1), min(cert_r1, default=float("nan")), max(cert_r1, default=float("nan")), med(cert_gap)))
    L.append("        searching launches (%d): ROLE 0 median %.1f us (sum %.1f), ROLE 1 (sum + solve) median %.1f us"
             % (len(srch_r0), med(srch_r0), sum(srch_r0), med(srch_r1)))
    L.append("")
    L.append("[cert] launch: certified lanes / skipped tiles [/ tiles searched in line, * = certified regime]")
    L.append("        " + cert_line.strip())
    for l in timeline:
        L.append("        " + l)
    L.append("")
    text = "\n".join(L) + "\n"
    sys.stdout.write(text)
    with open(a.out, "a") as f:
        f.write(text)


if __name__ == "__main__":
    main()
