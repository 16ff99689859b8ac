"""Per-kernel breakdown of ONE registration from an ncu launch list (gpu__time_duration.sum CSV).
usage: python tools/launch_breakdown.py launches.csv [iteration_kernel_launches_per_registration]"""
import csv
import sys
from collections import OrderedDict


def main():
    path = sys.argv[1]
    n_it = int(sys.argv[2]) if len(sys.argv) > 2 else 62  # 31 iterations x 2 instances (searching / certified+sum)
    lines = [l for l in open(path) if not l.startswith("==")]
    rows = [(r["Kernel Name"].split("(")[0].replace("void ", "")[:48], float(r["Metric Value"].replace(",", "")) / 1000)
            for r in csv.DictReader(lines) if r.get("Metric Name") == "gpu__time_duration.sum"]
    idx = [i for i, r in enumerate(rows) if "icp_iteration" in r[0]]
    runs, cur = [], [idx[0]]
    for a, b in zip(idx, idx[1:]):
        if b - a > 20:
            runs.append(cur)
            cur = [b]
        else:
            cur.append(b)
    runs.append(cur)
    full = [r for r in runs if len(r) == n_it]
    last = full[-1]
    # a registration starts at the bounds_init kernel of the target index build before its first iteration
    s = last[0]
    while s > 0 and "bounds_init" not in rows[s][0]:
        s -= 1
    s0 = s - 1
    while s0 > 0 and "bounds_init" not in rows[s0][0]:
        s0 -= 1
    e = last[-1] + 2
    while e < len(rows) and "compact" in rows[e][0]:
        e += 1
    seg = rows[s0:e]
    print("searching instance, us per launch:       ", [round(rows[i][1], 1) for i in last if rows[i][0].rstrip().endswith(", 0>")])
    print("certified / sum+solve instance, us per launch:", [round(rows[i][1], 1) for i in last if rows[i][0].rstrip().endswith(", 1>")])
    agg = OrderedDict()
    for n, t in seg:
        k = agg.setdefault(n, [0, 0.0])
        k[0] += 1
        k[1] += t
    tot = sum(t for _, t in seg)
    print("one registration: %d launches, %.1f us summed kernel time" % (len(seg), tot))
    for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("  %-50s x%-3d %8.1f us  %5.1f%%" % (n, c, t, 100 * t / tot))


if __name__ == "__main__":
    main()
