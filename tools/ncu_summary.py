#!/usr/bin/env python3
"""Summarise an .ncu-rep into a small markdown file for profiles/.
usage: tools/ncu_summary.py prof.ncu-rep profiles/name.md "title / command line"
"""
import csv
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"), ("launch__block_size", "block"), ("launch__registers_per_thread", "regs/thread"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM write"),
    ("lts__t_bytes.sum", "L2 bytes"), ("lts__t_sector_hit_rate.pct", "L2 hit rate"),
    ("l1tex__t_sector_hit_rate.pct", "L1 hit rate"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "active threads / instruction"),
    ("sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", "fp64 pipe"),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "xu pipe"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu pipe"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu pipe"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma pipe"),
]


def run(args):
    return subprocess.run(["ncu"] + args, capture_output=True, text=True).stdout


def main():
    rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else ""
    raw = list(csv.reader(run(["-i", rep, "--page", "raw", "--csv"]).splitlines()))
    hdr, units = raw[0], raw[1]
    lines = ["# " + title, "", "source: `%s` (ncu --set full --clock-control none --import-source on)" % rep, ""]
    for r in raw[2:]:
        d = dict(zip(hdr, r))
        lines += ["## " + d.get("Kernel Name", "?"), "", "| metric | value |", "|---|---|"]
        for k, label in KEYS:
            if k in d and d[k] != "":
                lines.append("| %s (`%s`) | %s %s |" % (label, k, d[k], units[hdr.index(k)]))
        stalls = []
        for k in hdr:
            if "issue_stalled" in k and k.endswith("_per_warp_active.pct"):
                try:
                    stalls.append((float(d[k]), k.split("issue_stalled_")[1].replace("_per_warp_active.pct", "")))
                except ValueError:
                    pass
        stalls.sort(reverse=True)
        if stalls:
            lines += ["", "warp stall reasons (% of active warps, top 6): " +
                      ", ".join("%s %.1f" % (n, v) for v, n in stalls[:6])]
        lines.append("")
    src = list(csv.reader(run(["-i", rep, "--page", "source", "--csv", "--print-source", "sass"]).splitlines()))
    hi = [i for i, r in enumerate(src) if r and r[0] == "Address"]
    if hi:
        h = src[hi[0]]
        end = hi[1] - 1 if len(hi) > 1 else len(src)
        data = [r for r in src[hi[0] + 1:end] if len(r) > 5]
        ci, ie = h.index("Warp Stall Sampling (All Samples)"), h.index("Instructions Executed")
        tot = sum(int(r[ci]) for r in data if r[ci].isdigit())
        tote = sum(int(r[ie]) for r in data if r[ie].isdigit())
        lines += ["## hottest SASS (first kernel instance): stall samples / executions", "",
                  "total samples %d, total warp instructions %d" % (tot, tote), "", "```"]
        for r in sorted(data, key=lambda r: -int(r[ci]) if r[ci].isdigit() else 0)[:14]:
            lines.append("%7s %10s  %s" % (r[ci], r[ie], r[1].strip()[:90]))
        lines.append("--- TMA / mbarrier instructions (executions) ---")
        for r in data:
            if any(t in r[1] for t in ("UBLKCP", "SYNCS.", "CREDUX")):
                lines.append("%7s %10s  %s" % (r[ci], r[ie], r[1].strip()[:90]))
        lines.append("```")
    open(out, "w").write("\n".join(lines) + "\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
