#!/usr/bin/env python
"""Summarise ncu outputs into small text files.
  python tools/ncu_summary.py launches gpurun_out/launches.csv            -> per-kernel count / total / share
  python tools/ncu_summary.py full gpurun_out/prof.ncu-rep                -> key counters per captured kernel (needs ncu here)
"""
import csv
import io
import re
import subprocess
import sys
from collections import OrderedDict, defaultdict


def short(name):
    m = re.match(r"(?:void )?(?:\w+::)*(\w+)", name)
    return m.group(1) if m else name


def launches(path):
    rows = [r for r in csv.reader(l for l in open(path, errors="ignore") if l.startswith('"'))]
    hdr = rows[0]
    ik, im, iv = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value")
    iu = hdr.index("Metric Unit")
    tot, cnt = defaultdict(float), defaultdict(int)
    for r in rows[1:]:
        if r[im] != "gpu__time_duration.sum":
            continue
        v = float(r[iv].replace(",", ""))
        u = r[iu]
        v_us = v / 1e3 if u in ("ns", "nsecond") else (v if u in ("us", "usecond") else v * 1e3 if u in ("ms", "msecond") else v)
        tot[short(r[ik])] += v_us
        cnt[short(r[ik])] += 1
    total = sum(tot.values())
    print(f"{'kernel':26s} {'launches':>8s} {'total_us':>12s} {'avg_us':>10s} {'share':>7s}")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"{k:26s} {cnt[k]:8d} {v:12.1f} {v / cnt[k]:10.2f} {100 * v / total:6.1f}%")
    print(f"{'TOTAL':26s} {sum(cnt.values()):8d} {total:12.1f}")


KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "smsp__cycles_active.avg", "sm__cycles_elapsed.avg.per_second", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "sm__inst_executed_pipe_fp64.sum", "smsp__inst_executed.sum"]


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr = rows[0]
    ik = hdr.index("Kernel Name")
    cols = OrderedDict((k, hdr.index(k)) for k in KEYS if k in hdr)
    units = rows[1]
    for r in rows[2:]:
        print(f"== {short(r[ik])}  (id {r[0]})")
        for k, i in cols.items():
            print(f"   {k:90s} {r[i]:>18s} {units[i]}")


if __name__ == "__main__":
    (launches if sys.argv[1] == "launches" else full)(sys.argv[2])
