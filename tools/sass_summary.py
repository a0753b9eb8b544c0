#!/usr/bin/env python
"""Static SASS evidence: per-kernel counts of the mnemonics that show which hardware paths libvxs.so uses
(DMMA16 = mma.sync.m16n8k{4,8,16}.f64, DMMA8 = mma.sync.m8n8k4.f64, UBLKCP = cp.async.bulk, SYNCS = mbarrier, LDGSTS = cp.async, RED/ATOM .F64).  No GPU needed:
    python tools/sass_summary.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "voxel_slam_b200", "lib", "libvxs.so")
PAT = {"DMMA16": r"\bDMMA\.16x8x", "DMMA8": r"\bDMMA\.8x8x4", "UBLKCP": r"UBLKCP", "SYNCS": r"\bSYNCS", "LDGSTS": r"LDGSTS", "RED.F64": r"(RED|REDG|ATOM|ATOMG)\.E\.ADD\.F64", "BAR": r"\bBAR\.", "DFMA": r"\bDFMA",
       "LDG": r"\bLDG", "STG": r"\bSTG", "LDS": r"\bLDS", "STS": r"\bSTS"}


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    cur, arch = None, set()
    size, cnt = collections.Counter(), collections.defaultdict(collections.Counter)
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"arch = (\S+)", line)
        if m:
            arch.add(m.group(1))
        if cur is None or not re.search(r"^\s+/\*[0-9a-f]{4,6}\*/", line):
            continue
        size[cur] += 1
        for k, p in PAT.items():
            if re.search(p, line):
                cnt[cur][k] += 1
    names = list(size)
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    rows = []
    for mangled, d in zip(names, dem):
        d = d.replace("(anonymous namespace)::", "")
        d = re.sub(r"^void ", "", d)
        d = re.sub(r"\((?!.*\().*$", "", d) if d.count("(") == 1 else re.sub(r"\(.*$", "", d)
        rows.append((d, size[mangled], cnt[mangled]))
    rows.sort(key=lambda r: -r[1])
    keys = list(PAT)
    print(f"SASS mnemonic counts per kernel of voxel_slam_b200/lib/libvxs.so (cuobjdump -sass; cubin arch {sorted(arch)}; STATIC instruction counts, not executed counts)")
    print("produced by tools/sass_summary.py.  DMMA16 = mma.sync.m16n8k{4,8,16}.f64 (Hopper fp64 tensor shapes), DMMA8 = mma.sync.m8n8k4.f64 (Ampere shape),\n"
          "UBLKCP = cp.async.bulk (1-D TMA), SYNCS = mbarrier ops, LDGSTS = cp.async,")
    print("RED.F64 = fp64 reduction atomics.\n")
    print("%-44s %7s " % ("kernel", "instrs") + " ".join("%7s" % k for k in keys))
    tot = collections.Counter()
    for d, n, c in rows:
        tot.update(c)
        print("%-44s %7d " % (d[:44], n) + " ".join("%7d" % c[k] for k in keys))
    print("\n%-44s %7d " % ("total (%d kernels)" % len(rows), sum(size.values())) + " ".join("%7d" % tot[k] for k in keys))
    # ---- registers / stack / static shared memory per kernel (cuobjdump -res-usage)
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines()
    rr = []
    for i, l in enumerate(res):
        m = re.match(r"\s*Function (\S+):", l)
        if m and i + 1 < len(res):
            r = dict(re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", res[i + 1]))
            rr.append((m.group(1), int(r.get("REG", 0)), int(r.get("STACK", 0)), int(r.get("SHARED", 0))))
    dem = subprocess.run(["c++filt"], input="\n".join(n for n, *_ in rr), capture_output=True, text=True).stdout.splitlines()
    seen, out = set(), []
    for (n, reg, stack, sh), d in zip(rr, dem):
        d = re.sub(r"^void ", "", d.replace("(anonymous namespace)::", ""))
        d = re.sub(r"\((?:[^()]|\([^()]*\))*\)\s*$", "", d)
        if (d, reg, stack, sh) not in seen:
            seen.add((d, reg, stack, sh)); out.append((d, reg, stack, sh))
    out.sort(key=lambda x: -x[1])
    print("\n\nResource usage (cuobjdump -res-usage): registers per thread, stack bytes per thread (local arrays / spills), STATIC shared memory bytes\n")
    print("%-44s %5s %6s %8s" % ("kernel", "REG", "STACK", "SHARED"))
    for d, reg, stack, sh in out:
        if reg >= 64 or stack:
            print("%-44s %5d %6d %8d" % (d[:44], reg, stack, sh))
    return 0


if __name__ == "__main__":
    sys.exit(main())
