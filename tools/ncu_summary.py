#!/usr/bin/env python
"""Summarise an Nsight Compute report into text: key section metrics, DRAM traffic, and (for kernels built with
-lineinfo) an instruction/stall breakdown per __syncthreads()-delimited phase.  Usage:
    python tools/ncu_summary.py prof_lift_fwd_cols.ncu-rep > lift_forward_cols_kernel.txt
"""
import collections
import csv
import io
import subprocess
import sys


def ncu(args):
    return subprocess.run(["ncu", "-i", *args], capture_output=True, text=True).stdout


def main(path):
    details = ncu([path, "--page", "details"])
    keep = ("Duration", "DRAM Throughput", "Memory Throughput", "L2 Cache Throughput", "Compute (SM) Throughput", "Executed Ipc Active",
            "Issue Slots Busy", "No Eligible", "Eligible Warps", "Registers Per Thread", "Dynamic Shared Memory Per Block",
            "Theoretical Occupancy", "Achieved Occupancy", "Waves Per SM", "L1/TEX Hit Rate", "L2 Hit Rate", "Grid Size", "Block Size",
            "Block Limit Registers", "Block Limit Shared Mem")
    name = [l for l in details.splitlines() if "Context" in l and "Stream" in l]
    print("# report:", path)
    if name:
        print("# kernel:", name[0].strip())
    for line in details.splitlines():
        if any(k in line for k in keep) and "OPT" not in line and "INF" not in line:
            print("   ", " ".join(line.split()))
    raw = list(csv.reader(io.StringIO(ncu([path, "--page", "raw", "--csv"]))))
    if len(raw) >= 3:
        hdr, units, vals = raw[0], raw[1], raw[2]
        want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sectors_op_red.sum",
                "lts__t_sectors_op_read.sum", "lts__t_sectors_op_write.sum", "smsp__inst_executed.sum",
                "launch__registers_per_thread", "sm__warps_active.avg.pct_of_peak_sustained_active",
                "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
                "smsp__sass_inst_executed_op_shared_ld.sum", "smsp__sass_inst_executed_op_shared_st.sum",
                "dram__throughput.avg.pct_of_peak_sustained_elapsed"]
        print("# raw metrics")
        for w in want:
            if w in hdr:
                i = hdr.index(w)
                print(f"    {w:62s} {vals[i]:>18s} {units[i]}")
    src = list(csv.reader(io.StringIO(ncu([path, "--page", "source", "--csv"]))))
    if len(src) > 3 and "Instructions Executed" in src[1]:
        hdr = src[1]
        ie, ss, sc = hdr.index("Instructions Executed"), hdr.index("# Samples"), hdr.index("Source")
        stall_cols = {n: hdr.index(n) for n in hdr if n.startswith("stall_") and "Not Issued" not in n}
        data = src[2:]
        tot = sum(int(r[ie] or 0) for r in data) or 1
        tots = sum(int(r[ss] or 0) for r in data) or 1
        print(f"# SASS phases (split at BAR.SYNC): total warp instructions {tot}, samples {tots}")
        seg, segs = 0, collections.defaultdict(lambda: dict(instr=0, samples=0, ops=collections.Counter(), stalls=collections.Counter()))
        for r in data:
            s = r[sc]
            S = segs[seg]
            n = int(r[ie] or 0)
            S["instr"] += n
            S["samples"] += int(r[ss] or 0)
            op = s.split()[0] if not s.startswith("@") else s.split()[1]
            S["ops"][op.split(".")[0]] += n
            for k, c in stall_cols.items():
                S["stalls"][k] += int(r[c] or 0)
            if "BAR.SYNC" in s:
                seg += 1
        for k, S in segs.items():
            print(f"  phase {k}: {S['instr'] / 1e6:7.2f} M warp-instr ({S['instr'] / tot * 100:5.1f} %), {S['samples'] / tots * 100:5.1f} % of samples")
            print("      ops   :", ", ".join(f"{o} {c / 1e6:.2f}M" for o, c in S["ops"].most_common(8)))
            print("      stalls:", ", ".join(f"{o[6:]} {c / tots * 100:.1f}%" for o, c in S["stalls"].most_common(5)))
        marks = collections.Counter()
        for r in data:
            for m in ("UTMALDG", "UTMASTG", "REDG", "FFMA2", "SYNCS", "MUFU.EX2", "LDS.128", "STS", "F2I"):
                if m in r[sc]:
                    marks[m] += int(r[ie] or 0)
        print("# marker instructions (warp-level executions):", dict(marks))


if __name__ == "__main__":
    main(sys.argv[1])
