#!/usr/bin/env python3
"""tools/ncu_summary.py -- condense an .ncu-rep (read here with `ncu -i`) into a few lines: duration, issue statistics,
warp stall reasons per issued instruction, instruction / branch counts, launch shape, DRAM bytes when the capture has them.
    python tools/ncu_summary.py x.ncu-rep [...] > x.txt"""
import csv
import subprocess
import sys

WANT = ("gpu__time_duration.sum", "smsp__cycles_active.avg", "sm__cycles_active.avg", "smsp__inst_executed.sum", "smsp__inst_issued.sum", "smsp__issue_active.avg.per_cycle_active",
        "smsp__inst_executed_op_branch.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "smsp__warps_eligible.avg.per_cycle_active", "smsp__average_warp_latency_per_inst_issued.ratio", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__inst_executed_op_shared_ld.sum", "smsp__inst_executed_op_shared_st.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed")

for path in sys.argv[1:]:
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    print("#", path)
    for r in rows[2:]:
        d = dict(zip(hdr, r)); u = dict(zip(hdr, units))
        print("== kernel %s  (launch id %s)" % (d["Kernel Name"][:110], d["ID"]))
        for k in WANT:
            if k in d and d[k] != "":
                print("   %-62s %s %s" % (k, d[k], u.get(k, "")))
        stalls = []
        for h in hdr:
            if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio") and "not_issued" not in h:
                try:
                    stalls.append((float(d[h].replace(",", "")), h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]))
                except ValueError:
                    pass
        if stalls:
            print("   warp cycles per issued instruction, by stall reason (sum = %.2f):" % sum(v for v, _ in stalls))
            for v, name in sorted(stalls, reverse=True):
                if v >= 0.005:
                    print("      %-24s %.3f" % (name, v))
