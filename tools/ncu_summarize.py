"""Compact text summary of an `ncu --set full` report: one block per captured launch with the metrics the roofline
arithmetic needs (duration, DRAM bytes, DRAM / tensor-pipe / SM utilisation, occupancy, registers) and the four largest
warp-stall reasons.

    python tools/ncu_summarize.py train.ncu-rep > train_summary.txt"""
import csv
import io
import re
import subprocess
import sys

KEEP = [
    "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "lts__t_sector_hit_rate.pct",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "sm__cycles_elapsed.max",
]


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    # header row = first row containing "Kernel Name"
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    head, units = rows[hi], rows[hi + 1]
    col = {n: i for i, n in enumerate(head)}
    stall_cols = [n for n in head if re.search(r"issue_stalled_.*_per_warp_active\.pct$", n)]
    if not stall_cols:
        stall_cols = [n for n in head if re.search(r"average_warps?_issue_stalled_.*per_issue_active", n)]
    print("# extracted from `ncu --set full --clock-control none` (raw page) of %s; one block per captured launch" % rep)
    for r in rows[hi + 2:]:
        if len(r) < len(head):
            continue
        print("----")
        print("%-80s %s" % ("Kernel Name", r[col["Kernel Name"]]))
        for k in KEEP:
            if k in col:
                print("%-80s %s %s" % (k, r[col[k]], units[col[k]]))
        stalls = []
        for n in stall_cols:
            try:
                stalls.append((float(r[col[n]].replace(",", "")), n))
            except ValueError:
                pass
        stalls.sort(reverse=True)
        for v, n in stalls[:4]:
            print("%-80s %.3f %s" % (n, v, units[col[n]]))


if __name__ == "__main__":
    main()
