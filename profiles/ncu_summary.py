#!/usr/bin/env python3
"""Summarise an .ncu-rep (read here, no GPU needed): per-kernel duration, DRAM /
L2 bytes and throughput, occupancy, top stall reasons.
usage: python profiles/ncu_summary.py prof.ncu-rep | prof_raw.csv"""
import csv
import subprocess
import sys

WANT = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sectors.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__waves_per_multiprocessor",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
    "lts__t_sectors_op_atom.sum", "lts__t_sectors_op_red.sum", "lts__t_sectors_op_read.sum", "lts__t_sectors_op_write.sum",
    "lts__t_sector_hit_rate.pct",
]


def main(path):
    # an .ncu-rep, or its `ncu -i rep --page raw --csv` export (much smaller than the report of a whole pass)
    out = open(path).read() if path.endswith(".csv") else \
        subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    ki = hdr.index("Kernel Name")
    stall_cols = [i for i, h in enumerate(hdr) if h.startswith("smsp__average_warps_issue_stalled") and h.endswith("_per_issue_active.ratio")]
    if not stall_cols:
        stall_cols = [i for i, h in enumerate(hdr) if h.startswith("smsp__average_warp_latency_issue_stalled") ]
    for r in rows[2:]:
        print("==", r[ki][:70])
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                print(f"   {w:68s} {r[i]:>16s} {units[i]}")
        st = sorted(((float(r[i].replace(',', '') or 0), hdr[i]) for i in stall_cols), reverse=True)[:6]
        for v, h in st:
            print(f"   stall {h.split('issue_stalled_')[-1][:40]:42s} {v:10.2f}")


if __name__ == "__main__":
    main(sys.argv[1])
