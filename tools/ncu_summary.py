#!/usr/bin/env python
"""Text summary of an `ncu --set full` report (DRAM bytes, duration, occupancy, stall samples per launch):

    python tools/ncu_summary.py step.ncu-rep "capture command / context" > ncu_step_summary.txt
"""
import csv
import io
import subprocess
import sys

WANT = ["dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum", "launch__block_size", "launch__grid_size",
        "launch__registers_per_thread", "sm__cycles_active.avg", "sm__cycles_active.max", "sm__cycles_elapsed.max",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct"]


def main():
    rep = sys.argv[1]
    ctx = sys.argv[2] if len(sys.argv) > 2 else ""
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    print(f"# ncu --set full --clock-control none --import-source on  ({ctx}); per launch, cache-control all (cold caches)")
    for r in rows[2:]:
        print(f"kernel: {r[hdr.index('Kernel Name')][:110]}")
        for w in WANT:
            if w in hdr:
                print(f"  {w} = {r[hdr.index(w)]} {units[hdr.index(w)]}")
        for i, h in enumerate(hdr):
            if "pcsamp_warps_issue_stalled" in h and "not_issued" not in h and r[i] not in ("0", ""):
                print(f"  {h} = {r[i]}")


if __name__ == "__main__":
    main()
