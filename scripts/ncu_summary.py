"""Summarise .ncu-rep files (read on the GPU-less host with `ncu -i`) into text tables."""
import csv
import subprocess
import sys

WANT = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum",
        "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__registers_per_thread", "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor",
        "smsp__average_warp_latency_issue_stalled_long_scoreboard.pct",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio"]
for rep in sys.argv[1:]:
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    print("# " + rep)
    for r in rows[2:]:
        print("-" * 100)
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                print("{:85s} {:>14s} {}".format(w, r[i][:70] if w == "Kernel Name" else r[i], units[i]))
