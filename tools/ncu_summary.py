"""Summarise an .ncu-rep (read here, no GPU needed) into a handful of metrics:
python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum",
        "lts__t_sectors.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__cycles_active.avg",
        "sm__cycles_elapsed.max", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem",
        "smsp__warps_eligible.avg.per_cycle_active", "smsp__issue_active.avg.pct_of_peak_sustained_active"]
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
for k, vals in enumerate(rows[2:]):
    name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
    print(f"# launch {k}: {name}   ({rep})")
    d = dict(zip(hdr, zip(vals, units)))
    for w in WANT:
        if w in d:
            print(f"{w:75s} {d[w][0]:>16s} {d[w][1]}")
    stalls = sorted(((float(v[0] or 0), h) for h, v in d.items() if "issue_stalled" in h and h.endswith("per_issue_active.ratio")), reverse=True)
    print("top stall reasons (warps per issue-active cycle): " + ", ".join(f"{h.split('issue_stalled_')[1].split('_per_')[0]}={x:.2f}" for x, h in stalls[:6]))
