#!/usr/bin/env python
"""Summarise an .ncu-rep (ncu --set full) into a small markdown table."""
import csv, subprocess, sys
WANT = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed.sum", "sm__cycles_elapsed.max"]
rep, title = sys.argv[1], sys.argv[2]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units = rows[0], rows[1]
print("# %s\n" % title)
for r in rows[2:]:
    name = r[hdr.index("Kernel Name")]
    print("Kernel: `%s`\n\n| metric | unit | value |\n|---|---|---|" % name[:160])
    for h, u, v in zip(hdr, units, r):
        if h in WANT:
            print("| %s | %s | %s |" % (h, u, v))
    print()
