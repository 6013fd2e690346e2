#!/usr/bin/env python
"""Turn ncu reports into small text summaries (kept under profiles/, outside version control).
usage: summarize_profiles.py <report.ncu-rep> <out.txt> "<title>"      (needs `ncu` on PATH; no GPU required)"""
import csv, os, re, subprocess, sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__inst_executed.sum", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "lts__t_sector_hit_rate.pct", "sm__inst_executed_pipe_tensor.sum"]


def main(rep, out, title):
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    with open(out, "w") as f:
        f.write("# %s\n# source: ncu --set full --clock-control none --import-source on (%s), H100\n" % (title, os.path.basename(rep)))
        for d in data:
            f.write("\nkernel: %s\n" % re.sub(r"\(.*", "", d[ki]))
            for k in KEYS:
                if k in hdr:
                    i = hdr.index(k); f.write("  %-70s %-14s %s\n" % (k, d[i], units[i]))
            for h in hdr:
                if "issue_stalled" in h and "per_issue_active" in h:
                    i = hdr.index(h)
                    try:
                        if float(d[i]) >= 0.3:
                            f.write("  %-70s %-14s\n" % (h.replace("smsp__average_warps_issue_stalled_", "stall:").replace("_per_issue_active.ratio", ""), d[i]))
                    except ValueError:
                        pass


if __name__ == "__main__":
    main(*sys.argv[1:4])
