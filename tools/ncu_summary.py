#!/usr/bin/env python
"""Summarise an .ncu-rep (captured with `ncu --set full`) into a small text file.
usage: python tools/ncu_summary.py prof.ncu-rep out.txt ["note"]"""
import csv, io, subprocess, sys

KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "smsp__sass_thread_inst_executed_op_dfma_pred_on.sum", "smsp__sass_thread_inst_executed_op_dadd_pred_on.sum",
        "smsp__sass_thread_inst_executed_op_dmul_pred_on.sum",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__average_warp_latency_per_inst_issued.ratio",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"]

def main():
    rep, out = sys.argv[1], sys.argv[2]
    note = sys.argv[3] if len(sys.argv) > 3 else ""
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write(f"# ncu --set full --clock-control none summary of {rep}\n# {note}\n")
        for r in rows[2:]:
            d = dict(zip(hdr, zip(units, r)))
            f.write(f"\n== {d['Kernel Name'][1]}  grid {d.get('launch__grid_size', ('', '?'))[1]} block {d.get('launch__block_size', ('', '?'))[1]}\n")
            for k in KEYS:
                if k in d:
                    f.write(f"{k:90s} {d[k][1]} {d[k][0]}\n")
            f.write("-- warp stall reasons (cycles per issued instruction)\n")
            for h in hdr:
                if "issue_stalled" in h and h.endswith("per_issue_active.ratio"):
                    v = float(d[h][1])
                    if v >= 0.01:
                        f.write(f"   {h.split('stalled_')[1].split('_per')[0]:24s} {v:.3f}\n")
    print(open(out).read())

main()
