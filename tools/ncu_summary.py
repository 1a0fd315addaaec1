#!/usr/bin/env python
"""Condense an `ncu --set full` report (read with `ncu -i X.ncu-rep --page raw --csv`) to the metrics the roofline
discussion uses, one block per profiled launch.  Usage: python tools/ncu_summary.py X.ncu-rep > X.txt"""
import csv
import subprocess
import sys

WANT = [
    ("duration_us", "gpu__time_duration.sum"),
    ("grid", "launch__grid_size"), ("block", "launch__block_size"), ("regs/thread", "launch__registers_per_thread"),
    ("smem/block dyn (B)", "launch__shared_mem_per_block_dynamic"),
    ("sm_cycles", "sm__cycles_elapsed.max"),
    ("tensor pipe active % (of elapsed)", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
    ("tensor pipe active % (realtime)", "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed"),
    ("tensor hmma inst %", "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active"),
    ("xu (MUFU) pipe %", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active"),
    ("fma pipe %", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"),
    ("fmaheavy pipe %", "sm__inst_executed_pipe_fmaheavy.avg.pct_of_peak_sustained_active"),
    ("alu pipe %", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"),
    ("issue slots busy %", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("eligible warps / cycle", "smsp__warps_eligible.avg.per_cycle_active"),
    ("achieved occupancy %", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("warp instructions", "smsp__inst_executed.sum"),
    ("dram read (MB)", "dram__bytes_read.sum"), ("dram write (MB)", "dram__bytes_write.sum"),
    ("dram throughput %", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    ("l2 hit rate %", "lts__t_sector_hit_rate.pct"),
    ("l1/tex->smem load throughput %", "l1tex__data_pipe_lsu_wavefronts_mem_shared.avg.pct_of_peak_sustained_elapsed"),
    ("sm throughput %", "sm__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("local load/store inst", "smsp__inst_executed_op_local_ld.sum"),
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(ln for ln in out.splitlines() if not ln.startswith("==")))
    hdr, units = rows[0], rows[1]
    ix = {h: i for i, h in enumerate(hdr)}
    print(f"# {path}: ncu --set full --clock-control none (one block per profiled launch)")
    for r in rows[2:]:
        name = r[ix["Kernel Name"]]
        print(f"\n## {name[:150]}")
        for label, key in WANT:
            if key in ix:
                print(f"  {label:36s} {r[ix[key]]:>16s} {units[ix[key]]}")
        stalls = [(float(r[i] or 0), h) for h, i in ix.items()
                  if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
        top = sorted(stalls, reverse=True)[:5]
        if top:
            print("  top stall reasons (warps stalled per issue):")
            for v, h in top:
                print(f"    {h[len('smsp__average_warps_issue_stalled_'):-len('_per_issue_active.ratio')]:28s} {v:8.2f}")


if __name__ == "__main__":
    main(sys.argv[1])
