#!/usr/bin/env python
"""Summarise an `ncu --set full` report: one block per captured launch with the metrics DESIGN.md quotes.

usage: python tools/ncu_summary.py report.ncu-rep [flops_or_bytes.json] > profiles/<name>_summary.txt
Reads the report through `ncu -i … --page raw --csv` (ncu must be on PATH)."""
import csv
import io
import subprocess
import sys

METRICS = [
    ("duration_us", "gpu__time_duration.sum"),
    ("grid", "launch__grid_size"),
    ("block", "launch__block_size"),
    ("regs/thread", "launch__registers_per_thread"),
    ("dyn smem B", "launch__shared_mem_per_block_dynamic"),
    ("dram read B", "dram__bytes_read.sum"),
    ("dram write B", "dram__bytes_write.sum"),
    ("dram % of peak", "dram__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L2 % of peak", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L2 hit %", "lts__t_sector_hit_rate.pct"),
    ("SM % of peak", "sm__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("tensor pipe % (elapsed)", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
    ("wgmma f16 path %", "sm__ops_path_tensor_op_hgmma_src_fp16_sparsity_off.avg.pct_of_peak_sustained_elapsed"),
    ("mma.sync f16->f32 path %", "sm__ops_path_tensor_op_hmma_src_fp16_dst_fp32_sparsity_off.avg.pct_of_peak_sustained_elapsed"),
    ("achieved occupancy %", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("ipc (active)", "smsp__inst_executed.avg.per_cycle_active"),
    ("stall long_scoreboard", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"),
    ("stall barrier", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"),
    ("stall no_instruction", "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio"),
    ("stall wait", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio"),
    ("stall short_scoreboard", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio"),
    ("stall math_throttle", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio"),
    ("stall mio_throttle", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio"),
]
UNIT_SCALE = {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "nsecond": 1e-3,
              "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    print("# %s  (ncu --set full --clock-control none; one replayed launch per block; times are cold-cache, serialised)" % rep)
    for r in rows[2:]:
        name = r[col["Kernel Name"]]
        print("\n== %s" % name[:150])
        dur = None
        dr = dw = 0.0
        for label, m in METRICS:
            if m not in col or r[col[m]] == "":
                continue
            try:
                v = float(r[col[m]].replace(",", ""))
            except ValueError:
                continue
            u = units[col[m]]
            if label == "duration_us":
                v *= UNIT_SCALE.get(u, 1.0)
                dur = v
            elif label.startswith("dram") and label.endswith("B"):
                v *= UNIT_SCALE.get(u, 1.0)
                if "read" in label:
                    dr = v
                else:
                    dw = v
            print("  %-26s %14.4g" % (label, v))
        if dur:
            print("  %-26s %14.4g   (dram read+write / duration)" % ("dram GB/s", (dr + dw) / dur * 1e-3))


if __name__ == "__main__":
    main()
