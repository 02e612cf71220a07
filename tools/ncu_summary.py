#!/usr/bin/env python
"""Condense an .ncu-rep (one profiled launch of the scan kernel) into the handful of
counters the design argues from.

    python tools/ncu_summary.py evidence_out/prof_full_glue10.ncu-rep [payload_bytes] > glue10_summary.txt
"""
import csv
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum",
    "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum",
    "memory_l1_wavefronts_shared_ideal",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum",
    "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__warps_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active",
    "launch__registers_per_thread", "launch__block_size", "launch__grid_size",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
    "sm__cycles_elapsed.max",
]


def main():
    rep = sys.argv[1]
    payload = float(sys.argv[2]) if len(sys.argv) > 2 else None
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        rec = dict(zip(hdr, r))
        print("# kernel:", rec.get("Kernel Name"), " grid", rec.get("Grid Size"), " block", rec.get("Block Size"))
        vals = {}
        for k in KEYS:
            if k in rec:
                u = units[hdr.index(k)]
                vals[k] = (rec[k], u)
                print("%-92s %s %s" % (k, rec[k], u))
        try:
            def num(k):
                return float(vals[k][0].replace(",", ""))
            dur_us = num("gpu__time_duration.sum") * {"us": 1, "ms": 1e3, "ns": 1e-3}.get(vals["gpu__time_duration.sum"][1], 1)
            scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1}
            traffic = num("dram__bytes_read.sum") * scale[vals["dram__bytes_read.sum"][1]] + \
                num("dram__bytes_write.sum") * scale[vals["dram__bytes_write.sum"][1]]
            print("derived: dram traffic per launch = %.0f bytes" % traffic)
            if payload:
                print("derived: algorithmic bytes per launch = %.0f ; traffic / algorithmic = %.4f" % (payload, traffic / payload))
                print("derived: payload / duration (under ncu, cold, not a bench number) = %.1f GB/s" % (payload / dur_us / 1e3))
                steps = payload / 32.0
                print("derived: shared wavefronts per warp-step (32 input bytes) = %.3f ; instructions per warp-step = %.2f" % (
                    num("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum") / steps, num("smsp__inst_executed.sum") / steps))
        except Exception as e:   # noqa: BLE001
            print("derived: (incomplete)", e)


if __name__ == "__main__":
    main()
