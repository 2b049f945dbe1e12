#!/usr/bin/env python
"""Summarise an Nsight Compute report (.ncu-rep, read without a GPU) into small files: a JSON of the headline
metrics of the dominant kernel plus an opcode / phase breakdown from the source page.
Usage: python tools/ncu_summary.py <report>.ncu-rep <output prefix>"""
from __future__ import annotations

import collections
import csv
import io
import json
import re
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "launch__waves_per_multiprocessor",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "smsp__inst_executed.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
    "sm__cycles_elapsed.max",
]


def ncu_csv(rep: str, page: str) -> list[list[str]]:
    out = subprocess.run(["ncu", "-i", rep, "--page", page, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main() -> None:
    rep, out_prefix = sys.argv[1], sys.argv[2]
    raw = ncu_csv(rep, "raw")
    hdr, units, vals = raw[0], raw[1], raw[2]
    col = {h: i for i, h in enumerate(hdr)}
    summary = {"report": rep, "kernel": vals[col["Kernel Name"]], "grid": vals[col["Grid Size"]],
               "block": vals[col["Block Size"]], "metrics": {}, "stall_cycles_per_issued_instruction": {}}
    for k in KEYS:
        if k in col:
            summary["metrics"][k] = {"value": vals[col[k]], "unit": units[col[k]]}
    for h, i in col.items():
        m = re.match(r"smsp__average_warps_issue_stalled_(\w+)_per_issue_active\.ratio", h)
        if m:
            try:
                v = float(vals[i])
            except ValueError:
                continue
            if v >= 0.02:
                summary["stall_cycles_per_issued_instruction"][m.group(1)] = round(v, 3)
    src = ncu_csv(rep, "source")
    shdr = src[1]
    ia, isrc, isamp = shdr.index("Instructions Executed"), shdr.index("Source"), shdr.index("# Samples")
    ops, samp = collections.Counter(), collections.Counter()
    hot = []  # (samples, executed, instruction text): where the stall samples sit
    phases, cur = [], {"instructions": 0, "samples": 0, "ffma2": 0}
    for r in src[2:]:
        if len(r) <= ia:
            continue
        s = r[isrc].strip()
        m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_]+)", s)
        op = m.group(2) if m else s[:10]
        n, sp = int(r[ia] or 0), int(r[isamp] or 0)
        ops[op] += n
        samp[op] += sp
        hot.append((sp, n, s[:70]))
        cur["instructions"] += n
        cur["samples"] += sp
        if op in ("FFMA2", "FFMA"):
            cur["ffma2"] += n
        if op == "BAR":
            phases.append(cur)
            cur = {"instructions": 0, "samples": 0, "ffma2": 0}
    phases.append(cur)
    tot, tots = sum(ops.values()), max(sum(samp.values()), 1)
    summary["warp_instructions_executed"] = tot
    summary["opcode_mix"] = [{"op": op, "share": round(n / tot, 4), "stall_sample_share": round(samp[op] / tots, 4)}
                             for op, n in ops.most_common(18)]
    summary["phases_between_barriers"] = [
        {"instructions_share": round(p["instructions"] / tot, 4), "sample_share": round(p["samples"] / tots, 4),
         "ffma2_share_of_phase": round(p["ffma2"] / max(p["instructions"], 1), 3)} for p in phases if p["instructions"] > tot * 0.002][:48]
    # ("ffma2" counts packed FFMA2, where the architecture has it, and scalar FFMA)
    summary["top_stall_instructions"] = [{"sample_share": round(sp / tots, 4), "executed": n, "sass": t}
                                         for sp, n, t in sorted(hot, reverse=True)[:24]]
    with open(out_prefix + ".json", "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary, indent=1)[:3000])


if __name__ == "__main__":
    main()
