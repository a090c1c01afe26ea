#!/usr/bin/env python
"""A JSON summary (stdout) of one `ncu --set full` report of the chain kernels (one launch each).

usage: tools/ncu_summary.py <report.ncu-rep> <blocks in the captured step> [note]
Per kernel: DRAM bytes read/written (dram__bytes_{read,write}.sum), rows, duration, executed warp
instructions per (block,channel) row, IPC, registers, and the algorithmic bytes per row of DESIGN.md §4.
"""
import csv
import json
import subprocess
import sys

rep, blocks = sys.argv[1], int(sys.argv[2])
note = sys.argv[3] if len(sys.argv) > 3 else ""
ch, N = 2, 2048
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
ALG = {"k_phaseA_transform": 8 * N, "k_phaseA_psy": 10 * N, "k_floor1_fit": 4 * N, "k_floor1_render": 2 * N, "k_cqn": 6 * N}
out = {"note": note or ("ncu --set full --clock-control none --import-source on, one un-split step of %d long stereo blocks "
                        "(%d (block,channel) rows per launch): the step's intermediates (%.1f GB) exceed the 50 MB L2"
                        % (blocks, blocks * ch, 30 * N * ch * blocks / 1e9)),
       "blocks": blocks, "kernels": {}}


def num(d, k):
    v = d.get(k, "")
    try:
        return float(v.replace(",", ""))
    except ValueError:
        return None


def scale(d, k):
    """value in base units: ncu prints e.g. Mbyte / Kbyte / usecond in the unit row"""
    v = num(d, k)
    if v is None:
        return None
    u = units[hdr.index(k)].lower()
    for pre, f in (("gbyte", 1e9), ("mbyte", 1e6), ("kbyte", 1e3), ("byte", 1.0), ("msecond", 1e6), ("usecond", 1e3), ("nsecond", 1.0), ("second", 1e9), ("ms", 1e6), ("us", 1e3), ("ns", 1.0), ("s", 1e9)):
        if u.startswith(pre):
            return v * f
    return v


for r in rows[2:]:
    d = dict(zip(hdr, r))
    name = d["Kernel Name"]
    key = next((k for k in ALG if k in name or (k == "k_phaseA_psy" and "k_phaseA_psy" in name) or (k == "k_cqn" and "k_cqn" in name)), None)
    if key is None or key in out["kernels"]:
        continue
    nrows = blocks * ch
    rd, wr = scale(d, "dram__bytes_read.sum"), scale(d, "dram__bytes_write.sum")
    inst = num(d, "smsp__inst_executed.sum")
    out["kernels"][key] = {
        "kernel_in_report": name.split("(")[0],
        "grid": d["Grid Size"], "block": d["Block Size"],
        "dram_bytes_read": rd, "dram_bytes_write": wr, "rows": nrows,
        "dram_bytes_per_row": (rd + wr) / nrows,
        "algorithmic_bytes_per_row": ALG[key],
        "traffic_over_algorithmic": (rd + wr) / nrows / ALG[key],
        "gpu_time_ns": scale(d, "gpu__time_duration.sum"),
        "warp_instructions_per_row": inst / nrows,
        "ipc": num(d, "sm__inst_executed.avg.per_cycle_active"),
        "issue_slot_utilisation": (num(d, "sm__inst_executed.avg.per_cycle_active") or 0) / 4.0,
        "registers": num(d, "launch__registers_per_thread"),
        "achieved_occupancy_pct": num(d, "sm__warps_active.avg.pct_of_peak_sustained_active"),
        "shared_wavefronts_per_row": (num(d, "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum") or 0) / nrows,
        "shared_bank_conflict_wavefronts_per_row": ((num(d, "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum") or 0) +
                                                    (num(d, "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_st.sum") or 0)) / nrows,
    }
print(json.dumps(out, indent=1))
