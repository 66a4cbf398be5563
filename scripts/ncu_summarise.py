#!/usr/bin/env python
"""Reads the .ncu-rep files of scripts/ncu_capture.sh (no GPU needed) and writes, per kernel, the handful of
metrics the roofline discussion needs to profiles/ncu_<name>.csv plus one table profiles/NCU_SUMMARY.md."""
import csv
import io
import os
import re
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum", "l1tex__t_bytes.sum",
    "lts__t_sectors_srcunit_tex_aperture_peer.sum", "lts__t_sectors_srcunit_tex_aperture_peer_op_read.sum",
    "lts__t_sectors_srcunit_tex_aperture_peer_op_write.sum", "sm__inst_executed.sum", "smsp__cycles_active.avg",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_barrier_per_warp_active.pct", "smsp__warp_issue_stalled_membar_per_warp_active.pct",
    "smsp__warp_issue_stalled_lg_throttle_per_warp_active.pct",
]


def raw_rows(rep):
    if rep.endswith(".csv"):  # already exported on the GPU box (scripts/ncu_capture.sh)
        out = open(rep).read()
    else:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rd = list(csv.reader(io.StringIO(out)))
    if len(rd) < 3:
        return [], []
    return rd[0], rd[2:]


def main():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    reps = sys.argv[1:] or [os.path.join(root, "gpurun_out", f) for f in ("ncu_ep_raw.csv", "ncu_coll_raw.csv")]
    os.makedirs(os.path.join(root, "profiles"), exist_ok=True)
    table = []
    for rep in reps:
        if not os.path.exists(rep):
            continue
        hdr, rows = raw_rows(rep)
        if not hdr:
            continue
        col = {h: i for i, h in enumerate(hdr)}
        name_i = col.get("Kernel Name")
        seen = {}
        for r in rows:
            name = r[name_i]
            short = re.sub(r"\(.*", "", name).replace("void ", "").replace("ub::", "")
            grid = r[col["launch__grid_size"]] if "launch__grid_size" in col else "?"
            key = f"{short}@{grid}"
            if key in seen:
                continue
            seen[key] = 1
            vals = {k: r[col[k]] for k in KEEP if k in col}
            fn = re.sub(r"[^A-Za-z0-9_]+", "_", key).strip("_")[:80]
            with open(os.path.join(root, "profiles", f"ncu_{fn}.csv"), "w") as f:
                w = csv.writer(f)
                w.writerow(["kernel", name])
                for k in hdr:
                    if k in col and (k in KEEP or k.startswith(("launch__", "smsp__warp_issue_stalled", "dram__", "lts__t_sectors_srcunit_tex_aperture"))):
                        w.writerow([k, r[col[k]]])
            table.append((key, vals))
    with open(os.path.join(root, "profiles", "NCU_SUMMARY.md"), "w") as f:
        f.write("# ncu --set full summaries (1 H100, one-rank communicator, benchmarks/ncu_targets.py)\n\n")
        f.write("Durations under ncu are serialised and cold-cache: compare shares and percentages, not absolutes.\n\n")
        f.write("| kernel@grid | us | regs | warps active % | DRAM % of peak | DRAM read MB | DRAM write MB | long-scoreboard stall % | barrier stall % |\n")
        f.write("|---|---:|---:|---:|---:|---:|---:|---:|---:|\n")

        def g(v, k, scale=1.0, fmt="{:.1f}"):
            try:
                return fmt.format(float(v.get(k, "nan").replace(",", "")) * scale)
            except Exception:
                return "-"

        for key, v in table:
            f.write(f"| {key} | {g(v, 'gpu__time_duration.sum', 1e-3)} | {g(v, 'launch__registers_per_thread', 1, '{:.0f}')} | "
                    f"{g(v, 'sm__warps_active.avg.pct_of_peak_sustained_active')} | {g(v, 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed')} | "
                    f"{g(v, 'dram__bytes_read.sum', 1e-6)} | {g(v, 'dram__bytes_write.sum', 1e-6)} | "
                    f"{g(v, 'smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct')} | {g(v, 'smsp__warp_issue_stalled_barrier_per_warp_active.pct')} |\n")
    print(f"{len(table)} kernels summarised")


if __name__ == "__main__":
    main()
