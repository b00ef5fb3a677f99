#!/usr/bin/env python3
"""ncu_summary.py <raw.csv> <out_summary.csv> [--traffic out.json --frames F --points P --tag TEXT]

Distils `ncu -i X.ncu-rep --page raw --csv` (hundreds of columns) into one row per kernel launch with the columns the
roofline discussion uses, and optionally writes the per-kernel DRAM bytes per launch (dram__bytes_read.sum +
dram__bytes_write.sum) as a traffic file that bench.py scales to its own batch (`roofline.traffic`, B/point).
"""
import argparse
import csv
import json
import re

COLS = ["Kernel Name", "Block Size", "Grid Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "launch__registers_per_thread", "launch__cluster_dim_x",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "sm__throughput.avg.pct_of_peak_sustained_elapsed"]

# kernel name -> the stage name bench.py uses
STAGES = [(r"k_front_cluster", "k_front"), (r"k_bin_hist", "k_bin_hist"), (r"k_bin_scan", "k_bin_scan"), (r"k_scatter", "k_scatter"),
          (r"k_fit_resident", "k_fit_S"), (r"k_fit_warp<\(bool\)1, \(int\)1|k_fit_warp<1, 1", "k_fit_M"), (r"k_fit_warp<", "k_fit_L1"),
          (r"k_fit_cta<4096|k_fit_cta<\(int\)4096", "k_fit_L2"), (r"k_fit_cta<8192|k_fit_cta<\(int\)8192", "k_fit_L3"),
          (r"k_fit_patch<4|k_fit_patch<\(int\)4", "k_fit_L1"), (r"k_fit_patch<8|k_fit_patch<\(int\)8", "k_fit_L2"),
          (r"k_fit_patch<16|k_fit_patch<\(int\)16", "k_fit_L3"), (r"k_fit_big", "k_fit_X"), (r"k_gle", "k_gle"), (r"k_order", "k_order"),
          (r"k_emit", "k_emit"), (r"k_gather_xyz", "k_gather_xyz"), (r"k_repack|k_pad_xyz", "k_repack")]


def to_bytes(v, unit):
    v = float(v)
    u = unit.lower()
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("raw")
    ap.add_argument("out")
    ap.add_argument("--traffic")
    ap.add_argument("--frames", type=int, default=0)
    ap.add_argument("--points", type=int, default=0)
    ap.add_argument("--tag", default="")
    a = ap.parse_args()
    rows = list(csv.reader(open(a.raw, newline="")))
    # skip ncu's "==PROF==" preamble lines if any
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    head, units, body = rows[hi], rows[hi + 1], rows[hi + 2:]
    idx = {c: head.index(c) for c in COLS if c in head}
    with open(a.out, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow([c for c in COLS if c in idx])
        w.writerow([units[idx[c]] for c in COLS if c in idx])
        for r in body:
            if len(r) == len(head):
                w.writerow([r[idx[c]] for c in COLS if c in idx])
    if a.traffic:
        t = {}
        for r in body:
            if len(r) != len(head):
                continue
            name = r[idx["Kernel Name"]]
            stage = next((s for pat, s in STAGES if re.search(pat, name)), None)
            if stage is None:
                continue
            rd = to_bytes(r[idx["dram__bytes_read.sum"]], units[idx["dram__bytes_read.sum"]])
            wr = to_bytes(r[idx["dram__bytes_write.sum"]], units[idx["dram__bytes_write.sum"]])
            e = t.setdefault(stage, {"frames": a.frames, "points": a.points, "dram_bytes": 0.0, "dram_read": 0.0, "dram_write": 0.0,
                                     "kernel": name.split("(")[0][:90], "launches": 0, "source": a.tag})
            e["dram_bytes"] += rd + wr
            e["dram_read"] += rd
            e["dram_write"] += wr
            e["launches"] += 1
        for e in t.values():   # mean per launch when a kernel was captured more than once
            for k in ("dram_bytes", "dram_read", "dram_write"):
                e[k] /= e["launches"]
            if a.points:
                e["bytes_per_point"] = round(e["dram_bytes"] / a.points, 3)
        json.dump(t, open(a.traffic, "w"), indent=1)


if __name__ == "__main__":
    main()
