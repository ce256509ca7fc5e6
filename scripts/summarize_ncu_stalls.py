#!/usr/bin/env python
"""Summarise `ncu --set full --import-source on` captures of single kernels (read here, without a GPU):
headline raw metrics + warp-stall sampling per reason + the instructions with the most samples.

    python scripts/summarize_ncu_stalls.py name=prof_x.ncu-rep ... > ncu_stalls.json
"""
import csv
import io
import json
import subprocess
import sys

RAW = ["gpu__time_duration.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
       "smsp__issue_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
       "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
       "lts__t_sector_hit_rate.pct", "launch__registers_per_thread", "sm__cycles_elapsed.max"]


def page(rep, which):
    out = subprocess.run(["ncu", "-i", rep, "--page", which, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    res = {}
    for arg in sys.argv[1:]:
        name, rep = arg.split("=", 1)
        raw = page(rep, "raw")
        hdr, units, vals = raw[0], raw[1], raw[-1]
        entry = {"kernel": vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "",
                 "raw": {k: f"{vals[hdr.index(k)]} {units[hdr.index(k)]}".strip() for k in RAW if k in hdr}}
        src = page(rep, "source")
        h = src[1]
        ix = {c: i for i, c in enumerate(h)}
        stall_cols = [c for c in h if c.startswith("stall_") and "Not Issued" not in c]
        rows = src[2:]
        tot = sum(int(r[ix["# Samples"]] or 0) for r in rows)
        agg = {c: sum(int(r[ix[c]] or 0) for r in rows) for c in stall_cols}
        entry["samples"] = tot
        entry["stall_pct"] = {k[6:]: round(100.0 * v / tot, 1) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:8]}
        top = sorted(rows, key=lambda r: -int(r[ix["# Samples"]] or 0))[:10]
        entry["top_instructions"] = [
            {"pct": round(100.0 * int(r[ix["# Samples"]] or 0) / tot, 1), "sass": " ".join(r[ix["Source"]].split()),
             "main_stall": max(stall_cols, key=lambda c: int(r[ix[c]] or 0))[6:]} for r in top]
        res[name] = entry
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
