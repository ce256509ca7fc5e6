"""Summarise ncu CSV logs into small summary files (a launch table, or the DRAM / L2 traffic of one step).
  python scripts/summarize_ncu.py launches <csv> <out.csv> "<title>"
  python scripts/summarize_ncu.py traffic  <csv> <out.json>"""
import collections
import csv
import json
import sys


def read(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    return list(csv.DictReader(lines))


def to_ms(v, unit):
    v = float(v.replace(",", ""))
    u = unit.lower()
    return v / 1e6 if u.startswith("ns") else v / 1e3 if u.startswith("us") else v * 1e3 if u in ("s", "second") else v


def to_bytes(v, unit):
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[unit.lower()]


def launches(path, out, title):
    agg = collections.defaultdict(lambda: [0, 0.0])
    for r in read(path):
        if r["Metric Name"] != "gpu__time_duration.sum":
            continue
        k = r["Kernel Name"].split("(")[0]
        agg[k][0] += 1
        agg[k][1] += to_ms(r["Metric Value"], r["Metric Unit"])
    tot = sum(v[1] for v in agg.values())
    rows = [f"# {title}", "# per-launch times under ncu are cold-cache and serialised: compare SHARES",
            "kernel,launches,total_ms,share"]
    for k, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        rows.append(f"{k},{n},{ms:.3f},{ms / tot:.4f}")
    open(out, "w").write("\n".join(rows) + "\n")
    print("\n".join(rows[:12]))


def traffic(path, out):
    per = collections.defaultdict(dict)
    for r in read(path):
        per[r["ID"]][r["Metric Name"]] = (r["Metric Value"], r["Metric Unit"])
        per[r["ID"]]["name"] = r["Kernel Name"].split("(")[0]
    n = 0
    tot = collections.Counter()
    for _id, m in per.items():
        if "dram__bytes_read.sum" not in m:
            continue
        n += 1
        tot["read"] += to_bytes(*m["dram__bytes_read.sum"])
        tot["write"] += to_bytes(*m["dram__bytes_write.sum"])
        tot["ms"] += to_ms(*m["gpu__time_duration.sum"])
        if "lts__t_bytes.sum" in m:
            tot["l2"] += to_bytes(*m["lts__t_bytes.sum"])
        k = "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"
        if k in m:
            tot["tensor_pct_x_ms"] += float(m[k][0]) * to_ms(*m["gpu__time_duration.sum"])
    res = {"kernel": "tc_igemm_kernel", "launches": n,
           "dram_bytes_per_launch": (tot["read"] + tot["write"]) / max(n, 1),
           "dram_read_bytes_total": tot["read"], "dram_write_bytes_total": tot["write"],
           "l2_bytes_total": tot["l2"], "ncu_time_ms_total": tot["ms"],
           "tensor_pipe_active_pct_time_weighted": tot["tensor_pct_x_ms"] / max(tot["ms"], 1e-9),
           "note": "one step of bench.py (batch 32), all tc_igemm launches; ncu serialises launches and runs them cold-cache"}
    json.dump(res, open(out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], sys.argv[4])
    else:
        traffic(sys.argv[2], sys.argv[3])
