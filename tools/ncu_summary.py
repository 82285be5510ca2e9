#!/usr/bin/env python
"""Turns an .ncu-rep (one kernel launch, --set full) into a small JSON summary for profiles/.
Usage: python tools/ncu_summary.py prof.ncu-rep profiles/NAME.json [--traffic-latest]"""
import csv
import json
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__issue_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__cycles_active.avg", "sm__cycles_elapsed.max",
]
STALL = "smsp__average_warp"


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    res = []
    for vals in rows[2:]:
        d = {}
        for h, u, v in zip(hdr, units, vals):
            if h in KEYS or h == "Kernel Name" or ("warp_issue_stalled" in h and h.endswith("_per_warp_active.pct")):
                try:
                    d[h] = {"value": float(v.replace(",", "")), "unit": u}
                except ValueError:
                    d[h] = v
        if "dram__bytes_read.sum" in d:
            scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}
            rd = d["dram__bytes_read.sum"]["value"] * scale[d["dram__bytes_read.sum"]["unit"]]
            wr = d["dram__bytes_write.sum"]["value"] * scale[d["dram__bytes_write.sum"]["unit"]]
            d["dram_bytes_per_launch"] = rd + wr
        stalls = {k: v["value"] for k, v in d.items() if isinstance(v, dict) and "warp_issue_stalled" in k}
        d["top_stalls"] = sorted(stalls.items(), key=lambda kv: -kv[1])[:6]
        for k in list(stalls):
            d.pop(k)
        res.append(d)
    json.dump({"source": rep, "launches": res}, open(out, "w"), indent=1)
    if "--traffic-latest" in sys.argv and res:
        json.dump({"dram_bytes_per_launch": res[0].get("dram_bytes_per_launch"), "from": out}, open("profiles/traffic_latest.json", "w"))
    print(json.dumps(res[0], indent=1)[:1500])


if __name__ == "__main__":
    main()
