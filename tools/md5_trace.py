#!/usr/bin/env python
"""Where the fused kernel's MD5 chains lose time to the compressors (GPU).

    python tools/build_variants.py md5_trace                       # here or anywhere nvcc is
    python tools/md5_trace.py --out DIR [--rounds 5] [--lib NAME=PATH ...]

Runs config 2 (1024 x 8 MiB random chunks, device-resident) in worker processes, one library each (SKYCHUNK_LIB),
alternating the untraced build (the in-tree libskychunk.so unless --lib says otherwise) and the traced one
(tools/bin/libskychunk_md5_trace.so).  Each worker times MD5-only, LZ4-only and fused passes, alternated, `--rounds`
times; the traced worker then reads the trace of its last fused pass.  For every MD5 warp the report gives

  * cycles per 64-byte block while a compressor CTA on its SM is still claiming blocks, and after that;
  * ring-wait cycles per block (the cp.async wait before round 2) in the same two windows;
  * the tail: the time from the warp's last chain block to the kernel's end.

DIR gets md5_trace_timing.jsonl (one line per worker), md5_trace_warps.jsonl (one line per MD5 warp) and
md5_trace_summary.json.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

TRACE_GROUPS, TRACE_STAMPS, TRACE_EVERY, TRACE_CTAS = 256, 512, 1024, 1024  # md5.cuh / skychunk.cu (SKY_MD5_TRACE)
FLAGS = {"md5": 2, "lz4": 1, "both": 0}


def dtypes():
    import numpy as np

    stamp = np.dtype([("t", "<u8"), ("clk", "<u4"), ("wait", "<u4")])
    md5 = np.dtype([("smid", "<u4"), ("warpid", "<u4"), ("cta", "<u4"), ("stamps", "<u4"), ("t0", "<u8"), ("t1", "<u8"),
                    ("c0", "<u4"), ("c1", "<u4"), ("wait", "<u4"), ("blocks", "<u4"), ("s", stamp, (TRACE_STAMPS,))])
    cta = np.dtype([("smid", "<u4"), ("digest", "<u4"), ("claims", "<u4"), ("pad", "<u4"), ("entry", "<u8"), ("first", "<u8"),
                    ("last", "<u8"), ("exhausted", "<u8")])
    assert md5.itemsize == 48 + 16 * TRACE_STAMPS and cta.itemsize == 48
    return md5, cta


# ------------------------------------------------------------------------------------------------ worker (one library)
def worker(a):
    import numpy as np
    import torch

    from skyplane_b200 import native

    n, chunk = a.chunks, a.chunk_mib << 20
    dev = torch.device("cuda", 0)
    stride = native.round16(chunk)
    d_in = torch.empty(n * stride + 64, dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(1000)
    for o in range(0, d_in.numel(), 1 << 28):
        e = min(d_in.numel(), o + (1 << 28))
        d_in[o:e] = torch.randint(0, 256, (e - o,), dtype=torch.uint8, device=dev, generator=g)
    bound = native.frame_bound(chunk)
    so = native.round16(bound)
    d_out = torch.empty(n * so + 64, dtype=torch.uint8, device=dev)
    ctx = native.Context(0, n * stride, n, 0)
    src_off, dst_off = [i * stride for i in range(n)], [i * so for i in range(n)]

    def run(fl):
        torch.cuda.synchronize()
        return ctx.process_device(d_in.data_ptr(), src_off, [chunk] * n, d_out.data_ptr(), dst_off, [bound] * n, FLAGS[fl], 0)

    for fl in FLAGS:  # warm-up
        run(fl)
    ms = {fl: [] for fl in FLAGS}
    digests = None
    for _ in range(a.rounds):
        for fl in ("md5", "lz4", "both"):  # the fused pass last: its trace is the one read below
            r = run(fl)
            ms[fl].append(r[2])
            if fl == "both":
                digests = r[1]
    line = {"lib": a.tag, "kernel_ms": ms, "median_ms": {k: statistics.median(v) for k, v in ms.items()},
            "digest0": digests[0].hex(), "chunks": n, "chunk_mib": a.chunk_mib}
    if a.fetch:
        L = native.lib()
        md5_t, cta_t = dtypes()
        md5 = np.zeros(TRACE_GROUPS, dtype=md5_t)
        ctas = np.zeros(TRACE_CTAS, dtype=cta_t)
        L.sky_md5_trace_fetch.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64]
        L.sky_md5_trace_fetch.restype = ctypes.c_int
        # the records of the last fused pass: clear them, run one more fused pass, read them
        rc = L.sky_md5_trace_fetch(0, md5.ctypes.data, md5.nbytes, ctas.ctypes.data, ctas.nbytes)
        assert rc == 0, rc
        r = run("both")
        line["traced_pass_ms"] = r[2]
        rc = L.sky_md5_trace_fetch(0, md5.ctypes.data, md5.nbytes, ctas.ctypes.data, ctas.nbytes)
        assert rc == 0, rc
        np.save(a.fetch + ".md5.npy", md5)
        np.save(a.fetch + ".cta.npy", ctas)
    ctx.close()
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------ analysis
def analyse(md5_path, cta_path, kernel_ms):
    """-> (per-warp rows, summary) from one traced fused pass."""
    import numpy as np

    md5 = np.load(md5_path)
    ctas = np.load(cta_path)
    used = ctas[ctas["entry"] > 0]
    warps = md5[md5["blocks"] > 0]
    t_start = int(used["entry"].min())
    t_end = int(max(used["exhausted"].max(), warps["t1"].max()))
    comp = used[used["digest"] == 0]
    comp_end = int(comp["exhausted"].max())  # the last compressor CTA found no more blocks
    rows = []
    for w in warps:
        mates = comp[comp["smid"] == w["smid"]]
        ex = int(mates["exhausted"].max()) if len(mates) else t_start  # the compressor beside it stops claiming here
        ts = [int(w["t0"])] + [int(x) for x in w["s"]["t"][: w["stamps"]]]
        cs = [int(w["c0"])] + [int(x) for x in w["s"]["clk"][: w["stamps"]]]
        ws = [0] + [int(x) for x in w["s"]["wait"][: w["stamps"]]]
        acc = {"during": [0, 0, 0], "after": [0, 0, 0], "straddle": [0, 0, 0]}  # blocks, cycles, wait cycles
        for k in range(1, len(ts)):
            win = "during" if ts[k] <= ex else ("after" if ts[k - 1] >= ex else "straddle")
            acc[win][0] += TRACE_EVERY
            acc[win][1] += (cs[k] - cs[k - 1]) & 0xFFFFFFFF
            acc[win][2] += (ws[k] - ws[k - 1]) & 0xFFFFFFFF
        total_cyc = (int(w["c1"]) - int(w["c0"])) & 0xFFFFFFFF
        ghz = total_cyc / max(1, int(w["t1"]) - int(w["t0"]))
        row = {"smid": int(w["smid"]), "cta": int(w["cta"]), "warpid": int(w["warpid"]), "blocks": int(w["blocks"]),
               "compressor_ctas_on_sm": int(len(mates)), "digest_ctas_on_sm": int(((used["smid"] == w["smid"]) & (used["digest"] == 1)).sum()),
               "start_ms": (int(w["t0"]) - t_start) / 1e6, "chain_ms": (int(w["t1"]) - int(w["t0"])) / 1e6,
               "sm_compress_end_ms": (ex - t_start) / 1e6, "tail_ms": (t_end - int(w["t1"])) / 1e6, "sm_ghz": ghz,
               "cycles_per_block": total_cyc / max(1, int(w["blocks"])), "wait_per_block": int(w["wait"]) / max(1, int(w["blocks"]))}
        for win, (b, c, wt) in acc.items():
            if win == "straddle":
                continue
            row[f"{win}_blocks"] = b
            row[f"{win}_cycles_per_block"] = c / b if b else None
            row[f"{win}_wait_per_block"] = wt / b if b else None
        # what the chain would have taken had the during-window blocks run at the after-window rate
        if acc["during"][0] and acc["after"][0]:
            r_after = acc["after"][1] / acc["after"][0]
            row["during_excess_ms"] = (acc["during"][1] - r_after * acc["during"][0]) / ghz / 1e6
            row["during_wait_excess_ms"] = (acc["during"][2] - acc["after"][2] / acc["after"][0] * acc["during"][0]) / ghz / 1e6
        rows.append(row)

    def mean(key):
        v = [r[key] for r in rows if r.get(key) is not None]
        return statistics.mean(v) if v else None

    summary = {"kernel_span_ms": (t_end - t_start) / 1e6, "traced_kernel_ms": kernel_ms, "compressors_end_ms": (comp_end - t_start) / 1e6,
               "md5_warps": len(rows), "compressor_ctas": int(len(comp)), "digest_ctas": int((used["digest"] == 1).sum()),
               "chain_ms_max": max(r["chain_ms"] for r in rows), "chain_ms_mean": mean("chain_ms"),
               "last_chain_end_ms": max(r["start_ms"] + r["chain_ms"] for r in rows),
               "chain_start_ms_max": max(r["start_ms"] for r in rows), "tail_ms_min": min(r["tail_ms"] for r in rows),
               "sm_ghz": mean("sm_ghz")}
    for key in ("cycles_per_block", "wait_per_block", "during_cycles_per_block", "after_cycles_per_block", "during_wait_per_block",
                "after_wait_per_block", "during_excess_ms", "during_wait_excess_ms", "sm_compress_end_ms"):
        summary[f"{key}_mean"] = mean(key)
    return rows, summary


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.applications.graphics"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return repr(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the records")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--chunks", type=int, default=1024)
    ap.add_argument("--chunk-mib", type=int, default=8)
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH: untraced builds to alternate with the traced one "
                    "(default: the in-tree libskychunk.so)")
    ap.add_argument("--trace-lib", default=str(ROOT / "tools" / "bin" / "libskychunk_md5_trace.so"))
    ap.add_argument("--pairs", type=int, default=2, help="alternations of the untraced and traced workers")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tag", default="", help=argparse.SUPPRESS)
    ap.add_argument("--fetch", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)

    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    libs = [tuple(s.split("=", 1)) for s in a.lib] or [("default", str(ROOT / "skyplane_b200" / "libskychunk.so"))]
    if not Path(a.trace_lib).exists():
        raise SystemExit(f"{a.trace_lib} is missing: run tools/build_variants.py md5_trace first")
    facts = {"gpu": gpu_facts()}
    print(json.dumps(facts), flush=True)
    lines = []
    for p in range(a.pairs):
        for tag, path in libs + [("md5_trace", a.trace_lib)]:
            fetch = str(out / "md5_trace") if (tag == "md5_trace" and p == a.pairs - 1) else ""
            cmd = [sys.executable, __file__, "--worker", "--tag", tag, "--rounds", str(a.rounds), "--chunks", str(a.chunks),
                   "--chunk-mib", str(a.chunk_mib)] + (["--fetch", fetch] if fetch else [])
            r = subprocess.run(cmd, capture_output=True, text=True, env={**os.environ, "SKYCHUNK_LIB": path}, cwd=str(ROOT))
            if r.returncode != 0:
                raise SystemExit(f"worker {tag} failed:\n{r.stderr[-3000:]}")
            line = json.loads(r.stdout.strip().splitlines()[-1])
            line["pair"] = p
            lines.append(line)
            print(json.dumps({k: line[k] for k in ("lib", "pair", "median_ms")}), flush=True)
    with open(out / "md5_trace_timing.jsonl", "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")
    traced = [x for x in lines if x["lib"] == "md5_trace"]
    rows, summary = analyse(str(out / "md5_trace.md5.npy"), str(out / "md5_trace.cta.npy"), traced[-1]["traced_pass_ms"])
    with open(out / "md5_trace_warps.jsonl", "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")

    def med(tag, fl):
        return statistics.median(v for x in lines if x["lib"] == tag for v in x["kernel_ms"][fl])

    summary["gpu"] = facts["gpu"]
    summary["timing_medians_ms"] = {tag: {fl: med(tag, fl) for fl in FLAGS} for tag in [t for t, _ in libs] + ["md5_trace"]}
    base = libs[0][0]
    summary["fused_minus_md5_ms"] = med(base, "both") - med(base, "md5")
    summary["traced_vs_untraced_fused"] = med("md5_trace", "both") / med(base, "both") - 1
    summary["traced_vs_untraced_md5"] = med("md5_trace", "md5") / med(base, "md5") - 1
    summary["digests_agree"] = len({x["digest0"] for x in lines}) == 1
    (out / "md5_trace_summary.json").write_text(json.dumps(summary, indent=1) + "\n")
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
