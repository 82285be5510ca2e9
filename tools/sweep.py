#!/usr/bin/env python
"""Kernel-only sweeps on one GPU (device-resident inputs): stage flags x workload x chunk size.
Writes one JSON line per configuration.  Used to fill profiles/ and DESIGN.md tables; not a bench line."""
import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from skyplane_b200 import native, synth  # noqa: E402


def make_input(workload, n_chunks, chunk_bytes, dev):
    stride = native.round16(chunk_bytes)
    buf = torch.empty(n_chunks * stride + 64, dtype=torch.uint8, device=dev)
    if workload == "random":
        g = torch.Generator(device=dev)
        g.manual_seed(1234)
        step = 1 << 28
        for o in range(0, buf.numel(), step):
            e = min(buf.numel(), o + step)
            buf[o:e] = torch.randint(0, 256, (e - o,), dtype=torch.uint8, device=dev, generator=g)
    elif workload == "zeros":
        buf.zero_()
    else:
        base = min(chunk_bytes, 16 << 20)
        pool = [synth.silesia_like_chunk(2000 + i, base) for i in range(8)]
        pool = [torch.frombuffer(bytearray((p * (chunk_bytes // base + 1))[:chunk_bytes]), dtype=torch.uint8).to(dev) for p in pool]
        for i in range(n_chunks):
            buf[i * stride : i * stride + chunk_bytes] = pool[i % len(pool)]
    return buf, stride


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-mib", type=int, default=2048)
    ap.add_argument("--sizes-mib", default="8")
    ap.add_argument("--workloads", default="random,silesia")
    ap.add_argument("--flags", default="lz4,md5,both")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--decode", action="store_true", help="also time the receiver-side decode + MD5 of the frames")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    FL = {"lz4": native.F_LZ4, "md5": native.F_MD5, "both": 0}
    for wl in a.workloads.split(","):
        for sz in a.sizes_mib.split(","):
            chunk_bytes = int(float(sz) * (1 << 20))
            n = max(1, (a.total_mib << 20) // chunk_bytes)
            d_in, stride = make_input(wl, n, chunk_bytes, dev)
            bound = native.frame_bound(chunk_bytes)
            so = native.round16(bound)
            d_out = torch.empty(n * so + 64, dtype=torch.uint8, device=dev)
            ctx = native.Context(0, n * stride, n, 0)
            src_off = [i * stride for i in range(n)]
            dst_off = [i * so for i in range(n)]
            for fl in a.flags.split(","):
                ms = []
                for it in range(a.iters + 1):
                    torch.cuda.synchronize()
                    out_lens, dg, kms = ctx.process_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, [bound] * n, FL[fl], 0)
                    if it:
                        ms.append(kms)
                k = statistics.median(ms)
                tot = n * chunk_bytes
                print(json.dumps({"workload": wl, "chunk_mib": float(sz), "chunks": n, "flags": fl, "kernel_ms": k, "raw_input_gbs": tot / k / 1e6,
                                  "ratio": (tot / sum(out_lens)) if sum(out_lens) else None, "per_stream_gbs": chunk_bytes / k / 1e6}), flush=True)
            if a.decode:
                # receiver side: decode the frames just produced (d_out) back into a fresh buffer + MD5 of the result
                out_lens, dg, _ = ctx.process_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, [bound] * n, 0, 0)
                d_back = torch.empty_like(d_in)
                ms = []
                for it in range(a.iters + 1):
                    st, dg2, kms = ctx.decode_device(d_out.data_ptr(), dst_off, out_lens, d_back.data_ptr(), src_off, [chunk_bytes] * n, 0)
                    if it:
                        ms.append(kms)
                ok = all(x == 0 for x in st) and dg2 == dg and bool(torch.equal(d_back[: n * stride - (stride - chunk_bytes)], d_in[: n * stride - (stride - chunk_bytes)]))
                k = statistics.median(ms)
                print(json.dumps({"workload": wl, "chunk_mib": float(sz), "chunks": n, "flags": "decode+md5", "kernel_ms": k,
                                  "raw_output_gbs": n * chunk_bytes / k / 1e6, "roundtrip_ok": ok}), flush=True)
                del d_back
            ctx.close()
            del d_in, d_out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
