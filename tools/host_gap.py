#!/usr/bin/env python
"""The host time between two device-path passes (GPU): where a bench.py step spends what its kernel does not.

    python tools/host_gap.py [--calls 20] [--chunks 1024] [--chunk-mib 8] [--per-value] [--out FILE]

Runs Context.process_device on config 2 (1024 x 8 MiB random chunks in HBM) the way bench.py does, `--calls` times
after a warm-up, and takes the host clock around each phase of each call:

  args     the Python side before the C call: the four offset / length lists become ctypes arrays (as Context.process_device
           builds them; --per-value: one ctypes argument per value, as it did before)
  call     sky_process_device itself: validation, batch metadata, its copies, the launch, the wait, the result copies
  results  the Python side after it: the lengths as a list, the digests as 16-byte slices

and CUDA events on the launching stream around each whole call (`step`).  `call - kernel` is the C side's host work and
its metadata copies plus the wake-up after the kernel; `step - kernel` is what one bench.py step pays beyond the kernel.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--chunks", type=int, default=1024)
    ap.add_argument("--chunk-mib", type=int, default=8)
    ap.add_argument("--out", default="")
    ap.add_argument("--per-value", action="store_true", help="time the phases with the conversions Context.process_device "
                    "made before it built its arrays in one call: one ctypes argument per value, one index per digest")
    a = ap.parse_args()

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
    lens, caps = [chunk] * n, [bound] * n
    stream = torch.cuda.current_stream().cuda_stream
    L = native.lib()

    def phased():
        """Context.process_device's own steps, one clock reading between each."""
        t0 = time.perf_counter()
        out = (ctypes.c_uint64 * n)()
        md5 = (ctypes.c_ubyte * (16 * n))()
        ms = ctypes.c_float(0)
        if a.per_value:  # one ctypes argument per value
            U = ctypes.c_uint64 * n
            arrays = (U(*src_off), U(*lens), U(*dst_off), U(*caps))
        else:
            arrays = tuple(native._u64_array(x, n) for x in (src_off, lens, dst_off, caps))
        t1 = time.perf_counter()
        rc = L.sky_process_device(ctx._h, n, d_in.data_ptr(), arrays[0], arrays[1], d_out.data_ptr(), arrays[2], arrays[3], 0, stream,
                                  out, md5, ctypes.byref(ms))
        t2 = time.perf_counter()
        assert rc == 0, rc
        if a.per_value:  # an index per digest
            raw = bytes(md5)
            res = list(out), [raw[16 * i: 16 * i + 16] for i in range(n)], ms.value
        else:
            res = out[:], native._digests(bytes(md5)), ms.value
        t3 = time.perf_counter()
        return res, (t1 - t0, t2 - t1, t3 - t2)

    def whole():
        return ctx.process_device(d_in.data_ptr(), src_off, lens, d_out.data_ptr(), dst_off, caps, 0, stream)

    for _ in range(3):
        whole()
    torch.cuda.synchronize()
    rows = {"args": [], "call": [], "results": [], "kernel": [], "step_phased": [], "step": []}
    for _ in range(a.calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res, (ta, tc, tr) = phased()
        e1.record()
        torch.cuda.synchronize()
        rows["args"].append(ta * 1e3)
        rows["call"].append(tc * 1e3)
        rows["results"].append(tr * 1e3)
        rows["kernel"].append(res[2])
        rows["step_phased"].append(e0.elapsed_time(e1))
        # the same call through Context.process_device, as bench.py makes it
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        whole()
        e3.record()
        torch.cuda.synchronize()
        rows["step"].append(e2.elapsed_time(e3))
    # back to back, as bench.py's timed loop runs them: one pair of events around all calls
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kms = []
    e0.record()
    for _ in range(a.calls):
        kms.append(whole()[2])
    e1.record()
    torch.cuda.synchronize()
    loop_step = e0.elapsed_time(e1) / a.calls
    med = {k: statistics.median(v) for k, v in rows.items()}
    summary = {"calls": a.calls, "phases": "per-value" if a.per_value else "current", "chunks": n, "chunk_mib": a.chunk_mib, "median_ms": med,
               "call_minus_kernel_ms": med["call"] - med["kernel"], "step_minus_kernel_ms": med["step"] - med["kernel"],
               "loop_step_ms": loop_step, "loop_kernel_ms": statistics.mean(kms), "loop_gap_ms": loop_step - statistics.mean(kms),
               "gpu": torch.cuda.get_device_name(0)}
    line = json.dumps(summary)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
