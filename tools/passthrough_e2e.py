#!/usr/bin/env python
"""Host-buffer path (sky_submit / sky_wait) with and without SKY_F_PASSTHROUGH, arms alternating in one process: e2e GB/s
of raw input on a random pool (BASELINE config 2: 8 MiB chunks), a Silesia-like pool (config 3's data, where no chunk should
pass through) and a 50/50 mix, the pinned host-copy ceilings measured in the same run (H2D alone, H2D + D2H at once), and
the receiver's time (sky_decode + MD5) for the payloads each arm produced.  One JSON line per measurement.

    python tools/passthrough_e2e.py --chunks 1024 --rounds 3 > profiles/h100_passthrough_e2e.jsonl
"""
import argparse
import hashlib
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from skyplane_b200 import native, synth  # noqa: E402


def gpu_line():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def copy_ceilings(seconds=1.0):
    """Pinned 1 GiB copies, no kernel: H2D alone, and H2D + D2H running at once (GB/s per direction)."""
    import torch

    n = 1 << 30
    h_in, h_out = torch.empty(n, dtype=torch.uint8).pin_memory(), torch.empty(n, dtype=torch.uint8).pin_memory()
    d_a, d_b = torch.empty(n, dtype=torch.uint8, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def rate(both):
        def go():
            with torch.cuda.stream(s1):
                d_a.copy_(h_in, non_blocking=True)
            if both:
                with torch.cuda.stream(s2):
                    h_out.copy_(d_b, non_blocking=True)
        go()
        torch.cuda.synchronize()
        reps, t0 = 0, time.perf_counter()
        while time.perf_counter() - t0 < seconds:
            go()
            reps += 1
            torch.cuda.synchronize()
        return n * reps / (time.perf_counter() - t0) / 1e9

    out = {"h2d_gbs": rate(False), "h2d_d2h_gbs": rate(True)}
    del h_in, h_out, d_a, d_b
    torch.cuda.empty_cache()
    return out


class Pool:
    def __init__(self, kind, n_pool, cb):
        self.cb, self.stride = cb, native.round16(cb)
        self.buf = native.PinnedBuffer(n_pool * self.stride)
        self.datas = []
        for i in range(n_pool):
            k = kind if kind != "mixed" else ("random" if i % 2 else "silesia")
            d = synth.random_chunk(7000 + i, cb) if k == "random" else synth.silesia_like_chunk(7000 + i, cb)
            self.buf.view[i * self.stride : i * self.stride + cb] = d
            self.datas.append(d)

    def addr(self, i):
        return self.buf.addr + (i % len(self.datas)) * self.stride


def stream(ctx, pool, outs, n_chunks, sub, flags):
    """n_chunks chunks of the pool through len(outs) slots, sub chunks per batch -> (seconds, chunks passed through, wire bytes)."""
    cb, bound = pool.cb, native.frame_need(pool.cb)
    inflight, passed, wire = [], 0, 0
    pt = bool(flags & native.F_PASSTHROUGH)

    def pop():
        nonlocal passed, wire
        t = inflight.pop(0)
        if pt:
            lens, _, _, comp, _ = ctx.wait_ex(t)
            passed += comp.count(False)
            wire += sum(ln if c else cb for ln, c in zip(lens, comp))
        else:
            lens, _, _ = ctx.wait(t)
            wire += sum(lens)

    t0 = time.perf_counter()
    for b in range(n_chunks // sub):
        if len(inflight) == len(outs):
            pop()
        out = outs[b % len(outs)]
        inflight.append(ctx.submit([pool.addr(b * sub + i) for i in range(sub)], [cb] * sub,
                                   [out.addr + i * native.round16(bound) for i in range(sub)], [bound] * sub, flags))
    while inflight:
        pop()
    return time.perf_counter() - t0, passed, wire


def decode_time(ctx, pool, flags, reps=3):
    """The receiver's side for one batch of the pool's chunks: the payloads one sky_submit(flags) makes, through sky_decode
    (frames with flags 0, chunks sent as themselves with SKY_F_MD5) -> best seconds of `reps`, digests checked."""
    n, cb, bound = len(pool.datas), pool.cb, native.frame_need(pool.cb)
    out = native.PinnedBuffer(n * native.round16(bound))
    dec = native.PinnedBuffer(n * native.round16(cb))
    try:
        t = ctx.submit([pool.addr(i) for i in range(n)], [cb] * n, [out.addr + i * native.round16(bound) for i in range(n)], [bound] * n, flags)
        lens, dg, _, comp, _ = ctx.wait_ex(t)
        frames = [i for i in range(n) if comp[i]]
        raws = [i for i in range(n) if not comp[i]]
        best = None
        for _ in range(reps):
            t0 = time.perf_counter()
            got = {}
            if frames:
                st, d, _ = ctx.decode([out.addr + i * native.round16(bound) for i in frames], [lens[i] for i in frames],
                                      [dec.addr + i * native.round16(cb) for i in frames], [cb] * len(frames), 0)
                got.update({i: (s, x) for i, s, x in zip(frames, st, d)})
            if raws:
                st, d, _ = ctx.decode([pool.addr(i) for i in raws], [cb] * len(raws), None, [cb] * len(raws), native.F_MD5)
                got.update({i: (s, x) for i, s, x in zip(raws, st, d)})
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        assert all(got[i] == (0, hashlib.md5(pool.datas[i]).digest()) == (0, dg[i]) for i in range(n))
        return best, len(raws)
    finally:
        out.close()
        dec.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--chunks", type=int, default=1024, help="chunks streamed per arm and pool")
    ap.add_argument("--chunk-mib", type=int, default=8)
    ap.add_argument("--pool", type=int, default=64, help="distinct chunks per pool (the stream cycles through them)")
    ap.add_argument("--sub", type=int, default=128, help="chunks per sky_submit")
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3, help="off / on alternations per pool")
    ap.add_argument("--pools", default="random,silesia,mixed")
    a = ap.parse_args()
    cb = a.chunk_mib << 20
    print(json.dumps({"gpu": gpu_line(), **copy_ceilings()}), flush=True)
    ctx = native.Context(0, a.sub * native.round16(cb), max(a.sub, a.pool), a.slots)
    outs = [native.PinnedBuffer(a.sub * native.round16(native.frame_need(cb))) for _ in range(a.slots)]
    base = native.F_LZ4 | native.F_MD5
    for kind in a.pools.split(","):
        pool = Pool(kind, a.pool, cb)
        stream(ctx, pool, outs, 2 * a.sub * a.slots, a.sub, base)  # warm-up of both arms' shapes
        stream(ctx, pool, outs, 2 * a.sub * a.slots, a.sub, base | native.F_PASSTHROUGH)
        for r in range(a.rounds):
            for arm, flags in (("off", base), ("on", base | native.F_PASSTHROUGH)):
                dt, passed, wire = stream(ctx, pool, outs, a.chunks, a.sub, flags)
                print(json.dumps({"pool": kind, "arm": arm, "round": r, "e2e_gbs": a.chunks * cb / dt / 1e9, "seconds": dt,
                                  "chunks": a.chunks, "chunk_mib": a.chunk_mib, "passed_through": passed,
                                  "wire_over_raw": wire / (a.chunks * cb)}), flush=True)
        for arm, flags in (("off", base), ("on", base | native.F_PASSTHROUGH)):
            dt, n_raw = decode_time(ctx, pool, flags)
            print(json.dumps({"pool": kind, "arm": arm, "receiver_decode_md5_ms": dt * 1e3, "chunks": len(pool.datas),
                              "receiver_gbs": len(pool.datas) * cb / dt / 1e9, "raw_payloads": n_raw}), flush=True)
        pool.buf.close()
    print(json.dumps({"gpu": gpu_line(), "after": copy_ceilings()}), flush=True)
    for o in outs:
        o.close()
    ctx.close()


if __name__ == "__main__":
    main()
