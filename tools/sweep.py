#!/usr/bin/env python
"""Kernel-only sweeps on one GPU (device-resident inputs): stage flags x workload x chunk size.
Writes one JSON line per configuration.  Used to fill profiles/ and DESIGN.md tables; not a bench line.
Flag sets: lz4, md5, both (the fused kernel), hc (SKY_F_HC: high-ratio frames + MD5), hc-lz4 (high-ratio frames only),
checksum / hc-checksum (SKY_F_CHECKSUM: frames with LZ4's content checksum, fast or high-ratio), hc3 .. hc9 and
hc3-checksum .. hc9-checksum (SKY_F_HC_LEVEL(3..9): the high-ratio mode at that level; hc5 makes hc's frames);
block-checksum, block-checksum-checksum, hc-block-checksum, hc-block-checksum-checksum and hc3-block-checksum ..
hc9-block-checksum (SKY_F_BLOCK_CHECKSUM: the same frames with LZ4's block checksums, alone or with the content checksum);
hc-linked, hc3-linked .. hc9-linked and their -checksum / -block-checksum forms (SKY_F_LINKED: the high-ratio frames with
linked blocks); hc-opt, hc3-opt .. hc9-opt and hc-linked-opt, hc3-linked-opt .. hc9-linked-opt (SKY_F_OPTIMAL: the same
frames from the optimal parse).
--decode-from liblz4[-linked][-checksums] times the receiver on liblz4's level-0 frames made on the host from the same
input: independent or linked blocks, without checksums or with block and content checksums.
--ref-ratio adds the reference's ratio (liblz4 level 0, linked blocks) on the distinct chunks; --liblz4-level9 times liblz4
level 9 with independent blocks on all of the host's cores (the rate the reference's sender would get from that level).
--verify also times SKY_F_VERIFY's check (sky_verify_device, check only) of every frame set right after it is made, in the
same iterations: kernel_ms (frames), verify_ms (their check) and kernel_plus_verify_ms; every status must be 0.
--decode-raw [--e2ee] is a sweep of its own, on the host path: Context.decode of `compress: false` payloads (the chunks
themselves, or with --e2ee their SecretBoxes) beside the LZ4 receive of the same chunks (their frames, or the frames' boxes),
alternated call by call: kernel_ms (device events) and call_ms (host clock around the synchronous call, copies included)."""
import argparse
import json
import multiprocessing as mp
import os
import statistics
import sys
import time
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


def pool_chunks(workload, chunk_bytes):
    """The distinct chunks make_input cycles through (Silesia-like workloads), as host bytes."""
    base = min(chunk_bytes, 16 << 20)
    return [(synth.silesia_like_chunk(2000 + i, base) * (chunk_bytes // base + 1))[:chunk_bytes] for i in range(8)]


def _level9_size(data):
    from tools import hc_model

    return len(hc_model.liblz4_frame(data, 9))


def liblz4_level9_all_cores(chunks, rounds=2):
    """liblz4 level 9, independent 64 KiB blocks, one chunk per process on every core: -> (GB/s of raw input, ratio)."""
    n = os.cpu_count() or 1
    work = [c for _ in range(rounds) for c in chunks]
    work = (work * (n // len(work) + 1))[: max(n, len(work))]
    with mp.get_context("fork").Pool(n) as pool:
        pool.map(_level9_size, work[:n])  # warm the workers (library load)
        t = time.perf_counter()
        sizes = pool.map(_level9_size, work, chunksize=1)
        dt = time.perf_counter() - t
    raw = sum(map(len, work))
    return {"liblz4_level9_indep_cores": n, "liblz4_level9_gbs": raw / dt / 1e9, "liblz4_level9_ratio": raw / sum(sizes)}


def liblz4_frames(d_in, stride, n, chunk_bytes, d_out, dst_off, linked, checksums):
    """liblz4 level-0 frames (linked or independent blocks; with block and content checksums if `checksums`) of the n device chunks,
    made on the host and copied to d_out at dst_off; the frames of the first 16 distinct chunks are kept for repeats (the
    Silesia-like input cycles through 8).  -> frame lengths."""
    import hashlib

    from tools import hc_model

    cache, lens = {}, []
    for i in range(n):
        data = d_in[i * stride : i * stride + chunk_bytes].cpu().numpy().tobytes()
        key = hashlib.sha1(data).digest()
        f = cache.get(key)
        if f is None:
            f = hc_model.liblz4_frame(data, 0, linked, content_checksum=checksums, block_checksum=checksums)
            if len(cache) < 16:
                cache[key] = f
        d_out[dst_off[i] : dst_off[i] + len(f)] = torch.frombuffer(bytearray(f), dtype=torch.uint8).to(d_out.device)
        lens.append(len(f))
    return lens


def decode_raw_sweep(total_mib, chunk_mib, iters, e2ee):
    """Time sky_decode on raw payloads and on LZ4 frames of the same random chunks (host buffers, pinned), alternated.
    The sender on the same ctx makes the payloads of 16 distinct chunks; the n payloads of a call cycle through them."""
    import hashlib
    import subprocess

    chunk_bytes = int(chunk_mib * (1 << 20))
    n = max(1, (total_mib << 20) // chunk_bytes)
    stride, n_pool = native.round16(chunk_bytes), min(16, n)
    room = native.round16(native.frame_bound(chunk_bytes) + native.BOX_OVERHEAD)
    src, frames, boxes, dst = (native.PinnedBuffer(k) for k in (n_pool * stride, n_pool * room, n_pool * room, n * stride))
    for i in range(n_pool):
        src.view[i * stride : i * stride + chunk_bytes] = synth.random_chunk(4000 + i, chunk_bytes)
    want = [hashlib.md5(src.view[i * stride : i * stride + chunk_bytes]).digest() for i in range(n_pool)]
    ctx = native.Context(0, n * stride, n, 1)
    key = bytes(range(32))
    ctx.set_e2ee_key(key)
    seal = native.F_E2EE if e2ee else 0
    src_addrs, lens = [src.addr + i * stride for i in range(n_pool)], [chunk_bytes] * n_pool
    nonces = os.urandom(24 * n_pool) if e2ee else None
    frame_lens, dg, _ = ctx.wait(ctx.submit(src_addrs, lens, [frames.addr + i * room for i in range(n_pool)], [room] * n_pool,
                                            native.F_LZ4 | native.F_MD5 | seal, nonces))
    assert dg == want
    if e2ee:
        box_lens, dg, _ = ctx.wait(ctx.submit(src_addrs, lens, [boxes.addr + i * room for i in range(n_pool)], [room] * n_pool,
                                              native.F_MD5 | seal, nonces))
        assert dg == want
    cyc = [i % n_pool for i in range(n)]
    dst_addrs = [dst.addr + i * stride for i in range(n)]
    legs = {"lz4": ([frames.addr + k * room for k in cyc], [frame_lens[k] for k in cyc], dst_addrs, seal),
            "raw": ([boxes.addr + k * room for k in cyc], [box_lens[k] for k in cyc], dst_addrs, native.F_MD5 | seal) if e2ee else
                   ([src.addr + k * stride for k in cyc], [chunk_bytes] * n, None, native.F_MD5)}
    kms, wall, ok = {k: [] for k in legs}, {k: [] for k in legs}, {k: True for k in legs}
    for it in range(iters + 1):
        for name, (addrs, plens, out, flags) in legs.items():
            t = time.perf_counter()
            st, dg, k = ctx.decode(addrs, plens, out, [chunk_bytes] * n, flags)
            w = (time.perf_counter() - t) * 1e3
            ok[name] = ok[name] and all(x == 0 for x in st) and dg == [want[k] for k in cyc]
            if out is not None:
                ok[name] = ok[name] and all(dst.view[i * stride : i * stride + chunk_bytes] == src.view[k * stride : k * stride + chunk_bytes]
                                            for i, k in list(enumerate(cyc))[:: max(1, n // 8)])
            if it:
                kms[name].append(k)
                wall[name].append(w)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        gpu = q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        gpu = torch.cuda.get_device_name(0)
    for name in legs:
        k = statistics.median(kms[name])
        print(json.dumps({"workload": "random", "chunk_mib": float(chunk_mib), "chunks": n, "distinct_chunks": n_pool, "path": "Context.decode (host buffers)",
                          "payload": ("box of " if e2ee else "") + ("lz4 frame" if name == "lz4" else "raw chunk"), "launches_per_call": {
                              "lz4": 5 if e2ee else 2, "raw": 4 if e2ee else 1}[name], "kernel_ms": k, "kernel_ms_min": min(kms[name]),
                          "kernel_ms_max": max(kms[name]), "kernel_ms_covers": "index + decode + MD5 (the box open is outside it)" if name == "lz4"
                          else ("open + MD5" if e2ee else "MD5"), "call_ms": statistics.median(wall[name]), "raw_output_gbs": n * chunk_bytes / k / 1e6,
                          "iters": iters, "all_ok": ok[name], "gpu": gpu}), flush=True)
    ctx.close()
    for b in (src, frames, boxes, dst):
        b.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-mib", type=int, default=2048)
    ap.add_argument("--sizes-mib", default="8")
    ap.add_argument("--workloads", default="random,silesia")
    ap.add_argument("--flags", default="lz4,md5,both")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--decode", action="store_true", help="also time the receiver-side decode + MD5 of the frames")
    ap.add_argument("--decode-from", default="both", help="flag set whose frames --decode times (both, hc, checksum, ...), or liblz4[-linked][-checksums] "
                    "(frames made on the host by liblz4: linked blocks, block and content checksums)")
    ap.add_argument("--ref-ratio", action="store_true", help="also the reference's ratio on the distinct chunks (CPU)")
    ap.add_argument("--liblz4-level9", action="store_true", help="also liblz4 level 9 on all host cores (CPU)")
    ap.add_argument("--verify", action="store_true", help="also time the frame check (SKY_F_VERIFY) of each flag set's frames")
    ap.add_argument("--decode-raw", action="store_true", help="only: Context.decode of raw (`compress: false`) payloads beside the LZ4 "
                    "receive of the same random chunks, alternated (--total-mib, the first of --sizes-mib, --iters)")
    ap.add_argument("--e2ee", action="store_true", help="with --decode-raw: the payloads are SecretBoxes")
    a = ap.parse_args()
    if a.decode_raw:
        return decode_raw_sweep(a.total_mib, float(a.sizes_mib.split(",")[0]), a.iters, a.e2ee)
    dev = torch.device("cuda", 0)
    FL = {"lz4": native.F_LZ4, "md5": native.F_MD5, "both": 0, "hc": native.F_HC, "hc-lz4": native.F_HC | native.F_LZ4,
          "checksum": native.F_CHECKSUM, "hc-checksum": native.F_HC | native.F_CHECKSUM}
    for lv in range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1):
        FL[f"hc{lv}"] = native.hc_level_flag(lv)
        FL[f"hc{lv}-checksum"] = native.hc_level_flag(lv) | native.F_CHECKSUM
        FL[f"hc{lv}-block-checksum"] = native.hc_level_flag(lv) | native.F_BLOCK_CHECKSUM
    for k in [k for k in FL if k.startswith("hc") and k != "hc-lz4"]:  # hc5-checksum -> hc5-linked-checksum
        head, _, tail = k.partition("-")
        FL[f"{head}-linked" + (f"-{tail}" if tail else "")] = FL[k] | native.F_LINKED
    for k in [k for k in FL if k.split("-")[0] in [f"hc{lv}" for lv in range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1)] + ["hc"]
              and k.removeprefix(k.split("-")[0]) in ("", "-linked")]:  # hc5 -> hc5-opt, hc5-linked -> hc5-linked-opt
        FL[f"{k}-opt"] = FL[k] | native.F_OPTIMAL
    FL.update({"block-checksum": native.F_BLOCK_CHECKSUM, "block-checksum-checksum": native.F_BLOCK_CHECKSUM | native.F_CHECKSUM,
               "hc-block-checksum": native.F_HC | native.F_BLOCK_CHECKSUM,
               "hc-block-checksum-checksum": native.F_HC | native.F_BLOCK_CHECKSUM | native.F_CHECKSUM})
    for wl in a.workloads.split(","):
        for sz in a.sizes_mib.split(","):
            chunk_bytes = int(float(sz) * (1 << 20))
            n = max(1, (a.total_mib << 20) // chunk_bytes)
            # (CPU legs first: their worker processes fork before this process has a CUDA context)
            if wl == "silesia" and (a.ref_ratio or a.liblz4_level9):
                import oracle.reflib as ref

                chunks = pool_chunks(wl, chunk_bytes)
                row = {"workload": wl, "chunk_mib": float(sz), "distinct_chunks": len(chunks)}
                if a.ref_ratio:
                    row["reference_ratio"] = sum(map(len, chunks)) / sum(len(ref.lz4f_compress(c)) for c in chunks)
                if a.liblz4_level9:
                    row.update(liblz4_level9_all_cores(chunks))
                print(json.dumps(row), flush=True)
            d_in, stride = make_input(wl, n, chunk_bytes, dev)
            bound = native.frame_need(chunk_bytes, checksum=True, block_checksum=True)  # (room for content and block checksums)
            so = native.round16(bound)
            d_out = torch.empty(n * so + 64, dtype=torch.uint8, device=dev)
            ctx = native.Context(0, n * stride, n, 0)
            src_off = [i * stride for i in range(n)]
            dst_off = [i * so for i in range(n)]
            for fl in a.flags.split(","):
                ms, vms, vok = [], [], True
                for it in range(a.iters + 1):
                    torch.cuda.synchronize()
                    out_lens, dg, kms = ctx.process_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, [bound] * n, FL[fl], 0)
                    if a.verify:  # the check of the frames just made, alternating with their making
                        xxh = None
                        if FL[fl] & native.F_CHECKSUM:  # the content checksums the frames carry, from behind their EndMarks
                            tail = [d_out[o + l - 4 : o + l].cpu().numpy().tobytes() for o, l in zip(dst_off, out_lens)]
                            xxh = [int.from_bytes(t, "little") for t in tail]
                        st, _, v = ctx.verify_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, out_lens,
                                                     None, xxh, FL[fl] or native.F_LZ4, 0)
                        vok = vok and all(x == 0 for x in st)
                        if it:
                            vms.append(v)
                    if it:
                        ms.append(kms)
                k = statistics.median(ms)
                tot = n * chunk_bytes
                row = {"workload": wl, "chunk_mib": float(sz), "chunks": n, "flags": fl, "kernel_ms": k, "raw_input_gbs": tot / k / 1e6,
                       "ratio": (tot / sum(out_lens)) if sum(out_lens) else None, "per_stream_gbs": chunk_bytes / k / 1e6}
                if a.verify:
                    v = statistics.median(vms)
                    row.update({"verify_ms": v, "kernel_plus_verify_ms": k + v, "verify_raw_gbs": tot / v / 1e6, "verify_all_ok": vok})
                print(json.dumps(row), flush=True)
            if a.decode:
                # receiver side: decode the frames just produced (d_out) back into a fresh buffer + MD5 of the result
                if a.decode_from.startswith("liblz4"):
                    out_lens = liblz4_frames(d_in, stride, n, chunk_bytes, d_out, dst_off, "-linked" in a.decode_from,
                                             a.decode_from.endswith("-checksums"))
                    dg = ctx.process_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, [bound] * n,
                                            native.F_MD5, 0)[1]
                else:
                    out_lens, dg, _ = ctx.process_device(d_in.data_ptr(), src_off, [chunk_bytes] * n, d_out.data_ptr(), dst_off, [bound] * n,
                                                         FL[a.decode_from], 0)
                d_back = torch.empty_like(d_in)
                ms = []
                for it in range(a.iters + 1):
                    st, dg2, kms = ctx.decode_device(d_out.data_ptr(), dst_off, out_lens, d_back.data_ptr(), src_off, [chunk_bytes] * n, 0)
                    if it:
                        ms.append(kms)
                ok = all(x == 0 for x in st) and dg2 == dg and bool(torch.equal(d_back[: n * stride - (stride - chunk_bytes)], d_in[: n * stride - (stride - chunk_bytes)]))
                k = statistics.median(ms)
                print(json.dumps({"workload": wl, "chunk_mib": float(sz), "chunks": n, "flags": "decode+md5", "frames_from": a.decode_from, "kernel_ms": k,
                                  "raw_output_gbs": n * chunk_bytes / k / 1e6, "roundtrip_ok": ok}), flush=True)
                del d_back
            ctx.close()
            del d_in, d_out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
