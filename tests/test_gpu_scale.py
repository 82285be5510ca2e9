"""GPU tests of the stage at the batch widths and sizes it admits beyond the rest of the suite.

(A) Wide batches of small ragged chunks: the widths are derived from the SM count, so that warps 1..3 of the sender's
digest CTAs and of the receiver's MD5 warps hash a group, and so that a warp takes a second group.  (B) The benchmark's
own batches over 4 GiB (BASELINE configs 2 and 3): every chunk's frame, digest and round trip, not just the first ones.
(C) Single chunks of 512 MiB (MD5's high length word) and over 4 GiB (64-bit block positions, XXH32's length mod 2^32,
64-bit content size, more than 65536 blocks).

Every expected value comes from the CPU: hashlib, liblz4 (which verifies block and content checksums), the sequential
twins of the compressors (tools/tile_model.py, tools/hc_model.py) and the C oracle's SecretBox.  The only comparison of
the GPU with itself is "the same bytes at another offset give the same frame", and that frame is checked against the
twin too.  Tests that need more free HBM or host memory than the machine has skip and say how much."""
import ctypes
import hashlib
import math
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import oracle.reflib as ref
from gpu_util import run_device
from skyplane_b200 import native, synth
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import hc_model  # noqa: E402
import tile_model  # noqa: E402
from test_checksum_format import with_content_checksum  # noqa: E402
from test_gpu_block_checksum import run_guarded  # noqa: E402
from test_gpu_receiver_conformance import guarded_decode  # noqa: E402
from test_gpu_verify import check_repair, parse_frame, run_verify  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800, method="thread")]

CK, BC, LZ4, MD5 = native.F_CHECKSUM, native.F_BLOCK_CHECKSUM, native.F_LZ4, native.F_MD5
HC3, LINKED = native.hc_level_flag(3), native.F_LINKED
BLOCK = native.BLOCK_BYTES
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
EDGE_LENS = [0, 1, 12, 13, 63, 64, 65535, 65536, 65537, 131073]
GIB = 1 << 30


# ------------------------------------------------------------------------------------------------ widths and fixtures
@pytest.fixture(scope="module")
def sm():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def sender_width(sm):  # digest CTAs = max(ceil(groups / 4), sm / 4): warps 1..3 get a group past sm / 4 groups
    return 32 * (sm // 4) + 1


def receiver_width(sm):  # one decode CTA per SM: group g goes to warp g / sm
    return 32 * sm + 1


def receiver_second_round(sm):  # past 4 * sm groups a receiver MD5 warp takes a second group
    return 128 * sm + 1


def sender_second_round(sm):  # digest CTAs are capped at the grid (2 per SM): past 8 * sm groups a warp takes a second
    return 256 * sm + 1


def groups(n):
    return -(-n // 32)


@pytest.fixture(scope="module")
def ctx(sm):
    c = native.Context(0, GIB, sender_second_round(sm), 0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def twin_opts():
    k = native.kernel_config()
    return tile_model.kernel_opts(k["lz4_entries"], k["seg_slots"], k["max_step_log"])


@pytest.fixture(scope="module")
def sources():
    """Four kinds of content the ragged chunks are sliced from: random, zeros, text, Silesia-like."""
    rng = np.random.default_rng(1234)
    text = b"".join(b"%d: it was the best of times, it was the worst of times, it was the age of %s;\n"
                    % (k, (b"wisdom", b"foolishness", b"belief")[k % 3]) for k in range(70000))
    return [rng.bytes(4 << 20), bytes(1 << 20), text[: 4 << 20], synth.silesia_like_chunk(77, 4 << 20)]


def ragged_chunks(sources, n, hi, seed):
    """n chunks: the edge lengths first, then lengths drawn log-uniformly up to `hi`, contents cycling through the four
    sources at seeded offsets."""
    rng = np.random.default_rng(seed)
    lens = EDGE_LENS + [int(math.exp(x)) for x in rng.uniform(0, math.log(hi), n - len(EDGE_LENS))]
    out = []
    for i, ln in enumerate(lens):
        src = sources[i % 4]
        o = int(rng.integers(0, len(src) - ln + 1))
        out.append(src[o : o + ln])
    return out


def fast_twin(data, opts, flags):
    f = tile_model.frame(data, opts, block_checksum=bool(flags & BC))
    return with_content_checksum(f, data) if flags & CK else f


def hc_twin(data, level, linked, flags=0):
    f = hc_model.frame(data, hc_model.kernel_opts(level=level), block_checksum=bool(flags & BC), linked=linked)
    return with_content_checksum(f, data) if flags & CK else f


def mismatches(got, want):
    return [i for i, (a, b) in enumerate(zip(got, want)) if a != b]


def assert_all(got, want, what):
    assert len(got) == len(want)
    bad = mismatches(got, want)
    assert not bad, f"{what}: {len(bad)} of {len(want)} differ, first at {bad[:8]}"


# ------------------------------------------------------------------------------------------------ (A) wide batches
@pytest.mark.parametrize("flags", [0, CK | BC], ids=["plain", "ck+bc"])
def test_fast_compressor_at_the_sender_width(ctx, sm, sources, twin_opts, flags):
    n = sender_width(sm)
    assert groups(n) > sm // 4  # more groups than digest CTAs: warps 1..3 of a digest CTA hash a group
    datas = ragged_chunks(sources, n, 256 << 10, seed=1)
    frames, digests = run_guarded(ctx, datas, flags)  # fails on any byte written outside [dst, dst + out_len)
    assert_all(digests, [hashlib.md5(d).digest() for d in datas], "digests")
    assert_all(frames, [fast_twin(d, twin_opts, flags) for d in datas], "frames against the tile twin")
    assert_all([ref.lz4f_decompress(f, len(d)) for d, f in zip(datas, frames)], datas, "liblz4's decode")


@pytest.mark.parametrize("level", [3, 9])
def test_linked_high_ratio_at_the_sender_width(ctx, sm, sources, level):
    n = sender_width(sm)
    assert groups(n) > sm // 4
    datas = ragged_chunks(sources, n, 256 << 10, seed=2)
    frames, digests = run_guarded(ctx, datas, native.hc_level_flag(level) | LINKED)
    assert_all(digests, [hashlib.md5(d).digest() for d in datas], "digests")
    assert_all(frames, [hc_twin(d, level, True) for d in datas], "frames against the hc twin")
    assert_all([ref.lz4f_decompress(f, len(d)) for d, f in zip(datas, frames)], datas, "liblz4's decode")


def test_md5_alone_at_the_sender_second_round(ctx, sm):
    n = sender_second_round(sm)
    assert groups(n) > 8 * sm  # more groups than four warps in every CTA of the grid
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 301, n)
    pool = rng.bytes(1 << 16)
    datas = [pool[int(o) : int(o) + int(ln)] for o, ln in zip(rng.integers(0, (1 << 16) - 300, n), lens)]
    _, digests, out_lens, _ = run_device(ctx, datas, flags=MD5)
    assert_all(digests, [hashlib.md5(d).digest() for d in datas], "digests")
    assert out_lens == [0] * n


def _flip_content_checksums(frames, rng):
    """~1 % of the frames, at seeded indices, with a bit of their content checksum (the last 4 bytes) flipped."""
    idx = sorted(set(int(i) for i in rng.choice(len(frames), max(1, len(frames) // 100), replace=False)))
    out = list(frames)
    for i in idx:
        f = bytearray(out[i])
        f[-1 - i % 4] ^= 1 << (i % 8)
        out[i] = bytes(f)
    return out, idx


@pytest.mark.parametrize("width", ["warps1-3", "second-round"])
def test_decode_at_the_receiver_widths(ctx, sm, sources, width):
    if width == "warps1-3":
        n, hi = receiver_width(sm), 128 << 10
        assert groups(n) > sm  # group sm lands on warp 1 of CTA 0
    else:
        n, hi = receiver_second_round(sm), 32 << 10
        assert groups(n) > 4 * sm  # group 4 * sm is a second group of warp 0 of CTA 0
    datas = ragged_chunks(sources, n, hi, seed=4)
    raws = [len(d) for d in datas]
    want = [hashlib.md5(d).digest() for d in datas]
    gpu, digests = run_guarded(ctx, datas, CK)
    assert_all(digests, want, "sender digests")
    lib = [hc_model.liblz4_frame(d, 0, linked=True, content_checksum=True) for d in datas]
    for name, frames in (("GPU frames", gpu), ("liblz4's linked frames", lib)):
        st, _ = guarded_decode(ctx, frames, raws, datas)  # bytes and MD5 of every ok chunk, guard bands, frame slab
        assert st == [native.D_OK] * n, f"{name}: {[(i, s) for i, s in enumerate(st) if s][:8]}"
    rng = np.random.default_rng(5)
    mixed = [g if i % 2 else l for i, (g, l) in enumerate(zip(gpu, lib))]
    flipped, idx = _flip_content_checksums(mixed, rng)
    expect = [None if i in set(idx) else d for i, d in enumerate(datas)]
    st, _ = guarded_decode(ctx, flipped, raws, expect)
    bad = set(idx)
    assert [i for i, s in enumerate(st) if s] == idx
    assert all(st[i] == native.D_CHECKSUM for i in bad) and all(s == native.D_OK for i, s in enumerate(st) if i not in bad)


def _mutate_for_verify(frame, data, k):
    """A changed literal (even k) or a zero offset (odd k, or no short literal run) in the middle one of the frame's
    sequences that have one -> (frame, status), or None when the frame has no compressed block"""
    f = parse_frame(frame, data)
    lits = [t + 1 for t in f.marks["token"] if 0 < frame[t] >> 4 < 15]
    if k % 2 == 0 and lits:
        p = lits[len(lits) // 2]
        return frame[:p] + bytes([frame[p] ^ 0x5A]) + frame[p + 1 :], native.D_MISMATCH
    if f.marks["offset"]:
        p = f.marks["offset"][len(f.marks["offset"]) // 2]
        return frame[:p] + b"\0\0" + frame[p + 2 :], native.D_CORRUPT
    return None


def check_verify_at_the_receiver_width(ctx, sm, sources, linked: bool):
    """Fast-path frames, or linked high-ratio level-3 frames, of one batch at the receiver's width: all pass, then ~1 % of
    them mutated fail with the expected codes and are repaired."""
    n = receiver_width(sm)
    assert groups(n) > sm
    datas = ragged_chunks(sources, n, 128 << 10, seed=6)
    frames, digests, _, _ = run_device(ctx, datas, LZ4 | MD5 | HC3 | LINKED if linked else 0)
    assert_all(digests, [hashlib.md5(d).digest() for d in datas], "digests")
    flags = native.F_HC | LINKED if linked else 0
    st, _, _ = run_verify(ctx, datas, frames, flags, repair=False)
    assert st == [0] * n, [(i, s) for i, s in enumerate(st) if s][:8]
    rng = np.random.default_rng(7)
    mutated, want = list(frames), [0] * n
    k = 0
    for i in rng.permutation(n):
        if k == max(1, n // 100):
            break
        m = _mutate_for_verify(frames[i], datas[i], k)
        if m is not None:
            mutated[i], want[i] = m
            k += 1
    assert k == max(1, n // 100)
    st, _, _ = run_verify(ctx, datas, mutated, flags, repair=False)
    assert_all(st, want, "statuses")
    assert {native.D_MISMATCH, native.D_CORRUPT} <= set(want)
    check_repair(ctx, datas, mutated, flags, st)  # failing frames become tile_model.assemble's stored-block frame


def test_verify_at_the_receiver_width(ctx, sm, sources):
    check_verify_at_the_receiver_width(ctx, sm, sources, linked=False)


def test_verify_linked_at_the_receiver_width(ctx, sm, sources):
    check_verify_at_the_receiver_width(ctx, sm, sources, linked=True)


def test_stage_host_path_at_the_receiver_width(sm, sources, twin_opts):
    """ChunkStage with one batch of max_chunks chunks: sealed frames and sealed raw chunks, opened and decoded back."""
    n = receiver_width(sm)
    assert groups(n) > sm
    datas = ragged_chunks(sources, n, 64 << 10, seed=8)
    stage = ChunkStage(0, max_batch_bytes=sum(native.round16(len(d)) for d in datas) + (16 << 20), max_chunks=n, n_slots=1)
    try:
        stage.set_e2ee_key(KEY)
        widths = []
        decode = stage.ctx.decode
        stage.ctx.decode = lambda addrs, *a, **k: (widths.append(len(addrs)), decode(addrs, *a, **k))[1]
        nonces = np.random.default_rng(9).bytes(24 * n)
        for compress in (True, False):
            slot = stage.begin()
            for d in datas:
                stage.add_bytes(slot, d)  # one batch of n chunks (raises if it does not fit)
            res = stage.collect(stage.launch(slot, compress=compress, encrypt=True, nonces=nonces))
            assert_all([r.md5 for r in res], [hashlib.md5(d).digest() for d in datas], "digests")
            boxes = [bytes(r.frame) for r in res]
            payloads = [fast_twin(d, twin_opts, 0) for d in datas] if compress else datas
            assert_all(boxes, [nonces[24 * i : 24 * i + 24] + oracle.secretbox_seal(KEY, nonces[24 * i : 24 * i + 24], p)
                               for i, p in enumerate(payloads)], "boxes")
            out = stage.decode(boxes, [len(d) for d in datas], encrypted=True, compressed=compress)
            assert_all([st for _, _, st in out], [native.D_OK] * n, "statuses")
            assert_all([data for data, _, _ in out], datas, "decoded chunks")
            assert_all([dg for _, dg, _ in out], [hashlib.md5(d).digest() for d in datas], "receiver digests")
        assert widths == [n, n]  # each decode was one launch of the whole batch
    finally:
        stage.close()


# ------------------------------------------------------------------------------------------------ memory guards
def _free_hbm():
    import torch

    return torch.cuda.mem_get_info()[0]


def _need_hbm(nbytes, what):
    free = _free_hbm()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GIB:.1f} GiB of free HBM, {free / GIB:.1f} GiB are free")


def _need_host(nbytes, what):
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    if avail < nbytes:
        pytest.skip(f"{what} needs {nbytes / GIB:.1f} GiB of host memory, {avail / GIB:.1f} GiB are available")


def _pattern_fill(ctx, dptr, nbytes):
    """Fill device memory with a byte pattern no chunk holds, so that bytes a kernel did not write cannot pass for its."""
    piece = bytearray(b"\xa5\x3c\x96\x0f" * (16 << 18))  # 64 MiB, writable: copied to the device without a host copy
    for o in range(0, nbytes, len(piece)):
        ctx.h2d(dptr + o, memoryview(piece)[: min(len(piece), nbytes - o)])


def _d2h(ctx, dptr, nbytes) -> bytearray:
    """Device bytes into one host bytearray (no second copy)."""
    buf = bytearray(nbytes)
    if nbytes:
        arr = (ctypes.c_char * nbytes).from_buffer(buf)
        ctx._check(native.lib().sky_memcpy_d2h(ctx._h, ctypes.addressof(arr), dptr, nbytes))
        del arr
    return buf


def _liblz4_restores(frame, data) -> bool:
    """liblz4's LZ4F_decompress of the whole frame into one buffer (it verifies block and content checksums) == data."""
    L = ref._lib()
    dctx = ctypes.c_void_p()
    L.LZ4F_createDecompressionContext(ctypes.byref(dctx), 100)
    try:
        n = len(data)
        out = bytearray(max(1, n))
        dst = (ctypes.c_char * len(out)).from_buffer(out)
        src = (ctypes.c_char * len(frame)).from_buffer(frame) if isinstance(frame, bytearray) else ctypes.c_char_p(bytes(frame))
        base_s, base_d = ctypes.cast(src, ctypes.c_void_p).value, ctypes.addressof(dst)
        so = do = 0
        while True:
            s, d = ctypes.c_size_t(len(frame) - so), ctypes.c_size_t(n - do)
            hint = L.LZ4F_decompress(dctx, base_d + do, ctypes.byref(d), base_s + so, ctypes.byref(s), None)
            if L.LZ4F_isError(hint):
                return False
            so, do = so + s.value, do + d.value
            if hint == 0:
                break
            if s.value == 0 and d.value == 0:
                return False
        del dst, src
        return so == len(frame) and do == n and memoryview(out)[:n] == memoryview(data)
    finally:
        L.LZ4F_freeDecompressionContext(dctx)


# ------------------------------------------------------------------------------------------------ (B) the bench's batches
BENCH = {2: (8 << 20, "random", 64), 3: (16 << 20, "silesia", 16)}


@pytest.fixture(scope="module", params=[2, 3], ids=["config2", "config3"])
def bench_pool(request):
    cb, kind, p = BENCH[request.param]
    pool = [synth.random_chunk(i, cb) for i in range(p)] if kind == "random" else \
           [synth.silesia_like_chunk(2000 + i, cb) for i in range(p)]  # bench.py's fill_device_input
    return request.param, cb, pool


def test_bench_batch_over_4gib(bench_pool, twin_opts):
    config, cb, pool = bench_pool
    n, p = 1024, len(pool)
    stride, ostride = native.round16(cb), native.round16(native.frame_bound(cb))
    _need_hbm(n * (stride + ostride) + 2 * GIB, f"config {config} ({n} x {cb >> 20} MiB)")
    ctx = native.Context(0, n * stride, n, 0)  # as bench.py sizes it
    try:
        # each pool chunk compressed alone at offset 0: the twin's frame, liblz4 restores it
        pool_frames, pool_dg, _, _ = run_device(ctx, pool)
        assert_all(pool_dg, [hashlib.md5(d).digest() for d in pool], "pool digests")
        assert_all(pool_frames, [tile_model.frame(d, twin_opts) for d in pool], "pool frames against the tile twin")
        assert all(ref.lz4f_decompress(f, cb) == d for d, f in zip(pool, pool_frames))
        if config == 2:
            assert_all(pool_frames, [oracle.lz4f_compress_indep(d) for d in pool], "pool frames against stored-block frames")
        hc_frames = None
        if config == 3:
            hc_frames, _, _, _ = run_device(ctx, pool, flags=LZ4 | HC3)
            assert_all(hc_frames, [hc_twin(d, 3, False) for d in pool], "pool hc frames against the hc twin")
        src_off = [i * stride for i in range(n)]
        dst_off = [i * ostride for i in range(n)]
        lens, caps = [cb] * n, [native.frame_bound(cb)] * n
        assert src_off[-1] >= 4 * GIB
        d_in, d_out = ctx.device_alloc(n * stride + 64), ctx.device_alloc(n * ostride + 64)
        try:
            pool_bufs = [bytearray(d) for d in pool]  # writable: copied to the device without a host copy

            def upload():
                for i in range(n):
                    ctx.h2d(d_in + src_off[i], pool_bufs[i % p])

            upload()
            for flags, want_frames in ((0, pool_frames), (LZ4 | HC3, hc_frames)):
                if want_frames is None:
                    continue
                if flags:
                    upload()  # the decode below wrote over the input
                out_lens, digests, _ = ctx.process_device(d_in, src_off, lens, d_out, dst_off, caps, flags)
                if not flags:
                    assert_all(digests, [pool_dg[i % p] for i in range(n)], "digests")
                assert_all(out_lens, [len(want_frames[i % p]) for i in range(n)], "frame lengths")
                bad = [i for i in range(n) if ctx.d2h(d_out + dst_off[i], out_lens[i]) != want_frames[i % p]]
                assert not bad, f"flags {flags:#x}: {len(bad)} frames differ from their pool chunk's, first at {bad[:8]}"
                if flags:
                    continue
                _pattern_fill(ctx, d_in, n * stride)
                st, dg, _ = ctx.decode_device(d_out, dst_off, out_lens, d_in, src_off, lens)
                assert_all(st, [native.D_OK] * n, "decode statuses")
                assert_all(dg, digests, "receiver digests")
                bad = [i for i in range(n) if _d2h(ctx, d_in + src_off[i], cb) != pool_bufs[i % p]]
                assert not bad, f"{len(bad)} decoded chunks differ from their pool chunk, first at {bad[:8]}"
        finally:
            ctx.device_free(d_in)
            ctx.device_free(d_out)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ (C) single big chunks
SIZES = [(1 << 29) + 13, (1 << 32) + BLOCK + 17]
TEXT_RUN = 3000


def _text_run():
    return b"".join(b"[%d] the quick brown fox jumps over the lazy dog; " % k for k in range(200))[:TEXT_RUN]


@pytest.fixture(scope="module", params=SIZES, ids=["512MiB+13", "4GiB+64KiB+17"])
def big(request):
    """-> (chunk as a bytearray, its MD5, the special block indices).  A 16 MiB Silesia-like piece repeated, with distinct
    random blocks at 0 (and, past 4 GiB, at 65535 and 65536) and a text run across byte 2^32, so that a linked match
    crosses from block 65535 into block 65536."""
    n = request.param
    _need_host(n + 2 * GIB, f"a {n} byte chunk")
    piece = synth.silesia_like_chunk(90, 16 << 20)
    buf = bytearray(piece) * (n // len(piece) + 1)
    del buf[n:]
    rng = np.random.default_rng(91)
    special = [0]
    buf[0:BLOCK] = rng.bytes(BLOCK)
    if n > 1 << 32:
        special += [65535, 65536]
        buf[65535 * BLOCK : 65537 * BLOCK] = rng.bytes(2 * BLOCK)
        t = _text_run()
        buf[(1 << 32) - len(t) : 1 << 32] = t
        buf[1 << 32 : (1 << 32) + len(t)] = t
    special.append((n - 1) // BLOCK)  # the short last block
    return buf, hashlib.md5(buf).digest(), special


def _companions(n=40):
    return [synth.silesia_like_chunk(300 + i, 1000 + 7919 * i) for i in range(n)]


def _block_key(j, special):
    return ("s", j) if j in special else ("p", j % 256)  # the piece repeats every 256 blocks


def _header(n, flags, linked):
    h = bytearray(tile_model.assemble(n, [], bool(flags & BC), linked)[:15])
    if flags & CK:
        h[4] |= 0x04
        h[14] = (oracle.xxh32(bytes(h[4:14])) >> 8) & 0xFF
    return bytes(h)


def _walk(frame, flags):
    """Block spans of a frame: [(compressed?, data start, size)], then the position after the EndMark."""
    mv, pos, out = memoryview(frame), 15, []
    while True:
        w = int.from_bytes(mv[pos : pos + 4], "little")
        if w == 0:
            return out, pos + 4
        out.append((not w & 0x80000000, pos + 4, w & 0x7FFFFFFF))
        pos += 4 + (w & 0x7FFFFFFF) + (4 if flags & BC else 0)


def _check_big_frame(frame, buf, special, flags, twin_block):
    """Header, content size, every block against the twin's block for its content (twin_block(j) -> block bytes in the
    frame), block checksums, EndMark and content checksum."""
    n = len(buf)
    linked = bool(flags & LINKED)
    assert bytes(frame[:15]) == _header(n, flags, linked)
    assert int.from_bytes(frame[6:14], "little") == n
    blocks, end = _walk(frame, flags)
    assert len(blocks) == -(-n // BLOCK)
    cache, bad = {}, []
    mv = memoryview(frame)
    for j, (comp, s, size) in enumerate(blocks):
        key = (_block_key(j - 1, special), _block_key(j, special)) if linked and j else _block_key(j, special)
        if key not in cache:
            cache[key] = twin_block(j)
        c, want = cache[key]
        if bool(c) != comp or mv[s : s + size] != want:
            bad.append(j)
        elif flags & BC and int.from_bytes(mv[s + size : s + size + 4], "little") != oracle.xxh32(want):
            bad.append(j)
    assert not bad, f"{len(bad)} of {len(blocks)} blocks differ from the twin's, first at {bad[:8]}"
    assert len(cache) < 600
    assert end + (4 if flags & CK else 0) == len(frame)
    if flags & CK:
        assert int.from_bytes(frame[end:], "little") == oracle.xxh32(buf)


def _run_big(ctx, chunks, flags):
    """sky_process_device over `chunks` (the first one big) -> (frames: big one as a bytearray, digests)"""
    ck, bc = bool(flags & CK), bool(flags & BC)
    src_off, dst_off, caps, ip, op = [], [], [], 0, 0
    for c in chunks:
        src_off.append(ip)
        dst_off.append(op)
        caps.append(native.frame_need(len(c), ck, bc))
        ip += native.round16(len(c))
        op += native.round16(caps[-1])
    d_in, d_out = ctx.device_alloc(ip + 64), ctx.device_alloc(op + 64)
    try:
        for c, o in zip(chunks, src_off):
            ctx.h2d(d_in + o, c)
        lens, digests, _ = ctx.process_device(d_in, src_off, [len(c) for c in chunks], d_out, dst_off, caps, flags)
        frames = [_d2h(ctx, d_out + dst_off[0], lens[0])] + [ctx.d2h(d_out + o, ln) for o, ln in zip(dst_off[1:], lens[1:])]
        return frames, digests
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)


BIG_MODES = [("plain", 0), ("ck", CK), ("bc", LZ4 | BC), ("hc3", LZ4 | HC3), ("hc3-linked", LZ4 | HC3 | LINKED)]


@pytest.fixture(scope="module")
def big_ctx():
    c = native.Context(0, GIB, 64, 0)
    yield c
    c.close()


@pytest.mark.parametrize("mode,flags", BIG_MODES, ids=[m for m, _ in BIG_MODES])
def test_big_chunk_frames(big_ctx, big, twin_opts, mode, flags):
    buf, md5, special = big
    n = len(buf)
    _need_hbm(2 * n + 2 * GIB, f"a {n} byte chunk and its frame")
    _need_host(2 * n + GIB, "the frame and liblz4's decode")
    comp = _companions()
    frames, digests = _run_big(big_ctx, [buf] + comp, flags)
    if flags & MD5 or not flags & LZ4:
        assert digests == [md5] + [hashlib.md5(c).digest() for c in comp]
    hc, linked = bool(flags & native.F_HC), bool(flags & LINKED)
    if hc:
        assert frames[1:] == [hc_twin(c, 3, linked, flags) for c in comp]
    else:
        assert frames[1:] == [fast_twin(c, twin_opts, flags) for c in comp]
    f = frames[0]
    assert _liblz4_restores(f, buf)
    if n < 1 << 32:  # the whole frame against the twin's
        data = bytes(buf)
        want = hc_twin(data, 3, linked, flags) if hc else fast_twin(data, twin_opts, flags)
        assert f == want
        return
    o_hc = hc_model.kernel_opts(level=3)

    def twin_block(j):
        blk = bytes(buf[j * BLOCK : (j + 1) * BLOCK])
        if not hc:
            return tile_model.blocks(blk, twin_opts)[0]
        if not linked or j == 0:
            return hc_model.blocks(blk, o_hc, linked=linked)[0]
        return hc_model.blocks(bytes(buf[(j - 1) * BLOCK : j * BLOCK]) + blk, o_hc, linked=True)[1]

    _check_big_frame(f, buf, special, flags, twin_block)
    if linked:  # the text run at the start of block 65536 is matched back across byte 2^32 into block 65535
        blocks, _ = _walk(f, flags)
        alone = hc_model.blocks(bytes(buf[65536 * BLOCK : 65537 * BLOCK]), o_hc)[0]
        assert blocks[65536][0] and alone[0] and blocks[65536][2] < alone[0]


def test_big_chunk_md5_alone(big_ctx, big):
    buf, md5, _ = big
    _need_hbm(2 * len(buf) + 2 * GIB, "the chunk and room for its frame")
    comp = _companions()
    _, digests, _, _ = run_device(big_ctx, [buf] + comp, flags=MD5)
    assert digests == [md5] + [hashlib.md5(c).digest() for c in comp]


def test_big_chunk_decode(big_ctx, big):
    """The GPU's frame and liblz4's own linked frame of the chunk, decoded in one batch with small companions."""
    buf, md5, _ = big
    n = len(buf)
    _need_hbm(4 * n + 2 * GIB, "the chunk, two frames and two outputs")
    _need_host(3 * n + GIB, "liblz4's frame and the decoded chunk")
    ctx, comp = big_ctx, _companions()
    lib = ref.lz4f_compress(buf)
    need, rn = native.frame_need(n), native.round16(n)
    d_in, d_f = ctx.device_alloc(rn + 64), ctx.device_alloc(native.round16(need) + native.round16(len(lib)) + (16 << 20))
    try:
        ctx.h2d(d_in, buf)
        (glen,), _, _ = ctx.process_device(d_in, [0], [n], d_f, [0], [need], LZ4)
        ctx.device_free(d_in)
        d_in = None
        comp_frames = [tile_model.frame(c) for c in comp]
        f_off = [0, native.round16(need)]
        ctx.h2d(d_f + f_off[1], lib)
        p = f_off[1] + native.round16(len(lib))
        for cf in comp_frames:
            f_off.append(p)
            ctx.h2d(d_f + p, cf)
            p += native.round16(len(cf))
        raws = [n, n] + [len(c) for c in comp]
        o_off, op = [], 0
        for r in raws:
            o_off.append(op)
            op += native.round16(r)
        d_o = ctx.device_alloc(op + 64)
        try:
            _pattern_fill(ctx, d_o, op)
            st, dg, _ = ctx.decode_device(d_f, f_off, [glen, len(lib)] + [len(cf) for cf in comp_frames], d_o, o_off, raws)
            assert st == [native.D_OK] * len(raws)
            assert dg == [md5, md5] + [hashlib.md5(c).digest() for c in comp]
            for k in (0, 1):
                assert _d2h(ctx, d_o + o_off[k], n) == buf, ("GPU frame", "liblz4 frame")[k]
            assert [ctx.d2h(d_o + o, len(c)) for o, c in zip(o_off[2:], comp)] == comp
        finally:
            ctx.device_free(d_o)
    finally:
        if d_in is not None:
            ctx.device_free(d_in)
        ctx.device_free(d_f)


def _first_literal(frame, start):
    """Position of the first literal byte of the compressed block whose data starts at `start`."""
    tok = frame[start]
    p = start + 1
    if tok >> 4 == 15:
        while frame[p] == 255:
            p += 1
        p += 1
    assert tok >> 4, "the block starts with a match"
    return p


def test_big_chunk_verify(big_ctx, big):
    buf, _, special = big
    n = len(buf)
    _need_hbm(2 * n + 2 * GIB, "the chunk and its frame")
    _need_host(3 * n + GIB, "the frames and liblz4's decode")
    ctx, comp = big_ctx, _companions()
    chunks = [buf] + comp
    src_off, f_off, caps, ip, fp = [], [], [], 0, 0
    for c in chunks:
        src_off.append(ip)
        f_off.append(fp)
        caps.append(native.frame_need(len(c)))
        ip += native.round16(len(c))
        fp += native.round16(caps[-1])
    lens = [len(c) for c in chunks]
    d_in, d_f = ctx.device_alloc(ip + 64), ctx.device_alloc(fp + 64)
    try:
        for c, o in zip(chunks, src_off):
            ctx.h2d(d_in + o, c)
        flen, _, _ = ctx.process_device(d_in, src_off, lens, d_f, f_off, caps, LZ4)
        st, fl2, _ = ctx.verify_device(d_in, src_off, lens, d_f, f_off, flen)
        assert st == [0] * len(chunks) and fl2 == flen
        # one literal changed in a block past 2^32 (the 512 MiB chunk: in its last full block)
        frame = _d2h(ctx, d_f, flen[0])
        blocks, _ = _walk(frame, 0)
        j = 65536 if n > 1 << 32 else len(blocks) - 2
        comp_blk, s, size = blocks[j]
        p = _first_literal(frame, s) if comp_blk else s + size // 2
        assert j * BLOCK >= (1 << 32 if n > 1 << 32 else 1 << 29) - BLOCK
        ctx.h2d(d_f + p, bytes([frame[p] ^ 0x21]))
        del frame
        st, fl2, _ = ctx.verify_device(d_in, src_off, lens, d_f, f_off, flen)
        assert st == [native.D_MISMATCH] + [0] * len(comp) and fl2 == flen
        st, fl2, _ = ctx.verify_device(d_in, src_off, lens, d_f, f_off, flen, caps)
        assert st == [native.D_MISMATCH] + [0] * len(comp)
        assert fl2 == [native.frame_need(n)] + flen[1:]
        repaired = _d2h(ctx, d_f, fl2[0])
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_f)
    # the stored-block frame, block by block (tile_model.assemble's layout), and liblz4 restores it
    assert bytes(repaired[:15]) == _header(n, 0, False)
    blocks, end = _walk(repaired, 0)
    mv, src = memoryview(repaired), memoryview(buf)
    assert end == len(repaired) and len(blocks) == -(-n // BLOCK)
    bad = [j for j, (c, s, size) in enumerate(blocks)
           if c or size != min(BLOCK, n - j * BLOCK) or mv[s : s + size] != src[j * BLOCK : j * BLOCK + size]]
    assert not bad, bad[:8]
    del mv, src
    assert _liblz4_restores(repaired, buf)


def test_big_chunk_e2ee(big):
    """The chunk sealed as it is (compress=False: the box holds more than 2^32 bytes), opened and digested on the GPU."""
    buf, md5, _ = big
    n = len(buf)
    _need_hbm(3 * n + 3 * GIB, "the stage's slabs")
    _need_host(4 * n + 2 * GIB, "the stage's pinned slabs, the box and the opened chunk")
    stage = ChunkStage(0, max_batch_bytes=native.round16(n) + (64 << 20), max_chunks=4, n_slots=1)
    try:
        stage.set_e2ee_key(KEY)
        comp = _companions(2)
        nonces = np.random.default_rng(12).bytes(24 * 3)
        slot = stage.begin()
        for c in [buf] + comp:
            stage.add_bytes(slot, c)
        res = stage.collect(stage.launch(slot, compress=False, encrypt=True, nonces=nonces))
        assert [r.md5 for r in res] == [md5] + [hashlib.md5(c).digest() for c in comp]
        box = bytearray(res[0].frame)
        del res
        want = bytearray(n + 16)  # tag | ciphertext from the C oracle
        L = oracle.lib()
        src, out = (ctypes.c_char * n).from_buffer(buf), (ctypes.c_char * len(want)).from_buffer(want)
        L.sky_oracle_secretbox_seal(ctypes.cast(ctypes.c_char_p(KEY), ctypes.c_void_p),
                                    ctypes.cast(ctypes.c_char_p(nonces[:24]), ctypes.c_void_p),
                                    ctypes.addressof(src), n, ctypes.addressof(out))
        del src, out
        assert len(box) == n + 40 and box[:24] == nonces[:24] and memoryview(box)[24:] == memoryview(want)
        del want
        got = stage.decode([box], [n], encrypted=True, compressed=False)
        (data, dg, st), = got
        assert st == native.D_OK and dg == md5 and data == buf
        del got, data
        box[40 + (1 << 32) + 5 if n > 1 << 32 else 40 + n - 3] ^= 0x10  # a ciphertext byte past 2^32 (or near the end)
        ((data, dg, st),) = stage.decode([box], [n], encrypted=True, compressed=False)
        assert st == native.D_AUTH and data is None
    finally:
        stage.close()
