"""GPU tests of SKY_F_VERIFY: the sender checks every frame against its chunk and sends a stored-block frame for one that
does not restore it.

Bars: (1) clean frames -- at edge lengths of five data kinds, under the fast path, high-ratio levels 3 and 9, content and
block checksums and E2EE, every status is 0 and payloads and digests equal those of the same batch without the flag;
(2) a status table of crafted frames through sky_verify_device, independent and linked (SKY_F_HC | SKY_F_LINKED), with the
earliest failing block's code winning in both directions, and short last blocks that liblz4 decodes against LZ4's
end-of-block rules refused; (3) over seeded structural mutants of GPU (fast, lazy and optimal parse), liblz4 and
generated frames, independent and linked, status 0 exactly when the reference predicate `restores` holds -- the stage's
frame descriptor, liblz4 (and, for frames without checksums, the strict oracle) decoding the whole mutant to the chunk,
and every block in the stage's layout and within the end-of-block rules; (4) with frame_cap every failing frame becomes
the stored-block frame the CPU assembles (linked FLG past one block under SKY_F_LINKED), which liblz4 decodes, and
frame_len follows; without it no byte changes, and with it nothing outside [frame, frame + cap) does (guard bytes between
frames, whole slab read back); (5) GatewayCompressHash(verify_frames=True) in the forked queue harness."""
import ctypes
import hashlib
import json
import os
import random
import struct
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

import lz4_craft as C
import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import hc_model  # noqa: E402
import tile_model  # noqa: E402
from test_checksum_format import with_content_checksum  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

BC, CK, V = native.F_BLOCK_CHECKSUM, native.F_CHECKSUM, native.F_VERIFY
LK = native.F_LINKED
LINKED = native.F_HC | LK  # what sky_verify_device is given for a batch of linked high-ratio frames
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
GAP = 256
LENS = [0, 1, 12, 13, 65535, 65536, 65537, 8 << 20]
CHECKSUMS = [0, CK, BC, CK | BC]


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 1 << 30, 4096, 0)
    yield c
    c.close()


def _pattern(n: int, seed: int) -> np.ndarray:
    return ((np.arange(n, dtype=np.uint32) * 167 + seed) & 0xFF).astype(np.uint8)


def kind_chunk(kind: str, n: int, seed: int) -> bytes:
    if kind == "random":
        return synth.random_chunk(seed, n)
    if kind == "silesia":
        return synth.silesia_like_chunk(seed, n)
    if kind == "zeros":
        return bytes(n)
    if kind == "period3":
        return (b"abc" * (n // 3 + 1))[:n]
    text = (b"it was the best of times, it was the worst of times; " * (n // 50 + 2))[: n // 2]  # half text, half random
    return text + np.random.default_rng(seed).bytes(n - len(text))


KINDS = ["random", "silesia", "zeros", "period3", "half"]


def stored_frame(data: bytes, flags: int) -> bytes:
    """The chunk's stored-block frame, assembled on the CPU: every block raw, with the flags' checksums, and the linked FLG
    past one block under F_LINKED."""
    f = tile_model.assemble(len(data), [(0, data[p : p + C.BLOCK]) for p in range(0, len(data), C.BLOCK)], bool(flags & BC),
                            bool(flags & LK))
    return with_content_checksum(f, data) if flags & CK else f


def stage_flg(n: int, flags: int) -> int:
    """FLG of the stage's frame of an n-byte chunk under `flags` (write_frame_header): 0x60 when empty, else 0x68 (content
    size), with B.Indep (0x20) clear under F_LINKED past one block; + 0x04 for F_CHECKSUM, + 0x10 for F_BLOCK_CHECKSUM."""
    flg = 0x60 if not n else 0x48 if flags & LK and n > C.BLOCK else 0x68
    return flg | (0x04 if flags & CK else 0) | (0x10 if flags & BC else 0)


def liblz4_whole(frame: bytes, n: int):
    """liblz4's decode of `frame` -> (bytes, consumed) or None where it rejects it."""
    L = ref._lib()
    dctx = ctypes.c_void_p()
    L.LZ4F_createDecompressionContext(ctypes.byref(dctx), 100)
    try:
        src = ctypes.create_string_buffer(frame, max(1, len(frame)))
        out = ctypes.create_string_buffer(max(1, n))
        so = do = 0
        while True:
            s = ctypes.c_size_t(len(frame) - so)
            d = ctypes.c_size_t(n - do)
            hint = L.LZ4F_decompress(dctx, ctypes.addressof(out) + do, ctypes.byref(d), ctypes.addressof(src) + so, ctypes.byref(s), None)
            if L.LZ4F_isError(hint):
                return None
            so += s.value
            do += d.value
            if hint == 0:
                return out.raw[:do], so
            if s.value == 0 and d.value == 0:
                return None
    finally:
        L.LZ4F_freeDecompressionContext(dctx)


def restores(frame: bytes, data: bytes, flags: int) -> bool:
    """The reference the frame check is held to: the stage accepts `frame` for `data` exactly when its FLG and BD are the
    ones the stage writes for the chunk and flags (stage_flg), liblz4 decodes the whole frame to `data` and consumes it, the
    strict oracle agrees (frames without checksums), and every block keeps the stage's layout and LZ4's end-of-block rules
    relative to its own decoded length (lz4_craft.conforms) -- rules liblz4 enforces in full-size blocks only."""
    if len(frame) < 6 or frame[4] != stage_flg(len(data), flags) or frame[5] != 0x40:
        return False
    got = liblz4_whole(frame, len(data))
    if got is None or got != (data, len(frame)):
        return False
    if not C.conforms(frame, len(data)):
        return False
    if flags & (CK | BC):
        return True
    try:
        out, info = oracle.lz4f_decode(frame, len(data), with_info=True)
    except ValueError:
        return False
    return out == data and info["consumed"] == len(frame)


def run_verify(ctx, datas, frames, flags, repair: bool):
    """sky_verify_device over `frames` (frame i checked against datas[i]) with GAP guard bytes around every frame region of
    frame_need bytes; the whole slab is read back.  -> (status, frames after, frame_len after)"""
    ck, bc = bool(flags & CK), bool(flags & BC)
    src_off, f_off, caps, ip, fp = [], [], [], 0, GAP
    for d, f in zip(datas, frames):
        src_off.append(ip)
        f_off.append(fp)
        caps.append(native.frame_need(len(d), ck, bc))
        ip += native.round16(len(d))
        fp += native.round16(max(len(f), caps[-1])) + GAP
    slab = _pattern(fp, 0x3C)
    for f, o in zip(frames, f_off):
        slab[o : o + len(f)] = np.frombuffer(f, np.uint8)
    d_in, d_f = ctx.device_alloc(ip + 64), ctx.device_alloc(fp)
    try:
        for d, o in zip(datas, src_off):
            if d:
                ctx.h2d(d_in + o, d)
        ctx.h2d(d_f, slab)
        xxh = [oracle.xxh32(d) for d in datas] if ck else None
        st, flen, _ = ctx.verify_device(d_in, src_off, [len(d) for d in datas], d_f, f_off, [len(f) for f in frames],
                                        caps if repair else None, xxh, flags)
        back = np.frombuffer(ctx.d2h(d_f, fp), np.uint8)
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_f)
    if not repair:
        assert np.array_equal(back, slab), "a check without frame_cap changed the frame slab"
        assert flen == [len(f) for f in frames]
    else:
        outside = np.ones(fp, bool)
        for o, cap in zip(f_off, caps):
            outside[o : o + cap] = False
        bad = np.flatnonzero((back != slab) & outside)
        assert bad.size == 0, f"{bad.size} bytes written outside [frame, frame + cap), first at slab byte {bad[0]}"
    return st, [back[o : o + n].tobytes() for o, n in zip(f_off, flen)], flen


def check_repair(ctx, datas, frames, flags, st):
    """With frame_cap: the same statuses, failing frames become the stored-block frame (liblz4 restores it), the others stay;
    run_verify checks the guard bytes."""
    st2, after, flen = run_verify(ctx, datas, frames, flags, repair=True)
    assert st2 == st
    for i, (d, f, s) in enumerate(zip(datas, frames, st)):
        if s == 0:
            assert after[i] == f and flen[i] == len(f)
        else:
            want = stored_frame(d, flags)
            assert after[i] == want and flen[i] == len(want) == native.frame_need(len(d), bool(flags & CK), bool(flags & BC)), i
            assert after[i][4] == stage_flg(len(d), flags) and ref.lz4f_decompress(after[i], len(d)) == d


# ------------------------------------------------------------------------------------------------ (1) clean frames
MODES = [("fast", {}), ("hc3", {"level": 3}), ("hc9", {"level": 9}), ("ck", {"checksum": True}), ("bc", {"block_checksum": True}),
         ("ck+bc", {"checksum": True, "block_checksum": True}), ("hc5+ck+bc", {"level": 5, "checksum": True, "block_checksum": True}),
         ("e2ee", {"encrypt": True}), ("e2ee+hc3+ck", {"encrypt": True, "level": 3, "checksum": True})]


@pytest.fixture(scope="module")
def stage():
    s = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=64, n_slots=2)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


@pytest.mark.parametrize("mode,opts", MODES, ids=[m[0] for m in MODES])
def test_clean_frames_pass_and_are_unchanged(stage, mode, opts):
    datas = [kind_chunk(k, n, 40 + i) for i, (k, n) in enumerate((k, n) for k in KINDS for n in LENS)]
    nonces = bytes(range(256)) * (24 * len(datas) // 256 + 1)
    nonces = nonces[: 24 * len(datas)] if opts.get("encrypt") else None
    plain = stage.process(datas, nonces=nonces, **opts)
    checked = stage.process(datas, nonces=nonces, verify=True, **opts)
    assert [r.verify_status for r in checked] == [0] * len(datas)
    assert [r.verify_status for r in plain] == [0] * len(datas)
    for d, a, b in zip(datas, plain, checked):
        assert bytes(b.frame) == bytes(a.frame) and b.md5 == a.md5 == hashlib.md5(d).digest()


def test_flag_rules(ctx):
    d_in, d_out = ctx.device_alloc(1 << 16), ctx.device_alloc(1 << 17)
    try:
        cap = native.frame_need(1000, True, True)
        for flags in (V, V | CK):  # the device path does not take the flag
            with pytest.raises(native.SkyChunkError) as e:
                ctx.process_device(d_in, [0], [1000], d_out, [0], [cap], flags)
            assert e.value.code == native.SKY_E_INVALID
        for flags, xxh in ((native.F_MD5, None), (CK, None), (0, [1]), (native.F_E2EE, None)):
            with pytest.raises(native.SkyChunkError) as e:
                ctx.verify_device(d_in, [0], [1000], d_out, [0], [cap], None, xxh, flags)
            assert e.value.code == native.SKY_E_INVALID
        with pytest.raises(native.SkyChunkError) as e:  # one byte short of the stored-block frame
            ctx.verify_device(d_in, [0], [1000], d_out, [0], [cap], [native.frame_need(1000) - 1], None, 0)
        assert e.value.code == native.SKY_E_CAPACITY
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)
    s = ChunkStage(0, max_batch_bytes=1 << 20, max_chunks=4, n_slots=1)
    try:
        buf = native.PinnedBuffer(1 << 16)
        with pytest.raises(native.SkyChunkError) as e:  # no frame to check
            s.ctx.submit([buf.addr], [100], None, None, native.F_MD5 | V)
        assert e.value.code == native.SKY_E_INVALID
        slot = s.begin()
        s.add_bytes(slot, b"q" * 5000)
        s.launch(slot)  # without the flag: no statuses to ask for, and the ticket stays valid
        assert native.lib().sky_wait(s.ctx._h, slot.ticket, None, None, (ctypes.c_int32 * 1)(), None, None) == native.SKY_E_INVALID
        (r,) = s.collect(slot)
        assert r.verify_status == 0 and ref.lz4f_decompress(bytes(r.frame), 5000) == b"q" * 5000
        t = s.ctx.submit([buf.addr], [100], [buf.addr + 4096], [native.frame_need(100)], V)  # alone: LZ4 + MD5 + verify
        lens, _, ver, _, _ = s.ctx.wait_ex(t)
        assert ver == [0] and lens[0] > 0
        buf.close()
    finally:
        s.close()


# ------------------------------------------------------------------------------------------------ (2) status table
def _lit_pos(b: C.Block) -> int:
    """A literal byte of the block's first sequence with 1..14 literals."""
    for t in b.marks["token"]:
        if 0 < b.data[t] >> 4 < 15:
            return t + 1
    raise AssertionError("no short literal run")


def _mutate(b: C.Block, pos: int, data: bytes) -> C.Block:
    return C.Block(b.data[:pos] + data + b.data[pos + len(data):], b.raw, b.marks)


def _craft(rng: random.Random, plan):
    """A chunk and its blocks from a plan: per block (size, None) for a stored block of random bytes, or (size, steps) for a
    compressed one, each step a literal count or an (offset, length) match, filled up to `size` with random literals.
    -> (chunk, blocks)"""
    buf, blocks = bytearray(), []
    for size, steps in plan:
        if steps is None:
            data = rng.randbytes(size)
            buf += data
            blocks.append(C.stored_block(data))
            continue
        w = C.BlockWriter(buf)
        for st in steps:
            w.literals(rng.randbytes(st)) if isinstance(st, int) else w.match(*st)
        blocks.append(w.literals(rng.randbytes(size - w.pos)).close())
    return bytes(buf), blocks


def _status_rows(rng: random.Random, linked: bool = False):
    """(name, chunk, frame, flags, status).  linked: the batch is SKY_F_HC | SKY_F_LINKED, so a frame of more than one
    block must carry the linked FLG (0x48) and its matches may reach back to the chunk's first byte."""
    rows = []
    mode = LINKED if linked else 0
    for ck in CHECKSUMS:
        flags = mode | ck
        kw = dict(content_size=True, block_checksum=bool(ck & BC), content_checksum=bool(ck & CK))

        def frame(blocks, content):  # the frame the stage writes around these blocks (FLG by stage_flg)
            return C.assemble_frame(blocks, content, linked=linked and len(content) > C.BLOCK, **kw)

        s = C.gen_stream(rng, 3 * C.BLOCK + 777, linked=linked, stored_p=0.0)
        n = len(s.content)
        tag = {0: "", CK: " ck", BC: " bc", CK | BC: " ck+bc"}[ck]
        good = frame(s.blocks, s.content)
        rows.append(("valid" + tag, s.content, good.data, flags, 0))
        blocks = list(s.blocks)
        blocks[1] = _mutate(blocks[1], _lit_pos(blocks[1]), bytes([blocks[1].data[_lit_pos(blocks[1])] ^ 0x01]))
        rows.append(("literal flipped" + tag, s.content, frame(blocks, s.content).data, flags, native.D_MISMATCH))
        blocks = list(s.blocks)
        blocks[2] = _mutate(blocks[2], blocks[2].marks["offset"][-1], b"\0\0")
        rows.append(("offset 0" + tag, s.content, frame(blocks, s.content).data, flags, native.D_CORRUPT))
        rows.append(("content size + 1" + tag, s.content, C.with_header(good.data, content_size=n + 1), flags, native.D_SIZE))
        rows.append(("truncated" + tag, s.content, good.data[:-1], flags, native.D_TRUNCATED))
        rows.append(("trailing byte" + tag, s.content, good.data + b"\0", flags, native.D_SIZE))
        other = C.gen_stream(rng, n, linked=linked, stored_p=0.3)
        rows.append(("other data, same length" + tag, s.content, frame(other.blocks, other.content).data, flags, native.D_MISMATCH))
        half = s.content[:50000], s.content[50000:100000]
        rows.append(("short middle block" + tag, s.content[:100000],
                     frame([C.stored_block(half[0]), C.stored_block(half[1])], s.content[:100000]).data, flags, native.D_LAYOUT))
        # a full block whose last match ends 3 bytes before its end (liblz4 needs 5 literals there)
        buf = bytearray()
        w = C.BlockWriter(buf)
        w.literals(rng.randbytes(40)).match(13, C.BLOCK - 43).literals(rng.randbytes(3))
        tail = bytes(buf)
        rows.append(("match into the last 5 bytes" + tag, tail, frame([w.close()], tail).data, flags, native.D_CORRUPT))
        # short last blocks that break an end-of-block rule: liblz4 decodes them, the check refuses them (short block: ...)
        head = s.content[: C.BLOCK] if linked else b""
        for name, blk, content in C.short_block_cases(rng, head, 1000):
            rows.append(("short block: " + name + tag, content, frame(s.blocks[:1] * bool(head) + [blk], content).data, flags,
                         native.D_CORRUPT))
        if not linked:
            rows.append(("linked FLG" + tag, s.content, C.assemble_frame(s.blocks, s.content, linked=True, **kw).data, flags,
                         native.D_BAD_HEADER))
            # offset into the previous block: decodes as a linked frame, not as an independent one
            buf = bytearray(s.content[: C.BLOCK])
            w = C.BlockWriter(buf)
            w.literals(rng.randbytes(30)).match(31, 10).literals(rng.randbytes(500))
            prev = bytes(buf)
            rows.append(("offset into the previous block" + tag, prev, frame([s.blocks[0], w.close()], prev).data, flags,
                         native.D_CORRUPT))
        else:
            rows.append(("independent FLG past one block" + tag, s.content, C.with_header(good.data, flg=good.data[4] | C.FLG_INDEP),
                         flags, native.D_BAD_HEADER))
            one = s.content[: C.BLOCK]
            rows.append(("linked FLG on one full block" + tag, one, C.assemble_frame(s.blocks[:1], one, linked=True, **kw).data, flags,
                         native.D_BAD_HEADER))
            crafted = [  # (name, plan, status): matches that reach across block starts, up to the chunk's first byte
                ("offset 65535 at q = 0 of block 1, to chunk byte 1", [(C.BLOCK, None), (C.BLOCK, [(65535, 100), 7, (9, 300)])], 0),
                ("offset q in block 0, to chunk byte 0", [(C.BLOCK, [30, (30, 20), 400, (100, 3000)]), (500, None)], 0),
                ("overlapping match straddling the block start", [(C.BLOCK, [100, (50, 2000)]), (C.BLOCK, [3, (10, 50), 9, (7, 600)])], 0),
                ("compressed block reading a stored block", [(C.BLOCK, None), (C.BLOCK, [5, (40000, 300), 100, (65000, 1000)]),
                                                            (C.BLOCK, [0, (65535, 4), 2, (60000, 5000)])], 0),
                ("short last block reading the full block before it", [(C.BLOCK, [20, (20, 700)]), (1000, [10, (5000, 200), 1, (1010, 64)])],
                 0),
            ]
            for name, plan, code in crafted:
                content, blocks = _craft(rng, plan)
                rows.append((name + tag, content, frame(blocks, content).data, flags, code))
            content, blocks = _craft(rng, [(C.BLOCK, [30, (30, 20), 400, (100, 3000)]), (500, None)])
            blocks[0] = _mutate(blocks[0], blocks[0].marks["offset"][0], struct.pack("<H", 31))
            rows.append(("offset q + 1 in block 0, before the chunk" + tag, content, frame(blocks, content).data, flags, native.D_CORRUPT))
            content, blocks = _craft(rng, [(C.BLOCK, [100, (50, 2000)]), (C.BLOCK, [100, (60, 3000)]), (777, None)])
            rows.append(("blocks 0 and 1 swapped" + tag, content, C.swap_blocks(frame(blocks, content), 0, 1), flags, native.D_MISMATCH))
        if ck & BC:
            rows.append(("block checksum" + tag, s.content, C.flip(good.data, good.marks["block_checksum"][6], 0x01), flags,
                         native.D_CHECKSUM))
        if ck & CK:
            rows.append(("content checksum" + tag, s.content, C.flip(good.data, good.marks["content_checksum"][0], 0x01), flags,
                         native.D_CHECKSUM))
    # earliest failing block: block 0 corrupt (its checksum right), blocks 1..3 with wrong checksums -- and the mirror image.
    # Four copies of each: every copy is another race between the failing blocks' status writes.
    for copy in range(4):
        s = C.gen_stream(rng, 4 * C.BLOCK, linked=linked, stored_p=0.0)
        for corrupt_first in (True, False):
            blocks = [(_mutate(b, b.marks["offset"][-1], b"\0\0") if (j == 0) == corrupt_first else b) for j, b in enumerate(s.blocks)]
            f = C.assemble_frame(blocks, s.content, linked=linked, content_size=True, block_checksum=True)
            data = bytearray(f.data)
            for j in range(4):
                if (j == 0) != corrupt_first:
                    data[f.spans[j][1] - 1] ^= 0x40  # the block's checksum
            rows.append((f"precedence, corrupt first={corrupt_first} #{copy}", s.content, bytes(data), mode | BC,
                         native.D_CORRUPT if corrupt_first else native.D_CHECKSUM))
        if linked:  # block 1's matches read a block 0 with a changed literal: block 0's MISMATCH wins whatever block 1 says
            content, blocks = _craft(rng, [(C.BLOCK, [10, (5, 100), 300, (200, 4000)]), (C.BLOCK, [(65535, 100), 10, (30000, 2000), 50, (65000, 500)]),
                                           (C.BLOCK, [0, (65535, 3000)])])
            p = _lit_pos(blocks[0]) + 3  # chunk byte 3, which block 1's first match reads
            blocks[0] = _mutate(blocks[0], p, bytes([blocks[0].data[p] ^ 0x10]))
            for b1 in ("passes", "checksum", "corrupt"):
                bl = list(blocks)
                if b1 == "corrupt":
                    bl[1] = _mutate(bl[1], bl[1].marks["offset"][-1], b"\0\0")
                f = C.assemble_frame(bl, content, linked=True, content_size=True, block_checksum=True)
                data = bytearray(f.data)
                if b1 == "checksum":
                    data[f.spans[1][1] - 1] ^= 0x40
                rows.append((f"precedence, block 1 reads a changed block 0, block 1 {b1} #{copy}", content, bytes(data), LINKED | BC,
                             native.D_MISMATCH))
    return rows


def check_status_table(ctx, linked: bool):
    """Every row of _status_rows: the reference agrees with its code, sky_verify_device reports it, and repair follows."""
    rows = _status_rows(random.Random(9), linked)
    for name, data, frame, flags, code in rows:
        assert restores(frame, data, flags) == (code == 0), name
        if name.startswith("short block: "):  # LZ4's end-of-block rules, kept where liblz4 does not ask for them
            assert liblz4_whole(frame, len(data)) == (data, len(frame)), name
    for flags in sorted({r[3] for r in rows}):
        sel = [r for r in rows if r[3] == flags]
        datas, frames = [r[1] for r in sel], [r[2] for r in sel]
        st, _, _ = run_verify(ctx, datas, frames, flags, repair=False)
        assert [(r[0], s) for r, s in zip(sel, st)] == [(r[0], r[4]) for r in sel]
        check_repair(ctx, datas, frames, flags, st)


def test_status_table_and_repair(ctx):
    check_status_table(ctx, linked=False)


def test_linked_status_table_and_repair(ctx):
    """The table under SKY_F_HC | SKY_F_LINKED: sky_verify_linked_index_kernel, sky_verify_linked_kernel and
    sky_verify_linked_settle_kernel."""
    check_status_table(ctx, linked=True)


# ------------------------------------------------------------------------------------------------ (3) differential
def parse_frame(frame: bytes, content: bytes) -> C.Frame:
    """A well-formed frame (independent or linked blocks) -> lz4_craft's Frame with its structural byte positions."""
    flg = frame[4]
    hl = C.header_len(flg)
    bc, ck = bool(flg & C.FLG_BLOCK_CHK), bool(flg & C.FLG_CONTENT_CHK)
    marks = {"magic": [0, 1, 2, 3], "flg": [4], "bd": [5], "size": list(range(6, hl - 1)) if flg & C.FLG_SIZE else [], "hc": [hl - 1],
             "block_word": [], "token": [], "ext": [], "offset": [], "raw_data": [], "end_mark": [], "block_checksum": [],
             "content_checksum": []}
    spans, ip = [], hl
    while True:
        w = struct.unpack_from("<I", frame, ip)[0]
        if w == 0:
            break
        s, size = ip, w & 0x7FFFFFFF
        marks["block_word"] += list(range(ip, ip + 4))
        ip += 4
        if not w & 0x80000000:
            p, end = ip, ip + size
            while True:
                marks["token"].append(p)
                tok = frame[p]
                p += 1
                ll = tok >> 4
                if ll == 15:
                    while True:
                        marks["ext"].append(p)
                        p += 1
                        ll += frame[p - 1]
                        if frame[p - 1] != 255:
                            break
                p += ll
                if p >= end:
                    break
                marks["offset"].append(p)
                p += 2
                if tok & 15 == 15:
                    while True:
                        marks["ext"].append(p)
                        p += 1
                        if frame[p - 1] != 255:
                            break
        ip += size
        if bc:
            marks["block_checksum"] += list(range(ip, ip + 4))
            ip += 4
        spans.append((s, ip))
    marks["end_mark"] = list(range(ip, ip + 4))
    if ck:
        marks["content_checksum"] = list(range(ip + 4, ip + 8))
    return C.Frame(frame, content, marks, spans, [], flg)


def _gpu_frames(datas, flags, linked):
    """The stage's frames of `datas`: independent -- the fast path, the high-ratio lazy parse at level 9 and the optimal
    parse at level 5; linked -- the lazy parse at levels 3 and 9 and the optimal parse at level 5."""
    s = ChunkStage(0, max_batch_bytes=16 << 20, max_chunks=64, n_slots=1)
    try:
        out = []
        modes = ((3, False), (9, False), (5, True)) if linked else ((None, False), (9, False), (5, True))
        for level, optimal in modes:
            res = s.process(datas, level=level, checksum=bool(flags & CK), block_checksum=bool(flags & BC), linked=linked,
                            optimal=optimal)
            out += [bytes(r.frame) for r in res]
        return out
    finally:
        s.close()


def _generated_frames(rng, sizes, flags, linked):
    """lz4_craft streams (30 % stored blocks) in the stage's frame: linked ones reach back as far as the chunk's first byte."""
    out = []
    for n in sizes:
        st = C.gen_stream(rng, n, linked=linked, stored_p=0.3)
        f = C.assemble_frame(st.blocks, st.content, linked=linked and n > C.BLOCK, content_size=n > 0, block_checksum=bool(flags & BC),
                             content_checksum=bool(flags & CK))
        out.append(parse_frame(f.data, st.content))
    return out


def check_mutants(ctx, linked: bool):
    """Seeded structural mutants of the bases, over the four checksum combinations: status 0 exactly where `restores`
    holds (and then liblz4 restores the chunk), every code a receiver code, and repair as in check_repair."""
    rng = random.Random(4243 + linked)
    # linked: up to four blocks, so splice, swap and dup change what a block's matches read before it
    sizes = (0, 3000, 65536, 70000, 131072, 140000, 180000, 200000) if linked else (0, 1, 50, 3000, 65536, 70000, 140000)
    datas = [kind_chunk(KINDS[i % len(KINDS)], n, 70 + i) for i, n in enumerate(sizes)]
    total, reached = 0, {}
    for ck in CHECKSUMS:
        flags = (LINKED if linked else 0) | ck
        bases = [parse_frame(f, d) for f, d in zip(_gpu_frames(datas, flags, linked), datas * 3)]
        bases += [parse_frame(hc_model.liblz4_frame(d, lvl, linked=linked, content_checksum=bool(ck & CK), block_checksum=bool(ck & BC)), d)
                  for d in datas for lvl in (0, 9)]
        if linked:
            bases += _generated_frames(rng, sizes[1:], flags, linked)
        for b in bases:
            assert restores(b.data, b.content, flags)
        mut, src, names = [], [], []
        for _ in range(560):
            f = rng.choice(bases)
            name, m = C.random_mutant(rng, f, bases)
            mut.append(m)
            src.append(f.content)
            names.append(name)
        mut += [b.data for b in bases]
        src += [b.content for b in bases]
        names += ["base"] * len(bases)
        st, _, _ = run_verify(ctx, src, mut, flags, repair=False)
        bad = [(nm, s) for nm, m, d, s in zip(names, mut, src, st) if (s == 0) != restores(m, d, flags)]
        assert not bad, bad[:20]
        passed = [(m, d) for m, d, s in zip(mut, src, st) if s == 0]
        assert all(liblz4_whole(m, len(d)) == (d, len(m)) for m, d in passed)  # status 0 => liblz4 restores the chunk
        assert all(s in native.D_NAMES and s not in (native.D_AUTH, native.D_UNSUPPORTED) for s in st), sorted(set(st))
        check_repair(ctx, src, mut, flags, st)
        total += len(mut) - len(bases)
        for s in st:
            reached[s] = reached.get(s, 0) + 1
    print(f"{'linked' if linked else 'independent'}: {total} mutants, statuses {dict(sorted(reached.items()))}")
    assert total >= 2000
    assert {0, native.D_CORRUPT, native.D_MISMATCH, native.D_SIZE, native.D_TRUNCATED, native.D_LAYOUT, native.D_BAD_HEADER,
            native.D_CHECKSUM} <= set(reached), reached


def test_mutants_differential_and_repair(ctx):
    check_mutants(ctx, linked=False)


def test_linked_mutants_differential_and_repair(ctx):
    check_mutants(ctx, linked=True)


# ------------------------------------------------------------------------------------------------ (5) operator
DRIVER = r"""
import json, sys
from pathlib import Path
from skyplane_b200.harness import run_stream
base = Path(sys.argv[1]); n_req = int(sys.argv[2])
files = sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))
lens = [p.stat().st_size for p in files]
res = run_stream(base / "chunks", files, lens, n_req, n_workers=1, max_batch_chunks=8, max_batch_bytes=64 << 20, keep_frames=True,
                 verify_frames=True, block_checksum=True)
print("RESULT " + json.dumps(res))
"""


def test_operator_with_verify_frames():
    base = Path(tempfile.mkdtemp(prefix="skyb200_verify_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [synth.random_chunk(0, 8 << 20), synth.silesia_like_chunk(1, 8 << 20), b"", b"x" * 13, synth.silesia_like_chunk(2, (1 << 20) + 77)]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        n_req = 20
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), str(n_req)], capture_output=True, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        assert res["frame_verify"] == {}  # no complete record carries frame_verify_status
        for rec in res["records"]:
            data = pool[rec["pool_index"]]
            assert rec["md5"] == hashlib.md5(data).hexdigest()
            assert ref.lz4f_decompress(Path(rec["frame_path"]).read_bytes(), len(data)) == data
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
