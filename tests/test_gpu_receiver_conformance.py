"""GPU receiver against crafted, generated and mutated LZ4 frames and SecretBoxes.

Every device decode goes through `guarded_decode`: frames and output regions sit in slabs with >= 256 guard bytes
between them, pre-filled with a pattern, and after each batch the whole output slab and the whole frame slab are read
back.  Nothing outside a chunk's [out, out + raw_len) may change, the frames must be untouched, and every ok chunk must
hold exactly the expected bytes with their MD5.  Expected bytes come from the frame generator (tests/lz4_craft.py) or,
for mutants, from the strict oracle (frames without checksums) or liblz4 (checksummed frames) -- never from the GPU."""
import hashlib
import math
import random

import numpy as np
import pytest

import lz4_craft as C
import oracle
import oracle.reflib as ref
from skyplane_b200 import native

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300, method="thread")]

GAP = 256
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 1 << 30, 4096, 0)
    yield c
    c.close()


def _pattern(n: int, seed: int) -> np.ndarray:
    return ((np.arange(n, dtype=np.uint32) * 167 + seed) & 0xFF).astype(np.uint8)


def guarded_decode(ctx, frames, raw_lens, expect):
    """Decode `frames` on the device with guard bytes around every frame and output region.  expect[i]: the bytes
    chunk i must decode to if the GPU accepts it, or None if it must not be accepted.  -> (status, outputs)"""
    f_off, o_off, fp, op = [], [], GAP, GAP
    for f, r in zip(frames, raw_lens):
        f_off.append(fp)
        o_off.append(op)
        fp += native.round16(len(f)) + GAP
        op += native.round16(r) + GAP
    fslab = _pattern(fp, 0x3C)
    for f, o in zip(frames, f_off):
        fslab[o : o + len(f)] = np.frombuffer(f, np.uint8)
    oslab = _pattern(op, 0x5B)
    d_f, d_o = ctx.device_alloc(fp), ctx.device_alloc(op)
    try:
        ctx.h2d(d_f, fslab)
        ctx.h2d(d_o, oslab)
        st, dg, _ = ctx.decode_device(d_f, f_off, [len(f) for f in frames], d_o, o_off, list(raw_lens))
        fback = np.frombuffer(ctx.d2h(d_f, fp), np.uint8)
        oback = np.frombuffer(ctx.d2h(d_o, op), np.uint8)
    finally:
        ctx.device_free(d_f)
        ctx.device_free(d_o)
    assert np.array_equal(fback, fslab), "the decoder wrote into the frame slab"
    outside = np.ones(op, bool)
    for o, r in zip(o_off, raw_lens):
        outside[o : o + r] = False
    bad = np.flatnonzero((oback != oslab) & outside)
    if bad.size:
        i = int(np.searchsorted(o_off, bad[0], side="right")) - 1
        pytest.fail(f"{bad.size} guard bytes changed, first at slab byte {bad[0]} (behind chunk {i}, status {st[max(i, 0)]})")
    outs = []
    for i, (o, r) in enumerate(zip(o_off, raw_lens)):
        if st[i] != native.D_OK:
            outs.append(None)
            continue
        out = oback[o : o + r].tobytes()
        assert expect[i] is not None, f"chunk {i}: accepted by the GPU, rejected by the reference"
        assert out == expect[i], f"chunk {i}: decoded bytes differ from the reference's"
        assert dg[i] == hashlib.md5(out).digest(), f"chunk {i}: digest"
        outs.append(out)
    return st, outs


def reference_decode(frame: bytes, raw_len: int):
    """The reference's bytes for a (possibly mutated) frame, or None where it rejects it: liblz4 for frames whose FLG
    carries a checksum bit, the strict oracle otherwise."""
    try:
        if len(frame) > 4 and frame[4] & (C.FLG_BLOCK_CHK | C.FLG_CONTENT_CHK):
            out = ref.lz4f_decompress(frame, raw_len)
        else:
            out = oracle.lz4f_decode(frame, raw_len)
    except ValueError:  # OracleError is a ValueError
        return None
    return out if len(out) == raw_len else None


# ------------------------------------------------------------------------------------------------ sequence edges
def _edge_streams(rng: random.Random):
    """name -> (content, blocks, ok in an independent frame).  Block 0 is ordinary; the edge sits in block 1 (or 0)."""
    R = rng.randbytes
    cases = {}

    def two_blocks(fill):
        buf = bytearray()
        b0 = C.gen_stream(rng, C.BLOCK, linked=False, stored_p=0.0)
        buf += b0.content
        w = C.BlockWriter(buf)
        fill(w)
        return bytes(buf), [b0.blocks[0], w.close()]

    def offsets_31_32_33(w):
        w.literals(R(80))
        for off in (31, 32, 33):
            for ml in (4, 5, 31, 32, 33, 63, 64, 65, 95, 96, 97, 300):
                w.literals(R(rng.randrange(0, 3))).match(off, ml)
        w.literals(R(8))

    def match_len_32k(w):
        w.literals(R(256))
        for off in (1, 2, 7, 16, 31, 32, 33, 64, 200):
            for k in range(1, 6):
                for d in (-1, 0, 1):
                    w.literals(R(1)).match(off, 32 * k + d)
        w.literals(R(6))

    def length_fields(w):
        w.literals(R(64))
        for v in C.LEN_EDGES:
            w.literals(R(v)).match(rng.randrange(1, 65), C.MIN_MATCH + v)
        w.literals(R(C.LEN_EDGES[-1]))

    def reach_block_start(w):  # offset == position in the block: the oldest byte an independent block may use
        w.literals(R(50)).match(50, 20)
        w.literals(R(10)).match(w.pos, 4)
        w.literals(R(3)).match(w.pos, 300)
        w.literals(R(7))

    def before_block_start(w):  # one byte further: the last byte of block 0, legal only when blocks are linked
        w.literals(R(30)).match(31, 10)
        w.literals(R(9))

    def match_to_block_end(w):  # the last match ends at the block end; a zero-literal last sequence follows
        w.literals(R(40)).match(13, 77)
        w.literals(R(5)).match(1, 33)

    for name, fill in [("offsets_31_32_33", offsets_31_32_33), ("match_len_32k", match_len_32k), ("length_fields", length_fields),
                       ("reach_block_start", reach_block_start), ("before_block_start", before_block_start),
                       ("match_to_block_end", match_to_block_end)]:
        content, blocks = two_blocks(fill)
        cases[name] = (content, blocks, name != "before_block_start")

    # a match that reaches exactly byte 0 of the chunk, in block 0
    buf = bytearray()
    w = C.BlockWriter(buf)
    w.literals(R(100)).match(100, 40).literals(R(2)).match(w.pos, 64)
    w.literals(R(6)).match(7, C.BLOCK - w.pos - 12).literals(R(12))  # the rest of a full-size block
    assert w.pos == C.BLOCK
    tail = R(3000)
    cases["reach_chunk_byte0"] = (bytes(buf) + tail, [w.close(), C.stored_block(tail)], True)

    # a full-size block whose last match ends exactly at its end, then a zero-literal sequence, then another block
    buf = bytearray()
    w = C.BlockWriter(buf)
    w.literals(R(1000)).match(1000, 30000)
    w.literals(R(17)).match(32, C.BLOCK - w.pos - 40)
    w.literals(R(17)).match(1, C.BLOCK - w.pos)
    assert w.pos == C.BLOCK
    b1 = C.gen_stream(rng, 5000, stored_p=0.0)
    cases["full_block_match_to_end"] = (bytes(buf) + b1.content, [w.close(), b1.blocks[0]], True)
    return cases


def test_sequence_edges_linked_and_independent(ctx):
    rng = random.Random(2024)
    frames, raws, expect, want = [], [], [], []
    for name, (content, blocks, indep_ok) in _edge_streams(rng).items():
        for linked in (False, True):
            for opts in ({}, {"content_size": True, "block_checksum": True, "content_checksum": True}):
                f = C.assemble_frame(blocks, content, linked=linked, **opts)
                ok = linked or indep_ok
                frames.append(f.data)
                raws.append(len(content))
                expect.append(content if ok else None)
                want.append((name, linked, bool(opts), native.D_OK if ok else native.D_CORRUPT))
                if ok and not opts:
                    assert oracle.lz4f_decode(f.data, len(content)) == content, name
    st, _ = guarded_decode(ctx, frames, raws, expect)
    got = [(n, l, o, s) for (n, l, o, _), s in zip(want, st)]
    assert got == want


# ------------------------------------------------------------------------------------------------ random valid streams
def _random_batch(rng: random.Random, n: int):
    frames, raws, expect = [], [], []
    specials = [0, 0, 1, 5, 12, 13, 65535, 65536, 65537, 131072, 1 << 20]
    for i in range(n):
        size = specials[i] if i < len(specials) else int(math.exp(rng.uniform(0, math.log(1100000))))
        linked = rng.random() < 0.4
        conforming = rng.random() < 0.7
        opts = {"content_size": rng.random() < 0.5}
        if rng.random() < 0.3:
            opts.update(block_checksum=rng.random() < 0.7, content_checksum=rng.random() < 0.7)
        s = C.gen_stream(rng, size, linked=linked, conforming=conforming)
        frames.append(s.frame(**opts).data)
        raws.append(size)
        expect.append(s.content)
    return frames, raws, expect


def test_random_valid_streams(ctx):
    rng = random.Random(77)
    for b in range(3):
        frames, raws, expect = _random_batch(rng, 110)
        st, _ = guarded_decode(ctx, frames, raws, expect)
        assert st == [native.D_OK] * len(frames), [(i, s) for i, s in enumerate(st) if s]


# ------------------------------------------------------------------------------------------------ status table
def _set(frame: bytes, pos: int, data: bytes) -> bytes:
    return frame[:pos] + data + frame[pos + len(data):]


def _status_table(rng: random.Random):
    s = C.gen_stream(rng, 150000, stored_p=0.0)  # 64 KiB + 64 KiB + 18928, all compressed
    f, fs = s.frame(), s.frame(content_size=True)
    n = len(s.content)
    rows = []  # (name, frame, raw_len, status)
    for v in (0x00, 0x80, 0xC0):
        rows.append((f"version {v >> 6:02b}", C.with_header(f.data, flg=(f.flg & 0x3F) | v), n, native.D_BAD_HEADER))
    rows.append(("FLG reserved bit", C.with_header(f.data, flg=f.flg | C.FLG_RESERVED), n, native.D_BAD_HEADER))
    for bit in (0x01, 0x02, 0x04, 0x08, 0x80):
        rows.append((f"BD reserved bit {bit:#x}", C.with_header(f.data, bd=C.BD_64K | bit), n, native.D_BAD_HEADER))
    for bsid in range(8):
        if bsid != 4:
            rows.append((f"block size id {bsid}", C.with_header(f.data, bd=bsid << 4), n,
                         native.D_BAD_HEADER if bsid < 4 else native.D_LAYOUT))
    rows.append(("header checksum", C.flip(f.data, 6, 0x10), n, native.D_BAD_HEADER))
    rows.append(("dictID", C.with_header(f.data, flg=f.flg | C.FLG_DICT, dict_id=0x12345678), n, native.D_UNSUPPORTED))
    for cs in (n + 1, n - 1, 0, n + C.BLOCK):
        rows.append((f"content size {cs}", C.with_header(fs.data, content_size=cs), n, native.D_SIZE))
    for size in (C.BLOCK + 1, 0x7FFFFFFF):
        rows.append((f"block word {size:#x}", C.resize_block(f, 0, size), n, native.D_CORRUPT))
    half = s.content[:50000], s.content[50000:100000]
    short = C.assemble_frame([C.stored_block(half[0]), C.stored_block(half[1])], s.content[:100000])
    rows.append(("short stored block not last", short.data, 100000, native.D_LAYOUT))
    rows.append(("early EndMark", C.set_word(f.data, C.block_word_pos(f, 2), 0), n, native.D_SIZE))
    rows.append(("extra block", C.dup_block(f, 2), n, native.D_SIZE))
    rows.append(("missing EndMark", C.drop_end_mark(f), n, native.D_TRUNCATED))
    for k in (0, len(f.marks["offset"]) // 2, -1):
        rows.append((f"offset 0 #{k}", _set(f.data, f.marks["offset"][k], b"\0\0"), n, native.D_CORRUPT))
    fc = s.frame(block_checksum=True, content_checksum=True)
    rows.append(("block checksum", C.flip(fc.data, fc.marks["block_checksum"][5], 0x01), n, native.D_CHECKSUM))
    rows.append(("content checksum", C.flip(fc.data, fc.marks["content_checksum"][0], 0x01), n, native.D_CHECKSUM))
    # the expected raw length off by one byte or one block on valid frames
    tail = s.content[2 * C.BLOCK:]
    stored_last = C.assemble_frame(s.blocks[:2] + [C.stored_block(tail)], s.content)
    full = C.gen_stream(rng, 2 * C.BLOCK, stored_p=0.0)
    table = {  # frame -> status for raw_len + 1, - 1, + 65536, - 65536
        "last block compressed": (f.data, n, [native.D_LAYOUT, native.D_CORRUPT, native.D_SIZE, native.D_SIZE]),
        "with content size": (fs.data, n, [native.D_SIZE] * 4),
        "last block stored": (stored_last.data, n, [native.D_LAYOUT, native.D_LAYOUT, native.D_SIZE, native.D_SIZE]),
        "two full blocks": (full.frame().data, 2 * C.BLOCK, [native.D_SIZE, native.D_CORRUPT, native.D_SIZE, native.D_SIZE]),
        "linked, two full blocks": (C.gen_stream(rng, 2 * C.BLOCK, linked=True, stored_p=0.0).frame().data, 2 * C.BLOCK,
                                    [native.D_SIZE, native.D_CORRUPT, native.D_SIZE, native.D_SIZE]),
    }
    for name, (frame, r, codes) in table.items():
        for d, code in zip((1, -1, C.BLOCK, -C.BLOCK), codes):
            rows.append((f"{name}: raw_len {d:+d}", frame, r + d, code))
    rows.append(("empty frame: raw_len 1", C.stored_frame(b"").data, 1, native.D_SIZE))
    return rows


def test_status_table(ctx):
    rng = random.Random(5)
    rows = _status_table(rng)
    good = C.gen_stream(rng, 70000, stored_p=0.0)
    gf = good.frame().data
    frames, raws, expect = [gf], [len(good.content)], [good.content]
    for _, frame, r, _ in rows:
        frames += [frame, gf]
        raws += [r, len(good.content)]
        expect += [None, good.content]
    st, _ = guarded_decode(ctx, frames, raws, expect)
    assert st[0::2] == [native.D_OK] * (len(rows) + 1)
    assert [(name, s) for (name, *_), s in zip(rows, st[1::2])] == [(name, code) for name, _, _, code in rows]


# ------------------------------------------------------------------------------------------------ prefixes
def _prefix_lengths(rng: random.Random, f: C.Frame, sample: int = 40):
    n = len(f.data)
    first_data = f.spans[0][0] + 4 if f.spans else n
    cuts = set(range(0, min(first_data, n - 1) + 1))
    for b in [s for span in f.spans for s in span] + [f.marks["end_mark"][0], n - 4]:
        cuts.update(range(max(0, b - 8), min(n, b + 9)))
    cuts.update(rng.sample(range(n), min(sample, n)))
    cuts.discard(n)
    return sorted(cuts)


def _prefix_bases(rng: random.Random):
    s = C.gen_stream(rng, 150000, stored_p=0.3)
    l = C.gen_stream(rng, 140000, linked=True)
    return [s.frame(), s.frame(content_size=True), s.frame(block_checksum=True, content_checksum=True),
            l.frame(content_size=True, content_checksum=True), C.stored_frame(b""), C.stored_frame(b"", content_size=True),
            C.stored_frame(b"", content_checksum=True), C.stored_frame(rng.randbytes(300))]


def test_every_proper_prefix_is_truncated(ctx):
    rng = random.Random(31)
    frames, raws, expect = [], [], []
    for f in _prefix_bases(rng):
        for k in _prefix_lengths(rng, f):
            frames += [f.data[:k], f.data]
            raws += [len(f.content)] * 2
            expect += [None, f.content]
    st, _ = guarded_decode(ctx, frames, raws, expect)
    assert st[1::2] == [native.D_OK] * (len(frames) // 2)
    bad = [(len(fr), s) for fr, s in zip(frames[0::2], st[0::2]) if s != native.D_TRUNCATED]
    assert not bad, bad[:20]


# ------------------------------------------------------------------------------------------------ random mutants
def _mutation_bases(rng: random.Random):
    bases = []
    for size in (0, 1, 50, 3000, 65536, 70000, 140000):
        for linked in (False, True):
            for opts in ({}, {"content_size": True}, {"block_checksum": True, "content_checksum": True}):
                s = C.gen_stream(rng, size, linked=linked, conforming=bool(opts.get("block_checksum")) or rng.random() < 0.5)
                bases.append(s.frame(**opts))
    return bases


def test_random_mutants_differential(ctx):
    rng = random.Random(4242)
    bases = _mutation_bases(rng)
    pool = [b for b in bases if len(b.content) <= 70000]
    for batch in range(3):
        frames, raws, expect, names = [], [], [], []
        first = rng.choice(pool)
        frames.append(first.data)
        raws.append(len(first.content))
        expect.append(first.content)
        for _ in range(1000):
            f = rng.choice(bases)
            name, m = C.random_mutant(rng, f, bases)
            nb = rng.choice(pool)
            frames += [m, nb.data]
            raws += [len(f.content), len(nb.content)]
            expect += [reference_decode(m, len(f.content)), nb.content]
            names.append(name)
        st, _ = guarded_decode(ctx, frames, raws, expect)
        assert st[0::2] == [native.D_OK] * (len(names) + 1)  # every neighbour
        assert all(s in native.D_NAMES and s != native.D_AUTH for s in st[1::2]), sorted(set(st[1::2]))


# ------------------------------------------------------------------------------------------------ status precedence
def _precedence_frame(rng: random.Random, linked: bool, corrupt_first: bool) -> C.Frame:
    """16 compressed 64 KiB blocks with block checksums.  corrupt_first: block 0 has a zero offset in its last
    sequence (and a correct checksum over it), blocks 1..15 a wrong checksum; otherwise the mirror image."""
    s = C.gen_stream(rng, 16 * C.BLOCK, linked=linked, stored_p=0.0)
    corrupt = [0] if corrupt_first else list(range(1, 16))
    blocks = []
    for j, b in enumerate(s.blocks):
        if j in corrupt:
            o = b.marks["offset"][-1]
            b = C.Block(b.data[:o] + b"\0\0" + b.data[o + 2:], False, b.marks)
        blocks.append(b)
    f = C.assemble_frame(blocks, s.content, linked=linked, block_checksum=True, content_checksum=True)
    for j in range(16):
        if j not in corrupt:
            f.data = C.flip(f.data, f.marks["block_checksum"][4 * j + 2], 0x40)
    return f


@pytest.mark.parametrize("linked", [False, True], ids=["independent", "linked"])
def test_status_is_the_earliest_failing_blocks(ctx, linked):
    rng = random.Random(8 + linked)
    good = [C.gen_stream(rng, size, linked=linked) for size in (100000, 16 * C.BLOCK, 3000)]
    frames, raws, expect, want = [], [], [], []
    for copy in range(4):
        for corrupt_first, code in ((True, native.D_CORRUPT), (False, native.D_CHECKSUM)):
            f = _precedence_frame(rng, linked, corrupt_first)
            for g in good:
                frames.append(g.frame(block_checksum=True).data)
                raws.append(len(g.content))
                expect.append(g.content)
                want.append(native.D_OK)
            frames.append(f.data)
            raws.append(len(f.content))
            expect.append(None)
            want.append(code)
    st, _ = guarded_decode(ctx, frames, raws, expect)
    assert st == want


# ------------------------------------------------------------------------------------------------ SecretBox
def _box_lengths():
    return sorted(set(range(0, 201)) | {4096 * k + d for k in (1, 2, 3) for d in (-17, -16, -15, -1, 0, 1, 15, 16, 17)} | {65551})


def _box_payloads(rng: random.Random):
    """(plaintext, raw_len, expected status, expected bytes): stored-block frames of an exact length where one exists,
    other plaintexts (not frames) for the lengths no frame has."""
    out = []
    for n in _box_lengths():
        if n == 11 or n >= 16:
            payload = rng.randbytes(n - 15) if n >= 16 else b""
            out.append((C.stored_frame(payload).data, len(payload), native.D_OK, payload))
        else:
            out.append((rng.randbytes(n), 0, native.D_TRUNCATED if n < 11 else native.D_BAD_HEADER, None))
    big = [rng.randbytes(C.BLOCK) for _ in range(16)]
    content = b"".join(big)
    out.append((C.assemble_frame([C.stored_block(b) for b in big], content).data, len(content), native.D_OK, content))
    return out


@pytest.fixture(scope="module")
def stage():
    from skyplane_b200.stage import ChunkStage

    s = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=512, n_slots=1)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


def test_secretbox_open_at_every_length_class(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    rng = random.Random(606)
    box = nacl_secret.SecretBox(KEY)
    items = _box_payloads(rng)
    boxes = [bytes(box.encrypt(p, rng.randbytes(24))) for p, *_ in items]
    assert all(len(b) == len(p) + 40 for b, (p, *_) in zip(boxes, items))
    out = stage.decode(boxes, [r for _, r, _, _ in items], encrypted=True)
    got = [(len(p), st, data == want) for (p, _, _, want), (data, _, st) in zip(items, out)]
    assert got == [(len(p), code, True) for p, _, code, _ in items]
    # the last ciphertext byte and the last tag byte are covered by the tag
    tampered, raws = [], []
    for b, (p, r, _, _) in zip(boxes, items):
        if p:
            tampered.append(C.flip(b, len(b) - 1, 0x01))
            raws.append(r)
        tampered.append(C.flip(b, 39, 0x80))
        raws.append(r)
    out = stage.decode(tampered, raws, encrypted=True)
    assert all(st == native.D_AUTH and data is None for data, _, st in out)


def test_secretbox_seal_at_every_length_class(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    rng = random.Random(607)
    box = nacl_secret.SecretBox(KEY)
    datas = [rng.randbytes(n) for n in _box_lengths()] + [rng.randbytes(1048651)]
    nonces = rng.randbytes(24 * len(datas))
    res = stage.process(datas, compress=False, encrypt=True, nonces=nonces)
    for i, (d, r) in enumerate(zip(datas, res)):
        assert bytes(r.frame) == bytes(box.encrypt(d, nonces[24 * i : 24 * i + 24])), len(d)


def test_every_proper_prefix_of_a_box_is_rejected(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    rng = random.Random(608)
    box = nacl_secret.SecretBox(KEY)
    small = C.stored_frame(rng.randbytes(300))
    s = C.gen_stream(rng, 150000)
    large = s.frame(content_checksum=True)
    items = []  # (box or a proper prefix of it, raw_len, the frame's content if whole)
    for f in (small, large):
        b = bytes(box.encrypt(f.data, rng.randbytes(24)))
        cuts = range(len(b)) if len(b) < 1000 else sorted(set(range(64)) | set(rng.sample(range(len(b)), 150)) |
                                                        set(range(len(b) - 40, len(b))))
        items += [(b[:k], len(f.content), None) for k in cuts] + [(b, len(f.content), f.content)]
    out = stage.decode([b for b, _, _ in items], [r for _, r, _ in items], encrypted=True)
    for (b, _, whole), (data, _, st) in zip(items, out):
        if whole is not None:
            assert st == native.D_OK and data == whole
        else:
            assert st == native.D_AUTH and data is None, len(b)
