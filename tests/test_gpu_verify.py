"""GPU tests of SKY_F_VERIFY: the sender checks every frame against its chunk and sends a stored-block frame for one that
does not restore it.

Bars: (1) clean frames -- at edge lengths of five data kinds, under the fast path, high-ratio levels 3 and 9, content and
block checksums and E2EE, every status is 0 and payloads and digests equal those of the same batch without the flag;
(2) a status table of crafted frames through sky_verify_device, with the earliest failing block's code winning in both
directions; (3) over seeded structural mutants of GPU and liblz4 frames, status 0 exactly when liblz4 (and, for frames
without checksums, the strict oracle) decodes the whole mutant to the chunk and its descriptor is the stage's; (4) with
frame_cap every failing frame becomes the stored-block frame the CPU assembles, which liblz4 decodes, and frame_len follows;
without it no byte changes, and with it nothing outside [frame, frame + cap) does (guard bytes between frames, whole slab
read back); (5) GatewayCompressHash(verify_frames=True) in the forked queue harness."""
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
    """The chunk's stored-block frame, assembled on the CPU: every block raw, with the flags' checksums."""
    f = tile_model.assemble(len(data), [(0, data[p : p + C.BLOCK]) for p in range(0, len(data), C.BLOCK)], bool(flags & BC))
    return with_content_checksum(f, data) if flags & CK else f


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
    """Do liblz4 and (for frames without checksums) the strict oracle decode the whole frame to `data`, with the stage's
    frame descriptor?"""
    if len(frame) < 6 or frame[4] != (0x68 if data else 0x60) | (0x04 if flags & CK else 0) | (0x10 if flags & BC else 0) or frame[5] != 0x40:
        return False
    got = liblz4_whole(frame, len(data))
    if got is None or got != (data, len(frame)):
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
    """With frame_cap: the same statuses, failing frames become the stored-block frame (liblz4 restores it), the others stay."""
    st2, after, flen = run_verify(ctx, datas, frames, flags, repair=True)
    assert st2 == st
    for i, (d, f, s) in enumerate(zip(datas, frames, st)):
        if s == 0:
            assert after[i] == f and flen[i] == len(f)
        else:
            want = stored_frame(d, flags)
            assert after[i] == want and flen[i] == len(want) == native.frame_need(len(d), bool(flags & CK), bool(flags & BC)), i
            assert ref.lz4f_decompress(after[i], len(d)) == d


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
        with pytest.raises(native.SkyChunkError) as e:
            s.ctx.wait_verify(slot.ticket)
        assert e.value.code == native.SKY_E_INVALID
        (r,) = s.collect(slot)
        assert r.verify_status == 0 and ref.lz4f_decompress(bytes(r.frame), 5000) == b"q" * 5000
        t = s.ctx.submit([buf.addr], [100], [buf.addr + 4096], [native.frame_need(100)], V)  # alone: LZ4 + MD5 + verify
        lens, _, ver, _ = s.ctx.wait_verify(t)
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


def _status_rows(rng: random.Random):
    """(name, chunk, frame, flags, status)"""
    rows = []
    for flags in CHECKSUMS:
        kw = dict(content_size=True, block_checksum=bool(flags & BC), content_checksum=bool(flags & CK))
        s = C.gen_stream(rng, 3 * C.BLOCK + 777, stored_p=0.0)
        n = len(s.content)
        tag = {0: "", CK: " ck", BC: " bc", CK | BC: " ck+bc"}[flags]
        good = C.assemble_frame(s.blocks, s.content, **kw)
        rows.append(("valid" + tag, s.content, good.data, flags, 0))
        blocks = list(s.blocks)
        blocks[1] = _mutate(blocks[1], _lit_pos(blocks[1]), bytes([blocks[1].data[_lit_pos(blocks[1])] ^ 0x01]))
        rows.append(("literal flipped" + tag, s.content, C.assemble_frame(blocks, s.content, **kw).data, flags, native.D_MISMATCH))
        blocks = list(s.blocks)
        blocks[2] = _mutate(blocks[2], blocks[2].marks["offset"][-1], b"\0\0")
        rows.append(("offset 0" + tag, s.content, C.assemble_frame(blocks, s.content, **kw).data, flags, native.D_CORRUPT))
        rows.append(("content size + 1" + tag, s.content, C.with_header(good.data, content_size=n + 1), flags, native.D_SIZE))
        rows.append(("truncated" + tag, s.content, good.data[:-1], flags, native.D_TRUNCATED))
        rows.append(("trailing byte" + tag, s.content, good.data + b"\0", flags, native.D_SIZE))
        other = C.gen_stream(rng, n, stored_p=0.3)
        rows.append(("other data, same length" + tag, s.content, C.assemble_frame(other.blocks, other.content, **kw).data, flags,
                     native.D_MISMATCH))
        half = s.content[:50000], s.content[50000:100000]
        rows.append(("short middle block" + tag, s.content[:100000],
                     C.assemble_frame([C.stored_block(half[0]), C.stored_block(half[1])], s.content[:100000], **kw).data, flags,
                     native.D_LAYOUT))
        rows.append(("linked FLG" + tag, s.content, C.assemble_frame(s.blocks, s.content, linked=True, **kw).data, flags,
                     native.D_BAD_HEADER))
        # offset into the previous block: decodes as a linked frame, not as an independent one
        buf = bytearray(s.content[: C.BLOCK])
        w = C.BlockWriter(buf)
        w.literals(rng.randbytes(30)).match(31, 10).literals(rng.randbytes(500))
        prev = bytes(buf)
        rows.append(("offset into the previous block" + tag, prev, C.assemble_frame([s.blocks[0], w.close()], prev, **kw).data, flags,
                     native.D_CORRUPT))
        # a full block whose last match ends 3 bytes before its end (liblz4 needs 5 literals there)
        buf = bytearray()
        w = C.BlockWriter(buf)
        w.literals(rng.randbytes(40)).match(13, C.BLOCK - 43).literals(rng.randbytes(3))
        tail = bytes(buf)
        rows.append(("match into the last 5 bytes" + tag, tail, C.assemble_frame([w.close()], tail, **kw).data, flags, native.D_CORRUPT))
        if flags & BC:
            rows.append(("block checksum" + tag, s.content, C.flip(good.data, good.marks["block_checksum"][6], 0x01), flags,
                         native.D_CHECKSUM))
        if flags & CK:
            rows.append(("content checksum" + tag, s.content, C.flip(good.data, good.marks["content_checksum"][0], 0x01), flags,
                         native.D_CHECKSUM))
    # earliest failing block: block 0 corrupt (its checksum right), blocks 1..3 with wrong checksums -- and the mirror image
    s = C.gen_stream(rng, 4 * C.BLOCK, stored_p=0.0)
    for corrupt_first in (True, False):
        blocks = [(_mutate(b, b.marks["offset"][-1], b"\0\0") if (j == 0) == corrupt_first else b) for j, b in enumerate(s.blocks)]
        f = C.assemble_frame(blocks, s.content, content_size=True, block_checksum=True)
        data = bytearray(f.data)
        for j in range(4):
            if (j == 0) != corrupt_first:
                data[f.spans[j][1] - 1] ^= 0x40  # the block's checksum
        rows.append((f"precedence, corrupt first={corrupt_first}", s.content, bytes(data), BC,
                     native.D_CORRUPT if corrupt_first else native.D_CHECKSUM))
    return rows


def test_status_table_and_repair(ctx):
    rows = _status_rows(random.Random(9))
    for name, data, frame, flags, code in rows:  # the references agree with every row but one: a short block before the last
        if not name.startswith("short middle block"):  # is LZ4, but not the stage's layout (64 KiB blocks, only the last short)
            assert restores(frame, data, flags) == (code == 0), name
    for flags in CHECKSUMS:
        sel = [r for r in rows if r[3] == flags]
        datas, frames = [r[1] for r in sel], [r[2] for r in sel]
        st, _, _ = run_verify(ctx, datas, frames, flags, repair=False)
        assert [(r[0], s) for r, s in zip(sel, st)] == [(r[0], r[4]) for r in sel]
        check_repair(ctx, datas, frames, flags, st)


# ------------------------------------------------------------------------------------------------ (3) differential
def parse_frame(frame: bytes, content: bytes) -> C.Frame:
    """A well-formed independent-block frame -> lz4_craft's Frame with its structural byte positions."""
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


def _gpu_frames(ctx, datas, flags):
    s = ChunkStage(0, max_batch_bytes=16 << 20, max_chunks=64, n_slots=1)
    try:
        out = []
        for level in (None, 9):
            res = s.process(datas, level=level, checksum=bool(flags & CK), block_checksum=bool(flags & BC))
            out += [bytes(r.frame) for r in res]
        return out
    finally:
        s.close()


def test_mutants_differential_and_repair(ctx):
    rng = random.Random(4243)
    sizes = (0, 1, 50, 3000, 65536, 70000, 140000)
    datas = [kind_chunk(KINDS[i % len(KINDS)], n, 70 + i) for i, n in enumerate(sizes)]
    total = 0
    for flags in CHECKSUMS:
        bases = [parse_frame(f, d) for f, d in zip(_gpu_frames(ctx, datas, flags), datas + datas)]
        bases += [parse_frame(hc_model.liblz4_frame(d, lvl, content_checksum=bool(flags & CK), block_checksum=bool(flags & BC)), d)
                  for d in datas for lvl in (0, 9)]
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
        assert all(s in native.D_NAMES and s not in (native.D_AUTH, native.D_UNSUPPORTED) for s in st), sorted(set(st))
        check_repair(ctx, src, mut, flags, st)
        total += len(mut) - len(bases)
    assert total >= 2000


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
