"""GPU tests of SKY_F_BLOCK_CHECKSUM: LZ4 block checksums (XXH32 of every block as stored) from the sender.

Bars: on the fast path and at high-ratio levels 3, 5 and 9, alone and with SKY_F_CHECKSUM, the frames equal the sequential
twin's with block checksums byte for byte at edge lengths; the digests are hashlib's; the frames decode with liblz4 (which
verifies the checksums), pyarrow and sky_decode; a flipped byte inside block j's data gives SKY_D_CHECKSUM and liblz4
rejects the frame; sealed payloads open with PyNaCl; pipelined slots filled to capacity still fit; MD5 alone with the
flag is SKY_E_INVALID; and no write lands outside [dst, dst + out_len) (256-byte guard bands between frames)."""
import hashlib
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle.reflib as ref
from skyplane_b200 import native
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import hc_model  # noqa: E402
import tile_model  # noqa: E402
from test_checksum_format import with_content_checksum  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

BC, CK = native.F_BLOCK_CHECKSUM, native.F_CHECKSUM
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
GAP = 256
LENS = [0, 1, 12, 13, 65535, 65536, 65537, 3 * 65536 + 100]
MODES = [("fast", 0, None), ("hc3", native.hc_level_flag(3), 3), ("hc5", native.hc_level_flag(5), 5), ("hc9", native.hc_level_flag(9), 9)]


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 1 << 30, 4096, 0)
    yield c
    c.close()


def _pattern(n: int, seed: int) -> np.ndarray:
    return ((np.arange(n, dtype=np.uint32) * 167 + seed) & 0xFF).astype(np.uint8)


def chunk(n: int, seed: int) -> bytes:
    """Half text, half random: compressed and stored blocks in one chunk."""
    rng = np.random.default_rng(seed)
    text = (b"it was the best of times, it was the worst of times; " * (n // 50 + 2))[: n // 2]
    return text + rng.bytes(n - len(text))


def run_guarded(ctx, chunks, flags):
    """sky_process_device with dst_cap = frame_need and GAP guard bytes around every frame region; fails on any byte written
    outside [dst, dst + out_len).  -> (frames, digests)"""
    ck, bc = bool(flags & CK), bool(flags & BC)
    src_off, dst_off, caps, ip, op = [], [], [], 0, GAP
    for c in chunks:
        src_off.append(ip)
        dst_off.append(op)
        caps.append(native.frame_need(len(c), ck, bc))
        ip += native.round16(len(c))
        op += native.round16(caps[-1]) + GAP
    slab = _pattern(op, 0x3C)
    d_in, d_out = ctx.device_alloc(ip + 64), ctx.device_alloc(op)
    try:
        for c, o in zip(chunks, src_off):
            if c:
                ctx.h2d(d_in + o, c)
        ctx.h2d(d_out, slab)
        lens, digests, _ = ctx.process_device(d_in, src_off, [len(c) for c in chunks], d_out, dst_off, caps, flags)
        back = np.frombuffer(ctx.d2h(d_out, op), np.uint8)
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)
    outside = np.ones(op, bool)
    for o, n, cap in zip(dst_off, lens, caps):
        assert n <= cap
        outside[o : o + n] = False
    bad = np.flatnonzero((back != slab) & outside)
    assert bad.size == 0, f"{bad.size} bytes written outside the frames, first at slab byte {bad[0]}"
    return [back[o : o + n].tobytes() for o, n in zip(dst_off, lens)], digests


def twin(data: bytes, level, ck: bool) -> bytes:
    f = (tile_model.frame(data, block_checksum=True) if level is None
         else hc_model.frame(data, hc_model.kernel_opts(level=level), block_checksum=True))
    return with_content_checksum(f, data) if ck else f


def decode(ctx, frames, raw_lens):
    f_off, o_off, fp, op = [], [], 0, 0
    for f, r in zip(frames, raw_lens):
        f_off.append(fp)
        o_off.append(op)
        fp += native.round16(len(f))
        op += native.round16(r)
    d_f, d_o = ctx.device_alloc(fp + 64), ctx.device_alloc(op + 64)
    try:
        for f, o in zip(frames, f_off):
            ctx.h2d(d_f + o, f)
        st, dg, _ = ctx.decode_device(d_f, f_off, [len(f) for f in frames], d_o, o_off, list(raw_lens))
        return [ctx.d2h(d_o + o, r) if s == 0 else None for o, r, s in zip(o_off, raw_lens, st)], dg, st
    finally:
        ctx.device_free(d_f)
        ctx.device_free(d_o)


@pytest.mark.parametrize("ck", [False, True], ids=["bc", "bc+checksum"])
@pytest.mark.parametrize("mode,hc_bits,level", MODES, ids=[m[0] for m in MODES])
def test_frames_equal_the_twin_and_decode(ctx, mode, hc_bits, level, ck):
    pa = pytest.importorskip("pyarrow")
    lens = LENS + ([8 << 20] if mode in ("fast", "hc5") else [(1 << 20) + 7])
    datas = [chunk(n, 100 + n % 97) for n in lens]
    flags = hc_bits | BC | (CK if ck else 0)
    frames, dg = run_guarded(ctx, datas, flags)
    assert dg == [hashlib.md5(d).digest() for d in datas]
    for d, f in zip(datas, frames):
        n = len(d)
        assert f == twin(d, level, ck), (mode, n)
        assert f[4] == (0x70 if not n else 0x78) | (0x04 if ck else 0)
        assert ref.lz4f_decompress(f, n) == d  # liblz4 verifies every block checksum (and the content checksum)
        if n:
            assert pa.decompress(f, decompressed_size=n, codec="lz4").to_pybytes() == d
    outs, dgd, st = decode(ctx, frames, [len(d) for d in datas])
    assert st == [0] * len(datas) and outs == datas and dgd == dg


def test_only_the_checksum_words_differ_from_the_plain_frame(ctx):
    datas = [chunk(n, 7) for n in (1, 65537, 5 * 65536)]
    plain, dg0 = run_guarded(ctx, datas, 0)
    frames, dg = run_guarded(ctx, datas, BC)
    assert dg == dg0
    for d, p, f in zip(datas, plain, frames):
        nblk = -(-len(d) // 65536)
        assert len(f) == len(p) + 4 * nblk
        pos_p, pos_f = 15, 15
        for _ in range(nblk):
            word = int.from_bytes(p[pos_p : pos_p + 4], "little")
            size = word & 0x7FFFFFFF
            blk = p[pos_p + 4 : pos_p + 4 + size]
            assert f[pos_f : pos_f + 4 + size] == p[pos_p : pos_p + 4 + size]
            assert f[pos_f + 4 + size : pos_f + 8 + size] == tile_model.xxh32(blk).to_bytes(4, "little")
            pos_p += 4 + size
            pos_f += 8 + size
        assert f[pos_f:] == p[pos_p:] == bytes(4)


@pytest.mark.parametrize("hc_bits", [0, native.hc_level_flag(5)], ids=["fast", "hc5"])
def test_a_flipped_block_byte_is_a_checksum_failure(ctx, hc_bits):
    data = chunk(6 * 65536 + 321, 3)
    (f,), _ = run_guarded(ctx, [data], hc_bits | BC)
    starts, pos = [], 15
    while True:
        size = int.from_bytes(f[pos : pos + 4], "little") & 0x7FFFFFFF
        if not size:
            break
        starts.append((pos + 4, size))
        pos += 8 + size
    assert len(starts) == 7
    bad = []
    for j, (s, size) in enumerate(starts):
        b = bytearray(f)
        b[s + (j * 7919) % size] ^= 0x20
        bad.append(bytes(b))
        with pytest.raises(ValueError):
            ref.lz4f_decompress(bytes(b), len(data))
    outs, _, st = decode(ctx, bad + [f], [len(data)] * (len(bad) + 1))
    assert st == [native.D_CHECKSUM] * len(bad) + [0] and outs[-1] == data


def test_sealed_frames_open_with_pynacl_and_decode():
    nacl = pytest.importorskip("nacl.secret")
    st = ChunkStage(0, max_batch_bytes=32 << 20, max_chunks=16, n_slots=1)
    try:
        st.set_e2ee_key(KEY)
        datas = [chunk(n, 11) for n in (0, 13, 65537, 4 << 20)]
        for level in (None, 5):
            res = st.process(datas, encrypt=True, block_checksum=True, checksum=True, level=level)
            box = nacl.SecretBox(KEY)
            for d, r in zip(datas, res):
                f = box.decrypt(bytes(r.frame))
                assert f == twin(d, level, True)
                assert ref.lz4f_decompress(f, len(d)) == d and r.md5 == hashlib.md5(d).digest()
    finally:
        st.close()


def test_pipelined_slots_filled_to_capacity_fit():
    """Slots filled with as many chunks as fit (every block stored, the most checksum words) take the flag, and hold
    exactly the batches they held before block checksums existed."""
    mb = 8 << 20
    st = ChunkStage(0, max_batch_bytes=mb, max_chunks=64, n_slots=2)
    try:
        rng = np.random.default_rng(5)
        for n in (65537, 1 << 20, mb):
            slot = st.begin()
            datas = []
            while st.fits(slot, n):
                datas.append(rng.bytes(n))
                st.add_bytes(slot, datas[-1])
            assert len(datas) == min(64, mb // n)
            st.launch(slot, block_checksum=True, checksum=True)
            slot2 = st.begin()
            st.add_bytes(slot2, datas[0])
            st.launch(slot2, block_checksum=True)
            res = st.collect(slot)
            res2 = st.collect(slot2)
            for d, r in zip(datas, res):
                assert bytes(r.frame) == twin(d, None, True)
            assert bytes(res2[0].frame) == twin(datas[0], None, False)
    finally:
        st.close()


def test_md5_alone_with_block_checksums_is_invalid(ctx):
    d_in, d_out = ctx.device_alloc(1 << 16), ctx.device_alloc(1 << 17)
    try:
        for flags in (native.F_MD5 | BC, native.F_MD5 | BC | CK):
            with pytest.raises(native.SkyChunkError) as e:
                ctx.process_device(d_in, [0], [1000], d_out, [0], [native.frame_need(1000, True, True)], flags)
            assert e.value.code == native.SKY_E_INVALID
        with pytest.raises(native.SkyChunkError) as e:  # one byte short of the block checksums' room
            ctx.process_device(d_in, [0], [1000], d_out, [0], [native.frame_need(1000, False, True) - 1], BC)
        assert e.value.code == native.SKY_E_CAPACITY
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)
