"""Host side of receiving `compress: false` chunks (no GPU): which flag sets `Context.decode` takes, how the gateway program
hands `"compress": false` to `GatewayDecompressVerify`, how `ChunkStage.decode(compressed=False)` stages payloads and calls the
library, and what the operator does with the files of such a transfer (with a stage double that computes with hashlib
and the oracle's SecretBox)."""
import hashlib
import multiprocessing as mp
import os

import pytest

import oracle
from skyplane_b200 import native
from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import ChecksumMismatchException, GatewayDecompressVerify
from skyplane_b200.stage import ChunkStage

KEY = bytes((5 * i + 1) & 0xFF for i in range(32))


def seal(data: bytes, key: bytes = KEY) -> bytes:
    nonce = os.urandom(24)
    return nonce + oracle.secretbox_seal(key, nonce, data)


# ------------------------------------------------------------------ flag rules
@pytest.mark.parametrize("flags", [0, native.F_LZ4, native.F_LZ4 | native.F_MD5, native.F_MD5, native.F_E2EE, native.F_LZ4 | native.F_E2EE,
                                   native.F_LZ4 | native.F_MD5 | native.F_E2EE, native.F_MD5 | native.F_E2EE])
def test_decode_takes_the_stage_bits_and_e2ee(flags):
    assert native.check_decode_flags(flags) == flags


@pytest.mark.parametrize("bad, name", [(native.F_HC, "F_HC"), (native.hc_level_flag(7), "F_HC"), (7 << native.HC_LEVEL_SHIFT, "level"),
                                       (native.F_CHECKSUM, "F_CHECKSUM"), (native.F_BLOCK_CHECKSUM, "F_BLOCK_CHECKSUM"),
                                       (native.F_VERIFY, "F_VERIFY"), (4, "0x4"), (1 << 20, "0x100000")])
@pytest.mark.parametrize("base", [0, native.F_MD5, native.F_MD5 | native.F_E2EE])
def test_decode_refuses_sender_options_by_name(bad, name, base):
    with pytest.raises(ValueError, match=name):
        native.check_decode_flags(base | bad)
    ctx = object.__new__(native.Context)  # (the check comes before the library is touched)
    ctx._h = None
    with pytest.raises(ValueError, match=name):
        ctx.decode([0], [0], None, [0], base | bad)


# ------------------------------------------------------------------ gateway program
def test_program_hands_compress_false_to_decompress_verify(tmp_path):
    from skyplane_b200.program import build_operator_graph

    def program(**fields):
        return [{"partitions": ["0"], "value": [{"op_type": "decompress_verify", "handle": "v", "num_gpus": 1, **fields,
                                                 "children": [{"op_type": "write_local", "handle": "w", "children": []}]}]}]

    ev, eq = mp.Event(), mp.Queue()
    off = build_operator_graph(program(compress=False), ChunkStore(tmp_path / "a"), "r", ev, eq).operators["decompress_verify_v"]
    on = build_operator_graph(program(compress=True), ChunkStore(tmp_path / "b"), "r", ev, eq).operators["decompress_verify_v"]
    default = build_operator_graph(program(), ChunkStore(tmp_path / "c"), "r", ev, eq).operators["decompress_verify_v"]
    assert isinstance(off, GatewayDecompressVerify) and off.use_compression is False
    assert on.use_compression is True and default.use_compression is True
    same = ("max_batch_chunks", "max_batch_bytes", "n_gpus", "remove_frames", "e2ee_key_bytes", "stale_retries", "n_processes", "handle")
    assert all(getattr(default, a) == getattr(on, a) == getattr(off, a) for a in same)


# ------------------------------------------------------------------ ChunkStage.decode(compressed=False) without a device
class _Buf:
    """A staging buffer with PinnedBuffer's face, in ordinary memory at a made-up address."""

    def __init__(self, addr, nbytes):
        self.addr, self.nbytes = addr, nbytes
        self.view = memoryview(bytearray(nbytes))


class _Slot:
    def __init__(self, in_bytes, out_bytes):
        self.inp, self.out = _Buf(0x10000000, in_bytes), _Buf(0x20000000, out_bytes)


class _Ctx:
    """Context.decode's face: checks the flags as the real one does, reads the payloads where the stage put them, 'computes'
    with hashlib and the oracle, writes opened chunks where the stage asked for them, and keeps every call for the test."""

    def __init__(self, slot):
        self.slot, self.calls = slot, []

    def _at(self, addr, n):
        for buf in (self.slot.inp, self.slot.out):
            if buf.addr <= addr and addr + n <= buf.addr + buf.nbytes:
                return buf, addr - buf.addr
        raise AssertionError(f"address {addr:#x} + {n} is outside the staging buffers")

    def decode(self, frame_addrs, frame_lens, dst_addrs, raw_lens, flags=0):
        native.check_decode_flags(flags)
        self.calls.append({"flags": flags, "n": len(frame_addrs), "dst": dst_addrs, "src_in_inp": [self._at(a, n)[0] is self.slot.inp
                                                                                                  for a, n in zip(frame_addrs, frame_lens)]})
        assert flags & native.F_MD5 and not flags & native.F_LZ4, "this double only receives raw chunks"
        st, dg = [], []
        for k, (a, n, r) in enumerate(zip(frame_addrs, frame_lens, raw_lens)):
            buf, off = self._at(a, n)
            data = bytes(buf.view[off : off + n])
            status = 0
            if flags & native.F_E2EE:
                try:
                    if n < 40:
                        raise ValueError("short box")
                    data = oracle.secretbox_open(KEY, data[:24], data[24:])
                except ValueError:
                    status = native.D_AUTH
            if status == 0 and len(data) != r:
                status = native.D_SIZE
            if status == 0 and flags & native.F_E2EE and r:
                dbuf, doff = self._at(dst_addrs[k], r)
                dbuf.view[doff : doff + r] = data
            st.append(status)
            dg.append(hashlib.md5(data).digest() if status == 0 else bytes(16))
        return st, dg, 0.0


def _stage(in_bytes=4096, out_bytes=8192, max_chunks=4):
    s = object.__new__(ChunkStage)
    slot = _Slot(in_bytes, out_bytes)
    s.ctx, s.max_chunks, s._slots, s._free = _Ctx(slot), max_chunks, [slot], [slot]
    return s, slot


def test_stage_decode_raw_stages_in_the_input_buffer_and_returns_no_bytes():
    s, slot = _stage()
    datas = [b"a" * 100, b"", b"b" * 17, os.urandom(1000)]
    out = s.decode(datas, [100, 0, 17, 999], compressed=False)
    (call,) = s.ctx.calls
    assert call["flags"] == native.F_MD5 and call["dst"] is None and all(call["src_in_inp"])
    assert [st for _, _, st in out] == [0, 0, 0, native.D_SIZE]
    assert all(data is None for data, _, _ in out)  # the caller holds the bytes
    assert [dg for _, dg, _ in out] == [hashlib.md5(d).digest() for d in datas[:3]] + [bytes(16)]
    assert bytes(slot.out.view) == bytes(slot.out.nbytes)  # nothing went through the frame buffer


def test_stage_decode_raw_encrypted_opens_boxes_and_returns_the_chunks():
    s, slot = _stage()
    datas = [b"x" * 300, b"", os.urandom(77)]
    boxes = [seal(d) for d in datas]
    forged = boxes[0][:60] + bytes([boxes[0][60] ^ 1]) + boxes[0][61:]
    out = s.decode(boxes + [forged, boxes[2]], [300, 0, 77, 300, 78], encrypted=True, compressed=False)
    assert [c["n"] for c in s.ctx.calls] == [4, 1]  # max_chunks per call
    assert all(c["flags"] == native.F_MD5 | native.F_E2EE and not any(c["src_in_inp"]) and c["dst"] is not None for c in s.ctx.calls)
    assert [(data, dg, st) for data, dg, st in out[:3]] == [(d, hashlib.md5(d).digest(), 0) for d in datas]
    assert out[3] == (None, bytes(16), native.D_AUTH) and out[4] == (None, bytes(16), native.D_SIZE)


def test_stage_decode_raw_batches_by_room_and_refuses_what_cannot_fit():
    s, slot = _stage(in_bytes=1024, max_chunks=64)
    datas = [bytes([i]) * 400 for i in range(5)]  # two fit 1024 bytes of input buffer at 16-byte steps, the third does not
    out = s.decode(datas, [400] * 5, compressed=False)
    assert [c["n"] for c in s.ctx.calls] == [2, 2, 1]
    assert [dg for _, dg, _ in out] == [hashlib.md5(d).digest() for d in datas]
    with pytest.raises(native.SkyChunkError) as e:
        s.decode([bytes(1025)], [1025], compressed=False)
    assert e.value.code == native.SKY_E_CAPACITY
    with pytest.raises(ValueError, match="raw lengths"):
        s.decode(datas, [400] * 4, compressed=False)
    s._free = []
    with pytest.raises(native.SkyChunkError) as e:
        s.decode(datas[:1], [400], compressed=False)
    assert e.value.code == native.SKY_E_BUSY


# ------------------------------------------------------------------ GatewayDecompressVerify(use_compression=False) and its files
def _operator(tmp_path, key=None, **kw):
    cs = ChunkStore(tmp_path)
    ev, eq = mp.Event(), mp.Queue()
    op = GatewayDecompressVerify("dv", "test:r", GatewayQueue(), None, ev, eq, cs, use_compression=False, e2ee_key_bytes=key, **kw)
    op.worker_id = 0
    op._stage, _ = _stage(in_bytes=1 << 16, out_bytes=1 << 17, max_chunks=8)
    return op, cs


def _req(cid, data, md5=True, length=None):
    return ChunkRequest(Chunk("k", "k", cid, len(data) if length is None else length, partition_id="0",
                              md5_hash=hashlib.md5(data).digest() if md5 else None))


def test_operator_digests_received_chunk_files_where_they_lie(tmp_path):
    op, cs = _operator(tmp_path, stale_retries=3)
    datas = {("%02x" % i) * 16: os.urandom(500 + i) for i in range(3)}
    datas["0e" * 16] = b""
    late, slow = "0a" * 16, "0b" * 16
    datas[late], datas[slow] = b"late " * 90, b"slow " * 70
    for cid, d in datas.items():
        if cid != late:
            cs.get_chunk_file_path(cid).write_bytes(d[: len(d) // 2] if cid == slow else d)
    reqs = [_req(cid, d, md5=cid != "00" * 16) for cid, d in datas.items()]
    before = {cid: os.stat(cs.get_chunk_file_path(cid)) for cid in datas if cid not in (late, slow)}
    done = op.process_batch(reqs)
    assert done == [cid not in (late, slow) for cid in datas]  # a missing file and a short one are re-queued
    for r, good in zip(reqs, done):
        if good:
            cid = r.chunk.chunk_id
            after = os.stat(cs.get_chunk_file_path(cid))
            assert (after.st_ino, after.st_mtime_ns) == (before[cid].st_ino, before[cid].st_mtime_ns)  # read, never rewritten
            assert r.chunk.md5_hash == hashlib.md5(datas[cid]).digest()
            assert not cs.get_compressed_file_path(cid).exists() and not cs.get_chunk_file_path(cid).with_name(f"{cid}.chunk.part").exists()
    cs.get_chunk_file_path(late).write_bytes(datas[late])
    with open(cs.get_chunk_file_path(slow), "ab") as f:
        f.write(datas[slow][len(datas[slow]) // 2:])
    assert op.process_batch(reqs[-2:]) == [True, True]
    # a file whose size stays wrong is rejected once it has been looked at stale_retries times
    stuck = "0c" * 16
    cs.get_chunk_file_path(stuck).write_bytes(b"q" * 10)
    r = _req(stuck, b"q" * 11)
    assert [op.process_batch([r]) for _ in range(3)] == [[False]] * 3
    with pytest.raises(ValueError, match="size mismatch"):
        op.process_batch([r])
    # right size, other bytes
    wrong = "0d" * 16
    cs.get_chunk_file_path(wrong).write_bytes(b"r" * 64)
    with pytest.raises(ChecksumMismatchException):
        op.process_batch([_req(wrong, b"s" * 64)])


def test_operator_opens_sealed_raw_payloads_and_writes_the_chunk(tmp_path):
    op, cs = _operator(tmp_path, key=KEY, stale_retries=2)
    datas = {("%02x" % (0x10 + i)) * 16: os.urandom(800 + 3 * i) for i in range(3)}
    datas["1e" * 16] = b""
    slow = "10" * 16
    boxes = {cid: seal(d) for cid, d in datas.items()}
    for cid, bx in boxes.items():
        cs.get_compressed_file_path(cid).write_bytes(bx[:-100] if cid == slow else bx)
    reqs = [_req(cid, d) for cid, d in datas.items()]
    assert op.process_batch(reqs) == [cid != slow for cid in datas]  # a short box fails authentication: it may still be arriving
    cs.get_compressed_file_path(slow).write_bytes(boxes[slow])
    assert op.process_batch(reqs[:1]) == [True]
    for cid, d in datas.items():
        assert cs.get_chunk_file_path(cid).read_bytes() == d and not cs.get_compressed_file_path(cid).exists()
    # an authentic box of another length is not "still arriving"; a box under another key is, until it has been seen often enough
    odd = "1a" * 16
    cs.get_compressed_file_path(odd).write_bytes(seal(b"z" * 50))
    with pytest.raises(ValueError, match="size mismatch"):
        op.process_batch([_req(odd, b"z" * 50, length=51)])
    other = "1b" * 16
    cs.get_compressed_file_path(other).write_bytes(seal(b"y" * 50, key=bytes(32)))
    r = _req(other, b"y" * 50)
    assert [op.process_batch([r]) for _ in range(2)] == [[False]] * 2
    with pytest.raises(ValueError, match="authentication"):
        op.process_batch([r])
    assert not cs.get_chunk_file_path(other).exists()
