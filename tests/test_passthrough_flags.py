"""Host side of sending incompressible chunks as themselves (SKY_F_PASSTHROUGH, no GPU): the flag's bit and refusals in
`native`, `ChunkStage`, the operators and the program loader; what `GatewayCompressHash(skip_incompressible=True)` writes and
reports for a mixed batch (with a context double that makes frames with the oracle's compressor); how
`GatewayDecompressVerify(skip_incompressible=True)` routes a mixed batch into decode calls (with a stage double); and the
sender's rule that maps a chunk's files to its wire header."""
import hashlib
import multiprocessing as mp
import os
import socket

import pytest

import oracle
from skyplane_b200 import native, stage as stage_mod, wire
from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash, GatewayDecompressVerify
from skyplane_b200.program import build_operator_graph
from skyplane_b200.stage import ChunkStage

KEY = bytes((3 * i + 7) & 0xFF for i in range(32))
ALL_FLAGS = (native.F_LZ4, native.F_MD5, native.F_E2EE, native.F_HC, native.F_CHECKSUM, native.F_BLOCK_CHECKSUM,
             native.F_VERIFY, native.F_LINKED, native.F_OPTIMAL)


def test_the_bit_is_free():
    assert native.F_PASSTHROUGH == 32768
    for f in ALL_FLAGS:
        assert not native.F_PASSTHROUGH & f
    for level in range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1):
        assert not native.F_PASSTHROUGH & native.hc_level_flag(level)
    assert not native.F_PASSTHROUGH & native.HC_LEVEL_MASK


# ------------------------------------------------------------------ refusals
@pytest.mark.parametrize("kw, match", [({"compress": False}, "needs compression"), ({"checksum": True}, "content checksum"),
                                       ({"block_checksum": True}, "block checksums")])
def test_native_refuses(kw, match):
    with pytest.raises(ValueError, match=match):
        native.check_passthrough(**kw)
    native.check_passthrough()  # compression, no checksums: fine
    flags = native.F_PASSTHROUGH | (native.F_MD5 if kw.get("compress") is False else native.F_LZ4 | native.F_MD5) \
        | (native.F_CHECKSUM if kw.get("checksum") else 0) | (native.F_BLOCK_CHECKSUM if kw.get("block_checksum") else 0)
    ctx = object.__new__(native.Context)  # (the check comes before the library is touched)
    ctx._h = None
    with pytest.raises(ValueError, match=match):
        ctx.submit([0], [1], [0], [64], flags)


@pytest.mark.parametrize("base", [0, native.F_MD5, native.F_MD5 | native.F_E2EE])
def test_decode_refuses_the_flag(base):
    with pytest.raises(ValueError, match="F_PASSTHROUGH"):
        native.check_decode_flags(base | native.F_PASSTHROUGH)


@pytest.mark.parametrize("kw, match", [({"compress": False}, "needs compression"), ({"checksum": True}, "content checksum"),
                                       ({"block_checksum": True}, "block checksums")])
def test_stage_refuses(kw, match):
    s = object.__new__(ChunkStage)
    slot = object.__new__(stage_mod._Slot)
    slot.reset()
    slot.lens = [10]
    with pytest.raises(ValueError, match=match):
        s.launch(slot, passthrough=True, **kw)
    with pytest.raises(ValueError, match=match):
        s.process([b"x" * 10], passthrough=True, **kw)


def _op_args(tmp_path):
    return ("h", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), ChunkStore(tmp_path))


@pytest.mark.parametrize("kw, match", [({"use_compression": False}, "needs compression"), ({"content_checksum": True}, "content checksum"),
                                       ({"block_checksum": True}, "block checksums")])
def test_operators_refuse(tmp_path, kw, match):
    with pytest.raises(ValueError, match=match):
        GatewayCompressHash(*_op_args(tmp_path), skip_incompressible=True, **kw)
    GatewayCompressHash(*_op_args(tmp_path), skip_incompressible=True, high_ratio=True, verify_frames=True, e2ee_key_bytes=KEY)
    with pytest.raises(ValueError, match="needs use_compression"):
        GatewayDecompressVerify(*_op_args(tmp_path), skip_incompressible=True, use_compression=False)


def _program(kind, **fields):
    child = {"op_type": "write_local", "handle": "w", "children": []}
    return [{"partitions": ["0"], "value": [{"op_type": kind, "handle": "x", "num_gpus": 1, **fields, "children": [child]}]}]


def test_program_loader_hands_the_field_on_and_refuses_bad_nodes(tmp_path):
    ev, eq = mp.Event(), mp.Queue()
    for kind, cls in (("compress_hash", GatewayCompressHash), ("decompress_verify", GatewayDecompressVerify)):
        on = build_operator_graph(_program(kind, skip_incompressible=True), ChunkStore(tmp_path / kind / "on"), "r", ev, eq).operators[f"{kind}_x"]
        off = build_operator_graph(_program(kind), ChunkStore(tmp_path / kind / "off"), "r", ev, eq).operators[f"{kind}_x"]
        assert isinstance(on, cls) and on.skip_incompressible is True and off.skip_incompressible is False
    for kind, fields in (("compress_hash", {"compress": False}), ("compress_hash", {"content_checksum": True}),
                         ("compress_hash", {"block_checksum": True}), ("decompress_verify", {"compress": False})):
        with pytest.raises(ValueError):
            build_operator_graph(_program(kind, skip_incompressible=True, **fields), ChunkStore(tmp_path / "bad"), "r", ev, eq)


# ------------------------------------------------------------------ the sender with a context double
class _Buf:
    def __init__(self, addr, nbytes):
        self.addr, self.nbytes = addr, nbytes
        self.view = memoryview(bytearray(nbytes))


class _Ctx:
    """Context's submit / wait_ex face over the doubles' buffers: frames from the oracle's compressor, boxes from its
    SecretBox, and the pass-through rule of include/skychunk.h."""

    def __init__(self, bufs):
        self.bufs, self.tickets, self.flags = bufs, {}, []

    def _at(self, addr, n):
        for buf in self.bufs:
            if buf.addr <= addr and addr + n <= buf.addr + buf.nbytes:
                return buf.view[addr - buf.addr : addr - buf.addr + n]
        raise AssertionError(f"address {addr:#x} + {n} is outside the staging buffers")

    def submit(self, src, lens, dst, caps, flags, nonces=None):
        assert flags & native.F_PASSTHROUGH and flags & native.F_LZ4
        self.flags.append(flags)
        out, dg, comp = [], [], []
        for k, (a, n, d, cap) in enumerate(zip(src, lens, dst, caps)):
            data = bytes(self._at(a, n))
            frame = oracle.lz4f_compress_indep(data)
            raw = len(frame) >= n
            payload = data if raw else frame
            if flags & native.F_E2EE:
                nonce = nonces[24 * k : 24 * k + 24]
                payload = nonce + oracle.secretbox_seal(KEY, nonce, payload)
            elif raw:
                payload = b""
            assert len(payload) <= cap
            self._at(d, len(payload))[:] = payload
            out.append(len(payload))
            dg.append(hashlib.md5(data).digest())
            comp.append(not raw)
        self.tickets[len(self.tickets) + 1] = (out, dg, None, comp, 0.0)
        return len(self.tickets)

    def wait_ex(self, ticket):
        return self.tickets.pop(ticket)


def _fake_stage(in_bytes=1 << 20, out_bytes=1 << 21):
    s = object.__new__(ChunkStage)
    slots = []
    for k in range(2):
        slot = object.__new__(stage_mod._Slot)
        slot.inp, slot.out = _Buf(0x10000000 * (2 * k + 1), in_bytes), _Buf(0x10000000 * (2 * k + 2), out_bytes)
        slot.reset()
        slots.append(slot)
    s.ctx = _Ctx([b for sl in slots for b in (sl.inp, sl.out)])
    s.max_chunks, s.max_batch_bytes, s._slots, s._free = 16, in_bytes // 2, slots, list(slots)
    return s


def _datas():
    return {"a0" * 16: os.urandom(100000), "a1" * 16: b"text, text, text; " * 400, "a2" * 16: b"", "a3" * 16: b"\x01",
            "a4" * 16: bytes(70000), "a5" * 16: os.urandom(65536)}


def _sender(tmp_path, key, **kw):
    cs = ChunkStore(tmp_path)
    op = GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), cs, skip_incompressible=True,
                             e2ee_key_bytes=key, **kw)
    op.worker_id = 0
    op._stage = _fake_stage()
    return op, cs


def _reqs(datas):
    return [ChunkRequest(Chunk("k", "k", cid, len(d), partition_id="0")) for cid, d in datas.items()]


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "e2ee"])
def test_sender_writes_the_payload_files_and_records_of_a_mixed_batch(tmp_path, key):
    op, cs = _sender(tmp_path, key)
    datas = _datas()
    for cid, d in datas.items():
        cs.get_chunk_file_path(cid).write_bytes(d)
    reqs = _reqs(datas)
    assert op.process_batch(reqs) == [True] * len(reqs)
    assert op._stage.ctx.flags == [native.F_LZ4 | native.F_MD5 | native.F_PASSTHROUGH | (native.F_E2EE if key else 0)]
    op._complete_many(0, reqs)
    records = {rec["chunk_id"]: rec for rec in cs.iter_status_records(cs.chunk_status_queue.get(timeout=10))}
    passed = {cid for cid, d in datas.items() if len(oracle.lz4f_compress_indep(d)) >= len(d)}
    assert passed == {"a0" * 16, "a2" * 16, "a3" * 16, "a5" * 16}
    for r in reqs:
        cid, d = r.chunk.chunk_id, datas[r.chunk.chunk_id]
        lz4, box = cs.get_compressed_file_path(cid), cs.get_box_file_path(cid)
        assert r.chunk.md5_hash == hashlib.md5(d).digest()
        rec = records[cid]
        assert rec.get("passed_through", False) == (cid in passed) and rec["uncompressed_size_bytes"] == len(d)
        if cid not in passed:
            frame = oracle.lz4f_compress_indep(d)
            got = lz4.read_bytes()
            assert (oracle.secretbox_open(KEY, got[:24], got[24:]) if key else got) == frame and not box.exists()
            assert rec["compressed_size_bytes"] == len(got)
        elif key:
            got = box.read_bytes()
            assert oracle.secretbox_open(KEY, got[:24], got[24:]) == d and not lz4.exists()
            assert rec["compressed_size_bytes"] == len(d) + native.BOX_OVERHEAD
        else:
            assert not lz4.exists() and not box.exists() and rec["compressed_size_bytes"] == len(d)
        assert cs.get_chunk_file_path(cid).read_bytes() == d


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "e2ee"])
def test_sink_sends_the_per_chunk_bit(tmp_path, key):
    a, b = socket.socketpair()
    op, cs = _sender(tmp_path, key, sink=lambda worker_id: a)
    datas = _datas()
    for cid, d in datas.items():
        cs.get_chunk_file_path(cid).write_bytes(d)
    try:
        assert op.process_batch(_reqs(datas)) == [True] * len(datas)
        a.shutdown(socket.SHUT_WR)
        for cid, d in datas.items():
            buf = bytearray(1 << 18)
            h, n = wire.recv_chunk(b, buf)
            payload = bytes(buf[:n])
            if key:
                payload = oracle.secretbox_open(KEY, payload[:24], payload[24:])
            assert h.chunk_id == cid and h.raw_data_len == len(d)
            assert h.is_compressed == (len(oracle.lz4f_compress_indep(d)) < len(d))
            assert (oracle.lz4f_decode(payload, len(d)) if h.is_compressed else payload) == d
        assert not any(p.suffix in (".lz4", ".box") for p in tmp_path.iterdir())
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ the receiver with a stage double
class _Stage:
    """ChunkStage.decode's face: keeps every call, 'decodes' with the oracle."""

    def __init__(self):
        self.calls = []

    def decode(self, frames, raw_lens, encrypted=False, compressed=True):
        self.calls.append({"n": len(frames), "encrypted": encrypted, "compressed": compressed})
        out = []
        for f, n in zip(frames, raw_lens):
            f = bytes(f)
            if encrypted:
                f = oracle.secretbox_open(KEY, f[:24], f[24:])
            data = oracle.lz4f_decode(f, n) if compressed else f
            out.append((data if compressed or encrypted else None, hashlib.md5(data).digest(), 0 if len(data) == n else native.D_SIZE))
        return out


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "e2ee"])
def test_receiver_routes_a_mixed_batch_into_one_decode_per_route(tmp_path, key):
    cs = ChunkStore(tmp_path)
    op = GatewayDecompressVerify("dv", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), cs, skip_incompressible=True,
                                 e2ee_key_bytes=key, stale_retries=2)
    op.worker_id = 0
    op._stage = _Stage()
    datas = _datas()
    late = "a9" * 16
    datas[late] = os.urandom(3000)
    passed = set()
    for cid, d in datas.items():
        if cid == late:
            continue  # its payload has not arrived
        frame = oracle.lz4f_compress_indep(d)
        raw = len(frame) >= len(d)
        payload = d if raw else frame
        if key:
            nonce = os.urandom(24)
            payload = nonce + oracle.secretbox_seal(KEY, nonce, payload)
        path = (cs.get_box_file_path(cid) if key else cs.get_chunk_file_path(cid)) if raw else cs.get_compressed_file_path(cid)
        path.write_bytes(payload)
        if raw:
            passed.add(cid)
    reqs = [ChunkRequest(Chunk("k", "k", cid, len(d), partition_id="0", md5_hash=hashlib.md5(d).digest())) for cid, d in datas.items()]
    assert op.process_batch(reqs) == [cid != late for cid in datas]
    calls = op._stage.calls
    assert sorted((c["compressed"], c["encrypted"], c["n"]) for c in calls) == [(False, key is not None, len(passed)),
                                                                                (True, key is not None, len(datas) - 1 - len(passed))]
    for cid, d in datas.items():
        if cid != late:
            assert cs.get_chunk_file_path(cid).read_bytes() == d
            assert not cs.get_compressed_file_path(cid).exists() and not cs.get_box_file_path(cid).exists()
    # a chunk sent as itself that is still arriving is re-queued, then rejected once its size stops changing
    if key is None:
        cs.get_chunk_file_path(late).write_bytes(datas[late][:100])
        r = reqs[-1]
        assert [op.process_batch([r]) for _ in range(2)] == [[False]] * 2
        with pytest.raises(ValueError, match="size mismatch"):
            op.process_batch([r])


# ------------------------------------------------------------------ the sender stub's rule (INTEGRATION §2)
def test_wire_payload_maps_each_file_state_to_its_header(tmp_path):
    cs = ChunkStore(tmp_path)
    cid = "ab" * 16
    cs.get_chunk_file_path(cid).write_bytes(b"chunk")
    assert cs.wire_payload(cid) == (cs.get_chunk_file_path(cid), False)  # sent as itself, unsealed
    cs.get_box_file_path(cid).write_bytes(b"box")
    assert cs.wire_payload(cid) == (cs.get_box_file_path(cid), False)  # the sealed chunk
    cs.get_box_file_path(cid).unlink()
    cs.get_compressed_file_path(cid).write_bytes(b"frame")
    assert cs.wire_payload(cid) == (cs.get_compressed_file_path(cid), True)  # a frame, or the box of a frame
    for path, is_compressed in ((cs.get_compressed_file_path(cid), True), (cs.get_chunk_file_path(cid), False)):
        a, b = socket.socketpair()
        try:
            got, want = cs.wire_payload(cid), path
            if path == cs.get_chunk_file_path(cid):
                cs.get_compressed_file_path(cid).unlink()
                got = cs.wire_payload(cid)
            wire.send_chunk(a, Chunk("k", "k", cid, 5), got[0].read_bytes(), 5, is_compressed=got[1])
            h, _ = wire.recv_chunk(b, bytearray(64))
            assert got[0] == want and h.is_compressed == is_compressed
        finally:
            a.close()
            b.close()
    ChunkStore(tmp_path)  # a restarted gateway starts with an empty chunk directory, boxes included
    assert not list(tmp_path.glob("*.chunk*"))
