"""CPU tests of the host side: reference-compatible types, queues, chunk store, the operator plugin
loop, the C-ABI surface, loud failure without a GPU, and the N>1 sharding logic over gloo."""
import ctypes
import json
import multiprocessing as mp
import os
import pickle
import queue
import re
import socket
import subprocess
import sys
import time
from pathlib import Path

import pytest

from skyplane_b200 import native
from skyplane_b200.chunk import Chunk, ChunkRequest, ChunkState, WireProtocolHeader
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayANDQueue, GatewayQueue
from skyplane_b200.operators import GatewayCompressHash, GatewayDecompressVerify, GatewayOperator
from skyplane_b200.sharding import shard_indices, shard_of_chunk_id

ROOT = Path(__file__).resolve().parent.parent


# ------------------------------------------------------------------ chunk.py parity with the reference
def test_wire_header_matches_reference_bytes(golden):
    g = golden["wire_headers"]
    assert WireProtocolHeader.length_bytes() == g["length_bytes"] == 53
    assert WireProtocolHeader.magic_hex() == g["magic"]
    assert WireProtocolHeader.protocol_version() == g["version"]
    for case in g["headers"]:
        h = WireProtocolHeader(**case["fields"])
        assert h.to_bytes().hex() == case["bytes_hex"]
        assert WireProtocolHeader.from_bytes(bytes.fromhex(case["bytes_hex"])) == h


def test_chunk_dicts_match_reference(golden):
    g = golden["wire_headers"]
    chunk = Chunk.from_dict(g["chunk_as_dict"])
    assert chunk.as_dict() == g["chunk_as_dict"]
    req = ChunkRequest(chunk=chunk, src_region="aws:us-east-1", dst_region="gcp:us-west1")
    assert req.as_dict() == g["chunk_request_as_dict"]
    hdr = chunk.to_wire_header(n_chunks_left_on_socket=5, wire_length=100, raw_wire_length=200, is_compressed=True)
    assert hdr.to_bytes().hex() == g["to_wire_header_hex"]
    assert [s.name for s in ChunkState] == g["chunk_states"]
    assert ChunkRequest.from_dict(g["chunk_as_dict"]).chunk == chunk
    assert ChunkState.from_str("COMPLETE") is ChunkState.complete and ChunkState.registered < ChunkState.complete


def test_wire_header_errors_and_socket():
    h = WireProtocolHeader("ab" * 16, 10, 20, True, 1)
    raw = bytearray(h.to_bytes())
    raw[0] ^= 0xFF
    with pytest.raises(ValueError, match="magic"):
        WireProtocolHeader.from_bytes(bytes(raw))
    raw = bytearray(h.to_bytes())
    raw[11] = 2
    with pytest.raises(ValueError, match="version"):
        WireProtocolHeader.from_bytes(bytes(raw))
    a, b = socket.socketpair()
    try:
        h.to_socket(a)
        assert WireProtocolHeader.from_socket(b) == h
    finally:
        a.close()
        b.close()


def test_md5_hash_json_and_pickle_paths():
    c = Chunk("s", "d", "00" * 16, 5, md5_hash=bytes(range(16)))
    with pytest.raises(TypeError):
        json.dumps(c.as_dict())  # the reference's JSON hop cannot carry raw bytes (SURVEY.md section 7.7)
    back = Chunk.from_json_dict(json.loads(json.dumps(c.as_json_dict())))
    assert back == c
    assert pickle.loads(pickle.dumps(ChunkRequest(c))).chunk.md5_hash == bytes(range(16))


# ------------------------------------------------------------------ queues + store
def test_gateway_queue_semantics():
    q = GatewayQueue(maxsize=4)
    q.register_handle("op")
    assert q.get_handles() == ["op"]
    with pytest.raises(queue.Empty):
        q.get_nowait("op")
    for i in range(3):
        q.put(i)
    time.sleep(0.05)
    assert q.get_batch_nowait(2) == [0, 1]
    assert q.get_batch_nowait(8) == [2]
    aq = GatewayANDQueue()
    aq.register_handle("a")
    aq.register_handle("b")
    aq.put("x")
    time.sleep(0.05)
    assert aq.get_nowait("a") == "x" and aq.get_nowait("b") == "x"
    with pytest.raises(ValueError):
        aq.put_nowait("y")


def test_chunk_store(tmp_path):
    (tmp_path / "stale.chunk").write_bytes(b"x")
    cs = ChunkStore(tmp_path)
    assert not (tmp_path / "stale.chunk").exists()
    q = GatewayQueue()
    cs.add_partition("0", q)
    with pytest.raises(ValueError):
        cs.add_partition("0", q)
    req = ChunkRequest(Chunk("s", "d", "ab" * 16, 3, partition_id="0"))
    size, ok = cs.add_chunk_request(req)
    assert ok
    rec = cs.chunk_status_queue.get(timeout=2)
    assert rec["state"] == "registered" and rec["chunk_id"] == "ab" * 16
    with pytest.raises(ValueError):
        cs.add_chunk_request(ChunkRequest(Chunk("s", "d", "cd" * 16, 3, partition_id="nope")))
    assert cs.get_chunk_file_path("ab" * 16) == tmp_path / ("ab" * 16 + ".chunk")
    assert cs.get_compressed_file_path("ab" * 16).name.endswith(".chunk.lz4")
    cs.log_chunk_state(req, ChunkState.complete, worker_id=1, operator_handle="h", metadata={"compressed_size_bytes": 1})
    rec = cs.chunk_status_queue.get(timeout=2)
    assert rec["state"] == "complete" and rec["compressed_size_bytes"] == 1 and rec["handle"] == "h"
    assert cs.remaining_bytes() > 0


# ------------------------------------------------------------------ operator plugin loop (no GPU involved)
class _Upper(GatewayOperator):
    """Toy operator: succeeds on the 2nd attempt for chunk ids starting with 'ff', raises for 'ee'."""

    def process(self, chunk_req, *args):
        cid = chunk_req.chunk.chunk_id
        if cid.startswith("ee"):
            raise RuntimeError("boom")
        if cid.startswith("ff") and chunk_req.chunk.mime_type is None:
            chunk_req.chunk.mime_type = "retried"
            return False
        chunk_req.chunk.dest_key = chunk_req.chunk.dest_key.upper()
        return True


def _drain(q, n, timeout=10.0):
    out, t0 = [], time.time()
    while len(out) < n and time.time() - t0 < timeout:
        try:
            out.append(q.get_nowait())
        except queue.Empty:
            time.sleep(0.01)
    return out


def test_operator_worker_loop_conventions(tmp_path):
    cs = ChunkStore(tmp_path)
    qin, qout = GatewayQueue(), GatewayQueue()
    err_ev, err_q = mp.Event(), mp.Queue()
    op = _Upper("up", "test:r", qin, qout, err_ev, err_q, cs, n_processes=2)
    op.start_workers()
    try:
        ids = ["%032x" % i for i in range(6)] + ["ff" + "0" * 30]
        for cid in ids:
            qin.put(ChunkRequest(Chunk("k", "dst", cid, 1, partition_id="0")))
        got = _drain(qout, len(ids))
        assert sorted(r.chunk.chunk_id for r in got) == sorted(ids)
        assert all(r.chunk.dest_key == "DST" for r in got)
        assert [r for r in got if r.chunk.chunk_id.startswith("ff")][0].chunk.mime_type == "retried"  # False -> re-queued
        states = {}
        t0 = time.time()
        while time.time() - t0 < 5 and sum(len(v) for v in states.values()) < 2 * len(ids) + 1:
            try:
                rec = cs.chunk_status_queue.get(timeout=0.2)
                states.setdefault(rec["chunk_id"], []).append(rec["state"])
            except queue.Empty:
                pass
        assert all(v[0] == "in_progress" and v[-1] == "complete" for v in states.values())
        qin.put(ChunkRequest(Chunk("k", "dst", "ee" + "0" * 30, 1)))
        t0 = time.time()
        while not err_ev.is_set() and time.time() - t0 < 5:
            time.sleep(0.01)
        assert err_ev.is_set() and "boom" in err_q.get(timeout=2)  # exception -> gateway-wide stop
    finally:
        op.stop_workers()


# ------------------------------------------------------------------ C ABI surface
def test_abi4_header_and_library_symbols_agree():
    hdr = (ROOT / "include" / "skychunk.h").read_text()
    declared = set(re.findall(r"SKY_API[^;]*?\b(sky_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(native.ABI_SYMBOLS) and len(declared) == len(native.ABI_SYMBOLS) == 24
    lib = native.lib()  # builds with nvcc if missing (cross-compiles without a GPU)
    for name in native.ABI_SYMBOLS:
        assert hasattr(lib, name), name
    out = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (sky_[a-z0-9_]+)", out))
    assert exported == declared
    m = re.search(r"#define SKY_ABI_VERSION (\d+)", hdr)
    assert lib.sky_abi_version() == int(m.group(1)) == 4


def test_frame_bound_and_strerror_without_gpu():
    import oracle

    for n in (0, 1, 65535, 65536, 65537, 8 << 20, (64 << 20) + 3):
        want = 11 if n == 0 else oracle.lz4f_bound(n)
        assert native.frame_bound(n) == want
    assert native.frame_bound(8 << 20) == 8389139
    assert b"no CUDA device" in native.lib().sky_strerror(native.SKY_E_NOGPU)


def test_library_carries_sm90a_code():
    out = subprocess.run(["cuobjdump", "-lelf", str(native.LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in out


@pytest.mark.skipif(native.device_count() > 0, reason="only meaningful on a box without a GPU")
def test_product_path_fails_loudly_without_gpu(tmp_path):
    with pytest.raises(native.SkyChunkError) as e:
        native.Context(0, 1 << 20, 4, 1)
    assert e.value.code == native.SKY_E_NOGPU
    from skyplane_b200.stage import ChunkStage

    with pytest.raises(native.SkyChunkError):
        ChunkStage()
    cs = ChunkStore(tmp_path)
    op = GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), cs)
    cid = "ab" * 16
    cs.get_chunk_file_path(cid).write_bytes(b"hello")
    with pytest.raises(native.SkyChunkError):  # no silent CPU path
        op.process(ChunkRequest(Chunk("s", "d", cid, 5)))


def test_product_package_never_imports_the_oracle():
    for p in (ROOT / "skyplane_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cuh", ".h"):
            text = p.read_text()
            assert "import oracle" not in text and "from oracle" not in text and "skyoracle" not in text, p


# ------------------------------------------------------------------ sharding + N>1 reduction over gloo
def test_shard_rules():
    assert shard_indices(10, 0, 4) == [0, 4, 8] and shard_indices(10, 3, 4) == [3, 7]
    all_idx = sorted(i for r in range(8) for i in shard_indices(1024, r, 8))
    assert all_idx == list(range(1024))
    assert shard_of_chunk_id("0" * 31 + "9", 8) == 1
    with pytest.raises(ValueError):
        shard_indices(4, 4, 4)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist

    from skyplane_b200.sharding import max_over_ranks, shard_indices, sum_over_ranks

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        mine = shard_indices(11, rank, world)
        elapsed = 1.0 + rank  # rank 1 is "slower"
        q.put((rank, mine, max_over_ranks(elapsed), sum_over_ranks(len(mine))))
    finally:
        dist.destroy_process_group()


def test_world_size_2_gloo_max_over_ranks():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=120) for _ in ps)
    for p in ps:
        p.join(60)
    assert res[0][1] == [0, 2, 4, 6, 8, 10] and res[1][1] == [1, 3, 5, 7, 9]
    assert res[0][2] == res[1][2] == 2.0  # MAX over ranks
    assert res[0][3] == res[1][3] == 11.0  # every unit counted once


# ------------------------------------------------------------------ GatewayCompressHash host logic with a stub stage (no GPU)
class _StubSlot:
    def __init__(self, cap):
        self.buf = bytearray(cap)
        self.reset()

    def reset(self):
        self.spans, self.used = [], 0

    def reserve(self, n):
        off = self.used
        self.spans.append((off, n))
        self.used += n
        return memoryview(self.buf)[off : off + n]


class _StubStage:
    """Test double with ChunkStage's staging API; 'computes' with hashlib + the oracle (tests may use the oracle)."""

    def __init__(self, cap=4 << 20, max_chunks=4, n_slots=2):
        self.max_batch_bytes, self.max_chunks = cap, max_chunks
        self._slots = [_StubSlot(cap) for _ in range(n_slots)]
        self._free = list(self._slots)
        self.launched = 0
        self.key = None

    def set_e2ee_key(self, key):
        self.key = key

    def begin(self):
        s = self._free.pop()
        s.reset()
        return s

    def release(self, slot):
        self._free.append(slot)

    def fits(self, slot, n):
        return len(slot.spans) < self.max_chunks and slot.used + n <= len(slot.buf)

    def launch(self, slot, compress=True, encrypt=False, nonces=None):
        self.launched += 1
        slot.compress, slot.encrypt = compress, encrypt
        return slot

    def collect(self, slot):
        import hashlib

        import oracle
        from skyplane_b200.stage import StageResult

        out = []
        for off, n in slot.spans:
            data = bytes(slot.buf[off : off + n])
            frame = oracle.lz4f_compress_indep(data) if slot.compress else data
            if slot.encrypt:
                nonce = os.urandom(24)
                frame = nonce + oracle.secretbox_seal(self.key, nonce, frame)
            out.append(StageResult(frame=memoryview(frame), md5=hashlib.md5(data).digest(), raw_len=n, comp_len=len(frame),
                                   is_compressed=slot.compress, is_encrypted=slot.encrypt))
        self._free.append(slot)
        return out

    def decode(self, frames, raw_lens, encrypted=False):
        import hashlib

        import oracle
        from skyplane_b200 import native

        out = []
        for f, n in zip(frames, raw_lens):
            try:
                if encrypted:
                    f = oracle.secretbox_open(self.key, bytes(f[:24]), bytes(f[24:])) if len(f) >= 40 else None
                    if f is None:
                        raise KeyError
                data = oracle.lz4f_decode(bytes(f), n)
                out.append((data, hashlib.md5(data).digest(), 0))
            except (KeyError, ValueError) as e:
                bad_auth = isinstance(e, KeyError) or "authentication" in str(e)
                out.append((None, b"\0" * 16, native.D_AUTH if bad_auth else native.D_TRUNCATED if len(f) < 15 + n // 300 else native.D_CORRUPT))
        return out

    def close(self):
        pass


class _StubbedCompressHash(GatewayCompressHash):
    def _get_stage(self):
        if self._stage is None:
            self._stage = _StubStage(cap=self.max_batch_bytes)
            if self.e2ee_key_bytes is not None:
                self._stage.set_e2ee_key(self.e2ee_key_bytes)
        return self._stage


def test_compress_hash_worker_loop_with_stub_stage(tmp_path):
    import hashlib

    import oracle

    cs = ChunkStore(tmp_path)
    qin, qout = GatewayQueue(), GatewayQueue()
    err_ev, err_q = mp.Event(), mp.Queue()
    op = _StubbedCompressHash("ch", "test:r", qin, qout, err_ev, err_q, cs, n_processes=1, max_batch_chunks=4, read_threads=2,
                               max_batch_bytes=4 << 20)
    datas = {("%02x" % i) * 16: os.urandom(1000 + 37 * i) + bytes(5000) for i in range(11)}
    datas["ee" * 16] = b""  # zero-length chunk (gateway_operator.py:544-548)
    late = "dd" * 16
    datas[late] = b"late chunk " * 500
    for cid, d in datas.items():
        if cid != late:
            cs.get_chunk_file_path(cid).write_bytes(d)
    op.start_workers()
    try:
        for cid, d in datas.items():
            qin.put(ChunkRequest(Chunk("k", "k", cid, len(d), partition_id="0")))
        got = _drain(qout, len(datas) - 1, timeout=20)
        assert len(got) == len(datas) - 1  # the late chunk keeps being re-queued (process -> False semantics)
        cs.get_chunk_file_path(late).write_bytes(datas[late])  # upstream finishes writing it
        got += _drain(qout, 1, timeout=20)
        assert sorted(r.chunk.chunk_id for r in got) == sorted(datas)
        for r in got:
            d = datas[r.chunk.chunk_id]
            assert r.chunk.md5_hash == hashlib.md5(d).digest()
            frame = cs.get_compressed_file_path(r.chunk.chunk_id).read_bytes()
            assert oracle.lz4f_decode(frame, len(d)) == d
            assert cs.get_chunk_file_path(r.chunk.chunk_id).exists()  # the stage never deletes the chunk file
        recs = []
        t0 = time.time()
        while time.time() - t0 < 5 and sum(1 for x in recs if x["state"] == "complete") < len(datas):
            try:
                recs.extend(cs.iter_status_records(cs.chunk_status_queue.get(timeout=0.2)))
            except queue.Empty:
                pass
        done = [x for x in recs if x["state"] == "complete"]
        assert len(done) == len(datas)
        assert all(x["uncompressed_size_bytes"] == len(datas[x["chunk_id"]]) and x["compressed_size_bytes"] > 0 for x in done)
        # a chunk larger than the staging slots does not stop the gateway: the stage is rebuilt with room for it
        big = "cc" * 16
        cs.get_chunk_file_path(big).write_bytes(bytes(5 << 20))
        qin.put(ChunkRequest(Chunk("k", "k", big, 5 << 20, partition_id="0")))
        (r,) = _drain(qout, 1, timeout=20)
        assert r.chunk.chunk_id == big and r.chunk.md5_hash == hashlib.md5(bytes(5 << 20)).digest() and not err_ev.is_set()
    finally:
        op.stop_workers()


def test_compress_false_passes_chunk_through_and_sink_sends_from_the_slot(tmp_path):
    """`compress: false` (gateway_daemon.py:235): digest only, is_compressed=False, no frame file; with a sink the payloads
    go out as WireProtocolHeader + bytes straight from the staging slot (gateway_operator.py:367-402)."""
    import hashlib
    import socket
    import threading

    from skyplane_b200 import wire

    cs = ChunkStore(tmp_path)
    qin, qout = GatewayQueue(), GatewayQueue()
    err_ev, err_q = mp.Event(), mp.Queue()
    a, b = socket.socketpair()
    op = _StubbedCompressHash("ch", "test:r", qin, qout, err_ev, err_q, cs, n_processes=1, max_batch_chunks=4, read_threads=2,
                               max_batch_bytes=4 << 20, use_compression=False, sink=lambda wid: a)
    datas = {("%02x" % i) * 16: os.urandom(3000 + i) for i in range(6)}
    for cid, d in datas.items():
        cs.get_chunk_file_path(cid).write_bytes(d)
    got_wire = {}

    def reader():
        buf = bytearray(1 << 20)
        for _ in datas:
            h, n = wire.recv_chunk(b, buf)
            got_wire[h.chunk_id] = (h, bytes(buf[:n]))

    t = threading.Thread(target=reader)
    t.start()
    op.start_workers()
    try:
        for cid, d in datas.items():
            qin.put(ChunkRequest(Chunk("k", "k", cid, len(d), partition_id="0")))
        got = _drain(qout, len(datas), timeout=20)
        t.join(10)
        assert not t.is_alive() and len(got) == len(datas)
        for r in got:
            d = datas[r.chunk.chunk_id]
            h, payload = got_wire[r.chunk.chunk_id]
            assert payload == d and h.is_compressed is False and h.data_len == h.raw_data_len == len(d)
            assert r.chunk.md5_hash == hashlib.md5(d).digest()
            assert not cs.get_compressed_file_path(r.chunk.chunk_id).exists()
    finally:
        op.stop_workers()
        a.close(); b.close()


class _StubbedDecompressVerify(GatewayDecompressVerify):
    def _get_stage(self):
        if self._stage is None:
            self._stage = _StubStage()
            if self.e2ee_key_bytes is not None:
                self._stage.set_e2ee_key(self.e2ee_key_bytes)
        return self._stage


def test_decompress_verify_batches_waits_for_partial_payloads_and_checks_json_digests(tmp_path):
    """ADVICE r1: a half-written payload is re-queued (not a gateway stop); a digest that crossed a JSON hop as hex is
    compared correctly; E2EE payloads are opened first."""
    import hashlib
    import json

    import oracle

    key = bytes(range(32))
    cs = ChunkStore(tmp_path)
    qin, qout = GatewayQueue(), GatewayQueue()
    err_ev, err_q = mp.Event(), mp.Queue()
    op = _StubbedDecompressVerify("dv", "test:r", qin, qout, err_ev, err_q, cs, n_processes=1, max_batch_chunks=8, e2ee_key_bytes=key)
    datas = {("%02x" % i) * 16: (b"payload %d " % i) * 400 for i in range(5)}
    boxes = {}
    for cid, d in datas.items():
        nonce = os.urandom(24)
        boxes[cid] = nonce + oracle.secretbox_seal(key, nonce, oracle.lz4f_compress_indep(d))
    slow = "04" * 16
    for cid, bx in boxes.items():
        cs.get_compressed_file_path(cid).write_bytes(bx[: len(bx) // 2] if cid == slow else bx)  # one payload is still arriving
    op.start_workers()
    try:
        for cid, d in datas.items():
            c = Chunk("k", "k", cid, len(d), partition_id="0", md5_hash=hashlib.md5(d).digest())
            req = ChunkRequest.from_dict(json.loads(json.dumps(c.as_json_dict())))  # the gateway API's JSON hop
            assert isinstance(req.chunk.md5_hash, bytes)
            qin.put(req)
        got = _drain(qout, 4, timeout=20)
        assert len(got) == 4 and not err_ev.is_set()
        with open(cs.get_compressed_file_path(slow), "ab") as f:  # the writer finishes
            f.write(boxes[slow][len(boxes[slow]) // 2:])
        got += _drain(qout, 1, timeout=20)
        assert sorted(r.chunk.chunk_id for r in got) == sorted(datas) and not err_ev.is_set()
        for r in got:
            assert cs.get_chunk_file_path(r.chunk.chunk_id).read_bytes() == datas[r.chunk.chunk_id]
        # a complete payload with a wrong digest still stops the gateway
        bad = "0f" * 16
        nonce = os.urandom(24)
        cs.get_compressed_file_path(bad).write_bytes(nonce + oracle.secretbox_seal(key, nonce, oracle.lz4f_compress_indep(b"x" * 100)))
        qin.put(ChunkRequest(Chunk("k", "k", bad, 100, partition_id="0", md5_hash=b"\1" * 16)))
        t0 = time.time()
        while not err_ev.is_set() and time.time() - t0 < 10:
            time.sleep(0.01)
        assert err_ev.is_set() and "ChecksumMismatch" in err_q.get(timeout=2)
    finally:
        op.stop_workers()


# ------------------------------------------------------------------ wire framing from staging buffers (SURVEY 8f row 2)
def test_wire_send_recv_roundtrip(golden):
    import threading

    import oracle
    from skyplane_b200 import wire
    from skyplane_b200.stage import StageResult

    datas = [os.urandom(70000), b"hello " * 5000, b""]
    chunks = [Chunk("k", "k", ("%02x" % (i + 1)) * 16, len(d)) for i, d in enumerate(datas)]
    results = []
    for d in datas:
        f = oracle.lz4f_compress_indep(d)
        results.append(StageResult(frame=memoryview(bytearray(f)), md5=b"\0" * 16, raw_len=len(d), comp_len=len(f)))
    a, b = socket.socketpair()
    try:
        t = threading.Thread(target=wire.send_results, args=(a, chunks, results))
        t.start()
        buf = bytearray(1 << 20)
        for i, (c, d, r) in enumerate(zip(chunks, datas, results)):
            hdr, n = wire.recv_chunk(b, buf)
            assert hdr.chunk_id == c.chunk_id and hdr.data_len == r.comp_len == n and hdr.raw_data_len == len(d)
            assert hdr.is_compressed and hdr.n_chunks_left_on_socket == len(chunks) - i - 1
            assert oracle.lz4f_decode(bytes(buf[:n]), len(d)) == d
        t.join()
        # byte-level: what goes on the wire starts with exactly the reference's header bytes
        case = golden["wire_headers"]["headers"][1]
        c = Chunk("s", "d", case["fields"]["chunk_id"], case["fields"]["raw_data_len"])
        payload = bytes(case["fields"]["data_len"])
        ta = threading.Thread(target=wire.send_chunk, args=(a, c, payload, case["fields"]["raw_data_len"]))
        ta.start()
        raw = bytearray()
        want = 53 + len(payload)
        while len(raw) < want:
            raw += b.recv(want - len(raw))
        ta.join()
        assert raw[:53].hex() == case["bytes_hex"]
        with pytest.raises(ValueError):
            tb = threading.Thread(target=wire.send_chunk, args=(a, c, b"x" * 100, 100))
            tb.start()
            try:
                wire.recv_chunk(b, bytearray(10))
            finally:
                b.recv(200)
                tb.join()
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ gateway-program loader (reference JSON schema)
class _Sink(GatewayOperator):
    """Terminal stand-in for send / write_object_store: records what it saw in a file."""

    def process(self, chunk_req, *args):
        with open(self.chunk_store.chunk_dir / f"{self.handle}.seen", "a") as f:
            f.write(chunk_req.chunk.chunk_id + " " + (chunk_req.chunk.md5_hash or b"").hex() + "\n")
        return True


def test_program_loader_wires_reference_schema(tmp_path):
    import hashlib

    from skyplane_b200.program import build_operator_graph

    program = [{
        "partitions": ["0", "1"],
        "value": [{
            "op_type": "compress_hash", "handle": "a", "num_gpus": 1, "compress": True,
            "children": [{"op_type": "mux_and", "handle": "b", "children": [
                {"op_type": "mux_or", "handle": "c", "children": [{"op_type": "send", "handle": "d", "children": []},
                                                                 {"op_type": "send", "handle": "e", "children": []}]},
                {"op_type": "write_local", "handle": "f", "children": []},
            ]}],
        }],
    }]
    cs = ChunkStore(tmp_path)
    ev, eq = mp.Event(), mp.Queue()
    sink = lambda op, kw: _Sink(**kw, n_processes=1)
    factories = {"send": sink, "write_local": sink,
                 "compress_hash": lambda op, kw: _StubbedCompressHash(**kw, n_processes=op["num_gpus"], max_batch_chunks=4, read_threads=1)}
    g = build_operator_graph(program, cs, "test:r", ev, eq, factories)
    assert set(g.operators) == {"compress_hash_a", "send_d", "send_e", "write_local_f"}
    assert g.num_required_terminal == {"0": 2, "1": 2}  # one branch through the mux_or, one through write_local
    assert sorted(g.terminal_operators["0"]) == ["send_d", "send_e", "write_local_f"] and g.n_processes == 4
    comp = g.operators["compress_hash_a"]
    assert isinstance(comp.output_queue, GatewayANDQueue) and sorted(comp.output_queue.get_handles()) == ["mux_or_c", "write_local_f"]
    assert g.operators["send_d"].input_queue is g.operators["send_e"].input_queue  # mux_or: either sender takes the chunk
    assert cs.chunk_requests["0"] is cs.chunk_requests["1"] is comp.input_queue
    with pytest.raises(ValueError, match="Unsupported op_type"):
        build_operator_graph([{"partitions": ["9"], "value": [{"op_type": "teleport", "handle": "x", "children": []}]}],
                             ChunkStore(tmp_path / "other"), "r", ev, eq)
    # run it: one chunk must reach write_local_f and exactly one of the two senders, with the digest attached
    data = b"program loader " * 4000
    cid = "5a" * 16
    cs.get_chunk_file_path(cid).write_bytes(data)
    g.start()
    try:
        cs.add_chunk_request(ChunkRequest(Chunk("k", "k", cid, len(data), partition_id="0")))
        t0 = time.time()
        seen = {}
        while time.time() - t0 < 20:
            seen = {h: (cs.chunk_dir / f"{h}.seen").read_text().split() for h in ("send_d", "send_e", "write_local_f")
                    if (cs.chunk_dir / f"{h}.seen").exists()}
            if "write_local_f" in seen and ("send_d" in seen or "send_e" in seen):
                break
            time.sleep(0.05)
        assert seen["write_local_f"] == [cid, hashlib.md5(data).hexdigest()]
        assert ("send_d" in seen) != ("send_e" in seen)
        assert not ev.is_set()
    finally:
        g.stop()


def test_read_local_ingest_skips_the_chunk_file(tmp_path):
    """src_type == "read_local": the byte range of the source object goes straight into the staging slot."""
    import hashlib

    import oracle

    cs = ChunkStore(tmp_path / "chunks")
    ev, eq = mp.Event(), mp.Queue()
    op = _StubbedCompressHash("ch", "r", GatewayQueue(), None, ev, eq, cs, max_batch_chunks=4, read_threads=2)
    op.worker_id = 0
    obj = tmp_path / "object.bin"
    blob = os.urandom(3000) + b"range " * 3000 + os.urandom(500)
    obj.write_bytes(blob)
    try:
        reqs = [ChunkRequest(Chunk(str(obj), "dst", ("%02x" % (i + 1)) * 16, ln, file_offset_bytes=off, multi_part=True, part_number=i + 1),
                             src_type="read_local") for i, (off, ln) in enumerate([(0, 3000), (3000, 18000), (21000, 500), (100, 0)])]
        late = ChunkRequest(Chunk(str(tmp_path / "missing.bin"), "dst", "ee" * 16, 10, file_offset_bytes=0), src_type="read_local")
        oks = op.process_batch(reqs + [late])
        assert oks == [True, True, True, True, False]  # a source that is not there yet -> retry, like a missing chunk file
        for r in reqs:
            off, ln = r.chunk.file_offset_bytes, r.chunk.chunk_length_bytes
            assert r.chunk.md5_hash == hashlib.md5(blob[off : off + ln]).digest()
            frame = cs.get_compressed_file_path(r.chunk.chunk_id).read_bytes()
            assert oracle.lz4f_decode(frame, ln) == blob[off : off + ln]
            assert not cs.get_chunk_file_path(r.chunk.chunk_id).exists()  # no tmpfs round trip
    finally:
        op.worker_exit(0)


def test_harness_stream_with_stub_operator(tmp_path):
    """The in-process gateway harness (ChunkStore + queues + forked workers) end to end, stage stubbed out."""
    import hashlib

    from skyplane_b200.harness import run_stream

    pool = tmp_path / "pool"
    pool.mkdir()
    datas = [os.urandom(20000), b"abc" * 30000, b"", os.urandom(100) * 50]
    files = []
    for k, d in enumerate(datas):
        f = pool / f"{k}.bin"
        f.write_bytes(d)
        files.append(f)
    res = run_stream(tmp_path / "chunks", files, [len(d) for d in datas], n_requests=30, n_workers=2, max_batch_chunks=4,
                     max_batch_bytes=4 << 20, keep_frames=True, window=8, timeout_s=60, warmup_requests=6, operator_cls=_StubbedCompressHash)
    assert len(res["records"]) == 30
    assert res["bytes"] == sum(len(datas[i % 4]) for i in range(6, 30)) or res["bytes"] > 0  # completions may reorder across workers
    assert res["status"] == {"registered": 30, "in_progress": 30, "complete": 30}
    assert res["uncompressed_bytes"] == sum(len(datas[r["pool_index"]]) for r in res["records"])
    for r in res["records"]:
        assert r["md5"] == hashlib.md5(datas[r["pool_index"]]).hexdigest()
        assert Path(r["frame_path"]).exists() and not (tmp_path / "chunks" / f"{r['chunk_id']}.chunk").exists()
    assert res["wall_s"] > 0


def test_local_operators_pipeline_from_program_json(tmp_path):
    """gen_data -> compress_hash -> write_local wired from a reference-schema program; wait-receive semantics."""
    import hashlib

    import oracle
    from skyplane_b200.local_operators import GatewayRandomDataGen, GatewayWaitReceiver
    from skyplane_b200.program import build_operator_graph

    cs = ChunkStore(tmp_path)
    ev, eq = mp.Event(), mp.Queue()
    # wait-receive: missing -> False, short -> False, complete -> True (gateway_operator.py:131-150)
    wr = GatewayWaitReceiver("receive_x", "r", GatewayQueue(), None, ev, eq, cs)
    req = ChunkRequest(Chunk("k", "k", "aa" * 16, 10))
    assert wr.process(req) is False
    cs.get_chunk_file_path("aa" * 16).write_bytes(b"12345")
    assert wr.process(req) is False
    cs.get_chunk_file_path("aa" * 16).write_bytes(b"1234567890")
    assert wr.process(req) is True
    with pytest.raises(ValueError):
        GatewayRandomDataGen("g", "r", GatewayQueue(), None, ev, eq, cs, size_mb=1, fill="ones")

    program = [{"partitions": ["0"], "value": [{"op_type": "gen_data", "handle": "g", "size_mb": 0.25, "fill": "random", "children": [
        {"op_type": "compress_hash", "handle": "c", "num_gpus": 1, "children": [{"op_type": "write_local", "handle": "w", "children": []}]}]}]}]
    g = build_operator_graph(program, cs, "r", ev, eq,
                             {"compress_hash": lambda op, kw: _StubbedCompressHash(**kw, n_processes=1, max_batch_chunks=4, read_threads=1)})
    assert list(g.operators) == ["gen_data_g", "compress_hash_c", "write_local_w"] and g.terminal_operators == {"0": ["write_local_w"]}
    g.start()
    try:
        ids = ["%032x" % (0xB200 + i) for i in range(5)]
        for cid in ids:
            cs.add_chunk_request(ChunkRequest(Chunk("gen", "gen", cid, 0, partition_id="0"), src_type="random", src_random_size_mb=1))
        done = set()
        t0 = time.time()
        while len(done) < len(ids) and time.time() - t0 < 30 and not ev.is_set():
            try:
                item = cs.chunk_status_queue.get(timeout=0.2)
            except queue.Empty:
                continue
            for rec in cs.iter_status_records(item):  # the batched operator ships its records as lists
                if rec["handle"] == "write_local_w" and rec["state"] == "complete":
                    done.add(rec["chunk_id"])
        assert done == set(ids) and not ev.is_set()
        for cid in ids:
            data = cs.get_chunk_file_path(cid).read_bytes()
            assert len(data) == 262144
            assert oracle.lz4f_decode(cs.get_compressed_file_path(cid).read_bytes(), len(data)) == data
    finally:
        g.stop()
