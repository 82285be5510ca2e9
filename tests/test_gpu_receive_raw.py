"""GPU tests of receiving `compress: false` chunks (the sender's SKY_F_MD5 rows) through the C ABI: sky_decode(SKY_F_MD5)
digests payloads that are the chunks themselves, sky_decode(SKY_F_MD5 | SKY_F_E2EE) opens their SecretBoxes first
(gateway_receiver.py:191-201 with is_compressed = False, and the hash check the reference leaves as a todo at :231).
Digests against hashlib, boxes against PyNaCl and the oracle, statuses, errors, launch counts, the other users of slot 0,
and the way from GatewayCompressHash over a socket into the receiver stage and GatewayDecompressVerify's workers."""
import ctypes
import hashlib
import itertools
import json
import multiprocessing as mp
import os
import shutil
import socket
import subprocess
import sys
import tempfile
import threading
from pathlib import Path

import numpy as np
import pytest

import oracle
from skyplane_b200 import native, synth, wire
from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash
from skyplane_b200.stage import ChunkStage

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300, method="thread")]
ROOT = Path(__file__).resolve().parent.parent
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
RNG = np.random.default_rng(2024)
RAW, RAW_BOX = native.F_MD5, native.F_MD5 | native.F_E2EE
GUARD = 0xA5


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 96 << 20, 512, 1)
    c.set_e2ee_key(KEY)
    yield c
    c.close()


def seal(data: bytes, key: bytes = KEY, nonce: bytes = None) -> bytes:
    nonce = nonce or RNG.bytes(24)
    return nonce + oracle.secretbox_seal(key, nonce, data)


def kinds(n):
    return [RNG.bytes(n), bytes(n), (b"abcdefg" * (n // 7 + 1))[:n], (b"the quick brown fox jumps over the lazy dog " * (n // 40 + 1))[:n],
            (b"lorem ipsum dolor " * (n // 36 + 1))[: n // 2] + RNG.bytes(n - n // 2)]


def sky_decode(ctx, payloads, raw_lens, flags, dst=True, checked=True):
    """sky_decode over ordinary host memory.  dst: every dst[i] is raw_lens[i] + 32 guard bytes (False: dst = NULL).
    -> (rc, status, digests, what the dst buffers hold afterwards, kernel_ms); checked: rc must be SKY_OK."""
    n = len(payloads)
    src = [(ctypes.c_ubyte * max(1, len(p))).from_buffer_copy(p or b"\0") for p in payloads]
    out = [(ctypes.c_ubyte * (r + 32)).from_buffer_copy(bytes([GUARD]) * (r + 32)) for r in raw_lens] if dst else None
    A, U = ctypes.c_void_p * n, ctypes.c_uint64 * n
    st, md5, ms = (ctypes.c_int32 * n)(), (ctypes.c_ubyte * (16 * n))(), ctypes.c_float(0)
    rc = native.lib().sky_decode(ctx._h, n, A(*map(ctypes.addressof, src)), U(*map(len, payloads)),
                                 A(*map(ctypes.addressof, out)) if dst else None, U(*raw_lens), flags, st, md5, ctypes.byref(ms))
    if checked:
        assert rc == native.SKY_OK, (rc, native.lib().sky_last_error(ctx._h))
    raw = bytes(md5)
    return rc, list(st), [raw[16 * i: 16 * i + 16] for i in range(n)], [bytes(o) for o in out] if dst else None, ms.value


def untouched(buf: bytes) -> bool:
    return buf == bytes([GUARD]) * len(buf)


# ------------------------------------------------------------------ digests
def test_raw_payloads_are_digested_and_nothing_is_written(ctx):
    lens = [0, 1, 55, 56, 63, 64, 65, 65535, 65536, 65537, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 8 << 20]
    datas = [d for n in lens for d in kinds(n)]  # ragged, in one batch
    want = [hashlib.md5(d).digest() for d in datas]
    before = ctx.launches
    _, st, dg, _, ms = sky_decode(ctx, datas, [len(d) for d in datas], RAW, dst=False)
    assert ctx.launches - before == 1  # the fused kernel's MD5 role, nothing else
    assert st == [0] * len(datas) and dg == want and ms > 0
    _, st, dg, out, _ = sky_decode(ctx, datas[:25], [len(d) for d in datas[:25]], RAW, dst=True)
    assert st == [0] * 25 and dg == want[:25] and all(untouched(o) for o in out)
    # the library's face in Python: the same call through Context.decode, dst None
    some = datas[40:50]
    bufs = [(ctypes.c_ubyte * max(1, len(d))).from_buffer_copy(d or b"\0") for d in some]
    st, dg, _ = ctx.decode([ctypes.addressof(b) for b in bufs], [len(d) for d in some], None, [len(d) for d in some], RAW)
    assert st == [0] * 10 and dg == want[40:50]


# ------------------------------------------------------------------ round trips with our sender: all four payload rows
@pytest.mark.parametrize("compress, encrypt", [(False, False), (False, True), (True, False), (True, True)])
def test_every_payload_the_sender_makes_has_a_receiver(compress, encrypt):
    stage = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=32, n_slots=2)
    try:
        stage.set_e2ee_key(KEY)
        datas = [synth.silesia_like_chunk(70 + i, (1 << 20) + 4321 * i) for i in range(3)] + [synth.random_chunk(9, 3 << 20), b"", b"tiny",
                                                                                              bytes(70000)]
        res = stage.process(datas, compress=compress, encrypt=encrypt)
        assert all(r.is_compressed == compress and r.is_encrypted == encrypt for r in res)
        out = stage.decode([bytes(r.frame) for r in res], [r.raw_len for r in res], encrypted=encrypt, compressed=compress)
        for d, r, (data, dg, st) in zip(datas, res, out):
            assert st == 0 and dg == r.md5 == hashlib.md5(d).digest()
            assert data == (None if not compress and not encrypt else d)  # a plain raw payload is the chunk: nothing to return
        if not compress and not encrypt:
            assert all(bytes(r.frame) == d for d, r in zip(datas, res))
    finally:
        stage.close()


# ------------------------------------------------------------------ boxes made on the CPU open on the GPU
def test_pynacl_boxes_of_raw_chunks_open_on_the_gpu(ctx):
    nacl_secret = pytest.importorskip("nacl.secret")
    box = nacl_secret.SecretBox(KEY)
    lens = list(range(0, 201, 7)) + [4096 * k + d for k in (1, 2, 3) for d in (-17, -16, -15, -1, 0, 1, 15, 16, 17)] + [65551, (1 << 20) + 5]
    datas = [RNG.bytes(n) for n in lens]
    boxes = []
    for d in datas:
        nonce = RNG.bytes(24)
        boxes.append(bytes(box.encrypt(d, nonce)))  # nonce | tag | ciphertext, what GatewaySender puts on the wire
        assert boxes[-1] == seal(d, nonce=nonce)
    before = ctx.launches
    _, st, dg, out, ms = sky_decode(ctx, boxes, lens, RAW_BOX)
    assert ctx.launches - before == 4  # keys, tag, xor, MD5
    assert st == [0] * len(lens) and ms > 0
    for d, g, o in zip(datas, dg, out):
        assert g == hashlib.md5(d).digest() and o[: len(d)] == d and untouched(o[len(d):]), len(d)


# ------------------------------------------------------------------ statuses
def test_a_payload_of_the_wrong_size_fails_alone(ctx):
    datas = [RNG.bytes(5000), RNG.bytes(70000), RNG.bytes(300), b"", RNG.bytes(1 << 20)]
    raws = [5000, 70001, 299, 1, 1 << 20]
    _, st, dg, out, _ = sky_decode(ctx, datas, raws, RAW)
    assert st == [0, native.D_SIZE, native.D_SIZE, native.D_SIZE, 0]
    assert dg == [hashlib.md5(datas[0]).digest(), bytes(16), bytes(16), bytes(16), hashlib.md5(datas[4]).digest()]
    assert all(untouched(o) for o in out)


def test_forged_truncated_and_missized_boxes(ctx):
    msg = RNG.bytes(3000)
    good = seal(msg)

    def flip(b, k, bit=1):
        return b[:k] + bytes([b[k] ^ bit]) + b[k + 1:]

    short = seal(RNG.bytes(30))  # 70 bytes: every proper prefix, those under the 40 bytes of nonce and tag included
    prefixes = [short[:k] for k in range(len(short))]
    one_more, one_less = seal(msg + b"!"), seal(msg[:-1])
    payloads = [good, flip(good, 1500), flip(good, 30, 0x80), flip(good, 0), good[:-1], seal(msg, key=bytes(32)),  # 0..5
                one_more, one_less, flip(one_more, 2000), flip(one_less, 39), seal(b""), good] + prefixes  # 6..11, then the prefixes
    raws = [3000] * 10 + [1, 3000] + [30] * len(prefixes)
    A, S = native.D_AUTH, native.D_SIZE
    _, st, dg, out, _ = sky_decode(ctx, payloads, raws, RAW_BOX)
    assert st[:12] == [0, A, A, A, A, A, S, S, A, A, S, 0]  # an authentic box of another length: SIZE; forged as well: AUTH
    assert st[12:] == [A] * len(prefixes)
    for k, (s, g, o) in enumerate(zip(st, dg, out)):
        if s == 0:
            assert o[:3000] == msg and untouched(o[3000:]) and g == hashlib.md5(msg).digest()
        else:
            assert untouched(o) and g == bytes(16), k  # no plaintext escaped, authentic or not


# ------------------------------------------------------------------ errors
def test_flag_and_argument_errors(ctx):
    data = RNG.bytes(1000)
    for base in (RAW, RAW_BOX, 0, native.F_E2EE):
        payload = seal(data) if base & native.F_E2EE else data
        for bad in (native.F_CHECKSUM, native.F_BLOCK_CHECKSUM, native.F_VERIFY, native.F_HC, native.hc_level_flag(4), 4, 8, 1 << 20):
            rc, *_ = sky_decode(ctx, [payload], [1000], base | bad, checked=False)
            assert rc == native.SKY_E_INVALID, (base, bad)
    assert sky_decode(ctx, [data], [1000], 0, dst=False, checked=False)[0] == native.SKY_E_INVALID  # frames decode into dst
    assert sky_decode(ctx, [seal(data)], [1000], RAW_BOX, dst=False, checked=False)[0] == native.SKY_E_INVALID  # so do boxes
    _, st, dg, _, _ = sky_decode(ctx, [data], [1000], RAW)  # the ctx still works
    assert st == [0] and dg == [hashlib.md5(data).digest()]
    with native.Context(0, 1 << 20, 8, 1) as small:
        assert sky_decode(small, [seal(data)], [1000], RAW_BOX, checked=False)[0] == native.SKY_E_NOKEY
        half = bytes(600 << 10)
        assert sky_decode(small, [half, half], [len(half)] * 2, RAW, checked=False)[0] == native.SKY_E_CAPACITY
        assert sky_decode(small, [b"x"] * 9, [1] * 9, RAW, checked=False)[0] == native.SKY_E_CAPACITY  # more chunks than max_chunks
        assert sky_decode(small, [half], [len(half)], RAW)[1] == [0]
    with native.Context(0, 1 << 20, 8, 0) as no_slabs:
        assert sky_decode(no_slabs, [data], [1000], RAW, checked=False)[0] == native.SKY_E_INVALID


# ------------------------------------------------------------------ slot 0 is shared: no call leaves anything behind for the next
def test_raw_decode_lz4_decode_and_submit_in_every_order():
    stage = ChunkStage(0, max_batch_bytes=32 << 20, max_chunks=16, n_slots=1)
    try:
        stage.set_e2ee_key(KEY)
        a = [synth.random_chunk(21, 1 << 20), b"", synth.silesia_like_chunk(22, 700001), RNG.bytes(65)]
        b = [synth.silesia_like_chunk(23, (2 << 20) + 17), RNG.bytes(123457)]
        c = [synth.silesia_like_chunk(24, 900000), RNG.bytes(5), b"", synth.random_chunk(25, 1 << 19)]
        d = [RNG.bytes(250001), RNG.bytes(4096), b""]
        frames_b = [bytes(r.frame) for r in stage.process(b)]
        boxes_d = [seal(x) for x in d]
        ops = {
            "raw": lambda: stage.decode(a, [len(x) for x in a[:3]] + [66], compressed=False),  # (its last chunk has the wrong size)
            "lz4": lambda: stage.decode(frames_b, [len(x) for x in b]),
            "submit": lambda: [(bytes(r.frame), r.md5, r.comp_len) for r in stage.process(c)],
            "raw_box": lambda: stage.decode(boxes_d, [len(x) for x in d], encrypted=True, compressed=False),
        }
        alone, cost = {}, {}
        for name, op in ops.items():
            before = stage.ctx.launches
            alone[name] = op()
            cost[name] = stage.ctx.launches - before
        assert cost == {"raw": 1, "lz4": 2, "submit": 1, "raw_box": 4}
        assert [x[1] for x in alone["raw"]] == [hashlib.md5(x).digest() for x in a[:3]] + [bytes(16)]
        assert [x[0] for x in alone["lz4"]] == b and [x[0] for x in alone["raw_box"]] == d
        for order in itertools.permutations(ops):
            before = stage.ctx.launches
            for name in order:
                assert ops[name]() == alone[name], (order, name)
            assert stage.ctx.launches - before == sum(cost.values())
    finally:
        stage.close()


# ------------------------------------------------------------------ sender -> socket -> receiver stage
@pytest.mark.parametrize("encrypt", [False, True])
def test_compress_false_from_the_sender_operator_over_a_socket_to_the_receiver_stage(tmp_path, encrypt):
    datas = [synth.silesia_like_chunk(80 + i, (1 << 20) + 999 * i) for i in range(3)] + [synth.random_chunk(4, 1 << 20), b"", b"z" * 13]
    cs = ChunkStore(tmp_path)
    a, b = socket.socketpair()
    ev, eq = mp.Event(), mp.Queue()
    op = GatewayCompressHash("ch", "r", GatewayQueue(), None, ev, eq, cs, use_compression=False, sink=lambda wid: a, max_batch_bytes=32 << 20,
                             max_batch_chunks=16, e2ee_key_bytes=KEY if encrypt else None)
    op.worker_id = 0
    recv_stage = ChunkStage(0, max_batch_bytes=32 << 20, max_chunks=16, n_slots=1)
    got = []

    def receiver():
        for _ in datas:
            buf = bytearray((2 << 20) + 64)
            h, n = wire.recv_chunk(b, buf)
            got.append((h, bytes(buf[:n])))

    t = threading.Thread(target=receiver)
    t.start()
    try:
        if encrypt:
            recv_stage.set_e2ee_key(KEY)
        reqs = []
        for i, d in enumerate(datas):
            cid = "%032x" % (0xC0FFEE00 + i)
            cs.get_chunk_file_path(cid).write_bytes(d)
            reqs.append(ChunkRequest(Chunk("src", "dst", cid, len(d), partition_id="0")))
        assert op.process_batch(reqs) == [True] * len(datas)
        t.join(60)
        assert not t.is_alive()
        out = recv_stage.decode([p for _, p in got], [h.raw_data_len for h, _ in got], encrypted=encrypt, compressed=False)
        for (h, payload), r, d, (data, dg, st) in zip(got, reqs, datas, out):
            assert h.chunk_id == r.chunk.chunk_id and h.is_compressed is False and h.raw_data_len == len(d)
            assert h.data_len == len(payload) == len(d) + (native.BOX_OVERHEAD if encrypt else 0)
            assert st == 0 and dg == r.chunk.md5_hash == hashlib.md5(d).digest()
            assert (data == d) if encrypt else (data is None and payload == d)
    finally:
        op.worker_exit(0)
        b.close()
        recv_stage.close()


# ------------------------------------------------------------------ GatewayDecompressVerify(use_compression=False) workers
DRIVER = r"""
import hashlib, json, multiprocessing as mp, os, sys, time
from pathlib import Path
import oracle
from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayDecompressVerify
base = Path(sys.argv[1]); key = bytes.fromhex(sys.argv[2]) if sys.argv[2] != "-" else None
pool = [p.read_bytes() for p in sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))]
store = ChunkStore(base / "dst")
qin, qout = GatewayQueue(), GatewayQueue()
ev, eq = mp.Event(), mp.Queue()
op = GatewayDecompressVerify("decompress_verify", "local:box", qin, qout, ev, eq, store, n_processes=1, use_compression=False,
                             e2ee_key_bytes=key, max_batch_chunks=8, max_batch_bytes=64 << 20)
def payload_of(data):
    if key is None:
        return data
    nonce = os.urandom(24)
    return nonce + oracle.secretbox_seal(key, nonce, data)
def payload_path(cid):
    return store.get_chunk_file_path(cid) if key is None else store.get_compressed_file_path(cid)
def request(cid, data):
    return ChunkRequest(Chunk("obj", "obj", cid, len(data), partition_id="0", md5_hash=hashlib.md5(data).digest()))
def drain(want, seconds):
    got, deadline = [], time.time() + seconds
    while len(got) < want and time.time() < deadline and not ev.is_set():
        got += qout.get_batch_nowait(16)
        time.sleep(0.01)
    return got
op.start_workers()
res = {}
try:
    ids = [f"{k:032x}" for k in range(len(pool))]
    for cid, data in zip(ids, pool):
        payload_path(cid).write_bytes(payload_of(data))
    stamps = {cid: os.stat(store.get_chunk_file_path(cid)).st_mtime_ns for cid in ids} if key is None else {}
    for cid, data in zip(ids, pool):
        qin.put(request(cid, data))
    done = drain(len(pool), 300)
    res["forwarded"] = sorted(r.chunk.chunk_id for r in done) == ids
    res["digests"] = all(r.chunk.md5_hash == hashlib.md5(pool[int(r.chunk.chunk_id, 16)]).digest() for r in done)
    res["chunk_files"] = all(store.get_chunk_file_path(cid).read_bytes() == data for cid, data in zip(ids, pool))
    res["payload_files_left"] = sum(store.get_compressed_file_path(cid).exists() for cid in ids)
    res["rewritten"] = sum(os.stat(store.get_chunk_file_path(cid)).st_mtime_ns != t for cid, t in stamps.items())
    # a payload that is still arriving: re-queued, then complete once it is whole
    slow, whole = "a" * 32, payload_of(pool[0])
    payload_path(slow).write_bytes(whole[: len(whole) // 2])
    qin.put(request(slow, pool[0]))
    res["early"] = len(drain(1, 1.5))
    with open(payload_path(slow), "ab") as f:
        f.write(whole[len(whole) // 2:])
    res["late"] = [r.chunk.chunk_id for r in drain(1, 120)] == [slow]
    res["error_before"] = ev.is_set()
    # a chunk whose bytes changed on the way: same length, other digest
    bad, data = "b" * 32, bytearray(pool[0])
    data[len(data) // 3] ^= 0x10
    payload_path(bad).write_bytes(payload_of(bytes(data)))
    qin.put(request(bad, pool[0]))
    ev.wait(120)
    res["error"] = eq.get(timeout=10) if ev.is_set() else None
finally:
    op.stop_workers()
print("RECV " + json.dumps(res), flush=True)
"""


@pytest.mark.parametrize("with_key", [False, True])
def test_decompress_verify_workers_receive_raw_chunks(with_key):
    base = Path(tempfile.mkdtemp(prefix="skyb200_raw_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [synth.silesia_like_chunk(5, 4 << 20), synth.random_chunk(6, 1 << 20), b"", b"x" * 13, synth.silesia_like_chunk(7, (1 << 20) + 77)]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), KEY.hex() if with_key else "-"], capture_output=True, text=True, env=env,
                           timeout=280)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RECV ")][-1][len("RECV "):])
        assert res["forwarded"] and res["digests"] and res["chunk_files"], res
        assert res["payload_files_left"] == 0 and res["rewritten"] == 0, res  # boxes are removed; received chunk files are left alone
        assert res["early"] == 0 and res["late"] and not res["error_before"], res
        assert res["error"] and "ChecksumMismatchException" in res["error"], res
    finally:
        shutil.rmtree(base, ignore_errors=True)
