"""GPU tests of sending incompressible chunks as themselves (SKY_F_PASSTHROUGH): through the C ABI on a mixed batch with the
fast compressor, high-ratio level 5 and high-ratio linked + optimal, each with and without E2EE and SKY_F_VERIFY, against
the same batch submitted without the flag; through ChunkStage; and end to end through GatewayCompressHash and
GatewayDecompressVerify (chunk files, and a socket sink read the way the reference's receiver reads it)."""
import ctypes
import functools
import hashlib
import multiprocessing as mp
import socket
import sys
import threading
from pathlib import Path

import numpy as np
import pytest

import oracle.reflib as ref
from skyplane_b200 import native, synth, wire
from skyplane_b200.chunk import Chunk, ChunkRequest, ChunkState
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash, GatewayDecompressVerify
from skyplane_b200.stage import ChunkStage
from test_linked_format import text

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools import hc_model as hm  # noqa: E402
from tools import tile_model as tm  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]

KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
GUARD = 64
FILL = 0xA5
MODES = {"fast": 0, "hc5": native.hc_level_flag(5), "hc-linked-optimal": native.F_HC | native.F_LINKED | native.F_OPTIMAL}
# the chunks at the pass-through edge, at the end of mixed_batch(): (compressor, chunk length, frame length - chunk length)
EDGE = [(mode, n, delta) for mode in MODES for n in (65536, 2 * 65536 + 100) for delta in (-1, 0, 1)]


def twin_frame_len(mode):
    """The length of `mode`'s frame of a chunk, from the compressor's sequential twin."""
    k = native.kernel_config()
    if mode == "fast":
        o = tm.kernel_opts(k["lz4_entries"], k["seg_slots"], k["max_step_log"])
        return lambda d: len(tm.frame(d, o))
    o = hm.Opts(native.hc_depth(5), k["hc_hash_bits"], k["hc_nice"])
    both = mode == "hc-linked-optimal"
    return lambda d: len(hm.frame(d, o, linked=both, optimal=both, seg=k["hc_opt_seg"]))


def at_the_edge(rng, mode, n, delta):
    """A random n-byte chunk with one zero run at offset 1000 whose `mode` frame is n + delta bytes: each byte of the run
    takes about one byte off the frame, so the run's length is stepped to the frame length wanted."""
    base, flen = rng.bytes(n), twin_frame_len(mode)
    z, seen = 300, set()
    while z not in seen:
        seen.add(z)
        d = base[:1000] + bytes(z) + base[1000 + z:]
        got = flen(d)
        if got == n + delta:
            return d
        z = max(1, z + max(-8, min(8, got - n - delta)))
    for z in range(max(1, min(seen) - 20), max(seen) + 20):  # the length skips a value near the step: walk the run
        d = base[:1000] + bytes(z) + base[1000 + z:]
        if flen(d) == n + delta:
            return d
    raise RuntimeError(f"no {n}-byte chunk with a {mode} frame of {n + delta} bytes")


@functools.lru_cache(maxsize=None)
def _mixed_batch():
    rng = np.random.default_rng(17)
    one_block = bytearray(rng.bytes(3 * 65536))
    one_block[65536:131072] = text(65536)
    near_miss = rng.bytes(200000) + bytes(24)
    return ([synth.random_chunk(1, (1 << 20) + 7), synth.silesia_like_chunk(2, (1 << 20) + 333), text(300001), b"", b"\x07",
             rng.bytes(65535), rng.bytes(65536), rng.bytes(65537), bytes(one_block), near_miss, synth.silesia_like_chunk(3, 65536)]
            + [at_the_edge(rng, *e) for e in EDGE])


def mixed_batch():
    """Random, Silesia-like, text, empty, 1 B, random at 64 KiB and one byte either side, a chunk whose only compressible
    part is one block (its frame is smaller), one whose compressible tail is too short to pay for the frame, and for each
    compressor in MODES, at one and at two blocks and a bit, chunks whose frame is one byte shorter than the chunk, as
    long, and one byte longer (EDGE): the first is sent compressed, the other two pass through."""
    return list(_mixed_batch())


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, max_batch_bytes=32 << 20, max_chunks=64, n_slots=2)
    c.set_e2ee_key(KEY)
    yield c
    c.close()


class Batch:
    """A batch's chunks in pinned memory, and pinned destinations with guard bytes on both sides of every dst[i]."""

    def __init__(self, datas, flags):
        self.datas = datas
        e2ee = bool(flags & native.F_E2EE)
        self.caps = [native.frame_need(len(d)) + (native.BOX_OVERHEAD if e2ee else 0) for d in datas]
        self.src_off, self.dst_off = [], []
        ip = op = 0
        for d, cap in zip(datas, self.caps):
            self.src_off.append(ip)
            ip += native.round16(len(d))
            op += GUARD
            self.dst_off.append(op)
            op += native.round16(cap) + GUARD
        self.src = native.PinnedBuffer(max(ip, 16))
        self.dst = native.PinnedBuffer(op)
        for d, o in zip(datas, self.src_off):
            self.src.view[o : o + len(d)] = d
        self.dst.view[:] = bytes([FILL]) * op

    def submit(self, ctx, flags, nonces=None):
        return ctx.submit([self.src.addr + o for o in self.src_off], [len(d) for d in self.datas],
                          [self.dst.addr + o for o in self.dst_off], self.caps, flags, nonces)

    def payload(self, i, n):
        return bytes(self.dst.view[self.dst_off[i] : self.dst_off[i] + n])

    def untouched(self, i, written):
        """The guard bytes around dst[i], and dst[i] beyond its first `written` bytes, still hold the fill."""
        lo, hi = self.dst_off[i] - GUARD, self.dst_off[i] + native.round16(self.caps[i]) + GUARD
        return bytes(self.dst.view[lo : self.dst_off[i]]) + bytes(self.dst.view[self.dst_off[i] + written : hi]) == \
            bytes([FILL]) * (hi - lo - written)

    def close(self):
        self.src.close()
        self.dst.close()


def sky_wait(ctx, t, n, verify, compressed):
    """sky_wait on ticket t with out_len and md5, and with verify[] / compressed[] when asked -> (rc, out_lens, digests,
    verify, compressed), None for an output not asked for."""
    out, md5 = (ctypes.c_uint64 * n)(), (ctypes.c_ubyte * (16 * n))()
    ver = (ctypes.c_int32 * n)() if verify else None
    comp = (ctypes.c_uint8 * n)() if compressed else None
    rc = native.lib().sky_wait(ctx._h, t, out, md5, ver, comp, None)
    return (rc, list(out), [bytes(md5[16 * i : 16 * i + 16]) for i in range(n)], None if ver is None else list(ver),
            None if comp is None else [bool(c) for c in comp])


def run(ctx, datas, flags, nonces=None):
    """-> (out_lens, digests, verify, compressed, payloads, guards intact) of one batch.  The batch is submitted once for
    each (verify, compressed) request sky_wait accepts for its ticket, and every one must complete it with the same
    results; without F_PASSTHROUGH compressed[i] is 1 exactly when the ticket has F_LZ4.  Before that, the requests the
    ticket refuses -- verify without F_VERIFY, no compressed with F_PASSTHROUGH -- must return SKY_E_INVALID and leave it
    waitable."""
    n = len(datas)
    forms = [(v, c) for v in (False, True) for c in (False, True)]
    allowed = [(v, c) for v, c in forms if (not v or flags & native.F_VERIFY) and (c or not flags & native.F_PASSTHROUGH)]
    got = []
    for form in allowed:
        b = Batch(datas, flags)
        try:
            t = b.submit(ctx, flags, nonces)
            for refused in (f for f in forms if f not in allowed):
                assert sky_wait(ctx, t, n, *refused)[0] == native.SKY_E_INVALID, refused
            rc, lens, dg, ver, comp = sky_wait(ctx, t, n, *form)
            assert rc == native.SKY_OK, form
            del ctx._inflight[t]
            got.append((lens, dg, ver, comp, [b.payload(i, k) for i, k in enumerate(lens)], all(b.untouched(i, k) for i, k in enumerate(lens))))
        finally:
            b.close()
    lens, dg, _, _, payloads, guards = got[0]
    ver = next((g[2] for g in got if g[2] is not None), None)
    comp = next(g[3] for g in got if g[3] is not None)
    assert all((g[0], g[1], g[4], g[5]) == (lens, dg, payloads, guards) and g[2] in (None, ver) and g[3] in (None, comp) for g in got)
    assert flags & native.F_PASSTHROUGH or comp == [bool(flags & native.F_LZ4)] * n
    return lens, dg, ver, comp, payloads, guards


@pytest.mark.parametrize("verify", [False, True], ids=["noverify", "verify"])
@pytest.mark.parametrize("e2ee", [False, True], ids=["plain", "e2ee"])
@pytest.mark.parametrize("mode", list(MODES))
def test_passthrough_against_the_same_batch_without_the_flag(ctx, mode, e2ee, verify):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = mixed_batch()
    base = native.F_LZ4 | native.F_MD5 | MODES[mode] | (native.F_VERIFY if verify else 0)
    nonces = np.random.default_rng(3).bytes(24 * len(datas)) if e2ee else None
    f_lens, _, f_ver, _, frames, _ = run(ctx, datas, base)  # the flag-off frames
    edge = [(n, delta, fl) for (m, n, delta), fl in zip(EDGE, f_lens[-len(EDGE):]) if m == mode]
    assert edge and all(fl == n + delta for n, delta, fl in edge), edge
    flags = base | native.F_PASSTHROUGH | (native.F_E2EE if e2ee else 0)
    lens, dg, ver, comp, payloads, guards = run(ctx, datas, flags, nonces)
    assert guards
    assert dg == [hashlib.md5(d).digest() for d in datas]
    assert comp == [fl < len(d) for fl, d in zip(f_lens, datas)]
    assert 0 < sum(comp) < len(datas), "the batch must mix chunks that pass through and chunks that do not"
    assert ver == (f_ver if verify else None)
    box = nacl_secret.SecretBox(KEY)
    for i, (d, c) in enumerate(zip(datas, comp)):
        if not e2ee:
            assert (lens[i], payloads[i]) == ((f_lens[i], frames[i]) if c else (0, b"")), i
            continue
        nonce = nonces[24 * i : 24 * i + 24]
        msg = frames[i] if c else d
        assert lens[i] == len(msg) + native.BOX_OVERHEAD
        assert payloads[i] == bytes(box.encrypt(msg, nonce)) and box.decrypt(payloads[i]) == msg, i


@pytest.mark.parametrize("e2ee", [False, True], ids=["plain", "e2ee"])
def test_two_slots_in_flight_and_repeats_agree(ctx, e2ee):
    datas = mixed_batch()
    flags = native.F_LZ4 | native.F_MD5 | native.F_PASSTHROUGH | (native.F_E2EE if e2ee else 0)
    nonces = bytes(range(24)) * len(datas) if e2ee else None
    one = run(ctx, datas, flags, nonces)
    assert one == run(ctx, datas, flags, nonces)  # deterministic
    a, b = Batch(datas, flags), Batch(datas[::-1], flags)
    try:
        ta, tb = a.submit(ctx, flags, nonces), b.submit(ctx, flags, nonces)  # both slots busy
        rb, ra = ctx.wait_ex(tb), ctx.wait_ex(ta)
        assert ra[:4] == one[:4] and [a.payload(i, n) for i, n in enumerate(ra[0])] == one[4]
        assert [x[::-1] for x in rb[:2]] == list(one[:2]) and rb[3][::-1] == one[3]
        assert [b.payload(i, n) for i, n in enumerate(rb[0])][::-1] == one[4]
    finally:
        a.close()
        b.close()


def test_refusals_and_wait_ex_on_other_tickets(ctx):
    L = native.lib()
    datas = [synth.random_chunk(4, 100000), synth.silesia_like_chunk(5, 100000)]
    b = Batch(datas, native.F_E2EE)
    try:
        n = len(datas)
        A, U = ctypes.c_void_p * n, ctypes.c_uint64 * n
        src, lens = A(*[b.src.addr + o for o in b.src_off]), U(*map(len, datas))
        dst, caps = A(*[b.dst.addr + o for o in b.dst_off]), U(*b.caps)
        t = ctypes.c_uint64()
        for bad in (native.F_MD5, native.F_MD5 | native.F_E2EE, native.F_CHECKSUM, native.F_BLOCK_CHECKSUM,
                    native.F_LZ4 | native.F_CHECKSUM | native.F_BLOCK_CHECKSUM):
            assert L.sky_submit(ctx._h, n, src, lens, dst, caps, bad | native.F_PASSTHROUGH, None, ctypes.byref(t)) == native.SKY_E_INVALID
        st = (ctypes.c_int32 * n)()
        assert L.sky_decode(ctx._h, n, dst, caps, src, lens, native.F_PASSTHROUGH, st, None, None) == native.SKY_E_INVALID
        d_in, d_out = ctx.device_alloc(1 << 20), ctx.device_alloc(1 << 20)
        try:
            for call in (lambda: ctx.process_device(d_in, [0], [100], d_out, [0], [native.frame_need(100)], native.F_PASSTHROUGH),
                         lambda: ctx.verify_device(d_in, [0], [100], d_out, [0], [50], flags=native.F_LZ4 | native.F_PASSTHROUGH)):
                with pytest.raises(native.SkyChunkError) as e:
                    call()
                assert e.value.code == native.SKY_E_INVALID
        finally:
            ctx.device_free(d_in)
            ctx.device_free(d_out)
        # wait_ex completes any ticket: compressed[i] is 1 exactly when the ticket makes frames
        for flags, want in ((0, True), (native.F_LZ4 | native.F_MD5, True), (native.F_MD5, False)):
            lens_, dg, ver, comp, _ = ctx.wait_ex(b.submit(ctx, flags))
            assert comp == [want] * n and ver is None and dg == [hashlib.md5(d).digest() for d in datas]
    finally:
        b.close()


@pytest.mark.parametrize("encrypt", [False, True], ids=["plain", "e2ee"])
def test_stage_results_per_chunk(encrypt):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = mixed_batch()
    s = ChunkStage(0, max_batch_bytes=32 << 20, max_chunks=64, n_slots=2)
    try:
        s.set_e2ee_key(KEY)
        off = s.process(datas)
        res = s.process(datas, encrypt=encrypt, passthrough=True, verify=True)
        for d, o, r in zip(datas, off, res):
            c = o.comp_len < len(d)
            assert r.is_compressed == c and r.is_encrypted == encrypt and r.md5 == hashlib.md5(d).digest() and r.verify_status == 0
            msg = bytes(o.frame) if c else d
            got = nacl_secret.SecretBox(KEY).decrypt(bytes(r.frame)) if encrypt else bytes(r.frame)
            assert got == msg and r.comp_len == len(r.frame)
        with pytest.raises(ValueError, match="content checksum"):
            s.process(datas[:1], passthrough=True, checksum=True)
    finally:
        s.close()


# ------------------------------------------------------------------ end to end through the operators
def _reqs(datas, prefix):
    return [ChunkRequest(Chunk("src", "dst", "%s%030x" % (prefix, i), len(d), partition_id="0")) for i, d in enumerate(datas)]


def _sender(tmp_path, datas, reqs, key, **kw):
    cs = ChunkStore(tmp_path / "send")
    for r, d in zip(reqs, datas):
        cs.get_chunk_file_path(r.chunk.chunk_id).write_bytes(d)
    op = GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), cs, use_compression=True,
                             skip_incompressible=True, e2ee_key_bytes=key, max_batch_bytes=32 << 20, n_slots=2, **kw)
    op.worker_id = 0
    return op, cs


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "e2ee"])
def test_operators_end_to_end_through_chunk_files(tmp_path, key):
    datas = mixed_batch()
    reqs = _reqs(datas, "aa")
    op, cs = _sender(tmp_path, datas, reqs, key)
    try:
        assert op.process_batch(reqs) == [True] * len(reqs)
        op._complete_many(0, reqs)
    finally:
        op.worker_exit(0)
    records = {}
    item = cs.chunk_status_queue.get(timeout=10)
    for rec in cs.iter_status_records(item):
        records[rec["chunk_id"]] = rec
    assert all(rec["state"] == ChunkState.complete.name for rec in records.values())
    rstore = ChunkStore(tmp_path / "recv")
    passed = 0
    for r, d in zip(reqs, datas):
        cid = r.chunk.chunk_id
        rec = records[cid]
        path, is_compressed = cs.wire_payload(cid)
        payload = path.read_bytes()
        assert rec["compressed_size_bytes"] == len(payload) and rec["uncompressed_size_bytes"] == len(d)
        assert rec.get("passed_through", False) == (not is_compressed)
        if not is_compressed:
            passed += 1
            assert path == (cs.get_box_file_path(cid) if key else cs.get_chunk_file_path(cid))
            assert not cs.get_compressed_file_path(cid).exists()
        # the receiving side: a frame (or its box) to .chunk.lz4, a sealed chunk to .chunk.box, a chunk to .chunk
        dest = rstore.get_compressed_file_path(cid) if is_compressed else (rstore.get_box_file_path(cid) if key else rstore.get_chunk_file_path(cid))
        dest.write_bytes(payload)
    assert 0 < passed < len(datas)
    rop = GatewayDecompressVerify("dv", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), rstore, skip_incompressible=True,
                                  e2ee_key_bytes=key, max_batch_bytes=32 << 20)
    rop.worker_id = 0
    try:
        assert rop.process_batch(reqs) == [True] * len(reqs)
    finally:
        rop.worker_exit(0)
    for r, d in zip(reqs, datas):
        cid = r.chunk.chunk_id
        assert rstore.get_chunk_file_path(cid).read_bytes() == d and r.chunk.md5_hash == hashlib.md5(d).digest()
        assert not rstore.get_compressed_file_path(cid).exists() and not rstore.get_box_file_path(cid).exists()


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "e2ee"])
def test_sink_headers_carry_the_per_chunk_bit_to_a_reference_style_receiver(tmp_path, key):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = mixed_batch()
    reqs = _reqs(datas, "bb")
    a, b = socket.socketpair()
    got = []

    def receiver():
        for _ in reqs:
            buf = bytearray(native.frame_need(max(map(len, datas))) + native.BOX_OVERHEAD)
            h, n = wire.recv_chunk(b, buf)
            got.append((h, bytes(buf[:n])))

    t = threading.Thread(target=receiver)
    t.start()
    op, _ = _sender(tmp_path, datas, reqs, key, sink=lambda worker_id: a)
    try:
        assert op.process_batch(reqs) == [True] * len(reqs)
        t.join(60)
        assert not t.is_alive()
    finally:
        op.worker_exit(0)  # (closes the sink socket)
        b.close()
    assert [h.chunk_id for h, _ in got] == [r.chunk.chunk_id for r in reqs]
    assert 0 < sum(h.is_compressed for h, _ in got) < len(datas)
    for (h, payload), d in zip(got, datas):
        # gateway_receiver.py:191-201: decrypt when keyed, lz4.frame.decompress only when the header says so
        data = bytes(nacl_secret.SecretBox(key).decrypt(payload)) if key else payload
        if h.is_compressed:
            data = ref.lz4f_decompress(data, h.raw_data_len)
        assert h.raw_data_len == len(d) and data == d and hashlib.md5(data).digest() == hashlib.md5(d).digest()
        assert h.is_compressed == (len(payload) - (native.BOX_OVERHEAD if key else 0) < len(d))
