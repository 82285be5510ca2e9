"""GPU tests of LZ4 content and block checksums (XXH32): SKY_F_CHECKSUM frames from the sender, and the receiver's
verification of checksummed frames from any liblz4 sender and from our own.

Sender bars: frames decode with liblz4 (checksums verified), pyarrow and sky_decode; the trailer is XXH32(chunk); apart
from FLG, the header checksum byte and the trailer, every byte equals the same batch's frame without the flag, and the
digests are the same -- on the fast and the high-ratio path, sealed in a SecretBox, through sky_process_device and through
pipelined slots.  Receiver bars: liblz4 frames with a content checksum, block checksums or both, linked and independent,
with and without E2EE, decode with the right digests; a flipped checksum or data byte gives SKY_D_CHECKSUM for that chunk
alone, and a frame cut inside its trailer SKY_D_TRUNCATED."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import hc_model  # noqa: E402
from test_checksum_format import with_content_checksum  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]

RNG = np.random.default_rng(64)
CK = native.F_CHECKSUM
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
LENS = [0, 1, 15, 16, 17, 63, 64, 65, 65535, 65536, 65537, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 8 << 20]


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 1 << 30, 4096, 0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def stage():
    s = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=64, n_slots=2)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


def kinds(n, rng=RNG):
    return {
        "random": rng.bytes(n),
        "zeros": bytes(n),
        "period7": (b"abcdefg" * (n // 7 + 1))[:n],
        "text": (b"it was the best of times, it was the worst of times; " * (n // 50 + 1))[:n],
        "half": (b"lorem ipsum dolor sit amet " * (n // 54 + 1))[: n // 2] + rng.bytes(n - n // 2),
    }


def run_device(ctx, chunks, flags, extra=4):
    """sky_process_device with dst_cap = sky_frame_bound(n) + extra. -> (frames, digests, out_lens)"""
    src_off, dst_off, caps, ip, op = [], [], [], 0, 0
    for c in chunks:
        src_off.append(ip)
        dst_off.append(op)
        caps.append(native.frame_bound(len(c)) + extra)
        ip += native.round16(len(c))
        op += native.round16(caps[-1])
    d_in, d_out = ctx.device_alloc(ip + 64), ctx.device_alloc(op + 64)
    try:
        for c, o in zip(chunks, src_off):
            if c:
                ctx.h2d(d_in + o, c)
        lens, digests, _ = ctx.process_device(d_in, src_off, [len(c) for c in chunks], d_out, dst_off, caps, flags)
        return [ctx.d2h(d_out + o, n) for o, n in zip(dst_off, lens)], digests, lens
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)


def decode_device(ctx, frames, raw_lens):
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
        st, dg, _ = ctx.decode_device(d_f, f_off, [len(f) for f in frames], d_o, o_off, raw_lens)
        return [ctx.d2h(d_o + o, r) if s == 0 else None for o, r, s in zip(o_off, raw_lens, st)], dg, st
    finally:
        ctx.device_free(d_f)
        ctx.device_free(d_o)


def check_checksummed(frame: bytes, plain: bytes, data: bytes):
    pa = pytest.importorskip("pyarrow")
    n = len(data)
    assert frame == with_content_checksum(plain, data), n
    assert frame[4] == (0x6C if n else 0x64) and len(frame) <= native.frame_bound(n) + 4
    assert frame[-4:] == oracle.xxh32(data).to_bytes(4, "little")
    assert ref.lz4f_decompress(frame, n) == data  # liblz4 verifies the content checksum
    if n:
        assert pa.decompress(frame, decompressed_size=n, codec="lz4").to_pybytes() == data


def roundtrip(ctx, flags, datas):
    plain, dg0, _ = run_device(ctx, datas, flags)
    frames, dg, lens = run_device(ctx, datas, flags | CK)
    assert dg == dg0 == [hashlib.md5(d).digest() for d in datas]
    for d, f, p, ln in zip(datas, frames, plain, lens):
        assert ln == len(f)
        check_checksummed(f, p, d)
    outs, dgd, st = decode_device(ctx, frames, [len(d) for d in datas])
    assert st == [0] * len(datas) and outs == datas and dgd == dg


@pytest.mark.parametrize("kind", ["random", "zeros", "period7", "text", "half"])
def test_checksum_frames_restore_every_length(ctx, kind):
    roundtrip(ctx, 0, [kinds(n)[kind] for n in LENS])


def test_checksum_frames_mixed_batch(ctx):
    datas = [RNG.bytes(int(n)) for n in RNG.integers(0, 400000, size=60)] + [synth.silesia_like_chunk(3, (3 << 20) + 5), b""]
    roundtrip(ctx, 0, datas)


def test_checksum_frames_high_ratio(ctx):
    datas = [kinds(n)["half"] for n in LENS] + [synth.silesia_like_chunk(4, 2 << 20)]
    roundtrip(ctx, native.F_HC, datas)


def test_flag_rules(ctx):
    datas = [synth.silesia_like_chunk(5, 300000), b"", b"abc" * 100]
    full = run_device(ctx, datas, native.F_LZ4 | native.F_MD5 | CK)
    assert run_device(ctx, datas, CK) == full  # alone: LZ4 + MD5 + checksum
    assert run_device(ctx, datas, native.F_LZ4 | CK)[0] == full[0]
    assert run_device(ctx, datas, native.F_HC | CK)[0] == run_device(ctx, datas, native.F_HC | native.F_LZ4 | native.F_MD5 | CK)[0]
    for flags, extra, code in ((native.F_MD5 | CK, 4, native.SKY_E_INVALID), (CK, 0, native.SKY_E_CAPACITY),
                               (native.F_HC | CK, 0, native.SKY_E_CAPACITY)):
        with pytest.raises(native.SkyChunkError) as e:
            run_device(ctx, datas, flags, extra)
        assert e.value.code == code
    n0 = ctx.launches
    run_device(ctx, datas, 0)
    n1 = ctx.launches
    run_device(ctx, datas, CK)
    n2 = ctx.launches
    run_device(ctx, datas, native.F_BLOCK_CHECKSUM, 4 * 5)  # (5 blocks in the longest chunk)
    assert n1 - n0 == 1 and n2 - n1 == 2  # the checksum epilogue only when asked for
    assert ctx.launches - n2 == 1  # block checksums need no epilogue: the compressor writes the final header


def test_e2ee_seals_the_checksummed_frame(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = [synth.silesia_like_chunk(30 + i, 300000 + 4321 * i) for i in range(3)] + [synth.random_chunk(9, 70000), b"", b"tiny"]
    nonces = RNG.bytes(24 * len(datas))
    box = nacl_secret.SecretBox(KEY)
    for hc in (False, True):
        plain = stage.process(datas, hc=hc)
        res = stage.process(datas, encrypt=True, nonces=nonces, hc=hc, checksum=True)
        for d, p, r in zip(datas, plain, res):
            frame = bytes(box.decrypt(bytes(r.frame)))
            check_checksummed(frame, bytes(p.frame), d)
            assert len(r.frame) <= native.frame_bound(len(d)) + 4 + native.BOX_OVERHEAD
            assert r.md5 == p.md5 == hashlib.md5(d).digest() and r.is_encrypted
        out = stage.decode([bytes(r.frame) for r in res], [len(d) for d in datas], encrypted=True)
        assert all(st == 0 and data == d and dg == hashlib.md5(d).digest() for d, (data, dg, st) in zip(datas, out))


def test_pipelined_slots_with_checksums():
    stage = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=64, n_slots=2)
    try:
        batch_a = [synth.silesia_like_chunk(20 + i, 2 << 20) for i in range(4)] + [b"", b"tiny"]
        batch_b = [synth.random_chunk(30 + i, (1 << 20) + i) for i in range(3)] + [kinds(100000)["text"]]
        plain_a, plain_b = stage.process(batch_a, hc=True), stage.process(batch_b)
        n0 = stage.ctx.launches
        sa, sb = stage.begin(), stage.begin()
        for c in batch_a:
            stage.add_bytes(sa, c)
        for c in batch_b:
            stage.add_bytes(sb, c)
        stage.launch(sa, hc=True, checksum=True)
        stage.launch(sb, checksum=True)
        rb, ra = stage.collect(sb), stage.collect(sa)
        for data, plain, res in ((batch_a, plain_a, ra), (batch_b, plain_b, rb)):
            for d, p, r in zip(data, plain, res):
                check_checksummed(bytes(r.frame), bytes(p.frame), d)
                assert r.md5 == hashlib.md5(d).digest() and r.comp_len == len(r.frame)
        assert stage.ctx.launches - n0 == 5  # HC + MD5/XXH kernel + epilogue, fused XXH kernel + epilogue
    finally:
        stage.close()


@pytest.mark.parametrize("size", [300, 4096, 65537])
def test_staging_reserves_the_trailer(size):
    """A slot filled to its byte limit: the input side binds first, as it did before the 4 bytes per chunk were
    reserved, and the full batch launches with checksums."""
    stage = ChunkStage(0, max_batch_bytes=1 << 20, max_chunks=4096, n_slots=1)
    try:
        slot = stage.begin()
        datas = []
        while stage.fits(slot, size):
            datas.append(RNG.bytes(size))
            stage.add_bytes(slot, datas[-1])
        assert len(datas) == slot.inp.nbytes // native.round16(size) and slot.out_used <= slot.out.nbytes
        stage.launch(slot, checksum=True)
        res = stage.collect(slot)
        assert len(res) == len(datas)
        for d, r in zip(datas[:: max(1, len(datas) // 16)], res[:: max(1, len(datas) // 16)]):
            assert ref.lz4f_decompress(bytes(r.frame), size) == d and r.md5 == hashlib.md5(d).digest()
    finally:
        stage.close()


LIBLZ4_MODES = [(linked, cc, bc) for linked in (False, True) for cc, bc in ((1, 0), (0, 1), (1, 1))]


@pytest.mark.parametrize("linked,content,block", LIBLZ4_MODES)
def test_receiver_verifies_liblz4_checksummed_frames(ctx, linked, content, block):
    datas = [d for n in (0, 1, 17, 65536, 65537, 200000) for d in kinds(n).values()] + [synth.silesia_like_chunk(40, 3 << 20)]
    frames = [hc_model.liblz4_frame(d, 0, linked, bool(content), bool(block)) for d in datas]
    assert all(f[4] & 0x14 == (0x04 if content else 0) | (0x10 if block else 0) for f in frames)
    outs, dg, st = decode_device(ctx, frames, [len(d) for d in datas])
    assert st == [0] * len(datas) and outs == datas
    assert dg == [hashlib.md5(d).digest() for d in datas]


def test_receiver_verifies_checksummed_boxes(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    box = nacl_secret.SecretBox(KEY)
    datas = [synth.silesia_like_chunk(41, 1 << 20), synth.random_chunk(42, 100000), b"", b"x" * 20]
    frames = [hc_model.liblz4_frame(d, 0, True, True, True) for d in datas]
    sealed = [bytes(box.encrypt(f, RNG.bytes(24))) for f in frames]
    out = stage.decode(sealed, [len(d) for d in datas], encrypted=True)
    assert all(st == 0 and data == d and dg == hashlib.md5(d).digest() for d, (data, dg, st) in zip(datas, out))


def test_tampered_checksums_fail_only_their_chunk(ctx):
    d = synth.silesia_like_chunk(43, 200000)
    r = synth.random_chunk(44, 200000)
    both = hc_model.liblz4_frame(d, 0, False, True, True)
    rand_content = hc_model.liblz4_frame(r, 0, False, True, False)  # stored blocks, content checksum only
    rand_block = hc_model.liblz4_frame(r, 0, False, False, True)
    hdr = 15

    def flip(f, k):
        b = bytearray(f)
        b[k] ^= 0x20
        return bytes(b)

    size0 = int.from_bytes(both[hdr : hdr + 4], "little") & 0x7FFFFFFF
    rsize0 = int.from_bytes(rand_block[hdr : hdr + 4], "little") & 0x7FFFFFFF
    frames = [
        both,
        flip(both, hdr + 4 + size0),  # block 0's checksum
        flip(both, len(both) - 2),  # the content trailer
        flip(rand_block, hdr + 4 + rsize0 // 2),  # a byte inside a stored block with a block checksum
        flip(rand_content, hdr + 4 + 1000),  # a byte inside a stored block: only the content checksum sees it
        both[:-2],  # cut inside the trailer
        rand_content,
    ]
    datas = [d, d, d, r, r, d, r]
    outs, dg, st = decode_device(ctx, frames, [len(x) for x in datas])
    C, T = native.D_CHECKSUM, native.D_TRUNCATED
    assert st == [0, C, C, C, C, T, 0], st
    assert outs[0] == d and outs[6] == r
    for f, x, s in zip(frames, datas, st):  # liblz4 rejects every frame we reject
        if s:
            with pytest.raises(ValueError):
                ref.lz4f_decompress(f, len(x))


DRIVER = r"""
import json, multiprocessing as mp, sys, time, traceback
from pathlib import Path
from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.harness import run_stream
from skyplane_b200.operators import GatewayDecompressVerify
base = Path(sys.argv[1]); n_req = int(sys.argv[2])
files = sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))
lens = [p.stat().st_size for p in files]
res = run_stream(base / "chunks", files, lens, n_req, n_workers=2, max_batch_chunks=8, max_batch_bytes=64 << 20, keep_frames=True,
                 content_checksum=True)
print("RESULT " + json.dumps(res), flush=True)
# the destination side: GatewayDecompressVerify workers get the frames, intact and with the trailer tampered with
store = ChunkStore(base / "dst")
qin, qout = GatewayQueue(), GatewayQueue()
ev, eq = mp.Event(), mp.Queue()
op = GatewayDecompressVerify("decompress_verify", "local:box", qin, qout, ev, eq, store, n_processes=1)
op.start_workers()
recv = {}
try:
    for k, rec in enumerate(res["records"][:6]):
        frame = Path(rec["frame_path"]).read_bytes()
        cid = f"{k:032x}"
        store.get_compressed_file_path(cid).write_bytes(frame)
        qin.put(ChunkRequest(Chunk(f"obj/{k}", f"obj/{k}", cid, lens[rec["pool_index"]], partition_id="0", md5_hash=bytes.fromhex(rec["md5"]))))
    done, deadline = 0, time.time() + 300
    while done < 6 and time.time() < deadline and not ev.is_set():
        done += len(qout.get_batch_nowait(16))
        time.sleep(0.01)
    recv["intact_done"] = done
    for k, rec in enumerate(res["records"][:6]):
        recv.setdefault("restored", []).append(store.get_chunk_file_path(f"{k:032x}").read_bytes() == files[rec["pool_index"]].read_bytes())
    rec = res["records"][0]
    frame = bytearray(Path(rec["frame_path"]).read_bytes())
    frame[-1] ^= 0x01
    cid = "f" * 32
    store.get_compressed_file_path(cid).write_bytes(bytes(frame))
    qin.put(ChunkRequest(Chunk("obj/t", "obj/t", cid, lens[rec["pool_index"]], partition_id="0", md5_hash=bytes.fromhex(rec["md5"]))))
    ev.wait(300)
    recv["error"] = eq.get(timeout=10) if ev.is_set() else None
finally:
    op.stop_workers()
print("RECV " + json.dumps(recv), flush=True)
"""


def test_operators_with_content_checksum_in_queue_harness():
    base = Path(tempfile.mkdtemp(prefix="skyb200_ck_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [synth.silesia_like_chunk(1, 8 << 20), synth.random_chunk(0, 1 << 20), b"", b"x" * 13, synth.silesia_like_chunk(2, (1 << 20) + 77)]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        n_req = 20
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), str(n_req)], capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])
        recv = json.loads([l for l in r.stdout.splitlines() if l.startswith("RECV ")][-1][len("RECV "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        for rec in res["records"]:
            data = pool[rec["pool_index"]]
            frame = Path(rec["frame_path"]).read_bytes()
            assert rec["md5"] == hashlib.md5(data).hexdigest()
            assert frame[4] == (0x6C if data else 0x64) and frame[-4:] == oracle.xxh32(data).to_bytes(4, "little")
            assert ref.lz4f_decompress(frame, len(data)) == data
        assert recv["intact_done"] == 6 and all(recv["restored"]), recv
        assert recv["error"] and "ChecksumMismatchException" in recv["error"], recv
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
