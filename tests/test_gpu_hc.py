"""GPU tests of the high-ratio mode (SKY_F_HC, csrc/lz4hc.cuh) through the C ABI, ChunkStage and GatewayCompressHash.

Bars: frames byte-identical to the sequential twin of the HC parse (tools/lz4hc_model.c); MD5 bit-exact; every frame decodes
with the strict oracle decoder, liblz4, pyarrow and sky_decode; ratio >= 1.12 x the reference's on 16 x 16 MiB Silesia-like.
"""
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
from gpu_util import run_device
from skyplane_b200 import native, synth
from skyplane_b200.stage import ChunkStage

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

RNG = np.random.default_rng(78)
HC = native.F_HC | native.F_LZ4 | native.F_MD5  # (= F_HC alone; spelled out so gpu_util fetches the frames)
KEY = bytes((5 * i + 1) & 0xFF for i in range(32))


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


def twin_opts():
    k = native.kernel_config()
    assert k["hc_depth"] and k["hc_hash_bits"] and k["hc_nice"]
    return hm.Opts(k["hc_depth"], k["hc_hash_bits"], k["hc_nice"])


def kinds(n, rng=RNG):
    return {
        "random": rng.bytes(n),
        "zeros": bytes(n),
        "period7": (b"abcdefg" * (n // 7 + 1))[:n],
        "text": (b"it was the best of times, it was the worst of times; " * (n // 50 + 1))[:n],
        "half": (b"lorem ipsum dolor sit amet " * (n // 54 + 1))[: n // 2] + rng.bytes(n - n // 2),
    }


def twin_set():
    a = RNG.bytes(1000)
    datas = [kinds(n)[k] for n in (13, 300, 4096, 65536, 65537, 200000) for k in ("zeros", "period7", "text", "half", "random")]
    datas += [synth.silesia_like_chunk(40 + i, (1 << 20) + 777 * i) for i in range(6)]
    datas += [a + bytes(60000) + a, RNG.bytes(300) + b"Q" * 65000, (RNG.bytes(70) * 1000)[:65536], RNG.bytes(40000) + synth.silesia_like_chunk(3, 90000)]
    datas += [kinds(n)[k] for n in (0, 1, 12, 13, 65535, 65536, 65537) for k in ("text", "half", "random")]
    return datas


def check_frame(frame: bytes, data: bytes, block_checksum: bool = False, linked: bool = False):
    """block_checksum: the frame has 4 more bytes per block, and the strict oracle decoder, which takes no checksums,
    does not read it; linked: a frame of more than one block has B.Indep clear."""
    n = len(data)
    assert len(frame) <= native.frame_bound(n) + (4 * -(-n // 65536) if block_checksum else 0)
    assert frame[5] == 0x40 and frame[4] == (0x68 if n else 0x60) & ~(0x20 if linked and n > 65536 else 0) | (0x10 if block_checksum else 0)
    if not block_checksum:
        out, info = oracle.lz4f_decode(frame, n, with_info=True)
        assert out == data and info["consumed"] == len(frame)
    assert ref.lz4f_decompress(frame, n) == data


def test_frames_equal_hc_twin_and_decode_everywhere(ctx, stage):
    """The parallel chain build, search and ballot parse are pinned to the sequential twin byte for byte; every frame
    decodes with four decoders, and sky_decode's digest of the decoded bytes equals the sender's."""
    pa = pytest.importorskip("pyarrow")
    o = twin_opts()
    datas = twin_set()
    frames, digests, lens, _ = run_device(ctx, datas, flags=HC)
    for i, (d, f, dg, ln) in enumerate(zip(datas, frames, digests, lens)):
        want = hm.frame(d, o)
        assert f == want, f"chunk {i} (len {len(d)}): GPU frame {len(f)} B != twin {len(want)} B"
        assert ln == len(f) and dg == hashlib.md5(d).digest()
        check_frame(f, d)
        if d:
            assert pa.decompress(f, decompressed_size=len(d), codec="lz4").to_pybytes() == d
    out = stage.decode(frames, [len(d) for d in datas])
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()


def test_flags_hc_alone_means_lz4_md5_hc(ctx):
    datas = [synth.silesia_like_chunk(5, 300000), b"", b"abc" * 100]
    full = run_device(ctx, datas, flags=HC)
    d_in = ctx.device_alloc(1 << 20)
    d_out = ctx.device_alloc(1 << 21)
    try:
        so, dof = [0, 300016, 300032], [0, 400000, 500000]
        for c, off in zip(datas, so):
            if c:
                ctx.h2d(d_in + off, c)
        lens, digests, _ = ctx.process_device(d_in, so, [len(c) for c in datas], d_out, dof, [native.frame_bound(len(c)) for c in datas], native.F_HC)
        assert lens == full[2] and digests == full[1]
        assert [ctx.d2h(d_out + o, n) for o, n in zip(dof, lens)] == full[0]
        lz4_only = run_device(ctx, datas, flags=native.F_HC | native.F_LZ4)
        assert lz4_only[0] == full[0] and all(dg == bytes(16) for dg in lz4_only[1])
        with pytest.raises(native.SkyChunkError) as e:
            ctx.process_device(d_in, so, [len(c) for c in datas], d_out, dof, [native.frame_bound(len(c)) for c in datas], native.F_MD5 | native.F_HC)
        assert e.value.code == native.SKY_E_INVALID
    finally:
        ctx.device_free(d_in)
        ctx.device_free(d_out)


def test_md5_and_hc_is_invalid_on_the_host_path(stage):
    slot = stage.begin()
    stage.add_bytes(slot, b"abc" * 1000)
    try:
        with pytest.raises(native.SkyChunkError) as e:
            stage.ctx.submit([slot.inp.addr], [3000], None, None, native.F_MD5 | native.F_HC)
        assert e.value.code == native.SKY_E_INVALID
        with pytest.raises(ValueError):
            stage.launch(slot, compress=False, hc=True)
    finally:
        stage.release(slot)


def test_ratio_on_silesia_like(ctx):
    datas = [synth.silesia_like_chunk(i, 16 << 20) for i in range(16)]
    frames, digests, _, _ = run_device(ctx, datas, flags=HC)
    fast, _, _, _ = run_device(ctx, datas)
    total, hc, fz = sum(map(len, datas)), sum(map(len, frames)), sum(map(len, fast))
    refsz = sum(len(ref.lz4f_compress(d)) for d in datas)
    print(f"ratio hc {total / hc:.3f} fast {total / fz:.3f} reference(linked) {total / refsz:.3f}")
    for d, f, dg in zip(datas, frames, digests):
        check_frame(f, d)
        assert dg == hashlib.md5(d).digest()
    assert total / hc >= 1.12 * total / refsz


def test_incompressible_frame_equals_fast_path(ctx):
    datas = [synth.random_chunk(3, 8 << 20), RNG.bytes(65537)]
    hc = run_device(ctx, datas, flags=HC)
    fast = run_device(ctx, datas)
    assert hc[0] == fast[0] and hc[1] == fast[1] and len(hc[0][0]) == native.frame_bound(8 << 20)


def test_run_to_run_determinism(ctx):
    datas = [synth.silesia_like_chunk(9, 3 << 20), kinds(200000)["half"], kinds(70000)["text"]]
    assert run_device(ctx, datas, flags=HC)[0] == run_device(ctx, datas, flags=HC)[0]


def test_multipart_sized_chunks(ctx):
    big = synth.silesia_like_chunk(80, 16 << 20) * 4  # 64 MiB, compressible: 1024 block rows
    odd = synth.random_chunk(81, (33 << 20) + 12345)
    datas = [big, odd, b"tail" * 1000]
    frames, digests, _, _ = run_device(ctx, datas, flags=HC)
    for d, f, dg in zip(datas, frames, digests):
        check_frame(f, d)
        assert dg == hashlib.md5(d).digest()
    fast, _, _, _ = run_device(ctx, datas)
    assert len(frames[1]) == native.frame_bound(len(odd)) and len(frames[0]) < len(fast[0])
    assert frames[2] == hm.frame(datas[2], twin_opts())


def test_e2ee_boxes_seal_the_twin_frame(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    o = twin_opts()
    datas = [synth.silesia_like_chunk(30 + i, 300000 + 4321 * i) for i in range(3)] + [synth.random_chunk(9, 70000), b"", b"tiny"]
    nonces = RNG.bytes(24 * len(datas))
    res = stage.process(datas, compress=True, encrypt=True, nonces=nonces, hc=True)
    box = nacl_secret.SecretBox(KEY)
    for i, (d, r) in enumerate(zip(datas, res)):
        assert bytes(r.frame) == bytes(box.encrypt(hm.frame(d, o), nonces[24 * i: 24 * i + 24]))
        assert r.md5 == hashlib.md5(d).digest() and r.is_compressed and r.is_encrypted
    out = stage.decode([bytes(r.frame) for r in res], [len(d) for d in datas], encrypted=True)
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()


def test_pipelined_slots_through_chunkstage():
    o = twin_opts()
    stage = ChunkStage(0, max_batch_bytes=64 << 20, max_chunks=64, n_slots=2)
    try:
        batch_a = [synth.silesia_like_chunk(20 + i, 2 << 20) for i in range(4)] + [b"", b"tiny"]
        batch_b = [synth.random_chunk(30 + i, (1 << 20) + i) for i in range(3)] + [kinds(100000)["text"]]
        sa, sb = stage.begin(), stage.begin()
        for c in batch_a:
            stage.add_bytes(sa, c)
        for c in batch_b:
            stage.add_bytes(sb, c)
        stage.launch(sa, hc=True)
        stage.launch(sb)  # a fast-path batch in flight beside the HC batch
        rb = stage.collect(sb)
        ra = stage.collect(sa)
        for d, r in zip(batch_a, ra):
            assert bytes(r.frame) == hm.frame(d, o) and r.md5 == hashlib.md5(d).digest() and r.comp_len == len(r.frame)
        for d, r in zip(batch_b, rb):
            check_frame(bytes(r.frame), d)
            assert r.md5 == hashlib.md5(d).digest()
        assert stage.ctx.launches == 3  # HC kernel + MD5-only fused kernel, then one fused kernel
    finally:
        stage.close()


DRIVER = r"""
import json, sys
from pathlib import Path
from skyplane_b200.harness import run_stream
base = Path(sys.argv[1]); n_req = int(sys.argv[2])
files = sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))
lens = [p.stat().st_size for p in files]
res = run_stream(base / "chunks", files, lens, n_req, n_workers=2, max_batch_chunks=8, max_batch_bytes=64 << 20, keep_frames=True, high_ratio=True)
print("RESULT " + json.dumps(res))
"""


def test_operator_high_ratio_in_queue_harness():
    base = Path(tempfile.mkdtemp(prefix="skyb200_hc_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [synth.silesia_like_chunk(1, 8 << 20), synth.random_chunk(0, 1 << 20), b"", b"x" * 13, synth.silesia_like_chunk(2, (1 << 20) + 77)]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        n_req = 25
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), str(n_req)], capture_output=True, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        assert res["uncompressed_bytes"] == res["bytes"] and 0 < res["compressed_bytes"] < res["bytes"]
        o = twin_opts()
        want = [hm.frame(d, o) for d in pool]
        for rec in res["records"]:
            data = pool[rec["pool_index"]]
            assert rec["md5"] == hashlib.md5(data).hexdigest()
            assert Path(rec["frame_path"]).read_bytes() == want[rec["pool_index"]]
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
