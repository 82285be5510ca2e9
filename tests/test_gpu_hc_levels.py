"""GPU tests of the high-ratio levels (SKY_F_HC_LEVEL(3..9), python-lz4's compression_level) through the C ABI, ChunkStage
and GatewayCompressHash.

Bars: at every level, with and without block checksums, linked blocks and the optimal parse, the frames are
byte-identical to the sequential twin (tools/lz4hc_model.c) at depth 2^(level-1); MD5 bit-exact; every frame decodes with
the strict oracle decoder (without block checksums), liblz4 and sky_decode; SKY_F_HC_LEVEL(5) is SKY_F_HC; on 16 x 16 MiB
Silesia-like chunks level 3 < 5 < 9 in ratio, and level 9 >= 1.02 x level 5.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth
from skyplane_b200.stage import ChunkStage
from test_checksum_format import with_content_checksum
from test_gpu_hc import check_frame, twin_set

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

LEVELS = range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1)
STAGES = native.F_LZ4 | native.F_MD5  # (spelled out: the same frames as the level flag alone)
KEY = bytes((7 * i + 3) & 0xFF for i in range(32))


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


def twin_opts(level):
    k = native.kernel_config()
    assert k["hc_max_level"] >= level
    return hm.Opts(native.hc_depth(level), k["hc_hash_bits"], k["hc_nice"])


def run_device(ctx, chunks, flags, extra=0):
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


@pytest.fixture(scope="module")
def datas():
    return twin_set()


# every HC kernel: id "<level>" is the plain frame, and each option adds its suffix ("5-bc-linked-opt")
HC_KERNELS = [pytest.param(level, bc, linked, optimal,
                           id="-".join([str(level)] + [s for s, on in (("bc", bc), ("linked", linked), ("opt", optimal)) if on]))
              for level in LEVELS for bc in (False, True) for linked in (False, True) for optimal in (False, True)]


def assert_frames_equal_twin(ctx, stage, datas, level, bc, linked, optimal, names=None):
    """One HC kernel's frames of `datas` against the sequential twin at depth 2^(level-1), byte for byte, with and
    without SKY_F_VERIFY (the frame check must pass every one unchanged); every frame decodes with liblz4 (and the oracle
    when it has no block checksums), and sky_decode restores the chunks with the sender's digests.  names[i] names chunk
    i in a failure."""
    o = twin_opts(level)
    flags = native.hc_level_flag(level) | STAGES
    flags |= (native.F_BLOCK_CHECKSUM if bc else 0) | (native.F_LINKED if linked else 0) | (native.F_OPTIMAL if optimal else 0)
    frames, digests, lens = run_device(ctx, datas, flags, extra=4 * -(-max(map(len, datas)) // 65536) if bc else 0)
    for i, (d, f, dg, ln) in enumerate(zip(datas, frames, digests, lens)):
        name = names[i] if names else f"chunk {i}"
        want = hm.frame(d, o, block_checksum=bc, linked=linked, optimal=optimal, seg=native.kernel_config()["hc_opt_seg"])
        assert f == want, f"level {level} flags {flags:#x} {name} (len {len(d)}): GPU frame {len(f)} B != twin {len(want)} B"
        assert ln == len(f) and dg == hashlib.md5(d).digest()
        check_frame(f, d, block_checksum=bc, linked=linked)
    out = stage.decode(frames, [len(d) for d in datas])
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()
    res = stage.process(datas, level=level, block_checksum=bc, linked=linked, optimal=optimal, verify=True)
    for i, (f, r) in enumerate(zip(frames, res)):
        assert r.verify_status == 0 and bytes(r.frame) == f, f"level {level} flags {flags:#x} verify: {names[i] if names else i}"


@pytest.mark.parametrize("level,bc,linked,optimal", HC_KERNELS)
def test_frames_equal_twin_at_every_level(ctx, stage, datas, level, bc, linked, optimal):
    """Every HC kernel -- each level with and without block checksums, linked blocks and the optimal parse -- is pinned
    to the sequential twin at depth 2^(level-1) byte for byte (assert_frames_equal_twin)."""
    assert_frames_equal_twin(ctx, stage, datas, level, bc, linked, optimal)


def test_level5_is_the_default_high_ratio_mode(ctx, datas):
    default = run_device(ctx, datas, native.F_HC)
    assert run_device(ctx, datas, native.hc_level_flag(5)) == default
    assert run_device(ctx, datas, native.hc_level_flag(5) | STAGES) == default
    lz4_only = run_device(ctx, datas, native.hc_level_flag(7) | native.F_LZ4)
    assert lz4_only[0] == run_device(ctx, datas, native.hc_level_flag(7))[0] and all(dg == bytes(16) for dg in lz4_only[1])


def test_ratio_rises_with_level_on_silesia_like(ctx):
    datas = [synth.silesia_like_chunk(i, 16 << 20) for i in range(16)]
    total = sum(map(len, datas))
    ratio = {}
    for level in (3, 5, 9):
        frames, digests, _ = run_device(ctx, datas, native.hc_level_flag(level))
        for d, f, dg in zip(datas, frames, digests):
            check_frame(f, d)
            assert dg == hashlib.md5(d).digest()
        ratio[level] = total / sum(map(len, frames))
    print(f"ratio level 3 {ratio[3]:.4f} level 5 {ratio[5]:.4f} level 9 {ratio[9]:.4f}")
    assert ratio[3] < ratio[5] < ratio[9]
    assert ratio[9] >= 1.02 * ratio[5], ratio


def test_level9_with_content_checksum(ctx, stage):
    """The level-9 frame with LZ4's content checksum added; liblz4 and sky_decode verify it while decoding."""
    datas = [synth.silesia_like_chunk(50 + i, (1 << 20) + 999 * i) for i in range(3)] + [b"", b"abc" * 5, bytes(200000)]
    frames, digests, lens = run_device(ctx, datas, native.hc_level_flag(9) | native.F_CHECKSUM, extra=native.CHECKSUM_BYTES)
    o = twin_opts(9)
    for d, f, dg, ln in zip(datas, frames, digests, lens):
        assert f == with_content_checksum(hm.frame(d, o), d) and f[4] == (0x6C if d else 0x64)
        assert ln == len(f) and dg == hashlib.md5(d).digest()
        assert ref.lz4f_decompress(f, len(d)) == d
    out = stage.decode(frames, [len(d) for d in datas])
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()


def test_level3_e2ee_boxes_seal_the_twin_frame(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    o = twin_opts(3)
    datas = [synth.silesia_like_chunk(60 + i, 300000 + 777 * i) for i in range(3)] + [synth.random_chunk(4, 70000), b"", b"tiny"]
    nonces = bytes((3 * i + 1) & 0xFF for i in range(24 * len(datas)))
    res = stage.process(datas, encrypt=True, nonces=nonces, level=3)
    box = nacl_secret.SecretBox(KEY)
    for i, (d, r) in enumerate(zip(datas, res)):
        frame = box.decrypt(bytes(r.frame))
        assert frame == hm.frame(d, o) and bytes(r.frame)[:24] == nonces[24 * i: 24 * i + 24]
        assert oracle.lz4f_decode(frame, len(d)) == d and ref.lz4f_decompress(frame, len(d)) == d
        assert r.md5 == hashlib.md5(d).digest() and r.is_compressed and r.is_encrypted


def test_bad_level_fields_are_invalid(ctx, stage):
    datas = [synth.silesia_like_chunk(5, 300000), b"abc" * 100]
    lvl = lambda l: l << native.HC_LEVEL_SHIFT  # noqa: E731
    bad = [lvl(5), lvl(5) | native.F_LZ4, lvl(9) | STAGES | native.F_CHECKSUM, lvl(5) | native.F_MD5,
           native.hc_level_flag(5) | native.F_MD5] + [native.F_HC | lvl(l) for l in (1, 2, 10, 15)]
    for flags in bad:
        with pytest.raises(native.SkyChunkError) as e:
            run_device(ctx, datas, flags, extra=native.CHECKSUM_BYTES)
        assert e.value.code == native.SKY_E_INVALID, hex(flags)
    slot = stage.begin()
    stage.add_bytes(slot, datas[0])
    try:
        caps = [native.frame_bound(len(datas[0])) + native.CHECKSUM_BYTES + native.BOX_OVERHEAD]
        for flags in bad:
            with pytest.raises(native.SkyChunkError) as e:
                stage.ctx.submit([slot.inp.addr], [len(datas[0])], [slot.out.addr], caps, flags)
            assert e.value.code == native.SKY_E_INVALID, hex(flags)
    finally:
        stage.release(slot)
    # the context is still good after every refusal
    frames, digests, _ = run_device(ctx, datas, native.hc_level_flag(4))
    assert frames == [hm.frame(d, twin_opts(4)) for d in datas] and digests == [hashlib.md5(d).digest() for d in datas]


def test_chunkstage_process_level9(stage):
    o = twin_opts(9)
    datas = [synth.silesia_like_chunk(70 + i, (2 << 20) + 31 * i) for i in range(4)] + [synth.random_chunk(7, 100000), b"", b"x" * 13]
    res = stage.process(datas, level=9)
    for d, r in zip(datas, res):
        assert r.md5 == hashlib.md5(d).digest() and bytes(r.frame) == hm.frame(d, o) and r.comp_len == len(r.frame)


DRIVER = r"""
import json, sys
from pathlib import Path
from skyplane_b200.harness import run_stream
base = Path(sys.argv[1]); n_req = int(sys.argv[2])
files = sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))
lens = [p.stat().st_size for p in files]
res = run_stream(base / "chunks", files, lens, n_req, n_workers=2, max_batch_chunks=8, max_batch_bytes=64 << 20, keep_frames=True,
                 compression_level=9)
print("RESULT " + json.dumps(res))
"""


def test_operator_level9_in_queue_harness():
    base = Path(tempfile.mkdtemp(prefix="skyb200_hclv_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [synth.silesia_like_chunk(11, 8 << 20), synth.random_chunk(1, 1 << 20), b"", b"y" * 13, synth.silesia_like_chunk(12, (1 << 20) + 55)]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        n_req = 25
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), str(n_req)], capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        assert res["uncompressed_bytes"] == res["bytes"] and 0 < res["compressed_bytes"] < res["bytes"]
        o = twin_opts(9)
        want = [hm.frame(d, o) for d in pool]
        for rec in res["records"]:
            data = pool[rec["pool_index"]]
            assert rec["md5"] == hashlib.md5(data).hexdigest()
            assert Path(rec["frame_path"]).read_bytes() == want[rec["pool_index"]]
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
