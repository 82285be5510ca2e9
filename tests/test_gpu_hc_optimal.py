"""GPU tests of the high-ratio mode's optimal parse (SKY_F_HC | SKY_F_OPTIMAL) through the C ABI, ChunkStage and the
gateway operator.

Bars: at every level 3..9, independent and linked, with and without block and content checksums, the frames are
byte-identical to the twin (tools/lz4hc_model.c, hc_compress_block_opt, segments of sky_kernel_config(8) bytes) on the HC
tests' twin_set() plus text-like chunks long enough for segments and windows to matter; MD5 bit-exact; the strict oracle,
liblz4 and sky_decode restore every chunk; SKY_F_VERIFY passes every clean frame and sky_verify_device takes the flag; E2EE
boxes seal the twin frame; the flag's refusals leave the context usable; run-to-run determinism; on 16 x 16 MiB
Silesia-like chunks optimal level 5 beats lazy levels 5 and 6 on ratio; GatewayCompressHash(optimal_parse=True) writes the
twin's frames."""
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
from test_gpu_hc import twin_set
from test_gpu_hc_levels import run_device
from test_gpu_verify import run_verify
from test_linked_format import text, with_content_checksum

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

OPT, LK, BC, CK = native.F_OPTIMAL, native.F_LINKED, native.F_BLOCK_CHECKSUM, native.F_CHECKSUM
KEY = bytes((29 * i + 3) & 0xFF for i in range(32))
# the checksum flags each level runs with: every combination, at more than one level
LEVEL_CHECKSUMS = {3: 0, 4: BC, 5: CK, 6: BC | CK, 7: 0, 8: BC, 9: BC | CK}


def twin_opts(level):
    k = native.kernel_config()
    return hm.Opts(native.hc_depth(level), k["hc_hash_bits"], k["hc_nice"])


def twin(data: bytes, level: int, flags: int = 0) -> bytes:
    f = hm.frame(data, twin_opts(level), block_checksum=bool(flags & BC), linked=bool(flags & LK), optimal=True,
                 seg=native.kernel_config()["hc_opt_seg"])
    return with_content_checksum(f, data) if flags & CK else f


def extra(datas, flags):
    return (4 if flags & CK else 0) + (4 * -(-max(map(len, datas)) // 65536) if flags & BC else 0)


@pytest.fixture(scope="module")
def ctx():
    c = native.Context(0, 1 << 30, 4096, 0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def stage():
    s = ChunkStage(0, max_batch_bytes=96 << 20, max_chunks=128, n_slots=2)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


@pytest.fixture(scope="module")
def datas():
    return twin_set() + [text(n) for n in (2047, 2048, 2049, 2 << 20)] + [synth.silesia_like_chunk(83, 3 << 20)]


def test_kernel_config_reports_the_segment():
    assert native.kernel_config()["hc_opt_seg"] == hm.OPT_SEG == 2048


@pytest.mark.parametrize("linked", [False, True])
@pytest.mark.parametrize("level", sorted(LEVEL_CHECKSUMS))
def test_frames_equal_twin_at_every_level(ctx, stage, datas, level, linked):
    ck = LEVEL_CHECKSUMS[level]
    flags = native.hc_level_flag(level) | OPT | (LK if linked else 0) | ck
    frames, digests, lens = run_device(ctx, datas, flags, extra(datas, ck))
    for i, (d, f, dg, ln) in enumerate(zip(datas, frames, digests, lens)):
        want = twin(d, level, flags)
        assert f == want, f"level {level} linked {linked} flags {flags:#x} chunk {i} (len {len(d)}): GPU {len(f)} B != twin {len(want)} B"
        assert ln == len(f) and dg == hashlib.md5(d).digest()
        if not ck:
            assert oracle.lz4f_decode(f, len(d)) == d
        assert ref.lz4f_decompress(f, len(d)) == d
    out = stage.decode(frames, [len(d) for d in datas])
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()


def test_verify_passes_clean_frames(ctx, stage, datas):
    """SKY_F_VERIFY on optimal batches: every status 0, frames and digests as without the check; sky_verify_device takes
    the flag as a compressor bit."""
    for level, linked, ck in ((3, False, 0), (9, True, BC | CK), (5, True, 0)):
        kw = dict(level=level, linked=linked, optimal=True, checksum=bool(ck & CK), block_checksum=bool(ck & BC))
        plain = stage.process(datas, **kw)
        checked = stage.process(datas, verify=True, **kw)
        for d, p, c in zip(datas, plain, checked):
            assert c.verify_status == 0 and bytes(c.frame) == bytes(p.frame) == twin(d, level, ck | (LK if linked else 0))
            assert c.md5 == p.md5 == hashlib.md5(d).digest()
    for flags in (native.F_HC | OPT, native.F_HC | OPT | LK):
        frames = [twin(d, 5, flags) for d in datas]
        st, after, _ = run_verify(ctx, datas, frames, flags, repair=False)
        assert st == [0] * len(datas) and after == frames


def test_e2ee_boxes_seal_the_twin_frame(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = [text(300000), synth.silesia_like_chunk(62, 700001), synth.random_chunk(4, 70000), b"", b"tiny"]
    nonces = bytes((7 * i + 1) & 0xFF for i in range(24 * len(datas)))
    for linked in (False, True):
        res = stage.process(datas, encrypt=True, nonces=nonces, level=6, linked=linked, optimal=True)
        box = nacl_secret.SecretBox(KEY)
        for i, (d, r) in enumerate(zip(datas, res)):
            frame = box.decrypt(bytes(r.frame))
            assert frame == twin(d, 6, LK if linked else 0) and bytes(r.frame)[:24] == nonces[24 * i : 24 * i + 24]
            assert r.md5 == hashlib.md5(d).digest()


def test_flag_errors_leave_the_context_usable(ctx, stage):
    datas = [text(200000), b"abc" * 100]
    stages = native.F_LZ4 | native.F_MD5
    bad = [OPT, OPT | stages, OPT | native.F_LZ4, OPT | native.F_MD5, OPT | LK, OPT | CK, native.F_HC | OPT | native.F_MD5,
           native.hc_level_flag(5) | OPT | LK | native.F_MD5]
    for flags in bad:
        with pytest.raises(native.SkyChunkError) as e:
            run_device(ctx, datas, flags, extra=8)
        assert e.value.code == native.SKY_E_INVALID, hex(flags)
    slot = stage.begin()
    stage.add_bytes(slot, datas[0])
    try:
        caps = [native.frame_need(len(datas[0]), True, True) + native.BOX_OVERHEAD]
        for flags in bad:
            with pytest.raises(native.SkyChunkError) as e:
                stage.ctx.submit([slot.inp.addr], [len(datas[0])], [slot.out.addr], caps, flags)
            assert e.value.code == native.SKY_E_INVALID, hex(flags)
    finally:
        stage.release(slot)
    with pytest.raises(ValueError, match="F_OPTIMAL"):
        stage.ctx.decode([0], [1], None, [len(datas[0])], OPT)
    for base in (0, native.F_LZ4, native.F_MD5 | native.F_E2EE):  # the library refuses the bit before it reads anything
        assert native.lib().sky_decode(stage.ctx._h, 1, None, None, None, None, base | OPT, None, None, None) == native.SKY_E_INVALID
    frames, _, _ = run_device(ctx, datas, native.hc_level_flag(5) | OPT)
    assert frames == [twin(d, 5) for d in datas]


def test_deterministic_and_ratio_above_lazy_levels_5_and_6(ctx):
    """16 x 16 MiB Silesia-like chunks: optimal level 5 sends fewer bytes than lazy level 5 and lazy level 6, independent and
    linked; two runs give the same frames."""
    datas = [synth.silesia_like_chunk(100 + i, 16 << 20) for i in range(16)]
    raw = sum(map(len, datas))
    for lk in (0, LK):
        lazy5, _, _ = run_device(ctx, datas, native.hc_level_flag(5) | lk)
        lazy6, _, _ = run_device(ctx, datas, native.hc_level_flag(6) | lk)
        a, da, _ = run_device(ctx, datas, native.hc_level_flag(5) | lk | OPT)
        b, db, _ = run_device(ctx, datas, native.hc_level_flag(5) | lk | OPT)
        assert a == b and da == db
        r5, r6, ro = (raw / sum(map(len, f)) for f in (lazy5, lazy6, a))
        assert ro > r6 > r5, (lk, ro, r6, r5)
        assert ro / r5 >= 1.01, (lk, ro / r5)


DRIVER = r"""
import json, sys
from pathlib import Path
from skyplane_b200.harness import run_stream
base = Path(sys.argv[1]); n_req = int(sys.argv[2])
files = sorted((base / "pool").glob("*.bin"), key=lambda p: int(p.stem))
lens = [p.stat().st_size for p in files]
res = run_stream(base / "chunks", files, lens, n_req, n_workers=2, max_batch_chunks=8, max_batch_bytes=64 << 20, keep_frames=True,
                 compression_level=7, block_linked=True, optimal_parse=True)
print("RESULT " + json.dumps(res), flush=True)
"""


def test_operator_optimal_parse_writes_twin_frames():
    base = Path(tempfile.mkdtemp(prefix="skyb200_opt_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    try:
        (base / "pool").mkdir()
        pool = [text(8 << 20), synth.silesia_like_chunk(12, (1 << 20) + 55), synth.random_chunk(1, 1 << 20), b"", b"y" * 13]
        for k, d in enumerate(pool):
            (base / "pool" / f"{k}.bin").write_bytes(d)
        n_req = 15
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        r = subprocess.run([sys.executable, "-c", DRIVER, str(base), str(n_req)], capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        want = [twin(d, 7, LK) for d in pool]
        for rec in res["records"]:
            assert rec["md5"] == hashlib.md5(pool[rec["pool_index"]]).hexdigest()
            assert Path(rec["frame_path"]).read_bytes() == want[rec["pool_index"]]
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
