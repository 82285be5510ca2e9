"""GPU tests of the high-ratio mode's linked blocks (SKY_F_HC | SKY_F_LINKED, python-lz4's block_linked) through the C ABI,
ChunkStage and the gateway operators.

Bars: at every level 3..9 the frames are byte-identical to the linked twin (tools/lz4hc_model.c, hc_compress_block_linked)
on a ragged batch of edge lengths, 8 MiB Silesia-like and text-like chunks, with and without block and content checksums;
MD5 bit-exact; liblz4 and sky_decode restore every chunk; SKY_F_VERIFY passes clean linked frames unchanged (its status
table, mutants and repair on linked frames are in test_gpu_verify.py); E2EE boxes seal the twin frame; the flag's
refusals; run-to-run determinism; GatewayCompressHash(compression_level=5, block_linked=True) into GatewayDecompressVerify."""
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
from test_gpu_hc_levels import run_device
from test_linked_format import text, with_content_checksum

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

LK, BC, CK = native.F_LINKED, native.F_BLOCK_CHECKSUM, native.F_CHECKSUM
KEY = bytes((13 * i + 7) & 0xFF for i in range(32))
EDGE = [0, 1, 12, 13, 65535, 65536, 65537, 131089, (1 << 20) + 17]
# the checksum flags each level runs with: every combination, at more than one level
LEVEL_CHECKSUMS = {3: 0, 4: BC, 5: CK, 6: BC | CK, 7: 0, 8: BC, 9: BC | CK}


def twin_opts(level):
    k = native.kernel_config()
    return hm.Opts(native.hc_depth(level), k["hc_hash_bits"], k["hc_nice"])


def twin(data: bytes, level: int, flags: int = 0) -> bytes:
    f = hm.frame(data, twin_opts(level), block_checksum=bool(flags & BC), linked=True)
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
    s = ChunkStage(0, max_batch_bytes=96 << 20, max_chunks=64, n_slots=2)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


@pytest.fixture(scope="module")
def datas():
    out = [text(n) for n in EDGE] + [synth.silesia_like_chunk(n % 97, n) for n in EDGE[3:]]
    out += [synth.silesia_like_chunk(80, 8 << 20), text(8 << 20), synth.random_chunk(3, 200000)]
    return out


@pytest.mark.parametrize("level", sorted(LEVEL_CHECKSUMS))
def test_frames_equal_linked_twin_at_every_level(ctx, stage, datas, level):
    ck = LEVEL_CHECKSUMS[level]
    flags = native.hc_level_flag(level) | LK | ck
    frames, digests, lens = run_device(ctx, datas, flags, extra(datas, ck))
    for i, (d, f, dg, ln) in enumerate(zip(datas, frames, digests, lens)):
        want = twin(d, level, ck)
        assert f == want, f"level {level} chunk {i} (len {len(d)}): GPU frame {len(f)} B != twin {len(want)} B"
        assert ln == len(f) and dg == hashlib.md5(d).digest()
        assert f[4] == (0x60 if not d else 0x68 if len(d) <= 65536 else 0x48) | (0x10 if ck & BC else 0) | (0x04 if ck & CK else 0)
        assert ref.lz4f_decompress(f, len(d)) == d
    out = stage.decode(frames, [len(d) for d in datas])
    for d, (data, dg, st) in zip(datas, out):
        assert st == 0 and data == d and dg == hashlib.md5(d).digest()


def test_linked_frames_are_smaller_on_text_and_deterministic(ctx):
    datas = [text(4 << 20), synth.silesia_like_chunk(81, 8 << 20)]
    indep, _, _ = run_device(ctx, datas, native.hc_level_flag(5))
    a, da, _ = run_device(ctx, datas, native.hc_level_flag(5) | LK)
    b, db, _ = run_device(ctx, datas, native.hc_level_flag(5) | LK)
    assert a == b and da == db
    assert len(a[0]) < len(indep[0]) and len(a[1]) <= len(indep[1])
    for d, f in zip(datas, a):
        assert oracle.lz4f_decode(f, len(d)) == d


def test_verify_passes_clean_linked_frames(stage, datas):
    """SKY_F_VERIFY on linked batches: every status 0, frames and digests as without the check."""
    for level, ck in ((3, 0), (9, BC | CK)):
        kw = dict(level=level, linked=True, checksum=bool(ck & CK), block_checksum=bool(ck & BC))
        plain = stage.process(datas, **kw)
        checked = stage.process(datas, verify=True, **kw)
        for d, p, c in zip(datas, plain, checked):
            assert c.verify_status == 0 and bytes(c.frame) == bytes(p.frame) == twin(d, level, ck) and c.md5 == p.md5


def test_e2ee_boxes_seal_the_linked_twin_frame(stage):
    nacl_secret = pytest.importorskip("nacl.secret")
    datas = [text(300000), synth.silesia_like_chunk(61, 700001), synth.random_chunk(4, 70000), b"", b"tiny"]
    nonces = bytes((5 * i + 2) & 0xFF for i in range(24 * len(datas)))
    res = stage.process(datas, encrypt=True, nonces=nonces, level=7, linked=True)
    box = nacl_secret.SecretBox(KEY)
    for i, (d, r) in enumerate(zip(datas, res)):
        frame = box.decrypt(bytes(r.frame))
        assert frame == twin(d, 7) and bytes(r.frame)[:24] == nonces[24 * i : 24 * i + 24]
        assert ref.lz4f_decompress(frame, len(d)) == d and r.md5 == hashlib.md5(d).digest()


def test_linked_flag_errors(ctx, stage):
    datas = [text(200000), b"abc" * 100]
    stages = native.F_LZ4 | native.F_MD5
    bad = [LK, LK | stages, LK | native.F_LZ4, LK | native.F_MD5, LK | native.F_CHECKSUM, native.F_HC | LK | native.F_MD5,
           native.hc_level_flag(5) | LK | native.F_MD5]
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
    frames, _, _ = run_device(ctx, datas, native.hc_level_flag(5) | LK)
    with pytest.raises(ValueError, match="F_LINKED"):
        stage.ctx.decode([0], [len(frames[0])], None, [len(datas[0])], LK)
    for base in (0, native.F_LZ4, native.F_MD5 | native.F_E2EE):  # the library refuses the bit before it reads anything
        assert native.lib().sky_decode(stage.ctx._h, 1, None, None, None, None, base | LK, None, None, None) == native.SKY_E_INVALID
    # the context is still good after every refusal
    assert frames == [twin(d, 5) for d in datas]


DRIVER = r"""
import json, multiprocessing as mp, sys, time
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
                 compression_level=5, block_linked=True)
print("RESULT " + json.dumps(res), flush=True)
store = ChunkStore(base / "dst")
qin, qout = GatewayQueue(), GatewayQueue()
ev, eq = mp.Event(), mp.Queue()
op = GatewayDecompressVerify("decompress_verify", "local:box", qin, qout, ev, eq, store, n_processes=1)
op.start_workers()
recv = {}
try:
    for k, rec in enumerate(res["records"][:6]):
        cid = f"{k:032x}"
        store.get_compressed_file_path(cid).write_bytes(Path(rec["frame_path"]).read_bytes())
        qin.put(ChunkRequest(Chunk(f"obj/{k}", f"obj/{k}", cid, lens[rec["pool_index"]], partition_id="0", md5_hash=bytes.fromhex(rec["md5"]))))
    done, deadline = 0, time.time() + 300
    while done < 6 and time.time() < deadline and not ev.is_set():
        done += len(qout.get_batch_nowait(16))
        time.sleep(0.01)
    recv["done"] = done
    recv["restored"] = [store.get_chunk_file_path(f"{k:032x}").read_bytes() == files[rec["pool_index"]].read_bytes()
                        for k, rec in enumerate(res["records"][:6])]
    recv["error"] = eq.get(timeout=1) if ev.is_set() else None
finally:
    op.stop_workers()
print("RECV " + json.dumps(recv), flush=True)
"""


def test_operator_block_linked_into_decompress_verify():
    base = Path(tempfile.mkdtemp(prefix="skyb200_lk_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
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
        recv = json.loads([l for l in r.stdout.splitlines() if l.startswith("RECV ")][-1][len("RECV "):])
        assert len(res["records"]) == n_req and res["status"].get("complete") == n_req
        want = [twin(d, 5) for d in pool]
        for rec in res["records"]:
            assert rec["md5"] == hashlib.md5(pool[rec["pool_index"]]).hexdigest()
            assert Path(rec["frame_path"]).read_bytes() == want[rec["pool_index"]]
        assert want[0][4] == 0x48
        assert recv["done"] == 6 and all(recv["restored"]) and recv["error"] is None, recv
    finally:
        import shutil

        shutil.rmtree(base, ignore_errors=True)
