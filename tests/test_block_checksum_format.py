"""CPU tests of SKY_F_BLOCK_CHECKSUM (LZ4's block checksums, XXH32 per block) that need no GPU: the sequential twins'
frames with block checksums against liblz4's own frames for the same preferences, the header's flag against native, the
staging room, and the argument rules of ChunkStage, GatewayCompressHash and the program loader."""
import multiprocessing as mp
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash
from skyplane_b200.stage import ChunkStage, _out_room

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model, tile_model  # noqa: E402

needs_liblz4 = pytest.mark.skipif(not ref.available(), reason="liblz4.so.1 not found")


def incompressible(n: int) -> bytes:
    return np.random.default_rng(n).bytes(n)


def stored(data: bytes):
    return [(0, data[i : i + 65536]) for i in range(0, len(data), 65536)]


def with_content_checksum(frame: bytes, data: bytes) -> bytes:
    dlen = 10 if data else 2
    f = bytearray(frame)
    f[4] |= 0x04
    f[4 + dlen] = (oracle.xxh32(bytes(f[4 : 4 + dlen])) >> 8) & 0xFF
    return bytes(f) + oracle.xxh32(data).to_bytes(4, "little")


@needs_liblz4
@pytest.mark.parametrize("ck", [False, True])
@pytest.mark.parametrize("n", [0, 1, 12, 13, 65535, 65536, 65537, 3 * 65536 + 5])
def test_stored_frames_equal_liblz4(n, ck):
    """Incompressible and empty chunks (every block stored): the whole frame is liblz4's with blockChecksumFlag = 1 (and
    contentChecksumFlag), byte for byte."""
    data = incompressible(n)
    ours = tile_model.assemble(n, stored(data), block_checksum=True)
    if ck:
        ours = with_content_checksum(ours, data)
    assert ours == hc_model.liblz4_frame(data, 0, content_checksum=ck, block_checksum=True)
    assert len(ours) == native.frame_need(n, ck, True)  # a stored frame takes all of it
    assert ref.lz4f_decompress(ours, n) == data


@needs_liblz4
def test_header_bytes_at_every_flg():
    """FLG and the header checksum byte for every combination of block / content checksum, empty or not."""
    for n in (0, 1000):
        data = incompressible(n)
        for bc in (False, True):
            for ck in (False, True):
                want = hc_model.liblz4_frame(data, 0, content_checksum=ck, block_checksum=bc)
                ours = tile_model.assemble(n, stored(data), block_checksum=bc)
                if ck:
                    ours = with_content_checksum(ours, data)
                hdr = 7 if n == 0 else 15
                assert ours[:hdr] == want[:hdr]
                assert ours[4] == (0x60 if n == 0 else 0x68) | (0x10 if bc else 0) | (0x04 if ck else 0)


@needs_liblz4
@pytest.mark.parametrize("level", [None, 3, 5, 9])
def test_twin_frames_decode_with_liblz4_and_pyarrow(level):
    pa = pytest.importorskip("pyarrow")
    text = (b"it was the best of times, it was the worst of times; " * 4000)[:150000] + incompressible(70000)
    f = (tile_model.frame(text, block_checksum=True) if level is None
         else hc_model.frame(text, hc_model.kernel_opts(level=level), block_checksum=True))
    plain = tile_model.frame(text) if level is None else hc_model.frame(text, hc_model.kernel_opts(level=level))
    assert len(f) == len(plain) + 4 * 4 and f[4] == 0x78
    assert ref.lz4f_decompress(f, len(text)) == text
    assert pa.decompress(f, decompressed_size=len(text), codec="lz4").to_pybytes() == text
    bad = bytearray(f)
    bad[15 + 4 + 10] ^= 1  # a byte of block 0's data
    with pytest.raises(ValueError):
        ref.lz4f_decompress(bytes(bad), len(text))


def test_header_flag_equals_native(tmp_path):
    src = tmp_path / "bc.c"
    src.write_text('#include <stdio.h>\n#include "skychunk.h"\n'
                   'int main(void) { printf("%u %u\\n", (unsigned)SKY_F_BLOCK_CHECKSUM, (unsigned)SKY_F_CHECKSUM); return 0; }\n')
    exe = tmp_path / "bc"
    subprocess.check_call(["gcc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    bc, ck = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert bc == native.F_BLOCK_CHECKSUM == 128 and ck == native.F_CHECKSUM
    others = native.F_LZ4 | native.F_MD5 | native.F_E2EE | native.F_HC | native.F_CHECKSUM | native.HC_LEVEL_MASK
    assert bc & others == 0


def test_frame_need_and_staging_room():
    for n in (0, 1, 65535, 65536, 65537, 8 << 20):
        nblk = -(-n // 65536)
        assert native.frame_need(n) == native.frame_bound(n)
        assert native.frame_need(n, checksum=True) == native.frame_bound(n) + 4
        assert native.frame_need(n, block_checksum=True) == native.frame_bound(n) + 4 * nblk
        assert native.frame_need(n, True, True) == native.frame_bound(n) + 4 + 4 * nblk
        assert _out_room(n) == native.round16(native.frame_need(n, True, True) + native.BOX_OVERHEAD)


def test_staging_slots_hold_every_batch_they_held_before():
    """The out slab grows by what block checksums can take: for chunk sizes that fill a slot, the count that fits is what
    fitted with the parent's room (frame_bound + content checksum + box, out slab without the block-checksum growth)."""
    for mb, mc in ((64 << 20, 64), (8 << 20, 256), (1 << 20, 16)):
        in_bytes = native.round16(mb) + 16 * mc
        old_out = mb + 4 * (mb // 65536 + 1) + 128 * mc
        new_out = old_out + 4 * (in_bytes // 65536 + 1) + 16 * mc
        for n in (1, 13, 65536, 65537, 100000, 1 << 20, mb // 3, mb):
            old_room = native.round16(native.frame_bound(n) + 4 + native.BOX_OVERHEAD)
            k_old = min(mc, in_bytes // native.round16(n) if n else mc, old_out // old_room)
            assert k_old * _out_room(n) <= new_out, (mb, mc, n, k_old)


class _Ctx:
    def __init__(self):
        self.calls = []

    def submit(self, src, lens, dst, caps, flags, nonces):
        self.calls.append((flags, caps))
        return len(self.calls)


def _stage_and_slot():
    stage = ChunkStage.__new__(ChunkStage)
    stage.ctx = _Ctx()
    slot = SimpleNamespace(lens=[200000], in_off=[0], out_off=[0], inp=SimpleNamespace(addr=1 << 20), out=SimpleNamespace(addr=2 << 24),
                           flags=0, ticket=None)
    return stage, slot


def test_chunkstage_launch_block_checksum():
    stage, slot = _stage_and_slot()
    base = native.F_MD5 | native.F_LZ4
    stage.launch(slot, block_checksum=True)
    stage.launch(slot, block_checksum=True, checksum=True, level=9, encrypt=True, nonces=bytes(24))
    stage.launch(slot)
    (f0, c0), (f1, c1), (f2, c2) = stage.ctx.calls
    assert f0 == base | native.F_BLOCK_CHECKSUM and c0 == [native.frame_bound(200000) + 16]
    assert f1 == base | native.F_BLOCK_CHECKSUM | native.F_CHECKSUM | native.hc_level_flag(9) | native.F_E2EE
    assert c1 == [native.frame_bound(200000) + 20 + native.BOX_OVERHEAD]
    assert f2 == base and c2 == [native.frame_bound(200000)]
    with pytest.raises(ValueError):
        stage.launch(slot, block_checksum=True, compress=False)
    with pytest.raises(ValueError):
        stage.process([b"x" * 100], block_checksum=True, compress=False)
    assert len(stage.ctx.calls) == 3


def _operator(tmp_path, **kw):
    return GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), ChunkStore(tmp_path), **kw)


def test_gateway_compress_hash_block_checksum(tmp_path):
    assert not _operator(tmp_path).block_checksum
    assert _operator(tmp_path, block_checksum=True).block_checksum
    op = _operator(tmp_path, block_checksum=True, content_checksum=True, compression_level=5)
    assert op.block_checksum and op.content_checksum
    with pytest.raises(ValueError):
        _operator(tmp_path, block_checksum=True, use_compression=False)


def test_program_json_block_checksum(tmp_path):
    from skyplane_b200.program import build_operator_graph

    def graph(**fields):
        prog = [{"partitions": ["0"], "value": [{"op_type": "compress_hash", "handle": "a", "num_gpus": 1, "children": [], **fields}]}]
        return build_operator_graph(prog, ChunkStore(tmp_path), "r", mp.Event(), mp.Queue()).operators["compress_hash_a"]

    assert not graph().block_checksum
    op = graph(block_checksum=True, high_ratio=True)
    assert op.block_checksum and op.high_ratio
    with pytest.raises(ValueError):
        graph(block_checksum=True, compress=False)
