"""CPU tests of the sequential twin's linked-block mode (tools/lz4_tile_model.c, tile_compress_block_linked): LZ4 frames
whose blocks after a chunk's first may match into the previous 64 KiB window (FLG B.Indep clear past one block).  Its frames decode with
liblz4, pyarrow and the strict oracle, its matches do reach across block starts, its header bytes are liblz4's own for the
same preferences, and every block is a function of the chunk's source bytes alone."""
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import synth

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model, tile_model  # noqa: E402

needs_liblz4 = pytest.mark.skipif(not ref.available(), reason="liblz4.so.1 not found")

LENS = [0, 1, 12, 13, 65535, 65536, 65537, 131071, 131072, 131073, (1 << 20) + 17]


def text(n: int) -> bytes:
    """Repetitive text whose repeats lie further apart than a block's start: lines drawn from a small vocabulary."""
    rng = np.random.default_rng(n)
    words = [b"chunk", b"frame", b"block", b"offset", b"window", b"literal", b"match", b"sequence", b"gateway", b"region"]
    out = bytearray()
    while len(out) < n:
        out += b" ".join(words[int(k)] for k in rng.integers(0, len(words), size=int(rng.integers(3, 9)))) + b";\n"
        out += rng.bytes(int(rng.integers(0, 24)))
    return bytes(out[:n])


def data_for(n: int, kind: str) -> bytes:
    if kind == "text":
        return text(n)
    if kind == "silesia":
        return synth.silesia_like_chunk(n % 97, n)
    return np.random.default_rng(n).bytes(n)


def sequences(block: bytes):
    """(position in the block, offset) of every match of one LZ4 block."""
    ip = op = 0
    out = []
    while ip < len(block):
        tok = block[ip]
        ip += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                b = block[ip]
                ip += 1
                ll += b
                if b != 255:
                    break
        ip += ll
        op += ll
        if ip >= len(block):
            break
        off = block[ip] | (block[ip + 1] << 8)
        ip += 2
        ml = tok & 15
        if ml == 15:
            while True:
                b = block[ip]
                ip += 1
                ml += b
                if b != 255:
                    break
        out.append((op, off))
        op += ml + 4
    return out


def with_content_checksum(frame: bytes, data: bytes) -> bytes:
    dlen = 10 if data else 2
    f = bytearray(frame)
    f[4] |= 0x04
    f[4 + dlen] = (oracle.xxh32(bytes(f[4 : 4 + dlen])) >> 8) & 0xFF
    return bytes(f) + oracle.xxh32(data).to_bytes(4, "little")


@needs_liblz4
@pytest.mark.parametrize("kind", ["text", "silesia", "random"])
@pytest.mark.parametrize("n", LENS)
def test_linked_frames_decode(n, kind):
    pa = pytest.importorskip("pyarrow")
    data = data_for(n, kind)
    for bc in (False, True):
        f = tile_model.frame(data, block_checksum=bc, linked=True)
        assert f[4] == (0x60 if n == 0 else 0x68 if n <= 65536 else 0x48) | (0x10 if bc else 0)
        if not bc:  # (the strict oracle takes no checksums)
            assert oracle.lz4f_decode(f, n) == data
        assert ref.lz4f_decompress(f, n) == data
        if n:
            assert pa.decompress(f, decompressed_size=n, codec="lz4").to_pybytes() == data
        assert len(f) <= oracle.lz4f_bound(n) + (4 * -(-n // 65536) if bc else 0)


def test_block_zero_is_the_independent_block():
    """A chunk's first block has no window: it is the independent block, byte for byte, and a one-block chunk's frame is
    the independent frame (FLG 0x68, as liblz4 writes it for one block whatever blockMode asks for)."""
    data = text(65536 + 4000)
    ind, lnk = tile_model.blocks(data, tile_model.kernel_opts()), tile_model.blocks(data, tile_model.kernel_opts(), linked=True)
    assert ind[0] == lnk[0]
    one = text(50000)
    assert tile_model.frame(one, linked=True) == tile_model.frame(one)
    assert tile_model.frame(data, linked=True)[4] == 0x48


def test_matches_reach_into_the_previous_block():
    """On text, blocks after the first take matches whose source lies before their own start (and never beyond the
    64 KiB window), and the linked frame is smaller than the independent one."""
    data = text(4 * 65536)
    blks = tile_model.blocks(data, tile_model.kernel_opts(), linked=True)
    across = 0
    for j, (c, b) in enumerate(blks):
        assert c, "text blocks compress"
        for pos, off in sequences(b):
            assert 1 <= off <= 65535
            if off > pos:
                assert j > 0, "block 0 has no window to reach into"
                across += 1
    assert across > 0
    assert len(tile_model.frame(data, linked=True)) < len(tile_model.frame(data))


def test_blocks_depend_on_source_bytes_only():
    """Block j of a linked chunk is a function of the chunk's bytes up to its own end: compressing the chunk cut after
    block j gives the same blocks 0..j, so blocks still compress in parallel."""
    data = synth.silesia_like_chunk(21, 6 * 65536)
    full = tile_model.blocks(data, tile_model.kernel_opts(), linked=True)
    for j in (1, 3, 5):
        assert tile_model.blocks(data[: (j + 1) * 65536], tile_model.kernel_opts(), linked=True) == full[: j + 1]


@needs_liblz4
def test_empty_and_stored_frames_equal_liblz4():
    """Empty chunks and incompressible ones (every block stored): the whole frame is liblz4's with blockMode = linked,
    byte for byte, for every combination of block and content checksums -- B.Indep clear only past one block."""
    for n in (0, 1, 13, 65536, 65537, 3 * 65536 + 5):
        data = data_for(n, "random")
        for bc in (False, True):
            for ck in (False, True):
                ours = tile_model.assemble(n, [(0, data[i : i + 65536]) for i in range(0, n, 65536)], block_checksum=bc, linked=True)
                if ck:
                    ours = with_content_checksum(ours, data)
                want = hc_model.liblz4_frame(data, 0, linked=True, content_checksum=ck, block_checksum=bc)
                assert ours == want, (n, bc, ck)
                assert ours[4] == (0x60 if n == 0 else 0x68 if n <= 65536 else 0x48) | (0x10 if bc else 0) | (0x04 if ck else 0)
                assert ref.lz4f_decompress(ours, n) == data


@needs_liblz4
def test_linked_ratio_on_text():
    """The window is worth it where repeats span blocks: a 40000-byte text repeated is stored about once with linked
    blocks, but once per block start with independent ones; on Silesia-like chunks linked frames are never larger."""
    t = text(40000) * 26
    assert len(tile_model.frame(t, linked=True)) * 2 <= len(tile_model.frame(t))
    s = synth.silesia_like_chunk(0, 2 << 20)
    assert len(tile_model.frame(s, linked=True)) <= len(tile_model.frame(s))
