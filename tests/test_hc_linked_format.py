"""CPU tests of the high-ratio mode's linked blocks (SKY_F_HC | SKY_F_LINKED) on its sequential twin
(tools/lz4hc_model.c, hc_compress_block_linked), and of the flag's rules on the host side.  The twin's linked frames
decode with liblz4, pyarrow and the strict oracle, their header bytes are liblz4's own for the same preferences, their
matches do reach into the previous block and never beyond 65535 bytes, and with no window the twin is the independent one."""
import ctypes
import multiprocessing as mp
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.stage import ChunkStage
from test_linked_format import data_for, sequences, text, with_content_checksum

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

needs_liblz4 = pytest.mark.skipif(not ref.available(), reason="liblz4.so.1 not found")

LENS = [0, 1, 12, 13, 65535, 65536, 65537, 131089, (1 << 20) + 17]
CHECKSUMS = [(False, False), (False, True), (True, False), (True, True)]  # (block, content)


def linked_flg(n: int, bc: bool = False, ck: bool = False) -> int:
    return (0x60 if n == 0 else 0x68 if n <= 65536 else 0x48) | (0x10 if bc else 0) | (0x04 if ck else 0)


def twin_frame(data: bytes, level: int, bc: bool = False, ck: bool = False) -> bytes:
    f = hm.frame(data, hm.kernel_opts(level=level), block_checksum=bc, linked=True)
    return with_content_checksum(f, data) if ck else f


@needs_liblz4
@pytest.mark.parametrize("level", [3, 5, 9])
@pytest.mark.parametrize("n", LENS)
def test_linked_frames_decode(n, level):
    pa = pytest.importorskip("pyarrow")
    for kind in ("text", "silesia"):
        data = data_for(n, kind)
        for bc, ck in CHECKSUMS:
            f = twin_frame(data, level, bc, ck)
            assert f[4] == linked_flg(n, bc, ck)
            if not (bc or ck):  # (the strict oracle takes no checksums)
                assert oracle.lz4f_decode(f, n) == data
            assert ref.lz4f_decompress(f, n) == data
            if n:
                assert pa.decompress(f, decompressed_size=n, codec="lz4").to_pybytes() == data
            assert len(f) <= oracle.lz4f_bound(n) + 4 * ck + 4 * -(-n // 65536) * bc


def test_no_window_is_the_independent_block():
    """hist = 0 is hc_compress_block byte for byte, and so is a chunk's first block in a linked frame."""
    L = hm.lib()
    o = hm.kernel_opts(level=5)
    a, b = ctypes.create_string_buffer(65536 + 4096), ctypes.create_string_buffer(65536 + 4096)
    for n in (0, 5, 13, 4000, 65535, 65536):
        for blk in (text(n), synth.silesia_like_chunk(3, n), data_for(n, "random")):
            ca = L.hc_compress_block(blk, len(blk), a, ctypes.byref(o))
            src = ctypes.create_string_buffer(blk, len(blk) + 1)
            cb = L.hc_compress_block_linked(ctypes.addressof(src), len(blk), 0, b, ctypes.byref(o))
            assert ca == cb and a.raw[:ca] == b.raw[:cb]
    data = text(3 * 65536 + 100)
    assert hm.blocks(data, o, linked=True)[0] == hm.blocks(data, o)[0]


@needs_liblz4
def test_one_block_empty_and_stored_frames_equal_liblz4():
    """Empty and incompressible chunks (every block stored) give liblz4's linked frame byte for byte in every checksum
    combination; a chunk of one block gets liblz4's header for the same preferences -- the independent FLG -- and is the
    independent high-ratio frame."""
    for n in (0, 1, 13, 65536, 65537, 3 * 65536 + 5):
        data = data_for(n, "random")
        for bc, ck in CHECKSUMS:
            want = hm.liblz4_frame(data, 5, linked=True, content_checksum=ck, block_checksum=bc)
            assert twin_frame(data, 5, bc, ck) == want, (n, bc, ck)
    for n in (1, 13, 4000, 65536):
        data = text(n)
        for bc, ck in CHECKSUMS:
            ours = twin_frame(data, 5, bc, ck)
            hdr = 7 + 8
            assert ours[:hdr] == hm.liblz4_frame(data, 5, linked=True, content_checksum=ck, block_checksum=bc)[:hdr]
            indep = hm.frame(data, hm.kernel_opts(level=5), block_checksum=bc)
            assert ours == (with_content_checksum(indep, data) if ck else indep)


def test_matches_reach_into_the_previous_block():
    data = text(4 * 65536)
    for level in (3, 5, 9):
        across = 0
        for j, (c, b) in enumerate(hm.blocks(data, hm.kernel_opts(level=level), linked=True)):
            assert c, "text blocks compress"
            for pos, off in sequences(b):
                assert 1 <= off <= 65535
                if off > pos:
                    assert j > 0, "block 0 has no window to reach into"
                    across += 1
        assert across > 0, level


def test_blocks_depend_on_source_bytes_only():
    data = synth.silesia_like_chunk(21, 6 * 65536)
    o = hm.kernel_opts(level=5)
    full = hm.blocks(data, o, linked=True)
    for j in (1, 3, 5):
        assert hm.blocks(data[: (j + 1) * 65536], o, linked=True) == full[: j + 1]


def test_linked_ratio_on_the_study_set():
    """4 x 4 MiB Silesia-like chunks at level 5: linked frames are >= 1.04 x smaller than independent ones (1.045)."""
    o = hm.kernel_opts(level=5)
    indep = linked = 0
    for i in range(4):
        d = synth.silesia_like_chunk(10 + i, 4 << 20)
        indep += len(hm.frame(d, o))
        linked += len(hm.frame(d, o, linked=True))
    assert indep / linked >= 1.04, indep / linked


# ------------------------------------------------------------------ flag rules, no GPU
@pytest.mark.parametrize("base", [0, native.F_MD5, native.F_LZ4 | native.F_E2EE])
def test_decode_refuses_linked_by_name(base):
    with pytest.raises(ValueError, match="F_LINKED"):
        native.check_decode_flags(base | native.F_LINKED)
    ctx = object.__new__(native.Context)  # (the check comes before the library is touched)
    ctx._h = None
    with pytest.raises(ValueError, match="F_LINKED"):
        ctx.decode([0], [0], None, [0], base | native.F_LINKED)


@pytest.mark.parametrize("kw", [{}, {"level": 2}, {"level": 0}, {"compress": False}])
def test_linked_needs_the_high_ratio_mode(kw):
    stage = object.__new__(ChunkStage)  # (the check comes before the library is touched)
    with pytest.raises(ValueError, match="linked"):
        stage.launch(SimpleNamespace(lens=[100]), linked=True, **kw)
    with pytest.raises(ValueError, match="linked"):
        stage.process([b"x" * 100], linked=True, **kw)


def test_program_hands_block_linked_to_compress_hash(tmp_path):
    from skyplane_b200.operators import GatewayCompressHash
    from skyplane_b200.program import build_operator_graph

    def program(**fields):
        return [{"partitions": ["0"], "value": [{"op_type": "compress_hash", "handle": "c", "num_gpus": 1, **fields,
                                                 "children": [{"op_type": "write_local", "handle": "w", "children": []}]}]}]

    ev, eq = mp.Event(), mp.Queue()
    on = build_operator_graph(program(compression_level=5, block_linked=True), ChunkStore(tmp_path / "a"), "r", ev, eq)
    default = build_operator_graph(program(compression_level=5), ChunkStore(tmp_path / "b"), "r", ev, eq)
    on, default = on.operators["compress_hash_c"], default.operators["compress_hash_c"]
    assert isinstance(on, GatewayCompressHash) and on.block_linked is True and default.block_linked is False
    assert on.compression_level == default.compression_level == 5
    for fields in ({"block_linked": True}, {"block_linked": True, "compression_level": 1}, {"block_linked": True, "compress": False}):
        with pytest.raises(ValueError, match="block_linked"):
            build_operator_graph(program(**fields), ChunkStore(tmp_path / "c"), "r", ev, eq)
