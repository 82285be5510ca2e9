"""CPU tests of the high-ratio levels (SKY_F_HC_LEVEL, python-lz4's compression_level 3..9) that need no GPU: the header's
level field against native, the sequential twin's ratio and frames at every level, and the argument rules of
ChunkStage, GatewayCompressHash and the program loader."""
import multiprocessing as mp
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402

LEVELS = range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1)


def test_header_level_macro_equals_native(tmp_path):
    """SKY_F_HC_LEVEL(l) as a C compiler expands it, for every value the 4-bit field holds."""
    src = tmp_path / "levels.c"
    src.write_text('#include <stdio.h>\n#include "skychunk.h"\n'
                   'int main(void) { for (int l = 0; l < 16; l++) printf("%u\\n", (unsigned)SKY_F_HC_LEVEL(l)); return 0; }\n')
    exe = tmp_path / "levels"
    subprocess.check_call(["gcc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [native.F_HC | (l << native.HC_LEVEL_SHIFT) for l in range(16)]
    assert all(got[l] & native.HC_LEVEL_MASK == l << 8 for l in range(16))
    assert native.HC_LEVEL_MASK & (native.F_LZ4 | native.F_MD5 | native.F_E2EE | native.F_HC | native.F_CHECKSUM) == 0
    for l in LEVELS:
        assert native.hc_level_flag(l) == got[l]
    for bad in (0, 1, 2, 10, 15, True, 5.0):
        with pytest.raises(ValueError):
            native.hc_level_flag(bad)


def test_kernel_config_reads_levels():
    k = native.kernel_config()
    assert k["hc_max_level"] == native.HC_MAX_LEVEL == 9
    assert k["hc_depth"] == native.hc_depth(native.HC_DEFAULT_LEVEL) == 16  # the default level's depth, as before levels
    assert [native.hc_depth(l) for l in LEVELS] == [4, 8, 16, 32, 64, 128, 256]
    assert [hm.kernel_opts(level=l).depth for l in LEVELS] == [4, 8, 16, 32, 64, 128, 256]
    assert hm.kernel_opts(level=5).depth == hm.kernel_opts().depth
    with pytest.raises(ValueError):
        hm.kernel_opts(level=10)


@pytest.mark.skipif(not ref.available(), reason="liblz4.so.1 not found")
def test_twin_ratio_rises_with_level_and_frames_decode():
    """2 x 1 MiB Silesia-like: every level's frames decode with the strict oracle and liblz4, and each level is strictly
    smaller than the one below."""
    datas = [synth.silesia_like_chunk(10 + i, 1 << 20) for i in range(2)] + [b"", b"abc", bytes(70000)]
    raw = sum(map(len, datas))
    ratios = []
    for l in LEVELS:
        frames = [hm.frame(d, hm.kernel_opts(level=l)) for d in datas]
        for d, f in zip(datas, frames):
            assert oracle.lz4f_decode(f, len(d)) == d
            assert ref.lz4f_decompress(f, len(d)) == d
            assert len(f) <= native.frame_bound(len(d))
        ratios.append(raw / sum(map(len, frames)))
    assert all(a < b for a, b in zip(ratios, ratios[1:])), ratios
    assert hm.frame(datas[0], hm.kernel_opts(level=5)) == hm.frame(datas[0])


def test_hc_flags_follow_python_lz4_levels():
    F = native.hc_flags
    assert F() == 0 and F(hc=True) == native.F_HC  # no level: today's flags
    for l in LEVELS:
        assert F(l) == F(l, hc=True) == native.hc_level_flag(l)
    for l in (0, 1, 2):
        assert F(l) == 0  # python-lz4's fast levels: the fast compressor
        with pytest.raises(ValueError):
            F(l, hc=True)
    for bad in (-1, 10, 12, 16):
        with pytest.raises(ValueError):
            F(bad)
    for l in (0, 3, 9):
        with pytest.raises(ValueError):
            F(l, compress=False)
    for bad in (True, 5.0, "5"):
        with pytest.raises(ValueError):
            F(bad)
    assert F(None, compress=False) == 0


class _Ctx:
    def __init__(self):
        self.flags = []

    def submit(self, src, lens, dst, caps, flags, nonces):
        self.flags.append(flags)
        return len(self.flags)


def _stage_and_slot():
    """A ChunkStage whose context only records what launch() submits (no device)."""
    stage = ChunkStage.__new__(ChunkStage)
    stage.ctx = _Ctx()
    slot = SimpleNamespace(lens=[1000], in_off=[0], out_off=[0], inp=SimpleNamespace(addr=1 << 20), out=SimpleNamespace(addr=2 << 20),
                           flags=0, ticket=None)
    return stage, slot


def test_chunkstage_launch_level_flags():
    stage, slot = _stage_and_slot()
    base = native.F_MD5 | native.F_LZ4
    stage.launch(slot)
    stage.launch(slot, hc=True)
    stage.launch(slot, level=9)
    stage.launch(slot, hc=True, level=3, checksum=True)
    stage.launch(slot, level=1)
    assert stage.ctx.flags == [base, base | native.F_HC, base | native.hc_level_flag(9),
                               base | native.hc_level_flag(3) | native.F_CHECKSUM, base]
    assert slot.flags == base
    for kw in ({"level": 10}, {"level": -1}, {"level": 2, "hc": True}, {"level": 5, "compress": False}, {"level": 0, "compress": False}):
        with pytest.raises(ValueError):
            stage.launch(slot, **kw)
    with pytest.raises(ValueError):
        stage.process([b"x" * 100], level=12)
    assert len(stage.ctx.flags) == 5


def _operator(tmp_path, **kw):
    return GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), ChunkStore(tmp_path), **kw)


def test_gateway_compress_hash_levels(tmp_path):
    assert _operator(tmp_path).compression_level is None
    assert _operator(tmp_path, compression_level=9).compression_level == 9
    assert _operator(tmp_path, compression_level=4, high_ratio=True).compression_level == 4
    assert _operator(tmp_path, compression_level=0).compression_level == 0
    for kw in ({"compression_level": 10}, {"compression_level": -1}, {"compression_level": 2, "high_ratio": True},
               {"compression_level": 9, "use_compression": False}, {"compression_level": "9"}):
        with pytest.raises(ValueError):
            _operator(tmp_path, **kw)


def test_program_json_compression_level(tmp_path):
    from skyplane_b200.program import build_operator_graph

    def graph(**fields):
        prog = [{"partitions": ["0"], "value": [{"op_type": "compress_hash", "handle": "a", "num_gpus": 1, "children": [], **fields}]}]
        return build_operator_graph(prog, ChunkStore(tmp_path), "r", mp.Event(), mp.Queue()).operators["compress_hash_a"]

    assert graph().compression_level is None and not graph().high_ratio
    op = graph(high_ratio=True)
    assert op.high_ratio and op.compression_level is None  # level 5
    op = graph(compression_level=7, content_checksum=True)
    assert op.compression_level == 7 and op.content_checksum
    for fields in ({"compression_level": 11}, {"compression_level": 1, "high_ratio": True}, {"compression_level": 5, "compress": False}):
        with pytest.raises(ValueError):
            graph(**fields)
