"""CPU tests of the high-ratio mode's optimal parse (SKY_F_HC | SKY_F_OPTIMAL) on its sequential twin (tools/lz4hc_model.c,
hc_compress_block_opt), and of the flag's rules on the host side.  The twin's frames decode with liblz4, pyarrow and the
strict oracle at the HC tests' edge lengths, levels and checksum combinations, independent and linked; no match crosses a
parse segment's end; with one segment per block the parse is the cheapest one an exhaustive search finds among the same
candidates; the study set gains >= 1 % over the lazy parse."""
import ctypes
import multiprocessing as mp
import sys
from functools import lru_cache
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import lz4_craft as C
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

LENS = [0, 1, 12, 13, 2047, 2048, 2049, 65535, 65536, 65537, 131089, (1 << 20) + 17]
CHECKSUMS = [(False, False), (False, True), (True, False), (True, True)]  # (block, content)


def twin_frame(data: bytes, level: int, linked: bool, bc: bool = False, ck: bool = False, seg: int = hm.OPT_SEG) -> bytes:
    f = hm.frame(data, hm.kernel_opts(level=level), block_checksum=bc, linked=linked, optimal=True, seg=seg)
    return with_content_checksum(f, data) if ck else f


@needs_liblz4
@pytest.mark.parametrize("linked", [False, True])
@pytest.mark.parametrize("level", [3, 5, 9])
@pytest.mark.parametrize("n", LENS)
def test_optimal_frames_decode(n, level, linked):
    pa = pytest.importorskip("pyarrow")
    for kind in ("text", "silesia"):
        data = data_for(n, kind)
        for bc, ck in CHECKSUMS:
            f = twin_frame(data, level, linked, bc, ck)
            if not (bc or ck):  # (the strict oracle takes no checksums)
                assert oracle.lz4f_decode(f, n) == data
            assert ref.lz4f_decompress(f, n) == data
            if n:
                assert pa.decompress(f, decompressed_size=n, codec="lz4").to_pybytes() == data
            assert len(f) <= oracle.lz4f_bound(n) + 4 * ck + 4 * -(-n // 65536) * bc


@needs_liblz4
@pytest.mark.parametrize("seg", [0, 1024, hm.OPT_SEG, 8192])
def test_segment_sizes_give_valid_frames_and_no_match_crosses_a_segment(seg):
    data = text(300000) + synth.silesia_like_chunk(5, 300000) + bytes(70000) + text(9000) * 3
    for linked in (False, True):
        f = twin_frame(data, 5, linked, seg=seg)
        assert ref.lz4f_decompress(f, len(data)) == data
        for c, b in hm.blocks(data, hm.kernel_opts(level=5), linked, optimal=True, seg=seg):
            if not c:
                continue
            ms, _ = C.walk_block(b)
            assert [(pos, off) for pos, off, _ in ms] == sequences(b)
            for pos, _, ml in ms:
                assert pos + ml <= 65536
                if seg:
                    assert pos // seg == (pos + ml - 1) // seg, (seg, pos, ml)


def test_whole_block_segment_is_the_cheapest_parse():
    """seg = 0 (one segment per block): on small blocks the twin's block is the cheapest among every parse of the same
    candidates -- literals, and lengths 4 .. blen(p) at boff(p) that do not pass a long position, where the long match is
    taken as the lazy parse extends it -- found by an exhaustive search over (position, literal run) with exact sequence costs.  The twin keeps one
    literal run per position (liblz4's carried run), so it may lose a length byte where two runs tie; on these blocks it
    never does."""
    rng = np.random.default_rng(7)
    o = hm.kernel_opts(level=5)
    buf = ctypes.create_string_buffer(65536 + 4096)
    checked = 0
    for t in range(60):
        n = int(rng.integers(13, 600))
        alpha = int(rng.integers(2, 6))
        words = [bytes(rng.integers(97, 97 + alpha, int(rng.integers(3, 12)), dtype=np.uint8)) for _ in range(6)]
        data = b"".join(words[int(rng.integers(0, 6))] for _ in range(n))[:n]
        if t % 3 == 0:
            data = bytes(rng.integers(0, alpha, n, dtype=np.uint8))
        src = ctypes.create_string_buffer(data, len(data) + 1)
        c = hm.lib().hc_compress_block_opt(ctypes.addressof(src), len(data), 0, 0, buf, ctypes.byref(o))
        blen, boff = _search(data, o)
        best = _exhaustive(data, blen, boff, o.nice)
        if c:
            assert c == best, (t, n, c, best)
            checked += 1
        else:
            assert best > len(data) - 1
    assert checked >= 40


def _search(data: bytes, o):
    """The twin's search: sequential hash chains, nearest first, longest common prefix up to min(nice, matchlimit - p)."""
    L = len(data)
    mflimit, matchlimit = L - 12, L - 5
    head, chain = {}, {}
    blen, boff = [0] * (L + 1), [0] * (L + 1)
    for p in range(mflimit + 1):
        h = (int.from_bytes(data[p : p + 4], "little") * 2654435761 & 0xFFFFFFFF) >> (32 - o.hash_bits)
        chain[p] = head.get(h)
        head[h] = p
    for p in range(mflimit + 1):
        cap = min(o.nice, matchlimit - p)
        best = bo = 0
        c, k = chain[p], 0
        while k < o.depth and c is not None:
            ln = 0
            while ln < cap and data[p + ln] == data[c + ln]:
                ln += 1
            if ln > best:
                best, bo = ln, p - c
            if best == cap:
                break
            c, k = chain[c], k + 1
        if best >= 4:
            blen[p], boff[p] = best, bo
    return blen, boff


def _ext(x: int) -> int:
    return 1 + (x - 15) // 255 if x >= 15 else 0


def _exhaustive(data: bytes, blen, boff, nice: int) -> int:
    """Least block size over every parse with the twin's candidates and long-position rule, by exact costs."""
    L = len(data)
    mflimit, matchlimit = L - 12, L - 5
    sys.setrecursionlimit(100000)

    def long_len(p):
        ml = nice
        while p + ml < matchlimit and data[p + ml] == data[p - boff[p] + ml]:
            ml += 1
        return ml

    next_long = [L] * (L + 2)  # the first long position at or after p
    for p in range(L - 1, -1, -1):
        next_long[p] = p if p <= mflimit and blen[p] == nice and L - p >= nice else next_long[p + 1]

    @lru_cache(maxsize=None)
    def best(p: int, run: int) -> int:
        """bytes of everything from p on, with `run` literals open before p"""
        if p == L or p > mflimit:
            ll = run + L - p
            return 1 + _ext(ll) + ll
        if blen[p] == nice and L - p >= nice:  # a long position: its extended match is taken
            ml = long_len(p)
            return 1 + _ext(run) + run + 2 + _ext(ml - 4) + best(p + ml, 0)
        out = best(p + 1, run + 1)
        for ml in range(4, min(blen[p], next_long[p + 1] - p) + 1):  # (no match skips a long position)
            out = min(out, 1 + _ext(run) + run + 2 + _ext(ml - 4) + best(p + ml, 0))
        return out

    return best(0, 0)


def test_optimal_ratio_on_the_study_set():
    """4 x 4 MiB Silesia-like chunks at level 5: the optimal parse sends >= 1.010 x fewer bytes than the lazy parse,
    independent (1.016 x) and linked (1.021 x)."""
    o = hm.kernel_opts(level=5)
    for linked in (False, True):
        lazy = opt = 0
        for i in range(4):
            d = synth.silesia_like_chunk(10 + i, 4 << 20)
            lazy += len(hm.frame(d, o, linked=linked))
            opt += len(hm.frame(d, o, linked=linked, optimal=True))
        assert lazy / opt >= 1.010, (linked, lazy / opt)


# ------------------------------------------------------------------ flag rules, no GPU
def test_flag_bit_is_its_own():
    others = (native.F_LZ4 | native.F_MD5 | native.F_E2EE | native.F_HC | native.F_CHECKSUM | native.F_BLOCK_CHECKSUM
              | native.HC_LEVEL_MASK | native.F_VERIFY | native.F_LINKED)
    assert native.F_OPTIMAL == 16384 and not native.F_OPTIMAL & others
    header = (ROOT / "include" / "skychunk.h").read_text()
    assert "#define SKY_F_OPTIMAL 16384u" in header


@pytest.mark.parametrize("base", [0, native.F_MD5, native.F_LZ4 | native.F_E2EE])
def test_decode_refuses_optimal_by_name(base):
    with pytest.raises(ValueError, match="F_OPTIMAL"):
        native.check_decode_flags(base | native.F_OPTIMAL)
    ctx = object.__new__(native.Context)  # (the check comes before the library is touched)
    ctx._h = None
    with pytest.raises(ValueError, match="F_OPTIMAL"):
        ctx.decode([0], [0], None, [0], base | native.F_OPTIMAL)


@pytest.mark.parametrize("kw", [{}, {"level": 2}, {"level": 0}, {"compress": False}, {"linked": True}])
def test_optimal_needs_the_high_ratio_mode(kw):
    stage = object.__new__(ChunkStage)  # (the check comes before the library is touched)
    with pytest.raises(ValueError, match="optimal|linked"):
        stage.launch(SimpleNamespace(lens=[100]), optimal=True, **kw)
    with pytest.raises(ValueError, match="optimal|linked"):
        stage.process([b"x" * 100], optimal=True, **kw)


def test_program_hands_optimal_parse_to_compress_hash(tmp_path):
    from skyplane_b200.operators import GatewayCompressHash
    from skyplane_b200.program import build_operator_graph

    def program(**fields):
        return [{"partitions": ["0"], "value": [{"op_type": "compress_hash", "handle": "c", "num_gpus": 1, **fields,
                                                 "children": [{"op_type": "write_local", "handle": "w", "children": []}]}]}]

    ev, eq = mp.Event(), mp.Queue()
    on = build_operator_graph(program(compression_level=7, optimal_parse=True), ChunkStore(tmp_path / "a"), "r", ev, eq)
    default = build_operator_graph(program(compression_level=7), ChunkStore(tmp_path / "b"), "r", ev, eq)
    on, default = on.operators["compress_hash_c"], default.operators["compress_hash_c"]
    assert isinstance(on, GatewayCompressHash) and on.optimal_parse is True and default.optimal_parse is False
    for fields in ({"optimal_parse": True}, {"optimal_parse": True, "compression_level": 1}, {"optimal_parse": True, "compress": False}):
        with pytest.raises(ValueError, match="optimal_parse"):
            build_operator_graph(program(**fields), ChunkStore(tmp_path / "c"), "r", ev, eq)
