"""The receiver tests' frame corpus (tests/lz4_craft.py), checked on the CPU before any GPU sees it: generated streams
decode to the generator's bytes with the strict oracle, conforming ones with liblz4 (and pyarrow where installed),
lenient ones are rejected by liblz4 where they break an end-of-block rule, each targeted mutator does what the
receiver tests' tables assume, and the block-rule walker (conforms) passes every frame liblz4 and the twins make and
refuses the short-block and offset-0 frames liblz4 still decodes."""
import random
import struct

import pytest

import lz4_craft as C
import oracle
import oracle.reflib as ref

SIZES = [0, 1, 4, 5, 12, 13, 100, 4096, 65535, 65536, 65537, 131072, 200001]


def _streams(conforming: bool):
    rng = random.Random(1 if conforming else 2)
    for size in SIZES:
        for linked in (False, True):
            yield C.gen_stream(rng, size, linked=linked, conforming=conforming)


def test_block_assembler_writes_tokens_extensions_and_offsets():
    lit = bytes(range(15))
    b = C.encode_block([(lit, 1, 19), (b"", 0x0114, 4 + 270)], b"z" * 270)
    assert b.data[:2] == bytes([0xFF, 0]) and b.data[2:17] == lit and b.data[17:19] == b"\x01\x00" and b.data[19] == 0
    assert b.data[20] == 0x0F and b.data[21:23] == b"\x14\x01" and b.data[23:25] == bytes([255, 0])
    assert b.data[25] == 0xF0 and b.data[26:28] == bytes([255, 0]) and b.data[28:] == b"z" * 270
    assert b.marks == {"token": [0, 20, 25], "ext": [1, 19, 23, 24, 26, 27], "offset": [17, 21]}
    w = C.BlockWriter(bytearray())  # the same two matches with enough history for offset 0x114, decoded by the oracle
    w.literals(lit).match(1, 19).literals(bytes(300)).match(0x0114, 274).literals(b"z" * 270)
    blk = w.close()
    assert blk.data[: 20] == b.data[:20]
    assert oracle.lz4f_decode(C.assemble_frame([blk], bytes(w.buf)).data, 2000) == bytes(w.buf)


def test_frame_header_matches_liblz4():
    data = bytes(range(256)) * 300
    theirs = ref.lz4f_compress(data)  # linked blocks, content size on
    hdr = C.make_header(C.flags(linked=True, content_size=True), C.BD_64K, len(data))
    assert theirs[: len(hdr)] == hdr
    assert C.with_header(theirs, flg=theirs[4]) == theirs and C.repair_hc(theirs) == theirs
    assert C.stored_frame(b"").data == b"\x04\x22\x4d\x18" + C.make_header(C.flags())[4:] + C.END_MARK
    assert len(C.stored_frame(b"x" * 185).data) == 200


@pytest.mark.parametrize("conforming", [True, False], ids=["conforming", "lenient"])
def test_generated_streams_decode_to_the_generators_bytes(conforming):
    pa = None
    try:
        import pyarrow as pa
    except ImportError:
        pass
    for s in _streams(conforming):
        assert len(s.blocks) == -(-len(s.content) // C.BLOCK) and all(len(b.data) <= C.BLOCK for b in s.blocks)
        for opts in ({}, {"content_size": True}):
            f = s.frame(**opts)
            assert oracle.lz4f_decode(f.data, len(s.content)) == s.content
        for opts in ({}, {"content_size": True, "block_checksum": True, "content_checksum": True}):
            f = s.frame(**opts)
            if conforming:
                assert ref.lz4f_decompress(f.data, len(s.content)) == s.content
                if pa is not None:
                    assert pa.Codec("lz4").decompress(f.data, decompressed_size=len(s.content)).to_pybytes() == s.content
            elif s.violations:  # a full-size block breaks an end-of-block rule: liblz4 refuses the frame
                with pytest.raises(ValueError):
                    ref.lz4f_decompress(f.data, len(s.content))


def test_lenient_streams_break_the_rules_in_every_full_compressed_block():
    for s in _streams(False):
        full = [j for j, b in enumerate(s.blocks) if not b.raw and (j + 1) * C.BLOCK <= len(s.content)]
        assert s.violations == full
    assert any(s.violations for s in _streams(False))
    assert not any(s.violations for s in _streams(True))


def _base():
    rng = random.Random(9)
    s = C.gen_stream(rng, 150000, stored_p=0.0)
    return s, s.frame(), s.frame(content_size=True), s.frame(block_checksum=True, content_checksum=True)


def _oracle_code(frame, cap):
    try:
        return oracle.lz4f_decode(frame, cap)
    except oracle.OracleError as e:
        return e.code


E_TRUNC, E_HDR, E_BLKSZ, E_CORRUPT, E_SIZE, E_UNSUP = -1, -3, -4, -5, -7, -8


def test_targeted_mutators_do_what_the_tables_say():
    s, f, fs, fc = _base()
    n, c = len(s.content), s.content
    blk = [c[j * C.BLOCK : (j + 1) * C.BLOCK] for j in range(3)]
    cases = [  # (mutant, what the strict oracle returns: bytes or an error code)
        (C.with_header(f.data, flg=f.flg & 0x3F), E_HDR),
        (C.with_header(f.data, flg=f.flg | C.FLG_RESERVED), E_HDR),
        (C.with_header(f.data, bd=C.BD_64K | 0x01), E_HDR),
        (C.with_header(f.data, bd=0x30), E_HDR),
        (C.with_header(f.data, bd=0x50), c),  # 256 KiB maximum: a valid frame (the GPU receiver only takes 64 KiB)
        (C.flip(f.data, 6, 0x10), E_HDR),
        (C.with_header(f.data, flg=f.flg | C.FLG_DICT, dict_id=7), E_UNSUP),
        (C.with_header(fs.data, content_size=n + 1), E_SIZE),
        (C.resize_block(f, 0, C.BLOCK + 1), E_BLKSZ),
        (C.set_word(f.data, C.block_word_pos(f, 2), 0), c[: 2 * C.BLOCK]),
        (C.set_word(fs.data, C.block_word_pos(fs, 2), 0), E_SIZE),
        (C.dup_block(f, 1), blk[0] + blk[1] + blk[1] + blk[2]),
        (C.swap_blocks(f, 0, 1), blk[1] + blk[0] + blk[2]),
        (C.drop_block(f, 0), blk[1] + blk[2]),
        (C.drop_block(fs, 0), E_SIZE),
        (C.drop_end_mark(f), E_TRUNC),
        (f.data + b"\x01\x02\x03", c),
        (f.data[: f.spans[1][0] + 7], E_TRUNC),
        (f.data[:-1], E_TRUNC),
        (f.data[: f.marks["offset"][3]] + b"\0\0" + f.data[f.marks["offset"][3] + 2 :], E_CORRUPT),
    ]
    other = C.gen_stream(random.Random(10), 70000, stored_p=0.0)
    of = other.frame()
    cases.append((C.splice_block(f, 1, of, 0), blk[0] + other.content[: C.BLOCK] + blk[2]))
    for i, (m, want) in enumerate(cases):
        assert _oracle_code(m, 4 * C.BLOCK) == want, i
    # checksums and the raw bit: liblz4 rejects checksum flips; a stored block's raw bit cleared is read as sequences
    for pos in (fc.marks["block_checksum"][1], fc.marks["content_checksum"][3]):
        with pytest.raises(ValueError, match="Checksum"):
            ref.lz4f_decompress(C.flip(fc.data, pos, 0x04), n)
    assert ref.lz4f_decompress(fc.data, n) == c
    st = C.assemble_frame([C.stored_block(blk[0]), C.stored_block(blk[1][:100])], blk[0] + blk[1][:100])
    assert _oracle_code(C.toggle_raw(st, 0), 4 * C.BLOCK) != blk[0] + blk[1][:100]
    assert struct.unpack_from("<I", C.resize_block(f, 1, 7), f.spans[1][0])[0] == 7


def test_random_mutants_are_reproducible_and_structural():
    s, f, fs, fc = _base()
    seen = set()
    for seed in range(300):
        a = C.random_mutant(random.Random(seed), fc, [f, fs])
        assert a == C.random_mutant(random.Random(seed), fc, [f, fs]) and a[1] != fc.data
        seen.add(a[0].split(":")[0])
    assert seen >= {"flip", "flip_hc_fixed", "truncate", "trailing", "raw_bit", "size+1", "size-1", "size_65537", "drop", "dup",
                    "splice", "no_end_mark", "swap"}


def _twin_and_liblz4_frames():
    """Frames of edge-length chunks from liblz4 (levels 0 and 9) and the stage's CPU twins (fast, high-ratio lazy and
    optimal), independent and linked."""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    import hc_model as hm
    import tile_model

    from skyplane_b200 import synth

    for n in (0, 1, 12, 13, 400, 65535, 65536, 65537, 131072 + 999, 200001):
        for d in (synth.silesia_like_chunk(n % 89, n), (b"it was the best of times, it was the worst of times; " * (n // 50 + 1))[:n]):
            yield d, tile_model.frame(d)
            for linked in (False, True):
                for level in (0, 9):
                    yield d, hm.liblz4_frame(d, level, linked=linked)
                for level in (3, 9):
                    yield d, hm.frame(d, hm.kernel_opts(level=level), linked=linked)
                yield d, hm.frame(d, hm.kernel_opts(level=5), linked=linked, optimal=True)


def test_end_of_block_walker():
    """lz4_craft.conforms accepts every frame liblz4 and the twins make and every conforming stream, and rejects every
    lenient block -- short last blocks too, where liblz4 decodes the five short-block cases -- another layout, and offset 0,
    which liblz4 decodes where its output buffer happens to hold the right bytes."""
    for d, f in _twin_and_liblz4_frames():
        assert ref.lz4f_decompress(f, len(d)) == d and C.conforms(f, len(d)), (len(d), f[4])
    for s in _streams(True):
        assert C.conforms(s.frame(content_size=True).data, len(s.content))
    for s in _streams(False):  # every compressed block of a lenient stream long enough for a match breaks a rule
        bad = [j for j, b in enumerate(s.blocks) if not b.raw and C.walk_block(b.data)[0]]
        assert C.conforms(s.frame(block_checksum=True).data, len(s.content)) == (not bad)
    rng = random.Random(12)
    for head in (b"", rng.randbytes(C.BLOCK)):
        for want in (400, 1000, 65000):
            for name, blk, content in C.short_block_cases(rng, head, want):
                blocks = ([C.stored_block(head)] if head else []) + [blk]
                f = C.assemble_frame(blocks, content, linked=bool(head), content_size=True).data
                assert ref.lz4f_decompress(f, len(content)) == content, name
                assert oracle.lz4f_decode(f, len(content)) == content, name
                assert not C.conforms(f, len(content)), name
    buf = bytearray()  # the same end in a full block: liblz4 rejects it too
    w = C.BlockWriter(buf).literals(rng.randbytes(C.BLOCK - 304)).match(8, 300).literals(rng.randbytes(4))
    f = C.assemble_frame([w.close()], bytes(buf), content_size=True).data
    with pytest.raises(ValueError):
        ref.lz4f_decompress(f, C.BLOCK)
    assert not C.conforms(f, C.BLOCK)
    # layout: a short block before the last, or a block too many, is not the stage's layout
    c = rng.randbytes(100000)
    assert not C.conforms(C.assemble_frame([C.stored_block(c[:50000]), C.stored_block(c[50000:])], c).data, len(c))
    assert C.conforms(C.assemble_frame([C.stored_block(c[:C.BLOCK]), C.stored_block(c[C.BLOCK:])], c).data, len(c))
    assert not C.conforms(C.assemble_frame([C.stored_block(c[:C.BLOCK]), C.stored_block(c[C.BLOCK:]), C.stored_block(b"")], c).data,
                          len(c))
    # offset 0: liblz4 copies what its (zeroed) output buffer holds there, so on zeros it restores the chunk
    z = bytes(1000)
    f = C.assemble_frame([C.encode_block([(z[:100], 3, 300)], z[400:])], z, content_size=True)
    p = f.marks["offset"][0]
    zero = f.data[:p] + b"\0\0" + f.data[p + 2 :]
    assert ref.lz4f_decompress(zero, len(z)) == z and C.conforms(f.data, len(z)) and not C.conforms(zero, len(z))
