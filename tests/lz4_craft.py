"""A small LZ4 frame assembler, stream generator and frame mutator for the receiver tests.

Written from the LZ4 frame and block format descriptions, not from any decoder: the bytes a generated stream must
decode to come from the generator itself, which builds the output and the sequences that describe it together.

  * ``encode_block`` / ``assemble_frame`` write tokens, length extensions, little-endian offsets, block words, the
    EndMark and (optionally) block and content checksums; the header checksum byte is always recomputed.
  * ``gen_stream`` makes valid-by-construction streams in the receiver's layout (64 KiB blocks, only the last one
    short).  ``conforming`` streams keep LZ4's end-of-block rules (the last 5 bytes of a block are literals, the last
    match starts at least 12 bytes before the block end), so liblz4 accepts them; ``lenient`` streams end every
    compressed block with a sequence that breaks one of those rules, which liblz4 rejects in a full-size block.
  * ``conforms`` walks a frame's blocks (``walk_block``) for the receiver's layout, nonzero offsets and the end-of-block
    rules in every block, short ones too; ``short_block_cases`` makes short last blocks that break those rules and that
    liblz4 still decodes.
  * the mutators change one structural thing: a header field, a block word, a token, an extension byte, an offset,
    the EndMark, a checksum, whole blocks, or the frame's length.
"""
from __future__ import annotations

import random
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import oracle

MAGIC = 0x184D2204
BLOCK = 65536
MIN_MATCH = 4
LAST_LITERALS = 5  # a conforming block ends with at least this many literals
MF_LIMIT = 12      # ... and its last match starts at least this many bytes before the block end

FLG_VERSION, FLG_INDEP, FLG_BLOCK_CHK, FLG_SIZE, FLG_CONTENT_CHK, FLG_RESERVED, FLG_DICT = 0x40, 0x20, 0x10, 0x08, 0x04, 0x02, 0x01
BD_64K = 0x40
END_MARK = b"\x00\x00\x00\x00"

# length-field values around the 4-bit field's escape (15) and its first two 255-byte extensions
LEN_EDGES = (14, 15, 16, 269, 270, 271, 524, 525, 526)
OFFSET_EDGES = tuple(range(1, 41)) + (63, 64, 65, 4095, 4096, 65535)


# ------------------------------------------------------------------------------------------------ blocks
@dataclass
class Block:
    data: bytes                 # the block's payload: its sequences, or its bytes when stored raw
    raw: bool = False
    # positions inside `data` of each token, length-extension byte and 2-byte offset (compressed blocks)
    marks: Dict[str, List[int]] = field(default_factory=lambda: {"token": [], "ext": [], "offset": []})

    @property
    def word(self) -> int:
        return len(self.data) | (0x80000000 if self.raw else 0)


def _put_ext(out: bytearray, n: int) -> None:
    """Length extension of a 4-bit field that reads 15: n = length - 15 as 255-bytes and a final byte < 255."""
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)


def encode_block(seqs: Sequence[Tuple[bytes, int, int]], last_literals: bytes = b"") -> Block:
    """Sequences (literals, offset, match length >= 4), then the literal-only last sequence."""
    out = bytearray()
    marks: Dict[str, List[int]] = {"token": [], "ext": [], "offset": []}

    def put(lit: bytes, off: int, ml: int) -> None:
        ll, mf = len(lit), (ml - MIN_MATCH if off else 0)
        marks["token"].append(len(out))
        out.append((min(ll, 15) << 4) | min(mf, 15))
        if ll >= 15:
            s = len(out)
            _put_ext(out, ll - 15)
            marks["ext"].extend(range(s, len(out)))
        out.extend(lit)
        if off:
            marks["offset"].append(len(out))
            out.extend(struct.pack("<H", off))
            if mf >= 15:
                s = len(out)
                _put_ext(out, mf - 15)
                marks["ext"].extend(range(s, len(out)))

    for lit, off, ml in seqs:
        assert 1 <= off <= 65535 and ml >= MIN_MATCH
        put(lit, off, ml)
    put(last_literals, 0, 0)
    return Block(bytes(out), False, marks)


def stored_block(data: bytes) -> Block:
    return Block(bytes(data), True)


# ------------------------------------------------------------------------------------------------ frames
def header_checksum(desc: bytes) -> int:
    """HC byte: second byte of XXH32 (seed 0) over the frame descriptor (FLG .. dictID)."""
    return (oracle.xxh32(desc) >> 8) & 0xFF


def make_header(flg: int, bd: int = BD_64K, content_size: int = 0, dict_id: int = 0) -> bytes:
    desc = bytes([flg, bd])
    if flg & FLG_SIZE:
        desc += struct.pack("<Q", content_size)
    if flg & FLG_DICT:
        desc += struct.pack("<I", dict_id)
    return struct.pack("<I", MAGIC) + desc + bytes([header_checksum(desc)])


def header_len(flg: int) -> int:
    return 7 + (8 if flg & FLG_SIZE else 0) + (4 if flg & FLG_DICT else 0)


def flags(linked: bool = False, content_size: bool = False, block_checksum: bool = False, content_checksum: bool = False) -> int:
    return (FLG_VERSION | (0 if linked else FLG_INDEP) | (FLG_SIZE if content_size else 0) | (FLG_BLOCK_CHK if block_checksum else 0)
            | (FLG_CONTENT_CHK if content_checksum else 0))


def with_header(frame: bytes, flg: Optional[int] = None, bd: Optional[int] = None, content_size: Optional[int] = None,
                dict_id: int = 0) -> bytes:
    """Rebuild the header of `frame` with some fields changed and a valid HC byte; the body stays as it is."""
    old_flg = frame[4]
    old_size = struct.unpack_from("<Q", frame, 6)[0] if old_flg & FLG_SIZE else 0
    new_flg = old_flg if flg is None else flg
    hdr = make_header(new_flg, frame[5] if bd is None else bd, old_size if content_size is None else content_size, dict_id)
    return hdr + frame[header_len(old_flg):]


def repair_hc(frame: bytes) -> bytes:
    """Recompute the HC byte for whatever descriptor the (mutated) header now holds."""
    n = header_len(frame[4])
    return frame[: n - 1] + bytes([header_checksum(frame[4 : n - 1])]) + frame[n:]


@dataclass
class Frame:
    data: bytes
    content: bytes                                 # what the frame decodes to
    marks: Dict[str, List[int]]                    # structural byte positions inside `data`
    spans: List[Tuple[int, int]]                   # per block: [block word, end of its data and checksum)
    block_out: List[Tuple[int, int]]               # per block: its [start, end) in `content`
    flg: int = 0

    def __bytes__(self) -> bytes:
        return self.data

    def __len__(self) -> int:
        return len(self.data)


def assemble_frame(blocks: Sequence[Block], content: bytes, linked: bool = False, content_size: bool = False,
                   block_checksum: bool = False, content_checksum: bool = False, end_mark: bool = True) -> Frame:
    """Header + blocks (+ block checksums) + EndMark (+ content checksum).  `content` is what the blocks decode to."""
    flg = flags(linked, content_size, block_checksum, content_checksum)
    out = bytearray(make_header(flg, BD_64K, len(content)))
    hl = len(out)
    marks: Dict[str, List[int]] = {"magic": [0, 1, 2, 3], "flg": [4], "bd": [5], "size": list(range(6, hl - 1)) if content_size else [],
                                   "hc": [hl - 1], "block_word": [], "token": [], "ext": [], "offset": [], "raw_data": [],
                                   "end_mark": [], "block_checksum": [], "content_checksum": []}
    spans, block_out, pos = [], [], 0
    for b in blocks:
        s = len(out)
        marks["block_word"].extend(range(s, s + 4))
        out.extend(struct.pack("<I", b.word))
        base = len(out)
        for k in ("token", "ext", "offset"):
            marks[k].extend(base + i for i in b.marks[k])
        if b.raw and b.data:
            marks["raw_data"].extend((base, base + len(b.data) - 1))
        out.extend(b.data)
        if block_checksum:
            marks["block_checksum"].extend(range(len(out), len(out) + 4))
            out.extend(struct.pack("<I", oracle.xxh32(b.data)))
        spans.append((s, len(out)))
    if end_mark:
        marks["end_mark"] = list(range(len(out), len(out) + 4))
        out.extend(END_MARK)
    if content_checksum:
        marks["content_checksum"] = list(range(len(out), len(out) + 4))
        out.extend(struct.pack("<I", oracle.xxh32(content)))
    return Frame(bytes(out), bytes(content), marks, spans, block_out, flg)


def stored_frame(payload: bytes, **kw) -> Frame:
    """One stored block of n bytes: an (n + 15)-byte frame without content size or checksums."""
    return assemble_frame([stored_block(payload)] if payload else [], payload, **kw)


# ------------------------------------------------------------------------------------------------ generator
@dataclass
class Stream:
    content: bytes
    blocks: List[Block]
    linked: bool
    conforming: bool
    violations: List[int]  # full-size compressed blocks that break an end-of-block rule (lenient streams)

    def frame(self, content_size: bool = False, block_checksum: bool = False, content_checksum: bool = False) -> Frame:
        f = assemble_frame(self.blocks, self.content, self.linked, content_size, block_checksum, content_checksum)
        f.block_out = [(j * BLOCK, min(len(self.content), (j + 1) * BLOCK)) for j in range(len(self.blocks))]
        return f


def _lit_len(rng: random.Random) -> int:
    r = rng.random()
    if r < 0.25:
        return rng.choice(LEN_EDGES)
    if r < 0.55:
        return rng.randrange(0, 9)
    if r < 0.85:
        return rng.randrange(0, 64)
    if r < 0.95:
        return 32 * rng.randrange(1, 9) + rng.choice((-1, 0, 1))
    return rng.randrange(600, 4000)


def _match_len(rng: random.Random) -> int:
    r = rng.random()
    if r < 0.35:
        return max(MIN_MATCH, 32 * rng.randrange(1, 17) + rng.choice((-1, 0, 1)))
    if r < 0.6:
        return MIN_MATCH + rng.choice(LEN_EDGES)  # the match-length field sits at its escape / extension edges
    if r < 0.9:
        return rng.randrange(MIN_MATCH, 24)
    return rng.randrange(1000, 6000)


def _offset(rng: random.Random, hist: int, p: int, linked: bool) -> int:
    """hist = bytes a match may reach back (>= 1), p = position inside the current block."""
    top = min(65535, hist)
    r = rng.random()
    if r < 0.1:
        return top  # reaches the oldest byte it may: byte 0 of a linked chunk or of an independent block
    if linked and hist > p and r < 0.3:
        return rng.randrange(p + 1, top + 1)  # source starts in an earlier block
    cands = [o for o in OFFSET_EDGES if o <= top]
    if r < 0.85 or top <= 65:
        return rng.choice(cands)
    return rng.randrange(1, top + 1)


def _copy_match(buf: bytearray, off: int, ml: int) -> None:
    s = len(buf) - off
    if off >= ml:
        buf += buf[s : s + ml]
    else:
        buf += (bytes(buf[s:]) * (ml // off + 1))[:ml]


class BlockWriter:
    """One compressed block written by hand: literals and matches are applied to `buf` (the stream so far) as they are
    added, so the expected output is known without decoding anything."""

    def __init__(self, buf: bytearray):
        self.buf, self.start, self.seqs, self.lit = buf, len(buf), [], bytearray()

    @property
    def pos(self) -> int:  # position inside the block
        return len(self.buf) - self.start

    def literals(self, data: bytes) -> "BlockWriter":
        self.lit += data
        self.buf += data
        return self

    def match(self, off: int, ml: int) -> "BlockWriter":
        _copy_match(self.buf, off, ml)
        self.seqs.append((bytes(self.lit), off, ml))
        self.lit = bytearray()
        return self

    def close(self) -> Block:
        return encode_block(self.seqs, bytes(self.lit))


def _literals(rng: random.Random, n: int) -> bytes:
    if rng.random() < 0.5:
        return rng.randbytes(n)
    return bytes(rng.choice(b"abcdefgh ") for _ in range(n)) if n < 64 else (b"lorem ipsum dolor sit amet " * (n // 27 + 1))[:n]


def _compressed_block(rng: random.Random, buf: bytearray, want: int, linked: bool, conforming: bool) -> Tuple[Block, bool]:
    """Append `want` bytes to buf through sequences; returns the block and whether it breaks an end-of-block rule."""
    start = len(buf)
    low = 0 if linked else start
    seqs: List[Tuple[bytes, int, int]] = []
    p = 0
    while True:
        ll = _lit_len(rng)
        if start + p + ll - low == 0:
            ll += 1  # nothing to match against yet
        if p + ll > want - MF_LIMIT:
            break
        room = want - LAST_LITERALS - (p + ll)
        if room < MIN_MATCH:
            break
        ml = min(_match_len(rng), room)
        lit = _literals(rng, ll)
        buf += lit
        off = _offset(rng, len(buf) - low, p + ll, linked)
        _copy_match(buf, off, ml)
        seqs.append((lit, off, ml))
        p += ll + ml
    r = want - p
    violates = False
    if not conforming and r >= MIN_MATCH + (1 if start + p == low else 0):
        if rng.random() < 0.5:  # a match that ends exactly at the block end, then a zero-literal last sequence
            ml = rng.randrange(MIN_MATCH, r + 1 - (1 if start + p == low else 0))
            k = 0
        else:                   # a match that starts fewer than 12 bytes before the block end
            k = rng.randrange(MIN_MATCH, min(MF_LIMIT - 1, r) + 1)
            if start + want - k == low:
                k -= 1
            ml = rng.randrange(MIN_MATCH, k + 1)
            k -= ml
        ll = r - ml - k
        lit = _literals(rng, ll)
        buf += lit
        off = _offset(rng, len(buf) - low, p + ll, linked)
        _copy_match(buf, off, ml)
        seqs.append((lit, off, ml))
        p += ll + ml
        violates = True
    last = _literals(rng, want - p)
    buf += last
    return encode_block(seqs, last), violates


def gen_stream(rng: random.Random, size: int, linked: bool = False, conforming: bool = True, stored_p: float = 0.15) -> Stream:
    """A stream of `size` bytes in 64 KiB blocks (only the last one short); about `stored_p` of them stored raw."""
    buf = bytearray()
    blocks: List[Block] = []
    violations: List[int] = []
    for j in range((size + BLOCK - 1) // BLOCK):
        want = min(BLOCK, size - j * BLOCK)
        if rng.random() < stored_p:
            data = rng.randbytes(want) if rng.random() < 0.5 or not buf else (bytes(buf) * (want // len(buf) + 1))[:want]
            buf += data
            blocks.append(stored_block(data))
            continue
        b, v = _compressed_block(rng, buf, want, linked, conforming)
        blocks.append(b)
        if v and want == BLOCK:
            violations.append(j)
    assert len(buf) == size
    return Stream(bytes(buf), blocks, linked, conforming, violations)


def short_block_cases(rng: random.Random, head: bytes, want: int) -> List[Tuple[str, Block, bytes]]:
    """Last blocks of `want` (400 .. 65000) bytes behind the stream `head` that break an end-of-block rule: a 300-byte last
    match followed by 3 or 4 literals, and a 4-byte last match that starts 9, 10 or 11 bytes before the block end.  liblz4
    enforces these rules in blocks of (nearly) 64 KiB only and decodes all five here (3 literals only behind a match long
    enough for a length extension).  -> [(name, block, the whole stream's content)]"""
    assert 400 <= want <= 65000
    out = []
    for lits in (3, 4):
        buf = bytearray(head)
        w = BlockWriter(buf).literals(rng.randbytes(want - 300 - lits)).match(8, 300).literals(rng.randbytes(lits))
        out.append((f"long last match, then {lits} literals", w.close(), bytes(buf)))
    for k in (9, 10, 11):
        buf = bytearray(head)
        w = BlockWriter(buf).literals(rng.randbytes(want - k)).match(7, MIN_MATCH).literals(rng.randbytes(k - MIN_MATCH))
        out.append((f"4-byte match {k} bytes before the end", w.close(), bytes(buf)))
    return out


# ------------------------------------------------------------------------------------------------ end-of-block rules
def walk_block(block: bytes) -> Tuple[List[Tuple[int, int]], int]:
    """The sequences of one well-formed LZ4 block -> ([(output position, offset, length) of every match], decoded length)."""
    def length(i: int, n: int) -> Tuple[int, int]:
        if n == 15:
            while block[i] == 255:
                n += 255
                i += 1
            n += block[i]
            i += 1
        return i, n

    i = pos = 0
    matches = []
    while i < len(block):
        tok = block[i]
        i, ll = length(i + 1, tok >> 4)
        i += ll
        pos += ll
        if i >= len(block):
            break
        off = block[i] | block[i + 1] << 8
        i, ml = length(i + 2, tok & 15)
        matches.append((pos, off, ml + MIN_MATCH))
        pos += ml + MIN_MATCH
    return matches, pos


def conforms(frame: bytes, n: int) -> bool:
    """Does a well-formed frame of an n-byte chunk keep the stage's block layout and LZ4's block rules?  Every block decodes
    to min(64 KiB, n - its start) bytes, and in every compressed block each match has an offset of at least 1, starts at
    least MF_LIMIT bytes before the block's end and leaves at least LAST_LITERALS literals behind it -- relative to the
    block's own decoded length, so in a short last block too.  liblz4 asks for the end-of-block rules in full blocks only,
    and takes offset 0 as a copy of whatever its output buffer holds there."""
    try:
        flg = frame[4]
        ip, pos = header_len(flg), 0
        while True:
            w = struct.unpack_from("<I", frame, ip)[0]
            ip += 4
            if w == 0:
                return pos == n
            size, want = w & 0x7FFFFFFF, min(BLOCK, n - pos)
            if want <= 0 or ip + size > len(frame):
                return False
            if w & 0x80000000:
                if size != want:
                    return False
            else:
                matches, out = walk_block(frame[ip : ip + size])
                if out != want or any(off == 0 or q + MF_LIMIT > want or q + ml > want - LAST_LITERALS for q, off, ml in matches):
                    return False
            pos += want
            ip += size + (4 if flg & FLG_BLOCK_CHK else 0)
    except (IndexError, struct.error):
        return False


# ------------------------------------------------------------------------------------------------ mutators
def flip(frame: bytes, pos: int, mask: int = 0xFF) -> bytes:
    return frame[:pos] + bytes([frame[pos] ^ mask]) + frame[pos + 1:]


def set_word(frame: bytes, pos: int, word: int) -> bytes:
    return frame[:pos] + struct.pack("<I", word & 0xFFFFFFFF) + frame[pos + 4:]


def block_word_pos(f: Frame, k: int) -> int:
    return f.spans[k][0]


def toggle_raw(f: Frame, k: int) -> bytes:
    p = block_word_pos(f, k)
    return set_word(f.data, p, struct.unpack_from("<I", f.data, p)[0] ^ 0x80000000)


def resize_block(f: Frame, k: int, size: int) -> bytes:
    """Block k's size field set to `size` (the raw bit kept); the bytes behind it stay where they are."""
    p = block_word_pos(f, k)
    w = struct.unpack_from("<I", f.data, p)[0]
    return set_word(f.data, p, (w & 0x80000000) | size)


def _body(f: Frame, k: int) -> bytes:
    s, e = f.spans[k]
    return f.data[s:e]


def rebuild_blocks(f: Frame, order: Sequence[bytes]) -> bytes:
    """The frame with its block section replaced by `order` (each a block word + data + checksum span)."""
    first = f.spans[0][0] if f.spans else f.marks["end_mark"][0]
    tail = f.spans[-1][1] if f.spans else first
    return f.data[:first] + b"".join(order) + f.data[tail:]


def drop_block(f: Frame, k: int) -> bytes:
    return rebuild_blocks(f, [_body(f, i) for i in range(len(f.spans)) if i != k])


def dup_block(f: Frame, k: int) -> bytes:
    bodies = [_body(f, i) for i in range(len(f.spans))]
    return rebuild_blocks(f, bodies[: k + 1] + [bodies[k]] + bodies[k + 1:])


def swap_blocks(f: Frame, a: int, b: int) -> bytes:
    bodies = [_body(f, i) for i in range(len(f.spans))]
    bodies[a], bodies[b] = bodies[b], bodies[a]
    return rebuild_blocks(f, bodies)


def splice_block(f: Frame, k: int, other: Frame, m: int) -> bytes:
    bodies = [_body(f, i) for i in range(len(f.spans))]
    bodies[k] = _body(other, m)
    return rebuild_blocks(f, bodies)


def drop_end_mark(f: Frame) -> bytes:
    e = f.marks["end_mark"][0]
    return f.data[:e] + f.data[e + 4:]


STRUCTURAL = ("flg", "bd", "size", "hc", "block_word", "token", "ext", "offset", "end_mark", "block_checksum", "content_checksum")


def random_mutant(rng: random.Random, f: Frame, donors: Sequence[Frame]) -> Tuple[str, bytes]:
    """One seeded mutation of `f` at a structural position -> (description, frame bytes)."""
    kinds = [k for k in STRUCTURAL if f.marks.get(k)]
    nb = len(f.spans)
    ops = ["flip"] * 6 + ["flip_hc_fixed", "truncate", "trailing"]
    if nb:
        ops += ["raw_bit", "size_delta", "size_65537", "drop", "dup", "splice", "no_end_mark"]
    if nb > 1:
        ops.append("swap")
    op = rng.choice(ops)
    if op in ("flip", "flip_hc_fixed"):
        kind = rng.choice(kinds)
        pos = rng.choice(f.marks[kind])
        mask = rng.choice((0x01, 0x80, 0xFF, 1 << rng.randrange(8), rng.randrange(1, 256)))
        out = flip(f.data, pos, mask)
        if op == "flip_hc_fixed" and pos < header_len(f.flg) - 1:
            out = repair_hc(out) if header_len(out[4]) <= len(out) else out
        return f"{op}:{kind}@{pos}^{mask:#x}", out
    if op == "truncate":
        n = rng.randrange(0, len(f.data))
        return f"truncate:{n}", f.data[:n]
    if op == "trailing":
        return "trailing", f.data + rng.randbytes(rng.randrange(1, 9))
    k = rng.randrange(nb)
    if op == "raw_bit":
        return f"raw_bit:{k}", toggle_raw(f, k)
    if op == "size_delta":
        d = rng.choice((-1, 1))
        sz = (struct.unpack_from("<I", f.data, f.spans[k][0])[0] & 0x7FFFFFFF) + d
        return f"size{d:+d}:{k}", resize_block(f, k, max(0, sz))
    if op == "size_65537":
        return f"size_65537:{k}", resize_block(f, k, BLOCK + 1)
    if op == "drop":
        return f"drop:{k}", drop_block(f, k)
    if op == "dup":
        return f"dup:{k}", dup_block(f, k)
    if op == "splice":
        d = rng.choice([x for x in donors if x.spans] or [f])
        return f"splice:{k}", splice_block(f, k, d, rng.randrange(len(d.spans)))
    if op == "no_end_mark":
        return "no_end_mark", drop_end_mark(f)
    a, b = rng.sample(range(nb), 2)
    return f"swap:{a},{b}", swap_blocks(f, a, b)
