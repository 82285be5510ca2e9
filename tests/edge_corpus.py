"""A seeded corpus of short chunks built for the edges of the compressors' parses, where the kernels' lane-level shortcuts
meet their sequential twins' rules (tools/lz4_tile_model.c, tools/lz4hc_model.c) and natural data rarely goes.

Every chunk is random bytes with planted structure, tagged with the rule it targets, and carries what its twin must show
for the target to count as reached (test_edge_corpus.py checks that on the twins; test_gpu_edge_corpus.py runs the corpus
through every compressor kernel).  The geometry -- table entries, segment slots, stride cap, hash bits, stop length,
optimal-parse segment, depth per level -- is read from native.kernel_config(), not written down here.

Collisions are solved, not searched: the fast hash is hf = le32(s) * K1 + s[4] * K2 (mod 2^32) and the high-ratio hash
(le32(s) * K1) >> (32 - hash_bits), and K1 is odd, so le32(s) follows from any wanted hash and fifth byte.

Fields of Case.expect (all optional):
  fast_rejects    (n, positions): breaking the planted strings -- one byte at each position changed -- takes exactly n off
                  the fast twin's hits less the matches it accepts (tile_model_stats): each planted collision is a hit
                  the parse measured and rejected;
  fast_matches    [(block, pos, off, len)] matches the fast twin's blocks hold (pos = where the match starts in the block);
  fast_absent     the same form: matches they do not hold;
  near_mask       the fast twin's frame changes when its in-group candidates are restricted to this near_mask;
  hc_matches      {(level, linked, optimal): [(block, pos, off, len)]} matches the high-ratio twin's blocks hold;
  hc_absent       the same form: matches they do not hold;
  levels_differ   [(level_a, level_b)] the high-ratio twin's frames at these two levels differ;
  linked_offsets  [(block, offset)]: the linked level-5 twin's block holds a match at exactly this offset;
  linked_raw      a block the linked level-5 twin stores raw (no candidate lies inside the window);
  last_block      the length of the chunk's last block.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

from skyplane_b200 import native

K1, K2, M32 = 2654435761, 0x85EBCA6B, 0xFFFFFFFF
K1_INV = pow(K1, -1, 1 << 32)
BLOCK = 65536
LAST_LITERALS, MIN_MATCH = 5, 4
# a multiple of every stride, so that a slot's repeat one period back is a slot too, and more than 8 slots at the largest
# stride, so that the pad's hits come from the table, never from the in-group compares the near targets test
PAD_PERIOD = 256


@dataclass
class Case:
    tag: str
    data: bytes
    expect: Dict = field(default_factory=dict)


def geometry() -> dict:
    k = native.kernel_config()
    g = {key: k[key] for key in ("lz4_entries", "seg_slots", "max_step_log", "hc_hash_bits", "hc_nice", "hc_opt_seg")}
    g["depth"] = {lv: native.hc_depth(lv) for lv in range(native.HC_MIN_LEVEL, native.HC_MAX_LEVEL + 1)}
    return g


def le32(b) -> int:
    return int.from_bytes(bytes(b[:4]), "little")


def fast_hash(s) -> int:
    return (le32(s) * K1 + s[4] * K2) & M32


def fast_hashes(data: bytes) -> np.ndarray:
    """hf at every position p with p + 5 <= len(data)."""
    a = np.frombuffer(bytes(data), np.uint8).astype(np.uint64)
    n = len(a) - 4
    rd = a[:n] | a[1:n + 1] << 8 | a[2:n + 2] << 16 | a[3:n + 3] << 24
    return ((rd * K1 + a[4:n + 4] * K2) & M32).astype(np.uint64)


def solve_fast(hf: int, b4: int) -> bytes:
    """The 5-byte string with fast hash hf and fifth byte b4."""
    return (((hf - b4 * K2) * K1_INV) & M32).to_bytes(4, "little") + bytes([b4])


def hc_hash(s, bits: int) -> int:
    return ((le32(s) * K1) & M32) >> (32 - bits)


class Buf:
    """Random bytes with planted structure; `planted` marks the bytes the structure owns."""

    def __init__(self, rng, n: int):
        self.rng = rng
        self.b = bytearray(rng.bytes(n))
        self.planted = np.zeros(n, bool)

    def put(self, pos: int, s) -> None:
        self.b[pos:pos + len(s)] = bytes(s)
        self.planted[pos:pos + len(s)] = True

    def differ(self, pos: int, other: int) -> None:
        """b[pos] != other (a byte value)."""
        if self.b[pos] == other:
            self.b[pos] ^= 0x5A
        self.planted[pos] = True

    def protect(self, g, pairs, step: int = 1) -> None:
        """Keep the table entry each slot `src` leaves until slot `dst` looks it up, both in segments probed every `step`
        bytes (stride 1: a block's first two segments) whose groups start at multiples of 32 * step: redraw filler bytes
        under any slot of a group before dst's, after src, that shares its index."""
        for _ in range(1000):
            idx = (fast_hashes(self.bytes()) * g["lz4_entries"]) >> 32
            bad = []
            for src, dst in pairs:
                qs = np.arange(src + step, dst - dst % (32 * step), step)
                bad += qs[idx[qs] == idx[src]].tolist()
            if not bad:
                return
            for q in bad:
                free = [i for i in range(q, q + 5) if not self.planted[i]]
                if not free:
                    raise RuntimeError(f"slot {q} is all planted")
                self.b[free[0]] = int(self.rng.integers(256))
        raise RuntimeError("table entries keep colliding")

    def copy(self, src: int, dst: int, n: int) -> None:
        """b[dst:dst+n] = b[src:src+n], with the bytes either side different from the source's, so the match is exactly n."""
        self.put(dst, self.b[src:src + n])
        self.planted[src:src + n] = True
        self.differ(dst - 1, self.b[src - 1])
        self.differ(dst + n, self.b[src + n])

    def pad(self, start: int, end: int) -> None:
        """A PAD_PERIOD-byte random pattern repeated over [start, end): a block whose planted matches alone would not pay for
        their sequences is stored raw, and a stored block shows nothing of the parse."""
        pat = self.rng.bytes(PAD_PERIOD)
        self.put(start, (pat * ((end - start) // PAD_PERIOD + 1))[:end - start])

    def bytes(self) -> bytes:
        return bytes(self.b)


def collide(rng, hf: int, fixed: Dict[int, int], low_free: bool = False, differ: Dict[int, int] = {}) -> bytes:
    """A 5-byte string of fast hash hf (low_free: of any low hash byte, which neither the index nor the tag reads) whose
    bytes at the indices of `fixed` hold its values and at the indices of `differ` do not."""
    r = np.arange(1 << 16, dtype=np.uint64)
    h = (hf & ~0xFF) | (r & 0xFF) if low_free else np.full(1 << 16, hf, np.uint64)
    b4 = np.full(1 << 16, fixed[4], np.uint64) if 4 in fixed else r >> 8
    rd = (((h - b4 * K2) & M32) * K1_INV) & M32
    byte = lambda i: b4 if i == 4 else (rd >> np.uint64(8 * i)) & 0xFF  # noqa: E731
    ok = np.ones(1 << 16, bool)
    for i, v in fixed.items():
        ok &= byte(i) == v
    for i, v in differ.items():
        ok &= byte(i) != v
    good = np.flatnonzero(ok)
    if not len(good):
        raise RuntimeError("no collision with these bytes fixed")
    j = int(rng.choice(good))
    return int(rd[j]).to_bytes(4, "little") + bytes([int(b4[j])])


def _fixed(buf: Buf, pos: int) -> Dict[int, int]:
    return {i: buf.b[pos + i] for i in range(5) if buf.planted[pos + i]}


# ------------------------------------------------------------------------------------------------ fast compressor
def f1_false_hits(g, rng) -> List[Case]:
    """Table entries whose index and tag (hash bits 8..31) equal the probe's, for a string whose first k bytes agree with
    it, k = 0, 1, 2, three pairs in different groups of a block's first two segments.  (k = 3 is impossible for this
    hash: test_edge_corpus.py shows it.)  The parse must measure and reject each."""
    out = []
    for k in (0, 1, 2):
        buf = Buf(rng, 3000)
        pairs, breaks = [], []
        for j in range(3):
            a = 64 + 640 * j + 7 * k
            b = a + 320
            s = bytes(buf.b[a:a + 5])
            buf.put(a, s)
            buf.put(b, collide(rng, fast_hash(s), {i: s[i] for i in range(k)}, low_free=True, differ={k: s[k]}))
            pairs.append((a, b))
            breaks.append(b + k)
        buf.pad(420, 690)  # (in segment 0, so breaking the pairs leaves the stride schedule as it is)
        buf.protect(g, pairs)
        out.append(Case(f"F1 table false hit, {k} bytes agree", buf.bytes(), {"fast_rejects": (3, breaks)}))
    return out


def _quiet(g, data: bytes, nseg: int) -> bool:
    """No table or near hit in a block's first nseg segments, probed at the strides they have when none has a hit (the
    probe rule of tools/lz4_tile_model.c: a group looks the table up before its slots replace their entries)."""
    hf = fast_hashes(data)
    idx, tag = (hf * g["lz4_entries"]) >> 32, (hf >> 8) & 0xFFFF
    table = {}
    starts = _segment_starts(g, nseg + 1)
    for i in range(nseg):
        step = 1 << min(max(i - 1, 0), g["max_step_log"])
        slots = np.arange(starts[i], starts[i + 1], step)
        for grp in slots.reshape(-1, 32):
            h = hf[grp]
            for lane, p in enumerate(grp.tolist()):
                e = table.get(int(idx[p]))
                if (e is not None and e[1] == tag[p] and e[0] < p) or any(lane >= d and h[lane - d] == h[lane] for d in (3, 4, 8)):
                    return False
            for p in grp.tolist():
                table[int(idx[p])] = (p, int(tag[p]))
    return True


def _quiet_buf(g, rng, n: int, nseg: int) -> Buf:
    """n random bytes whose first nseg segments have no hit, so the later ones are probed at the strides planned for."""
    while True:
        buf = Buf(rng, n)
        if _quiet(g, buf.bytes(), nseg):
            return buf


def _quiet_block(g, rng, nseg: int) -> Buf:
    return _quiet_buf(g, rng, BLOCK, nseg)


def f2_near_slots(g, rng) -> List[Case]:
    """32-bit hash collisions 3, 4 and 8 slots back inside a group, at stride 1 and at stride 2 (segment 2 of a block
    whose segment 0 has no hit): the near candidate has the wrong bytes and must be rejected.  And the nearest-wins rule:
    an equal string 8 slots back with a colliding one 3 (or 4) slots back -- the nearer, wrong, candidate must win, so the
    equal string is never matched (with only the 8-slot compare it would be).  Equal strings 5, 6 and 7 slots back."""
    out = []
    for slog, base in ((0, 0), (1, 2 * g["seg_slots"])):
        step = 1 << slog
        # the pad goes where its hits decide no stride the planted strings' hits do not decide already, so that
        # breaking the strings (fast_rejects) leaves the stride schedule as it is
        pad = (300, 900) if slog == 0 else (base + 2000, base + 3500)
        for d in (3, 4, 8):
            buf = _quiet_buf(g, rng, base + 4200, 2 if slog else 0)
            breaks = []
            for j in range(4):
                p = base + (64 * j + 20) * step  # lane 20 of group 2j
                q = p - (d << slog)
                while True:  # (when the strings overlap, x must leave y a solution)
                    x = rng.bytes(5)
                    buf.put(p, x)
                    fixed = _fixed(buf, q)
                    try:
                        y = collide(rng, fast_hash(x), fixed)
                    except RuntimeError:
                        continue
                    if y != x:  # (an equal string would be a real match)
                        buf.put(q, y)
                        break
                breaks.append(q + min(set(range(5)) - set(fixed)))  # a byte of y that x does not share
            buf.pad(*pad)
            out.append(Case(f"F2 near collision {d} slots back, stride {step}", buf.bytes(), {"fast_rejects": (4, breaks)}))
        for d in (3, 4):
            buf = _quiet_buf(g, rng, base + 4200, 2 if slog else 0)
            breaks = []
            for j in range(4):
                p = base + (64 * j + 20) * step
                q = p - (d << slog)
                while True:
                    x = rng.bytes(5)
                    buf.put(p - (8 << slog), x)
                    buf.put(p, x)
                    fixed = _fixed(buf, q)
                    try:
                        y = collide(rng, fast_hash(x), fixed)
                    except RuntimeError:
                        continue
                    if y != x:  # (an equal string would be a real match)
                        buf.put(q, y)
                        break
                buf.differ(p + 5, buf.b[p - (8 << slog) + 5])
                breaks.append(q + min(set(range(5)) - set(fixed)))
            buf.pad(*pad)
            # broken, the nearer string is no candidate and the equal one 8 slots back is accepted: one rejection less each;
            # 4 slots back the colliding string is itself 4 slots after the far one, a second rejected near hit
            out.append(Case(f"F2 nearest of {d} and 8 slots back wins, stride {step}", buf.bytes(),
                            {"near_mask": 0x80, "fast_rejects": (4 * (2 if d == 4 else 1), breaks)}))
    # equal strings 5, 6 and 7 slots back: no near compare sees them, so inside a group they are not found at all, and
    # across a group boundary only the table finds them
    for d in (5, 6, 7):
        for across in (False, True):
            buf = Buf(rng, 4200)
            want = []
            for j in range(4):
                p = 64 * j + (34 if across else 20)  # lane 2 of an odd group: the string d back is in the group before
                x = rng.bytes(5)
                buf.put(p - d, x)
                buf.put(p, x)
                buf.differ(p + 5, buf.b[p - d + 5])
                buf.differ(p - 1, buf.b[p - d - 1])
                want.append((0, p, d, 5))
            buf.pad(2000, 3500)
            out.append(Case(f"F2 equal string {d} slots back, " + ("across a group boundary" if across else "inside a group"),
                            buf.bytes(), {"fast_matches" if across else "fast_absent": want}))
    return out


def _segment_starts(g, n: int = 8) -> List[int]:
    """Where a block's segments start when none of them has a hit (the stride doubles from the third segment on)."""
    starts, pos = [], 0
    for i in range(n):
        starts.append(pos)
        pos += g["seg_slots"] << min(max(i - 1, 0), g["max_step_log"])
    return starts


def f3_compare_window(g, rng) -> List[Case]:
    """Forward: matches of 4, 5, 22..26 and 300 bytes; matches cut by the segment end with 21..25 bytes of room, and by the
    block's last-literals limit with 21..25 bytes of room.  Backward: copies starting 0..9 bytes before a slot at the
    largest stride (the hit comes at the slot, the rest is backward extension, 8 bytes at most), and ones cut by the
    block start and by the previous match's end."""
    out = []
    seg = g["seg_slots"]
    for m in (4, 5, 22, 23, 24, 25, 26, 300):
        buf = Buf(rng, 2 * seg)
        src, dst = 40, 700 if m < 300 else 1400
        buf.copy(src, dst, m)
        buf.pad(1760, 2040)
        buf.protect(g, [(src, dst)])
        # (the fast probe hashes 5 bytes: a 4-byte repeat is not a candidate there)
        exp = {"fast_matches": [(0, dst, dst - src, m)]} if m > MIN_MATCH else {"hc_matches": {(5, False, False): [(0, dst, dst - src, m)]}}
        out.append(Case(f"F3 match of {m} bytes", buf.bytes(), exp))
    for room in (21, 22, 23, 24, 25):
        buf = Buf(rng, 2 * seg + 100)
        src, dst = 40, seg - room
        buf.copy(src, dst, room + 40)
        buf.pad(1300, 2000)
        buf.protect(g, [(src, dst)])
        out.append(Case(f"F3 match cut by the segment end, {room} bytes of room", buf.bytes(),
                        {"fast_matches": [(0, dst, dst - src, room)]}))
        n = 1500 + room
        buf = Buf(rng, n)
        dst = n - LAST_LITERALS - room
        buf.put(dst, buf.b[40:40 + n - dst])
        buf.planted[40:40 + n - dst] = True
        buf.differ(dst - 1, buf.b[39])
        buf.pad(300, 900)
        buf.protect(g, [(40, dst)])
        out.append(Case(f"F3 match cut by the last literals, {room} bytes of room", buf.bytes(),
                        {"fast_matches": [(0, dst, dst - 40, room)]}))
    # a random block's segments 0..4 have no hit, so segments 5 and 6 probe at the largest stride
    starts = _segment_starts(g)
    step = 1 << g["max_step_log"]
    s5, s6 = starts[5], starts[6]
    buf = _quiet_block(g, rng, 5)
    expect = []
    for back in range(10):  # source and copy one group apart in segment 6
        src = s6 + (64 + 64 * back) * step
        dst = src + 32 * step
        buf.copy(src - back, dst - back, back + 30)
        expect.append((0, dst - min(back, 8), dst - src, 30 + min(back, 8)))
    buf.pad(starts[7], starts[7] + 3000)
    buf.protect(g, [(s6 + (64 + 64 * back) * step, s6 + (96 + 64 * back) * step) for back in range(10)], step)
    out.append(Case("F3 backward extension of 0..9 bytes at the largest stride", buf.bytes(), {"fast_matches": expect}))
    # cut by the block start: the copy of the block's first bytes is found only at its byte c (the entries of positions
    # 0 .. c-1 are overwritten by strings of the same index and another tag), so the backward extension may take c bytes
    for c in (3, 7):
        for _ in range(100):  # (until no slot inside the copied bytes overwrites the entry it is found by)
            buf = Buf(rng, 2 * seg)
            dst = 1500
            buf.copy(c, dst, 40)
            buf.put(dst - c, buf.b[0:c])
            buf.planted[0:c] = True
            h0 = fast_hashes(buf.bytes())
            for i in range(c):
                buf.put(200 + 64 * i, collide(rng, int(h0[i]) ^ 0x100, {}))  # tag bit 0 flipped, same index
            buf.pad(1760, 2040)
            try:
                buf.protect(g, [(c, dst)])
                break
            except RuntimeError:
                pass
        out.append(Case(f"F3 backward extension cut by the block start, {c} bytes", buf.bytes(),
                        {"fast_matches": [(0, dst - c, dst - c, 40 + c)]}))
    # cut by the anchor: w[0:17] is a match found at its 5th byte (a slot), ending 3 bytes before the next slot; w[11:50]
    # is one found at that slot, whose 9 bytes before it agree, of which the 3 after the first match's end are taken
    buf = _quiet_block(g, rng, 5)
    w = rng.bytes(step + 34)  # w[4 + step] lands on the slot dst
    dst = s6 + 64 * step
    s1, s2 = s5 + 64 * step, s5 + 128 * step
    buf.put(s1 - 4, w[:step + 1])             # the first match: w[:step + 1], found at the slot holding w[4]
    buf.differ(s1 + step - 3, w[step + 1])
    buf.put(s2 - 9, w[step - 5:])             # the second: found at dst, agreeing 9 bytes back
    buf.differ(s2 - 10, w[step - 6])
    buf.put(dst - step - 4, w)
    buf.differ(dst - step - 5, buf.b[s1 - 5])
    buf.differ(dst + 30, buf.b[s2 + 30])
    buf.pad(starts[7], starts[7] + 3000)
    buf.protect(g, [(s1, dst - step), (s2, dst)], step)
    out.append(Case("F3 backward extension cut by the previous match", buf.bytes(),
                    {"fast_matches": [(0, dst - step - 4, dst - step - s1, step + 1), (0, dst - 3, dst - s2, 33)]}))
    return out


def f4_stride_and_tail(g, rng) -> List[Case]:
    """1..5 hit-less segments before hits at the stride they leave, on a slot and between two slots; last blocks of
    13..40 bytes."""
    out = []
    starts = _segment_starts(g)
    for quiet in range(1, 6):
        buf = _quiet_block(g, rng, quiet + 1)
        step = 1 << min(quiet, g["max_step_log"])
        s = starts[quiet + 1]
        src, on = s + 16 * step, s + 64 * step
        # between two slots: the copy starts half a stride before a slot, is found there and extended back to its start
        src2, slot2 = s + 128 * step, s + 192 * step
        between = slot2 - step // 2
        buf.copy(src, on, 80)
        buf.copy(src2 - step // 2, between, 80)
        buf.pad(starts[7], starts[7] + 3000)
        out.append(Case(f"F4 hits after {quiet} hit-less segments", buf.bytes(),
                        {"fast_matches": [(0, on, on - src, 80), (0, between, slot2 - src2, 80)]}))
    for t in (13, 14, 16, 17, 20, 24, 31, 40):
        out.append(Case(f"F4 last block of {t} bytes", bytes(300) + rng.bytes(BLOCK - 300) + (b"abcabcab" * 8)[:t], {"last_block": t}))
    return out


def f5_segment_bookkeeping(g, rng) -> List[Case]:
    """31, 32, 33, 64 and 65 matches in one segment (the parser emits 32 sequences at a time); literal runs of 14..17,
    269..271 and 524 bytes between matches; and a run carried across hit-less segments."""
    out = []
    seg = g["seg_slots"]
    for nseq in (31, 32, 33, 64, 65):
        for _ in range(100):  # (until no source's slot overwrites another's table entry)
            buf = Buf(rng, 2 * seg + 200)
            gap = (seg - 40) // nseq
            pairs, expect = [], []
            for i in range(nseq):
                src, dst = 8 + 12 * i, seg + 8 + gap * i  # sources in segment 0, the matches all in segment 1
                buf.copy(src, dst, 6)
                pairs.append((src, dst))
                expect.append((0, dst, dst - src, 6))
            buf.pad(2 * seg, 2 * seg + 190)
            try:
                buf.protect(g, pairs)
                break
            except RuntimeError:
                pass
        out.append(Case(f"F5 {nseq} matches in one segment", buf.bytes(), {"fast_matches": expect}))
    for run in (14, 15, 16, 17, 269, 270, 271, 524):
        for _ in range(100):  # (until no slot inside the copied bytes overwrites a source's entry)
            buf = Buf(rng, 2 * seg + 100)
            a, b = 100, 120 + run
            buf.copy(20, a, 20)
            buf.copy(60, b, 20)
            buf.pad(1300, 2000)
            try:
                buf.protect(g, [(20, a), (60, b)])
                break
            except RuntimeError:
                pass
        out.append(Case(f"F5 literal run of {run} bytes", buf.bytes(),
                        {"fast_matches": [(0, a, a - 20, 20), (0, b, b - 60, 20)]}))
    starts = _segment_starts(g)
    buf = Buf(rng, BLOCK)
    buf.copy(40, 300, 40)
    far = starts[6] + 64 * (1 << g["max_step_log"])
    buf.copy(far - 32 * (1 << g["max_step_log"]), far, 40)
    buf.pad(BLOCK - 3000, BLOCK)
    buf.protect(g, [(40, 300)])
    out.append(Case("F5 literal run carried across hit-less segments", buf.bytes(),
                    {"fast_matches": [(0, 300, 260, 40), (0, far, 32 * (1 << g["max_step_log"]), 40)]}))
    return out


# ------------------------------------------------------------------------------------------------ high-ratio compressor
def h1_depth(g, rng) -> List[Case]:
    """For each level: a 4-byte key whose longest continuation is at the depth-th and at the (depth+1)-th nearest
    occurrence, the nearer ones continuing with a wrong byte; once more with every other nearer occurrence replaced by a
    different key of the same hash, which uses up depth the same way."""
    out = []
    bits = g["hc_hash_bits"]
    for lv, depth in g["depth"].items():
        for place in (depth, depth + 1):
            for with_collisions in (False, True):
                for attempt in range(100):
                    key = rng.bytes(4)
                    hk = hc_hash(key, bits)
                    cont = rng.bytes(24)
                    n_occ = place
                    buf = Buf(rng, 240 + 12 * n_occ + 400)
                    occ = []
                    for j in range(n_occ):  # j = 0 farthest
                        p = 200 + 40 * (j > 0) + 12 * j
                        occ.append(p)
                        if j == 0:
                            buf.put(p, key + cont)
                            continue
                        k = key
                        if with_collisions and j % 2:
                            while True:
                                k = ((((hk << (32 - bits)) | int(rng.integers(1 << (32 - bits)))) * K1_INV) & M32).to_bytes(4, "little")
                                if k != key:
                                    break
                        buf.put(p, k + bytes([cont[0] ^ 0x33]) + rng.bytes(3))
                    probe = occ[-1] + 100
                    buf.put(probe, key + cont)
                    buf.differ(probe + 28, buf.b[occ[0] + 28])
                    buf.differ(probe - 1, buf.b[occ[0] - 1])
                    buf.pad(len(buf.b) - 250, len(buf.b) - 20)
                    data = buf.bytes()
                    a = np.frombuffer(data, np.uint8).astype(np.uint64)
                    n = len(a) - 3
                    h = ((a[:n] | a[1:n + 1] << 8 | a[2:n + 2] << 16 | a[3:n + 3] << 24) * K1 & M32) >> (32 - bits)
                    same = set(np.flatnonzero(h[:probe] == hk).tolist())
                    if same == set(occ):
                        break
                else:
                    raise RuntimeError("no H1 chunk")
                other = lv + 1 if place > depth else lv - 1
                exp = {}
                if native.HC_MIN_LEVEL <= other <= native.HC_MAX_LEVEL:
                    exp["levels_differ"] = [(lv, other)]
                else:  # the level next door does not exist: the match is (or is not) found at this level
                    exp["hc_matches" if place == depth else "hc_absent"] = {(lv, False, False): [(0, probe, probe - occ[0], 28)]}
                out.append(Case(f"H1 level {lv}: longest at the {place}-th nearest" + (", hash collisions between" if with_collisions else ""),
                                data, exp))
    return out


def h2_ties_and_cap(g, rng) -> List[Case]:
    """Equal-length candidates at different distances (the nearer one wins); matches of nice - 1, nice and nice + 1 bytes;
    positions whose cap is the block's last-literals limit rather than nice."""
    out = []
    nice = g["hc_nice"]
    buf = Buf(rng, 3000)
    s = rng.bytes(12)
    for p in (100, 250, 500):
        buf.put(p, s)
    buf.differ(500 + 12, buf.b[250 + 12])
    buf.differ(500 + 12, buf.b[100 + 12])
    buf.differ(250 + 12, buf.b[100 + 12])
    for p in (250, 500):
        buf.differ(p - 1, buf.b[100 - 1])
    buf.differ(499, buf.b[249])
    buf.pad(1500, 2900)
    out.append(Case("H2 equal-length candidates, the nearer wins", buf.bytes(), {"hc_matches": {(5, False, False): [(0, 500, 250, 12)]}}))
    for m in (nice - 1, nice, nice + 1):
        buf = Buf(rng, 3000)
        buf.copy(100, 1000, m)
        buf.pad(1500, 2900)
        out.append(Case(f"H2 match of {m} bytes", buf.bytes(), {"hc_matches": {(5, False, False): [(0, 1000, 900, m)]}}))
    for room in (nice - 2, nice - 1, nice, nice + 1):
        n = 2000
        buf = Buf(rng, n)
        dst = n - LAST_LITERALS - room
        buf.b[dst:] = buf.b[100:100 + n - dst]
        buf.differ(dst - 1, buf.b[99])
        buf.pad(300, 1500)
        out.append(Case(f"H2 cap at the last literals, {room} bytes of room", buf.bytes(),
                        {"hc_matches": {(5, False, False): [(0, dst, dst - 100, room)]}}))
    return out


def h3_linked_window(g, rng) -> List[Case]:
    """X + X: every candidate exactly 65536 back, none allowed.  X + X[1:] + tail: every candidate exactly 65535 back.  A key
    whose nearest occurrence is in the window and whose next one is 65536..65600 back.  Keys whose hash the window wrote
    but the block did not, and both."""
    out = []
    x = rng.bytes(BLOCK)
    out.append(Case("H3 X + X: candidates 65536 back", x + x, {"linked_raw": 1}))
    out.append(Case("H3 X + X[1:] + tail: candidates 65535 back", x + x[1:] + rng.bytes(300), {"linked_offsets": [(1, 65535)]}))
    for far in (65536, 65537, 65600):
        buf = Buf(rng, 2 * BLOCK + 2000)
        key = rng.bytes(40)
        probe = BLOCK + 1000
        buf.put(probe - far, key)             # too far back
        buf.put(probe - 30000, key[:20])      # in the window, shorter
        buf.put(probe, key)
        buf.differ(probe - 30000 + 20, key[20])
        buf.differ(probe - 1, buf.b[probe - far - 1])
        buf.differ(probe - 1, buf.b[probe - 30001])
        buf.pad(BLOCK + 20000, BLOCK + 24000)
        out.append(Case(f"H3 nearest in the window, next {far} back", buf.bytes(), {"linked_offsets": [(1, 30000)]}))
    buf = Buf(rng, 2 * BLOCK + 2000)
    key = rng.bytes(64)
    buf.put(BLOCK - 32, key)        # runs from the window into the block
    buf.put(BLOCK + 5000, key)
    buf.put(BLOCK + 9000, key)      # now the block has written the key's hash too: the nearer block copy wins
    buf.differ(BLOCK + 9000 + 64, buf.b[BLOCK + 5000 + 64])
    buf.differ(BLOCK + 9000 - 1, buf.b[BLOCK + 5000 - 1])
    buf.differ(BLOCK + 5000 - 1, buf.b[BLOCK - 33])
    buf.pad(BLOCK + 20000, BLOCK + 24000)
    out.append(Case("H3 a match from the window into the block", buf.bytes(), {"linked_offsets": [(1, 5032), (1, 4000)]}))
    return out


def h4_optimal(g, rng) -> List[Case]:
    """Long positions 31, 32 and 33 bytes before a parse segment's end, after a short match that reaches into the long one
    (so a parse that did not stop at the long position would take the short match longer); a long position right after
    a window start; literal runs crossing 15 and 270 inside a compressible segment; match lengths 18 and 19; a literal
    run across a segment start."""
    out = []
    nice, seg = g["hc_nice"], g["hc_opt_seg"]

    def fresh():
        buf = Buf(rng, 3 * seg)
        buf.pad(2 * seg + 104, 3 * seg - 100)
        return buf

    for r in (nice - 1, nice, nice + 1):
        buf = fresh()
        s1 = 2 * seg
        x = s1 - r
        long = rng.bytes(nice + 16)
        v = rng.bytes(5)
        buf.put(200, long)
        buf.differ(200 + nice + 16, buf.b[x + nice + 16])
        buf.put(400, v + long[:5])
        buf.differ(410, long[5])
        buf.put(x - 5, v + long)
        buf.differ(x - 6, buf.b[399])
        # at the long position the window stops and the long match is taken; 31 bytes before the end there is none, and
        # the short match's longer form, then the rest of the copy, costs the same and ends on the shorter last match
        exp = {"hc_matches" if r >= nice else "hc_absent": {(5, False, True): [(0, x, x - 200, r)]}}
        out.append(Case(f"H4 long position {r} bytes before a segment end", buf.bytes(), exp))
    buf = fresh()
    long = rng.bytes(2 * nice)
    buf.put(100, long)
    buf.put(1000, long + long[:nice])  # a long match, and a long position right where its window starts again
    buf.differ(100 + 2 * nice, long[0])
    buf.differ(1000 + 3 * nice, long[nice])
    out.append(Case("H4 long position at a window start", buf.bytes(),
                    {"hc_matches": {(5, False, True): [(0, 1000, 900, 2 * nice), (0, 1000 + 2 * nice, 2 * nice, nice)]}}))
    for run in (14, 15, 16, 269, 270, 271):
        buf = fresh()
        buf.copy(100, 600, 20)
        buf.copy(140, 620 + run, 20)
        out.append(Case(f"H4 literal run of {run} inside a compressible segment", buf.bytes(),
                        {"hc_matches": {(5, False, True): [(0, 600, 500, 20), (0, 620 + run, 480 + run, 20)]}}))
    for m in (18, 19):
        buf = fresh()
        buf.copy(100, 900, m)
        # 19 bytes need a length byte more than 18: a literal and the 18 bytes after it cost the same, and end shorter
        out.append(Case(f"H4 match of {m} bytes", buf.bytes(),
                        {"hc_matches": {(5, False, True): [(0, 900 + (m - 18), 800, 18)]}}))
    buf = fresh()
    buf.copy(100, seg - 300, 20)
    buf.copy(200, seg + 300, 20)
    out.append(Case("H4 literal run across a segment start", buf.bytes(),
                    {"hc_matches": {(5, False, True): [(0, seg - 300, seg - 400, 20), (0, seg + 300, seg + 100, 20)]}}))
    return out


TARGETS = [f1_false_hits, f2_near_slots, f3_compare_window, f4_stride_and_tail, f5_segment_bookkeeping,
           h1_depth, h2_ties_and_cap, h3_linked_window, h4_optimal]


def corpus(seed: int = 2026) -> List[Case]:
    g = geometry()
    rng = np.random.default_rng(seed)
    return [c for target in TARGETS for c in target(g, rng)]
