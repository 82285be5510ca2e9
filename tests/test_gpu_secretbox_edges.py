"""GPU SecretBox (XSalsa20-Poly1305, csrc/secretbox.cuh) at the values random boxes never reach, against the big-integer
reference in tests/secretbox_ref.py alone (pinned to PyNaCl, `cryptography` and the C oracle by test_secretbox_ref.py).

Every box here is crafted: its ciphertext is chosen, and the plaintext is that ciphertext XOR the reference keystream.
Boxes are opened by sky_decode(SKY_F_MD5 | SKY_F_E2EE) into guarded buffers, and the plaintexts are sealed through
ChunkStage.process(compress=False, encrypt=True), which must give the crafted box byte for byte.

  * Steered tags: ciphertexts solved so that Poly1305's accumulator h ends on 0..4 (where the tag kernel's unreduced sum
    is h + p and only its final subtraction makes the tag right), just below p, and on 2^128 - 1, 2^128, 2^129.
  * Carries when s is added: h chosen so that h + s carries out of each 32-bit tag word and out of 2^128.
  * Limb maxima: all-0xFF ciphertexts drive every 26-bit limb of every thread's partial sum to its largest value.
  * The tag comparison: each of the 128 tag bits flipped alone.
  * All-zero and all-0xFF keys and nonces, and nonces whose Salsa20 stream words are all 0xFF.
  * All of them in one ragged batch, between ordinary random boxes."""
import hashlib
import random
from dataclasses import dataclass
from typing import List, Optional

import pytest

import secretbox_ref as ref
from skyplane_b200 import native
from skyplane_b200.stage import ChunkStage
from test_gpu_receive_raw import RAW_BOX, sky_decode, untouched

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300, method="thread")]
P = ref.P
KEY = random.Random(2025).randbytes(32)
NONCE = random.Random(2026).randbytes(24)
TARGETS = [0, 1, 2, 3, 4, P - 6, P - 5, P - 1, (1 << 128) - 1, 1 << 128, 1 << 129]
NBLOCKS = [1, 2, 255, 256, 257, 511, 512, 513, 4097]  # the tag kernel runs 256 threads per box
TAILS = [0, 1, 15]  # bytes in a short last block (0: the message ends in a full block)


@dataclass
class Case:
    label: str
    nonce: bytes
    ct: bytes
    tag: bytes
    plain: Optional[bytes]  # None: the tag is not the ciphertext's, the box must not open

    @property
    def box(self) -> bytes:
        return self.nonce + self.tag + self.ct


def genuine(key: bytes, nonce: bytes, ct: bytes, label: str) -> Case:
    r, s = ref.poly_key(key, nonce)
    return Case(label, nonce, ct, ref.tag_of(ref.poly1305_h(r, ct), s), ref.xor(ct, ref.keystream(key, nonce, len(ct))))


def lengths():
    """(blocks, tail bytes) of the crafted messages: every block count ending in a full block, and from 2 blocks on a
    version whose last block is short."""
    return [(nb, t) for nb in NBLOCKS for t in TAILS if t == 0 or nb >= 2]


def msg_len(nb: int, tail: int) -> int:
    return 16 * nb if not tail else 16 * (nb - 1) + tail


def steered(key: bytes, nonce: bytes, nb: int, tail: int, h: int, rng: random.Random) -> Case:
    """A genuine box whose accumulator is h.  One block alone fixes m = h / r, so a one-block message looks for a nonce
    (a new r) under which m is a full block's value."""
    for k in range(256 if nb == 1 else 1):  # (steer always succeeds on two blocks or more)
        n = nonce[:23] + bytes([(nonce[23] + k) & 0xFF])
        r, _ = ref.poly_key(key, n)
        ct = ref.steer(r, rng.randbytes(msg_len(nb, tail)), h, rng=rng)
        if ct is not None:
            assert ref.poly1305_h(r, ct) == h
            return genuine(key, n, ct, f"h={h:#x} blocks={nb} tail={tail}")
    raise AssertionError(f"no nonce steers one block to h = {h:#x}")


def steered_cases(key: bytes, nonce: bytes, rng: random.Random) -> List[Case]:
    """Every target at every length; for h = 0..4 also the box that carries the tag of h + p (the right tag - 5 mod
    2^128), which is what a tag kernel without its final subtraction writes, and which must not open."""
    cases = []
    for h in TARGETS:
        for nb, tail in lengths():
            if h == 0 and nb == 1:
                continue  # unreachable: see ref.steer
            c = steered(key, nonce, nb, tail, h, rng)
            cases.append(c)
            if h < 5:
                _, s = ref.poly_key(key, c.nonce)
                assert ref.tag_of(h + P, s) == ((int.from_bytes(c.tag, "little") - 5) % (1 << 128)).to_bytes(16, "little")
                cases.append(Case(c.label + " tag(h+p)", c.nonce, c.ct, ref.tag_of(h + P, s), None))
    return cases


def carry_targets(s: int) -> List[int]:
    """h whose low word k sums with s's to exactly 2^32 (k = 0..3: a carry out of tag word k, out of 2^128 for k = 3),
    the h whose sum with s ripples through all four words to 2^128 (tag 0), that h + 2^128 and + 2^129, and
    2^128 - 1 - s (no carry at all: tag all ones)."""
    out = []
    for k in range(4):
        sk = (s >> (32 * k)) & ref.M32
        if sk:
            out.append(((1 << 32) - sk) << (32 * k))
    low = (1 << 128) - s if s else 1 << 128
    return out + [low % (1 << 128), low % (1 << 128) + (1 << 128), low % (1 << 128) + (1 << 129), (1 << 128) - 1 - s]


def carries_out_of(h: int, s: int, k: int) -> bool:
    m = 1 << (32 * (k + 1))
    return (h % m + s % m) >= m


def carry_cases(key: bytes, rng: random.Random) -> List[Case]:
    cases, reached = [], set()
    for i in range(3):  # three nonces: three values of s
        nonce = NONCE[:20] + bytes([i, 0xC0, 0xDE, 0x55])
        _, s = ref.poly_key(key, nonce)
        for h in carry_targets(s):
            reached |= {k for k in range(4) if carries_out_of(h, s, k)}
            for nb, tail in ((2, 0), (257, 0), (513, 15), (4097, 0)):
                cases.append(steered(key, nonce, nb, tail, h, rng))
                cases[-1].label += f" s={s:#x}"
    assert reached == {0, 1, 2, 3}  # each word's carry is reached, the one out of 2^128 included
    return cases


def limb_cases(key: bytes, nonce: bytes) -> List[Case]:
    """All-0xFF ciphertexts (every limb of every block at its largest), all-zero ones, and 0xFF blocks with a short
    0xFF or zero tail."""
    cases = []
    for nb, tail in lengths():
        n = msg_len(nb, tail)
        cases.append(genuine(key, nonce, b"\xff" * n, f"0xff*{n}"))
        cases.append(genuine(key, nonce, bytes(n), f"0x00*{n}"))
        if tail:
            cases.append(genuine(key, nonce, b"\xff" * (n - tail) + bytes(tail), f"0xff*{n - tail}+0x00*{tail}"))
    return cases


def flip_cases(base: Case) -> List[Case]:
    """The box itself and the 128 boxes that differ from it in one tag bit."""
    out = [base]
    for bit in range(128):
        tag = bytearray(base.tag)
        tag[bit // 8] ^= 1 << (bit % 8)
        out.append(Case(f"{base.label} tag bit {bit}", base.nonce, base.ct, bytes(tag), None))
    return out


def random_case(key: bytes, rng: random.Random) -> Case:
    """An ordinary box: random content of a ragged length, under one of a few nonces (whose streams the reference
    computes once)."""
    nonce = random.Random(rng.randrange(4)).randbytes(24)
    return genuine(key, nonce, rng.randbytes(rng.choice([0, 1, 17, 1000, 4096, 70001])), "random")


@pytest.fixture(scope="module")
def stage():
    s = ChunkStage(0, max_batch_bytes=48 << 20, max_chunks=1536, n_slots=1)
    s.set_e2ee_key(KEY)
    yield s
    s.close()


def check(stage: ChunkStage, cases: List[Case]):
    """Open every box on the GPU, and seal every genuine box's plaintext: each status, output, digest and box must be
    the reference's."""
    _, st, dg, out, _ = sky_decode(stage.ctx, [c.box for c in cases], [len(c.ct) for c in cases], RAW_BOX)
    for c, s, d, o in zip(cases, st, dg, out):
        if c.plain is not None:
            assert s == 0, c.label
            assert o[:len(c.plain)] == c.plain and untouched(o[len(c.plain):]), c.label
            assert d == hashlib.md5(c.plain).digest(), c.label
        else:
            assert s == native.D_AUTH, c.label
            assert untouched(o) and d == bytes(16), c.label  # no plaintext escapes a forged box
    sealed = [c for c in cases if c.plain is not None]
    res = stage.process([c.plain for c in sealed], compress=False, encrypt=True, nonces=b"".join(c.nonce for c in sealed))
    for c, r in zip(sealed, res):
        assert bytes(r.frame) == c.box, c.label
        assert r.md5 == hashlib.md5(c.plain).digest(), c.label


def test_steered_tags(stage):
    check(stage, steered_cases(KEY, NONCE, random.Random(1)))


def test_carries_when_s_is_added(stage):
    check(stage, carry_cases(KEY, random.Random(2)))


def test_limb_maxima(stage):
    check(stage, limb_cases(KEY, NONCE))


def tag_bit_cases(rng: random.Random) -> List[Case]:
    bases = [genuine(KEY, NONCE, rng.randbytes(1000), "random 1000"), steered(KEY, NONCE, 2, 1, 1, rng),
             genuine(KEY, NONCE, b"\xff" * (16 * 4097), "0xff*4097 blocks")]
    return [c for b in bases for c in flip_cases(b)]


def test_every_tag_bit_is_compared(stage):
    check(stage, tag_bit_cases(random.Random(3)))


KEYS = {"zero": bytes(32), "ones": b"\xff" * 32, "random": random.Random(2027).randbytes(32)}
NONCES = {"zero": bytes(24), "ones": b"\xff" * 24, "stream_words_ones": random.Random(2028).randbytes(16) + b"\xff" * 8}


@pytest.mark.parametrize("key_name", list(KEYS))
def test_edge_keys_and_nonces(key_name):
    """Each key in a Context of its own; under it the all-zero and all-0xFF nonces, and one whose nonce[16:24] (the
    Salsa20 input words next to the block counter) is all 0xFF."""
    key, rng = KEYS[key_name], random.Random(key_name)
    cases = []
    for nonce_name, nonce in NONCES.items():
        for n in (0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 4097, 16 * 4097 + 15):
            cases.append(genuine(key, nonce, rng.randbytes(n), f"{nonce_name} random {n}"))
        cases.append(genuine(key, nonce, b"\xff" * (16 * 4097), f"{nonce_name} 0xff*4097 blocks"))
        _, s = ref.poly_key(key, nonce)
        for h in (1, 4, P - 1, carry_targets(s)[-4]):  # (-4: the h whose sum with s ripples through every tag word)
            cases.append(steered(key, nonce, 513, 0, h, rng))
            cases[-1].label += f" {nonce_name}"
            cases.append(Case(cases[-1].label + " tag(h+p)", nonce, cases[-1].ct, ref.tag_of(h + P, s), None))
    st = ChunkStage(0, max_batch_bytes=8 << 20, max_chunks=128, n_slots=1)
    try:
        st.set_e2ee_key(key)
        check(st, cases)
    finally:
        st.close()


def test_mixed_batch(stage):
    """Every case above under the module's key, shuffled into one ragged batch with ordinary random boxes between
    them: each chunk's status, output, digest and seal must be its own."""
    rng = random.Random(4)
    crafted = (steered_cases(KEY, NONCE, random.Random(1)) + carry_cases(KEY, random.Random(2)) + limb_cases(KEY, NONCE)
               + tag_bit_cases(random.Random(3)))
    rng.shuffle(crafted)
    batch = []
    for c in crafted:
        batch.append(c)
        if rng.random() < 0.3:
            batch.append(random_case(KEY, rng))
    assert len(batch) <= stage.max_chunks and sum(len(c.box) for c in batch) <= stage.max_batch_bytes  # one batch
    check(stage, batch)
