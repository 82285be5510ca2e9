"""The big-integer SecretBox reference (tests/secretbox_ref.py) against PyNaCl, `cryptography`'s Poly1305 and the C
oracle, on random messages and on messages steered to the accumulator values random ones never reach.  The GPU
SecretBox edge tests compare with this reference alone, so it is pinned here, without a GPU."""
import random

import pytest

import oracle
import secretbox_ref as ref

P = ref.P
RNG = random.Random(1305)
LENS = [0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 4095, 4096, 4097, 65537]
# h (before s) where a Poly1305 implementation is usually wrong: the final subtraction (0..4 are h + p unreduced),
# just below p, and the bits 2^128 and 2^129 that s never reaches
TARGETS = [0, 1, 2, 3, 4, P - 6, P - 5, P - 1, (1 << 128) - 1, 1 << 128, 1 << 129]


def steered(key: bytes, nonce: bytes, n: int, target: int, rng: random.Random) -> bytes:
    """A ciphertext of n bytes (at least 32) whose Poly1305 accumulator under (key, nonce) is target."""
    r, _ = ref.poly_key(key, nonce)
    return ref.steer(r, rng.randbytes(n), target, rng=rng)


def test_reference_equals_pynacl_on_random_messages():
    nacl_secret = pytest.importorskip("nacl.secret")
    for n in LENS:
        key, nonce, msg = RNG.randbytes(32), RNG.randbytes(24), RNG.randbytes(n)
        box = bytes(nacl_secret.SecretBox(key).encrypt(msg, nonce))
        assert ref.seal(key, nonce, msg) == box, n
        assert ref.open(key, nonce, box[24:]) == msg
        assert ref.keystream(key, nonce, n) == ref.xor(msg, box[40:])
        for k in (24, 39, len(box) - 1):  # a tag byte, the last tag byte, the last ciphertext byte
            bad = bytearray(box)
            bad[k] ^= 0x80
            assert ref.open(key, nonce, bytes(bad[24:])) is None, (n, k)


def test_reference_equals_pynacl_on_steered_messages():
    nacl_secret = pytest.importorskip("nacl.secret")
    for target in TARGETS:
        for n in (32, 33, 47, 4096, 4111):
            key, nonce = RNG.randbytes(32), RNG.randbytes(24)
            ct = steered(key, nonce, n, target, RNG)
            msg = ref.xor(ct, ref.keystream(key, nonce, n))
            r, s = ref.poly_key(key, nonce)
            box = bytes(nacl_secret.SecretBox(key).encrypt(msg, nonce))
            assert box == nonce + ref.tag_of(target, s) + ct == ref.seal(key, nonce, msg), (target, n)
            if target < 5:  # the tag a Poly1305 without its final subtraction writes
                forged = nonce + ref.tag_of(target + P, s) + ct
                assert forged != box and ref.open(key, nonce, forged[24:]) is None
                with pytest.raises(Exception):
                    nacl_secret.SecretBox(key).decrypt(forged)


def _poly_keys():
    """r | s keys chosen at the arithmetic's ends: every clamp bit of r set (and every other bit too, which the clamp
    drops), r = 0, s = 0 and s = 2^128 - 1."""
    r_max, r_all = ref.CLAMP.to_bytes(16, "little"), b"\xff" * 16
    s_zero, s_max = bytes(16), b"\xff" * 16
    rand_r, rand_s = RNG.randbytes(16), RNG.randbytes(16)
    return [r + s for r in (r_max, r_all, bytes(16), rand_r) for s in (s_zero, s_max, rand_s)]


@pytest.mark.parametrize("key32", _poly_keys(), ids=lambda k: k.hex()[:8] + ".." + k.hex()[32:40])
def test_poly1305_equals_cryptography_for_chosen_keys(key32):
    poly = pytest.importorskip("cryptography.hazmat.primitives.poly1305")
    r = int.from_bytes(key32[:16], "little") & ref.CLAMP
    msgs = [RNG.randbytes(n) for n in (0, 1, 15, 16, 17, 64, 1000)] + [b"\xff" * 4096, b"\xff" * 4095, bytes(4096)]
    if r:
        msgs += [ref.steer(r, RNG.randbytes(n), t, rng=RNG) for t in TARGETS for n in (32, 47)]
    for m in msgs:
        assert ref.poly1305(key32, m) == poly.Poly1305.generate_tag(key32, m), len(m)
    if not r:  # r = 0: every message's tag is s
        assert all(ref.poly1305(key32, m) == key32[16:] for m in msgs)


def test_reference_equals_oracle():
    keys = [bytes(32), b"\xff" * 32, RNG.randbytes(32)]
    nonces = [bytes(24), b"\xff" * 24, RNG.randbytes(16) + b"\xff" * 8]
    for key in keys:
        for nonce in nonces:
            for n in (0, 1, 16, 17, 64, 65, 1000, 4097):
                msg = RNG.randbytes(n)
                boxed = oracle.secretbox_seal(key, nonce, msg)
                assert nonce + boxed == ref.seal(key, nonce, msg), (key[:1], nonce[:1], n)
                assert oracle.secretbox_open(key, nonce, boxed) == msg == ref.open(key, nonce, boxed)
    key, nonce = keys[2], nonces[2]
    r, s = ref.poly_key(key, nonce)
    for target in TARGETS:
        ct = steered(key, nonce, 4111, target, RNG)
        msg = ref.xor(ct, ref.keystream(key, nonce, len(ct)))
        assert oracle.secretbox_seal(key, nonce, msg) == ref.tag_of(target, s) + ct == ref.seal(key, nonce, msg)[24:]
        assert oracle.secretbox_open(key, nonce, ref.tag_of(target, s) + ct) == msg
        if target < 5:
            with pytest.raises(ValueError):
                oracle.secretbox_open(key, nonce, ref.tag_of(target + P, s) + ct)


def test_steer_reaches_its_target():
    rng = random.Random(7)
    for _ in range(40):
        r = int.from_bytes(rng.randbytes(16), "little") & ref.CLAMP
        for target in TARGETS + [rng.randrange(P)]:
            for n in (16, 32, 33, 47, 48, 16 * 257, 16 * 256 + 15):
                at = rng.randrange(n // 16)
                msg = rng.randbytes(n)
                got = ref.steer(r, msg, target, at=at, rng=rng)
                if got is None:  # nothing else to redraw
                    assert n == 16
                    continue
                assert len(got) == n and ref.poly1305_h(r, got) == target, (r, target, n, at)
    # a single block reaches a target for about a quarter of r, and never reaches 0
    hits = sum(ref.steer(int.from_bytes(rng.randbytes(16), "little") & ref.CLAMP, bytes(16), 1) is not None for _ in range(400))
    assert 50 < hits < 150
    assert all(ref.steer(int.from_bytes(rng.randbytes(16), "little") & ref.CLAMP, bytes(16), 0) is None for _ in range(20))
