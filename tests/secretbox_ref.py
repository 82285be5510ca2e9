"""XSalsa20-Poly1305 (NaCl's crypto_secretbox) written from the algorithm, on Python integers: the reference the GPU
SecretBox tests compare with.

Nothing here shares code or limb arithmetic with the CUDA kernels or the C oracle.  Salsa20 is the 20-round core over
32-bit words; Poly1305 is h = ((h + m_i) * r) mod 2^130 - 5 on big integers, then (h + s) mod 2^128.  `steer` builds
messages whose Poly1305 accumulator ends on a value of the caller's choice, which random messages reach with
probability about 2^-128: the final reduction, the carries of s and the limb maxima are all reached that way.

A box is PyNaCl's EncryptedMessage: nonce(24) | tag(16) | ciphertext.  The XSalsa20 stream's first 32 bytes are the
Poly1305 key (r | s); the message is XORed with the stream from byte 32 on."""
from __future__ import annotations

import random
from typing import Optional, Tuple

P = (1 << 130) - 5
M32 = 0xFFFFFFFF
SIGMA = (0x61707865, 0x3320646E, 0x79622D32, 0x6B206574)  # "expand 32-byte k"
CLAMP = 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF


def _words(b: bytes):
    return [int.from_bytes(b[i:i + 4], "little") for i in range(0, len(b), 4)]


def _rotl(x: int, n: int) -> int:
    return ((x << n) | (x >> (32 - n))) & M32


def _rounds(x: list) -> list:
    x = list(x)

    def qr(a, b, c, d):
        x[b] ^= _rotl((x[a] + x[d]) & M32, 7)
        x[c] ^= _rotl((x[b] + x[a]) & M32, 9)
        x[d] ^= _rotl((x[c] + x[b]) & M32, 13)
        x[a] ^= _rotl((x[d] + x[c]) & M32, 18)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(5, 9, 13, 1); qr(10, 14, 2, 6); qr(15, 3, 7, 11)  # columns
        qr(0, 1, 2, 3); qr(5, 6, 7, 4); qr(10, 11, 8, 9); qr(15, 12, 13, 14)  # rows
    return x


def _input(key: bytes, in16: bytes) -> list:
    k, n = _words(key), _words(in16)
    return [SIGMA[0], k[0], k[1], k[2], k[3], SIGMA[1], n[0], n[1], n[2], n[3], SIGMA[2], k[4], k[5], k[6], k[7], SIGMA[3]]


def hsalsa20(key: bytes, nonce16: bytes) -> bytes:
    """The XSalsa20 subkey: words 0, 5, 10, 15, 6, 7, 8, 9 of the Salsa20 rounds, without the feed-forward."""
    assert len(key) == 32 and len(nonce16) == 16
    x = _rounds(_input(key, nonce16))
    return b"".join(x[i].to_bytes(4, "little") for i in (0, 5, 10, 15, 6, 7, 8, 9))


def salsa20_block(key: bytes, nonce8: bytes, counter: int) -> bytes:
    """64 bytes of the Salsa20 stream: block `counter` (a 64-bit block number) under key and an 8-byte nonce."""
    assert len(key) == 32 and len(nonce8) == 8 and 0 <= counter < 1 << 64
    x0 = _input(key, nonce8 + counter.to_bytes(8, "little"))
    return b"".join(((a + b) & M32).to_bytes(4, "little") for a, b in zip(_rounds(x0), x0))


_STREAMS = {}


def xsalsa20(key: bytes, nonce: bytes, n: int) -> bytes:
    """The first n bytes of the XSalsa20 stream.  Kept per key and nonce and extended on demand: the tests ask for one
    stream many times."""
    assert len(key) == 32 and len(nonce) == 24
    key, nonce = bytes(key), bytes(nonce)
    got = _STREAMS.get((key, nonce), b"")
    if len(got) < n:
        sub = hsalsa20(key, nonce[:16])
        got += b"".join(salsa20_block(sub, nonce[16:], b) for b in range(len(got) // 64, (n + 63) // 64))
        _STREAMS[(key, nonce)] = got
    return got[:n]


def xor(a: bytes, b: bytes) -> bytes:
    """a XOR the first len(a) bytes of b."""
    n = len(a)
    return (int.from_bytes(a, "little") ^ int.from_bytes(b[:n], "little")).to_bytes(n, "little")


def keystream(key: bytes, nonce: bytes, n: int) -> bytes:
    """The n stream bytes an n-byte message is XORed with: bytes [32, 32 + n) of the XSalsa20 stream."""
    return xsalsa20(key, nonce, 32 + n)[32:]


def poly_key(key: bytes, nonce: bytes) -> Tuple[int, int]:
    """(r, s) of the box's one-time Poly1305 key: r clamped, both as integers."""
    k = xsalsa20(key, nonce, 32)
    return int.from_bytes(k[:16], "little") & CLAMP, int.from_bytes(k[16:], "little")


def blocks(msg: bytes):
    """Poly1305's block values: 16 bytes little-endian plus 2^(8 * length), so a full block lies in [2^128, 2^129)."""
    return [int.from_bytes(msg[i:i + 16], "little") + (1 << (8 * len(msg[i:i + 16]))) for i in range(0, len(msg), 16)]


def poly1305_h(r: int, msg: bytes) -> int:
    """The accumulator before s is added, fully reduced: in [0, p)."""
    h = 0
    for m in blocks(msg):
        h = (h + m) * r % P
    return h


def tag_of(h: int, s: int) -> bytes:
    return ((h + s) % (1 << 128)).to_bytes(16, "little")


def poly1305(key32: bytes, msg: bytes) -> bytes:
    """One-time authenticator of msg under any 32-byte key r | s (r is clamped here, as the algorithm says)."""
    assert len(key32) == 32
    r = int.from_bytes(key32[:16], "little") & CLAMP
    return tag_of(poly1305_h(r, msg), int.from_bytes(key32[16:], "little"))


def box_tag(key: bytes, nonce: bytes, ct: bytes) -> bytes:
    """The tag a box of ciphertext ct carries under key and nonce."""
    return poly1305(xsalsa20(key, nonce, 32), ct)


def seal(key: bytes, nonce: bytes, msg: bytes) -> bytes:
    """nonce | tag | ciphertext, PyNaCl's SecretBox(key).encrypt(msg, nonce)."""
    ct = xor(msg, keystream(key, nonce, len(msg)))
    return nonce + box_tag(key, nonce, ct) + ct


def open(key: bytes, nonce: bytes, tag_ct: bytes) -> Optional[bytes]:  # noqa: A001 (NaCl's name for it)
    """The plaintext of tag | ciphertext, or None if the tag is not the ciphertext's."""
    if len(tag_ct) < 16 or box_tag(key, nonce, tag_ct[16:]) != tag_ct[:16]:
        return None
    return xor(tag_ct[16:], keystream(key, nonce, len(tag_ct) - 16))


def steer(r: int, msg: bytes, target: int, at: int = 0, rng: Optional[random.Random] = None) -> Optional[bytes]:
    """msg with its full 16-byte block `at` solved mod p so that poly1305_h(r, result) == target.

    A full block's value has to lie in [2^128, 2^129), which about a quarter of the solutions do.  When it does not,
    another block (drawn by rng; a short last block keeps its length) is replaced with random bytes and block `at` is
    solved again.  A message of one block cannot be redrawn: then None, and the caller picks another r.  (A single
    block never reaches h = 0: p is prime, so m * r is 0 mod p only for r = 0.)"""
    assert 0 < r < P and 0 <= target < P and len(msg) >= 16 * (at + 1)
    rng = rng or random.Random(target ^ r)
    n = (len(msg) + 15) // 16
    others = [j for j in range(n) if j != at]
    w_inv = pow(pow(r, n - at, P), -1, P)  # block `at` enters h weighted by r^(n - at)
    msg = bytearray(msg)
    while True:
        msg[16 * at:16 * at + 16] = bytes(16)
        rest = poly1305_h(r, bytes(msg)) - (1 << 128) * pow(r, n - at, P)  # h without block at's value
        m = (target - rest) * w_inv % P
        if 1 << 128 <= m < 1 << 129:
            msg[16 * at:16 * at + 16] = (m - (1 << 128)).to_bytes(16, "little")
            return bytes(msg)
        if not others:
            return None
        j = rng.choice(others)
        msg[16 * j:16 * j + 16] = rng.randbytes(len(msg[16 * j:16 * j + 16]))
