"""Python face of tools/lz4_tile_model.c, the sequential CPU twin of the GPU block compressor (development / test tool,
not product code).  frame(data) assembles the LZ4 frame the GPU stage must emit byte for byte."""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
_SO = ROOT / "tools" / "bin" / "liblz4tile.so"
_SRC = ROOT / "tools" / "lz4_tile_model.c"
_lib = None


class Opts(ctypes.Structure):
    _fields_ = [("entries", ctypes.c_int), ("seg_slots", ctypes.c_int), ("max_step_log", ctypes.c_int), ("back_ext", ctypes.c_int),
                ("clip", ctypes.c_int), ("group_lag", ctypes.c_int), ("near_mask", ctypes.c_int)]


class Stats(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in ("probes", "hits", "accepted", "segments")]


def kernel_opts(entries: int = 4096, seg_slots: int = 1024, max_step_log: int = 4) -> Opts:
    """The options the kernel in skyplane_b200/csrc/lz4.cuh implements."""
    return Opts(entries, seg_slots, max_step_log, 1, 1, 1, 0x8C)


def lib():
    global _lib
    if _lib is None:
        _SO.parent.mkdir(exist_ok=True)
        if not _SO.exists() or _SO.stat().st_mtime < _SRC.stat().st_mtime:
            subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", str(_SO), str(_SRC)])
        _lib = ctypes.CDLL(str(_SO))
        _lib.tile_compress_block.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER(Opts)]
        _lib.tile_compress_block.restype = ctypes.c_uint32
        _lib.tile_compress_block_linked.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER(Opts), ctypes.c_uint32]
        _lib.tile_compress_block_linked.restype = ctypes.c_uint32
    return _lib


def _xxh32_small(b: bytes) -> int:  # XXH32, seed 0, inputs < 16 bytes (the frame descriptor)
    P1, P2, P3, P4, P5, M = 2654435761, 2246822519, 3266489917, 668265263, 374761393, 0xFFFFFFFF
    rotl = lambda x, s: ((x << s) | (x >> (32 - s))) & M  # noqa: E731
    h = (P5 + len(b)) & M
    i = 0
    while i + 4 <= len(b):
        h = (rotl((h + int.from_bytes(b[i:i + 4], "little") * P3) & M, 17) * P4) & M
        i += 4
    while i < len(b):
        h = (rotl((h + b[i] * P5) & M, 11) * P1) & M
        i += 1
    h ^= h >> 15
    h = (h * P2) & M
    h ^= h >> 13
    h = (h * P3) & M
    return h ^ (h >> 16)


SEED = 65536  # linked: positions of the previous window that seed a block's table (the rule DESIGN §4.2 measures)


def blocks(data: bytes, o: Opts, linked: bool = False, seed: int = SEED):
    """-> list of (compressed size or 0 when stored raw, block bytes as they appear in the frame).  linked:
    blocks after the first may match into the previous 64 KiB window, from a table seeded with its last `seed` positions."""
    L = lib()
    buf = ctypes.create_string_buffer(65536 + 4096)
    src = ctypes.create_string_buffer(bytes(data), len(data)) if linked else None
    out = []
    for pos in range(0, len(data), 65536):
        blk = data[pos:pos + 65536]
        if linked and pos:
            c = L.tile_compress_block_linked(ctypes.addressof(src) + pos, len(blk), buf, ctypes.byref(o), seed)
        else:
            c = L.tile_compress_block(blk, len(blk), buf, ctypes.byref(o))
        out.append((c, buf.raw[:c] if c else blk))
    return out


def assemble(n: int, blks, block_checksum: bool = False, linked: bool = False) -> bytes:
    """The stage's frame around an n-byte chunk's blocks [(compressed size or 0 when stored raw, block bytes)];
    block_checksum (SKY_F_BLOCK_CHECKSUM): FLG's B.Checksum bit, and u32le XXH32 of every block's bytes behind them;
    linked (linked-block mode): FLG's B.Indep bit clear when the chunk has more than one block -- liblz4 declares a frame
    of at most one block independent whatever blockMode asks for, and so does this header."""
    flg = (0x10 if block_checksum else 0) | (0 if linked and n > 65536 else 0x20)
    if not n:
        d = bytes([0x40 | flg, 0x40])
        return bytes([0x04, 0x22, 0x4D, 0x18]) + d + bytes([(_xxh32_small(d) >> 8) & 0xFF]) + bytes(4)
    d = bytes([0x48 | flg, 0x40]) + n.to_bytes(8, "little")
    fr = bytearray(bytes([0x04, 0x22, 0x4D, 0x18]) + d + bytes([(_xxh32_small(d) >> 8) & 0xFF]))
    for c, b in blks:
        fr += (c if c else (len(b) | 0x80000000)).to_bytes(4, "little") + b
        if block_checksum:
            fr += xxh32(b).to_bytes(4, "little")
    return bytes(fr + bytes(4))


def xxh32(b: bytes) -> int:
    """XXH32 (seed 0) of any input, from the project's C oracle."""
    import oracle

    return oracle.xxh32(b)


def frame(data: bytes, o: Opts | None = None, block_checksum: bool = False, linked: bool = False) -> bytes:
    return assemble(len(data), blocks(data, o or kernel_opts(), linked), block_checksum, linked)
