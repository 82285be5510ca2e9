"""Python face of tools/lz4hc_model.c, the sequential CPU twin of the high-ratio (SKY_F_HC) block compressor (development /
test tool, not product code).  frame(data) is the LZ4 frame the GPU stage must emit byte for byte with SKY_F_HC, and
frame(data, linked=True) the one it emits with SKY_F_HC | SKY_F_LINKED, and frame(data, optimal=True) the one it emits with
SKY_F_HC | SKY_F_OPTIMAL (parse segments of OPT_SEG bytes, sky_kernel_config(8))."""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

from tools import tile_model

ROOT = Path(__file__).resolve().parent.parent
_SO = ROOT / "tools" / "bin" / "liblz4hc.so"
_SRC = ROOT / "tools" / "lz4hc_model.c"
_lib = None


class Opts(ctypes.Structure):
    _fields_ = [("depth", ctypes.c_int), ("hash_bits", ctypes.c_int), ("nice", ctypes.c_int)]


def kernel_opts(depth: int = 16, hash_bits: int = 14, nice: int = 32, level: int | None = None) -> Opts:
    """The constants skyplane_b200/csrc/lz4hc.cuh is built with (sky_kernel_config(4), (5), (6)); `level` (3..9,
    SKY_F_HC_LEVEL) replaces the default level's depth with that level's, 2**(level - 1)."""
    if level is not None:
        if not 3 <= level <= 9:
            raise ValueError(f"high-ratio levels are 3..9, not {level}")
        depth = 1 << (level - 1)
    return Opts(depth, hash_bits, nice)


def lib():
    global _lib
    if _lib is None:
        _SO.parent.mkdir(exist_ok=True)
        if not _SO.exists() or _SO.stat().st_mtime < _SRC.stat().st_mtime:
            subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", str(_SO), str(_SRC)])
        _lib = ctypes.CDLL(str(_SO))
        _lib.hc_compress_block.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER(Opts)]
        _lib.hc_compress_block.restype = ctypes.c_uint32
        _lib.hc_compress_block_linked.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER(Opts)]
        _lib.hc_compress_block_linked.restype = ctypes.c_uint32
        _lib.hc_compress_block_opt.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p,
                                               ctypes.POINTER(Opts)]
        _lib.hc_compress_block_opt.restype = ctypes.c_uint32
    return _lib


WINDOW = 65536  # linked: source bytes before a block (after the chunk's first) that its matches may reach
OPT_SEG = 2048  # the kernel's optimal-parse segment (sky_kernel_config(8))


def blocks(data: bytes, o: Opts, linked: bool = False, optimal: bool = False, seg: int = OPT_SEG):
    """-> list of (compressed size or 0 when stored raw, block bytes as they appear in the frame).  linked: blocks after
    the first see the previous 64 KiB of the chunk (hc_compress_block_linked).  optimal: the optimal parse with segments
    of `seg` bytes, 0 = one per block (hc_compress_block_opt)."""
    L = lib()
    buf = ctypes.create_string_buffer(65536 + 4096)
    src = ctypes.create_string_buffer(bytes(data), len(data)) if (linked or optimal) else None
    out = []
    for pos in range(0, len(data), 65536):
        blk = data[pos:pos + 65536]
        if optimal:
            c = L.hc_compress_block_opt(ctypes.addressof(src) + pos, len(blk), min(pos, WINDOW) if linked else 0, seg, buf,
                                        ctypes.byref(o))
        elif linked:
            c = L.hc_compress_block_linked(ctypes.addressof(src) + pos, len(blk), min(pos, WINDOW), buf, ctypes.byref(o))
        else:
            c = L.hc_compress_block(blk, len(blk), buf, ctypes.byref(o))
        out.append((c, buf.raw[:c] if c else blk))
    return out


def frame(data: bytes, o: Opts | None = None, block_checksum: bool = False, linked: bool = False, optimal: bool = False,
          seg: int = OPT_SEG) -> bytes:
    return tile_model.assemble(len(data), blocks(data, o or kernel_opts(), linked, optimal, seg), block_checksum, linked)


def liblz4_frame(data: bytes, level: int, linked: bool = False, content_checksum: bool = False, block_checksum: bool = False) -> bytes:
    """liblz4's frame at compression `level` (>= 3: its HC search), 64 KiB blocks, independent unless `linked` -- what the
    high-ratio mode is compared with; with LZ4's content / block checksums (XXH32) when asked for."""
    import oracle.reflib as ref

    L = ref._lib()
    ptr, n, _keep = ref._addr(data)
    prefs = ref._prefs(n)
    prefs.compressionLevel = level
    prefs.frameInfo.blockMode = 0 if linked else 1
    prefs.frameInfo.contentChecksumFlag = int(content_checksum)
    prefs.frameInfo.blockChecksumFlag = int(block_checksum)
    cap = L.LZ4F_compressFrameBound(n, ctypes.byref(prefs))
    out = ctypes.create_string_buffer(cap)
    r = L.LZ4F_compressFrame(ctypes.cast(out, ctypes.c_void_p), cap, ptr, n, ctypes.byref(prefs))
    if L.LZ4F_isError(r):
        raise ValueError(L.LZ4F_getErrorName(r).decode())
    return out.raw[:r]
