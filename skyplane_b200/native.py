"""ctypes face of libskychunk.so (include/skychunk.h).  No torch, no numpy required.

The library is CUDA-only: if it is missing it is built with nvcc; if nvcc or a GPU is missing the
calls raise ``SkyChunkError`` -- there is deliberately no CPU fallback on the product path.
"""
from __future__ import annotations

import array
import ctypes
from pathlib import Path
from typing import Optional, Sequence

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libskychunk.so"

SKY_OK = 0
SKY_E_INVALID, SKY_E_NOGPU, SKY_E_CUDA, SKY_E_CAPACITY, SKY_E_BUSY, SKY_E_TICKET, SKY_E_NOMEM, SKY_E_NOKEY = -1, -2, -3, -4, -5, -6, -7, -8
F_LZ4, F_MD5, F_E2EE, F_HC, F_CHECKSUM, F_BLOCK_CHECKSUM = 1, 2, 16, 32, 64, 128
F_VERIFY = 1 << 12  # every frame is checked against its chunk on the GPU; one that fails is sent as its stored-block frame
F_LINKED = 1 << 13  # with F_HC only: linked blocks (python-lz4's block_linked), matches may reach into the previous 64 KiB
F_OPTIMAL = 1 << 14  # with F_HC only: the optimal parse (sequences chosen by their cost in bytes) over the same match search
# sky_submit only, with F_LZ4: a chunk whose frame is not smaller than the chunk is sent as itself (wait_ex says which)
F_PASSTHROUGH = 1 << 15
CHECKSUM_BYTES = 4  # F_CHECKSUM: the content checksum (u32le XXH32) behind the EndMark; F_BLOCK_CHECKSUM: as many per block
BLOCK_BYTES = 65536
# SKY_F_HC_LEVEL(l): the high-ratio level l (3..9: 2**(l - 1) chain candidates per position) in bits 8..11 of the flags;
# a level field of 0 with F_HC is the default level
HC_LEVEL_SHIFT = 8
HC_LEVEL_MASK = 0xF << HC_LEVEL_SHIFT
HC_MIN_LEVEL, HC_DEFAULT_LEVEL, HC_MAX_LEVEL = 3, 5, 9
BOX_OVERHEAD = 40
# sky_decode status codes
D_OK, D_BAD_HEADER, D_CORRUPT, D_SIZE, D_UNSUPPORTED, D_LAYOUT, D_TRUNCATED, D_AUTH, D_CHECKSUM = 0, -1, -2, -3, -4, -5, -6, -7, -8
D_MISMATCH = -9  # F_VERIFY: the frame is well formed but decodes to other bytes than its chunk
D_NAMES = {0: "ok", -1: "bad frame header", -2: "corrupt block", -3: "size mismatch", -4: "unsupported frame feature",
           -5: "unexpected block layout", -6: "truncated frame", -7: "box authentication failed", -8: "checksum mismatch",
           -9: "frame decodes to other bytes"}

# every symbol include/skychunk.h declares (tests check the .so exports exactly these)
ABI_SYMBOLS = (
    "sky_strerror", "sky_last_error", "sky_abi_version", "sky_device_count", "sky_device_pci_bus_id", "sky_kernel_config", "sky_frame_bound",
    "sky_ctx_create", "sky_ctx_destroy", "sky_pinned_alloc", "sky_pinned_free",
    "sky_submit", "sky_wait", "sky_set_e2ee_key", "sky_box_bound", "sky_process_device", "sky_verify_device",
    "sky_decode_device", "sky_decode",
    "sky_device_alloc", "sky_device_free", "sky_memcpy_h2d", "sky_memcpy_d2h", "sky_launch_count",
)


class SkyChunkError(RuntimeError):
    def __init__(self, code: int, detail: str = ""):
        self.code = code
        msg = f"libskychunk error {code}: {_strerror(code)}"
        if detail:
            msg += f" [{detail}]"
        super().__init__(msg)


_lib: Optional[ctypes.CDLL] = None


def _strerror(code: int) -> str:
    try:
        return lib().sky_strerror(code).decode()
    except Exception:
        return "?"


def lib() -> ctypes.CDLL:
    """Load (building first if needed) libskychunk.so."""
    global _lib
    if _lib is not None:
        return _lib
    import os

    from skyplane_b200 import build as _build

    override = os.environ.get("SKYCHUNK_LIB")  # tuning builds (tools/): same ABI, different kernel constants
    if override:
        L = ctypes.CDLL(override)
    else:
        if _build.needs_build():
            _build.build()
        L = ctypes.CDLL(str(LIB_PATH))
    vp, u64, u32, i32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int
    p_u64 = ctypes.POINTER(u64)
    L.sky_strerror.argtypes = [i32]
    L.sky_strerror.restype = ctypes.c_char_p
    L.sky_last_error.argtypes = [vp]
    L.sky_last_error.restype = ctypes.c_char_p
    L.sky_abi_version.argtypes = []
    L.sky_abi_version.restype = i32
    L.sky_device_count.argtypes = [ctypes.POINTER(i32)]
    L.sky_device_count.restype = i32
    L.sky_device_pci_bus_id.argtypes = [i32, ctypes.c_char_p, i32]
    L.sky_device_pci_bus_id.restype = i32
    L.sky_kernel_config.argtypes = [i32]
    L.sky_kernel_config.restype = u32
    L.sky_frame_bound.argtypes = [u64]
    L.sky_frame_bound.restype = u64
    L.sky_ctx_create.argtypes = [i32, u64, u32, u32, ctypes.POINTER(vp)]
    L.sky_ctx_create.restype = i32
    L.sky_ctx_destroy.argtypes = [vp]
    L.sky_ctx_destroy.restype = i32
    L.sky_pinned_alloc.argtypes = [u64]
    L.sky_pinned_alloc.restype = vp
    L.sky_pinned_free.argtypes = [vp]
    L.sky_pinned_free.restype = i32
    L.sky_submit.argtypes = [vp, u32, ctypes.POINTER(vp), p_u64, ctypes.POINTER(vp), p_u64, u32, ctypes.c_char_p, p_u64]
    L.sky_submit.restype = i32
    L.sky_set_e2ee_key.argtypes = [vp, ctypes.c_char_p]
    L.sky_set_e2ee_key.restype = i32
    L.sky_box_bound.argtypes = [u64]
    L.sky_box_bound.restype = u64
    L.sky_wait.argtypes = [vp, u64, p_u64, vp, ctypes.POINTER(ctypes.c_int32), vp, ctypes.POINTER(ctypes.c_float)]
    L.sky_wait.restype = i32
    L.sky_process_device.argtypes = [vp, u32, vp, p_u64, p_u64, vp, p_u64, p_u64, u32, vp, p_u64, vp, ctypes.POINTER(ctypes.c_float)]
    L.sky_process_device.restype = i32
    p_i32 = ctypes.POINTER(ctypes.c_int32)
    L.sky_decode_device.argtypes = [vp, u32, vp, p_u64, p_u64, vp, p_u64, p_u64, vp, p_i32, vp, ctypes.POINTER(ctypes.c_float)]
    L.sky_decode_device.restype = i32
    L.sky_verify_device.argtypes = [vp, u32, vp, p_u64, p_u64, vp, p_u64, p_u64, p_u64, ctypes.POINTER(ctypes.c_uint32), u32, vp, p_i32,
                                    ctypes.POINTER(ctypes.c_float)]
    L.sky_verify_device.restype = i32
    L.sky_decode.argtypes = [vp, u32, ctypes.POINTER(vp), p_u64, ctypes.POINTER(vp), p_u64, u32, p_i32, vp, ctypes.POINTER(ctypes.c_float)]
    L.sky_decode.restype = i32
    L.sky_device_alloc.argtypes = [vp, u64, ctypes.POINTER(vp)]
    L.sky_device_alloc.restype = i32
    L.sky_device_free.argtypes = [vp, vp]
    L.sky_device_free.restype = i32
    L.sky_memcpy_h2d.argtypes = [vp, vp, vp, u64]
    L.sky_memcpy_h2d.restype = i32
    L.sky_memcpy_d2h.argtypes = [vp, vp, vp, u64]
    L.sky_memcpy_d2h.restype = i32
    L.sky_launch_count.argtypes = [vp]
    L.sky_launch_count.restype = u64
    _lib = L
    return L


def device_pci_bus_id(device: int) -> str:
    """PCI bus id of CUDA device `device` in CUDA's own device order (honours CUDA_VISIBLE_DEVICES)."""
    buf = ctypes.create_string_buffer(32)
    rc = lib().sky_device_pci_bus_id(device, buf, 32)
    if rc != SKY_OK:
        raise SkyChunkError(rc)
    return buf.value.decode().lower()


def kernel_config() -> dict:
    """Compile-time constants of the loaded build (sky_kernel_config); the hc_* keys read 0 on a library without F_HC
    (hc_depth is the default level's; hc_max_level reads 0 on a library without levels)."""
    L = lib()
    return {"lz4_entries": L.sky_kernel_config(0), "warps": L.sky_kernel_config(1), "seg_slots": L.sky_kernel_config(2),
            "max_step_log": L.sky_kernel_config(3), "hc_depth": L.sky_kernel_config(4), "hc_hash_bits": L.sky_kernel_config(5),
            "hc_nice": L.sky_kernel_config(6), "hc_max_level": L.sky_kernel_config(7),
            "hc_opt_seg": L.sky_kernel_config(8)}


def hc_depth(level: int) -> int:
    """Chain candidates the high-ratio search walks per position at `level` (liblz4's hash-chain levels)."""
    return 1 << (level - 1)


def hc_level_flag(level: int) -> int:
    """SKY_F_HC_LEVEL(level): the flags of the high-ratio mode at `level` (3..9)."""
    if isinstance(level, bool) or not isinstance(level, int) or not HC_MIN_LEVEL <= level <= HC_MAX_LEVEL:
        raise ValueError(f"high-ratio levels are {HC_MIN_LEVEL}..{HC_MAX_LEVEL}, not {level!r}")
    return F_HC | (level << HC_LEVEL_SHIFT)


def hc_flags(level: Optional[int] = None, hc: bool = False, compress: bool = True) -> int:
    """python-lz4's ``compression_level`` (and the stage's ``hc`` switch) -> the flag bits that choose the compressor:
    0 (the fast path), F_HC (hc=True without a level: the default level 5) or hc_level_flag(level).  Levels 3..9 select the
    high-ratio mode at that level; 0..2 are the fast compressor, so they contradict hc=True.  A level with compress=False,
    or outside 0..9, is a ValueError (10..12 are liblz4's optimal parser, which the stage does not have)."""
    if level is None:
        return F_HC if hc else 0
    if isinstance(level, bool) or not isinstance(level, int):
        raise ValueError(f"compression_level must be an int, not {level!r}")
    if not compress:
        raise ValueError("compression_level selects how frames are compressed: it needs compression")
    if not 0 <= level <= HC_MAX_LEVEL:
        raise ValueError(f"compression_level {level} is not supported: 0..2 (fast) or {HC_MIN_LEVEL}..{HC_MAX_LEVEL} (high-ratio)")
    if level < HC_MIN_LEVEL:
        if hc:
            raise ValueError(f"compression_level {level} is the fast compressor: the high-ratio mode takes {HC_MIN_LEVEL}..{HC_MAX_LEVEL}")
        return 0
    return hc_level_flag(level)


def frame_bound(n: int) -> int:
    return int(lib().sky_frame_bound(n))


def frame_need(n: int, checksum: bool = False, block_checksum: bool = False) -> int:
    """Bytes an n-byte chunk's frame may take (dst_cap before any SecretBox): frame_bound(n), + 4 for the content checksum,
    + 4 per 64 KiB block for block checksums -- what sky_submit / sky_process_device require."""
    blocks = -(-n // BLOCK_BYTES)
    return frame_bound(n) + (CHECKSUM_BYTES if checksum else 0) + (CHECKSUM_BYTES * blocks if block_checksum else 0)


def check_passthrough(compress: bool = True, checksum: bool = False, block_checksum: bool = False):
    """F_PASSTHROUGH's rules, where the sender's options are chosen (so a bad combination fails when a stage call or an
    operator is set up, not in a worker): it chooses per chunk between the frame and the chunk, so it needs compression, and
    a chunk sent as itself cannot carry the LZ4 content or block checksums asked for.  ValueError otherwise."""
    if not compress:
        raise ValueError("pass-through chooses between a chunk's LZ4 frame and the chunk: it needs compression")
    if checksum:
        raise ValueError("pass-through does not combine with the content checksum: a chunk sent as itself has no LZ4 frame to carry it")
    if block_checksum:
        raise ValueError("pass-through does not combine with block checksums: a chunk sent as itself has no LZ4 frame to carry them")


def sender_flags(compress: bool = True, encrypt: bool = False, hc: bool = False, level: Optional[int] = None, checksum: bool = False,
                 block_checksum: bool = False, verify: bool = False, linked: bool = False, optimal: bool = False,
                 passthrough: bool = False) -> int:
    """The sky_submit flags of ChunkStage.launch's options, or a ValueError naming the option that breaks one of the
    sender's rules.  ChunkStage and GatewayCompressHash both ask it, so a bad combination fails when an operator is built or
    before a batch is staged, not in a worker.  Messages name each option by its program field and stage keyword."""
    for on, what in ((hc, "high_ratio (hc) selects how frames are compressed"),
                     (checksum, "content_checksum (checksum) is carried by the LZ4 frame"),
                     (block_checksum, "block_checksum is carried by the LZ4 frame"),
                     (verify, "verify_frames (verify) checks the LZ4 frames")):
        if on and not compress:
            raise ValueError(f"{what}: it needs compression")
    if passthrough:
        check_passthrough(compress, checksum, block_checksum)
    hc_bits = hc_flags(level, hc, compress)
    # the fast compressor has neither a linked-block mode (DESIGN §4.2) nor an optimal parse
    if linked and not hc_bits:
        raise ValueError("block_linked (linked) is a mode of the high-ratio compressor: it needs high_ratio (hc) or a "
                         "compression_level of 3..9")
    if optimal and not hc_bits:
        raise ValueError("optimal_parse (optimal) is a parse of the high-ratio compressor: it needs high_ratio (hc) or a "
                         "compression_level of 3..9")
    return (F_MD5 | (F_LZ4 if compress else 0) | (F_E2EE if encrypt else 0) | hc_bits | (F_CHECKSUM if checksum else 0)
            | (F_BLOCK_CHECKSUM if block_checksum else 0) | (F_VERIFY if verify else 0) | (F_LINKED if linked else 0)
            | (F_OPTIMAL if optimal else 0) | (F_PASSTHROUGH if passthrough else 0))


_DECODE_ONLY_SUBMIT = ((F_HC, "F_HC"), (HC_LEVEL_MASK, "a high-ratio level"), (F_CHECKSUM, "F_CHECKSUM"),
                       (F_BLOCK_CHECKSUM, "F_BLOCK_CHECKSUM"), (F_VERIFY, "F_VERIFY"), (F_LINKED, "F_LINKED"),
                       (F_OPTIMAL, "F_OPTIMAL"), (F_PASSTHROUGH, "F_PASSTHROUGH"))


def check_decode_flags(flags: int) -> int:
    """sky_decode takes the stage bits (F_LZ4, F_MD5) and F_E2EE only: a frame says itself which checksums it carries and
    whether its blocks are linked, and the compressor that made it does not matter to a decoder.  -> flags, or a ValueError naming the bit it does not take."""
    for bit, name in _DECODE_ONLY_SUBMIT:
        if flags & bit:
            raise ValueError(f"decode does not take {name}: it is a sender option (flags {flags:#x})")
    if flags & ~(F_LZ4 | F_MD5 | F_E2EE):
        raise ValueError(f"decode does not know flag bits {flags & ~(F_LZ4 | F_MD5 | F_E2EE):#x}")
    return flags


def round16(x: int) -> int:
    return (x + 15) & ~15


def _u64_array(values: Sequence[int], n: int):
    """(ctypes.c_uint64 * n)(*values), converted in one call through array.array rather than one argument per value
    (a 1024-chunk batch's four arrays took a few hundred microseconds per device-path call the slow way).  Same
    results: fewer than n values are padded with zeros, more is an IndexError, and negative values wrap."""
    U = ctypes.c_uint64 * n
    try:
        a = array.array("Q", values)
    except OverflowError:  # a negative value: let ctypes wrap it as it always has
        return U(*values)
    if len(a) > n:
        raise IndexError("too many initializers")
    if len(a) < n:
        a.frombytes(bytes(8 * (n - len(a))))
    return U.from_buffer(a)


def _digests(raw: bytes) -> list:
    """16-byte digests, one per chunk, from the n * 16 bytes the library wrote."""
    return [raw[i : i + 16] for i in range(0, len(raw), 16)]


def device_count() -> int:
    n = ctypes.c_int(0)
    rc = lib().sky_device_count(ctypes.byref(n))
    if rc != SKY_OK:
        return 0
    return n.value


class PinnedBuffer:
    """Page-locked host memory exposed as a writable memoryview (``.view``) and address (``.addr``)."""

    def __init__(self, nbytes: int):
        self.nbytes = int(nbytes)
        self.addr = lib().sky_pinned_alloc(self.nbytes)
        if not self.addr:
            raise SkyChunkError(SKY_E_NOMEM, "sky_pinned_alloc failed (no CUDA device?)")
        self._arr = (ctypes.c_ubyte * max(1, self.nbytes)).from_address(self.addr)
        self.view = memoryview(self._arr).cast("B")[: self.nbytes]

    def close(self):
        if self.addr:
            self.view.release()
            del self._arr
            lib().sky_pinned_free(self.addr)
            self.addr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context:
    """One sky_ctx: a GPU, its streams, metadata arrays and (n_slots > 0) staging slabs."""

    def __init__(self, device: int = 0, max_batch_bytes: int = 1 << 30, max_chunks: int = 1024, n_slots: int = 2):
        self._h = ctypes.c_void_p()
        self.device = device
        self.max_chunks = max_chunks
        self.max_batch_bytes = max_batch_bytes
        rc = lib().sky_ctx_create(device, max_batch_bytes, max_chunks, n_slots, ctypes.byref(self._h))
        if rc != SKY_OK:
            detail = lib().sky_last_error(None).decode()
            self._h = ctypes.c_void_p()
            raise SkyChunkError(rc, detail)
        self._inflight = {}

    # ------------------------------------------------------------------ helpers
    def _check(self, rc: int):
        if rc != SKY_OK:
            raise SkyChunkError(rc, lib().sky_last_error(self._h).decode())

    def close(self):
        if self._h:
            lib().sky_ctx_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self) -> int:
        return int(lib().sky_launch_count(self._h))

    # ------------------------------------------------------------------ host-buffer path
    def set_e2ee_key(self, key: Optional[bytes]):
        """32-byte SecretBox key for F_E2EE batches (None switches it off)."""
        if key is not None and len(key) != 32:
            raise ValueError("SecretBox keys are 32 bytes")
        self._check(lib().sky_set_e2ee_key(self._h, key))

    def submit(self, src_addrs: Sequence[int], src_lens: Sequence[int], dst_addrs: Optional[Sequence[int]], dst_caps: Optional[Sequence[int]],
               flags: int = 0, nonces: Optional[bytes] = None) -> int:
        """flags = F_MD5: digests only (dst may be None). | F_E2EE: dst receives sealed boxes; nonces = 24 bytes per chunk.
        | F_PASSTHROUGH: chunks whose frame does not shrink them are sent as themselves; complete the ticket with wait_ex."""
        if flags & F_PASSTHROUGH:
            check_passthrough((flags & (F_LZ4 | F_MD5)) != F_MD5, bool(flags & F_CHECKSUM), bool(flags & F_BLOCK_CHECKSUM))
        n = len(src_addrs)
        A = ctypes.c_void_p * n
        U = ctypes.c_uint64 * n
        args = (A(*src_addrs), U(*src_lens), A(*dst_addrs) if dst_addrs is not None else None, U(*dst_caps) if dst_caps is not None else None, nonces)
        if nonces is not None and len(nonces) != 24 * n:
            raise ValueError("need 24 nonce bytes per chunk")
        t = ctypes.c_uint64(0)
        self._check(lib().sky_submit(self._h, n, args[0], args[1], args[2], args[3], flags, nonces, ctypes.byref(t)))
        self._inflight[t.value] = (n, args, flags)  # keep the pointer arrays alive until wait()
        return t.value

    def wait(self, ticket: int):
        """-> (out_lens: list[int], digests: list[bytes], kernel_ms: float).  Refuses a ticket submitted with F_PASSTHROUGH
        (SKY_E_INVALID), which stays waitable for wait_ex."""
        out_lens, digests, _, _, ms = self._wait(ticket, False)
        return out_lens, digests, ms

    def wait_ex(self, ticket: int):
        """Completes any ticket, and the only wait for one submitted with F_PASSTHROUGH -> (out_lens, digests, verify,
        compressed, kernel_ms).  compressed[i]: True when chunk i's payload is its frame (or the box of its frame), False when
        it is the chunk (out_len 0 without F_E2EE: the caller holds the bytes) or the box of the chunk.  verify is None unless
        the ticket has F_VERIFY; verify[i] is then 0 or the D_* code of chunk i's frame as the compressor made it (its payload
        is the stored-block frame)."""
        out_lens, digests, ver, comp, ms = self._wait(ticket, True)
        return out_lens, digests, None if ver is None else list(ver), [bool(c) for c in comp], ms

    def _wait(self, ticket: int, ex: bool):
        """sky_wait with out_len and md5, and with verify (when the ticket has F_VERIFY) and compressed when `ex`."""
        n, _keep, flags = self._inflight[ticket]
        out = (ctypes.c_uint64 * n)()
        md5 = (ctypes.c_ubyte * (16 * n))()
        ver = (ctypes.c_int32 * n)() if ex and flags & F_VERIFY else None
        comp = (ctypes.c_uint8 * n)() if ex else None
        ms = ctypes.c_float(0)
        self._check(lib().sky_wait(self._h, ticket, out, md5, ver, comp, ctypes.byref(ms)))
        del self._inflight[ticket]
        return list(out), _digests(bytes(md5)), ver, comp, ms.value

    # ------------------------------------------------------------------ device-resident path
    def process_device(self, d_src: int, src_off: Sequence[int], src_len: Sequence[int], d_dst: int, dst_off: Sequence[int],
                       dst_cap: Sequence[int], flags: int = 0, stream: int = 0):
        """-> (out_lens, digests, kernel_ms). Pointers are raw device addresses (e.g. tensor.data_ptr())."""
        n = len(src_len)
        out = (ctypes.c_uint64 * n)()
        md5 = (ctypes.c_ubyte * (16 * n))()
        ms = ctypes.c_float(0)
        self._check(
            lib().sky_process_device(self._h, n, d_src, _u64_array(src_off, n), _u64_array(src_len, n), d_dst, _u64_array(dst_off, n),
                                     _u64_array(dst_cap, n), flags, stream or None, out, md5, ctypes.byref(ms))
        )
        return out[:], _digests(bytes(md5)), ms.value

    def verify_device(self, d_src: int, src_off: Sequence[int], src_len: Sequence[int], d_frames: int, frame_off: Sequence[int],
                      frame_len: Sequence[int], frame_cap: Optional[Sequence[int]] = None, content_xxh: Optional[Sequence[int]] = None,
                      flags: int = 0, stream: int = 0):
        """F_VERIFY's check of frames already in HBM against their chunks (sky_verify_device).  flags: the frame flags they
        were made with; content_xxh: the chunks' XXH32, exactly when flags has F_CHECKSUM.  frame_cap None: check only;
        otherwise failing frames are rewritten as stored-block frames.  -> (status, frame_len, kernel_ms)."""
        n = len(src_len)
        fl = _u64_array(frame_len, n)
        st = (ctypes.c_int32 * n)()
        ms = ctypes.c_float(0)
        self._check(lib().sky_verify_device(self._h, n, d_src, _u64_array(src_off, n), _u64_array(src_len, n), d_frames,
                                            _u64_array(frame_off, n), fl, _u64_array(frame_cap, n) if frame_cap is not None else None,
                                            (ctypes.c_uint32 * n)(*content_xxh) if content_xxh is not None else None, flags,
                                            stream or None, st, ctypes.byref(ms)))
        return list(st), list(fl), ms.value

    # ------------------------------------------------------------------ receiver side
    def decode_device(self, d_frames: int, frame_off: Sequence[int], frame_len: Sequence[int], d_out: int, out_off: Sequence[int],
                      raw_len: Sequence[int], stream: int = 0):
        """-> (status: list[int], digests: list[bytes], kernel_ms)."""
        n = len(frame_len)
        st = (ctypes.c_int32 * n)()
        md5 = (ctypes.c_ubyte * (16 * n))()
        ms = ctypes.c_float(0)
        self._check(lib().sky_decode_device(self._h, n, d_frames, _u64_array(frame_off, n), _u64_array(frame_len, n), d_out,
                                            _u64_array(out_off, n), _u64_array(raw_len, n), stream or None, st, md5, ctypes.byref(ms)))
        return list(st), _digests(bytes(md5)), ms.value

    def decode(self, frame_addrs: Sequence[int], frame_lens: Sequence[int], dst_addrs: Optional[Sequence[int]], raw_lens: Sequence[int],
               flags: int = 0):
        """Host buffers, synchronous. -> (status, digests, kernel_ms).  flags: the sender's stage bits (check_decode_flags).
        0: LZ4 frames; F_MD5: the payloads are the chunks themselves (`compress: false`), which are only digested -- nothing
        is written, dst_addrs may be None; | F_E2EE: the payloads are sealed boxes, and what they hold comes back in dst."""
        check_decode_flags(flags)
        n = len(frame_addrs)
        A = ctypes.c_void_p * n
        U = ctypes.c_uint64 * n
        st = (ctypes.c_int32 * n)()
        md5 = (ctypes.c_ubyte * (16 * n))()
        ms = ctypes.c_float(0)
        self._check(lib().sky_decode(self._h, n, A(*frame_addrs), U(*frame_lens), A(*dst_addrs) if dst_addrs is not None else None,
                                     U(*raw_lens), flags, st, md5, ctypes.byref(ms)))
        return list(st), _digests(bytes(md5)), ms.value

    # ------------------------------------------------------------------ torch-free device memory
    def device_alloc(self, nbytes: int) -> int:
        p = ctypes.c_void_p()
        self._check(lib().sky_device_alloc(self._h, nbytes, ctypes.byref(p)))
        return p.value

    def device_free(self, dptr: int):
        self._check(lib().sky_device_free(self._h, dptr))

    def h2d(self, dptr: int, data) -> None:
        mv = memoryview(data).cast("B")
        if mv.nbytes == 0:
            return
        buf = (ctypes.c_ubyte * mv.nbytes).from_buffer_copy(mv) if mv.readonly else (ctypes.c_ubyte * mv.nbytes).from_buffer(mv)
        self._check(lib().sky_memcpy_h2d(self._h, dptr, ctypes.addressof(buf), mv.nbytes))

    def d2h(self, dptr: int, nbytes: int) -> bytes:
        if nbytes == 0:
            return b""
        buf = (ctypes.c_ubyte * nbytes)()
        self._check(lib().sky_memcpy_d2h(self._h, ctypes.addressof(buf), dptr, nbytes))
        return bytes(buf)
