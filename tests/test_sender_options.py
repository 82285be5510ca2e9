"""The sender's options and their rules (native.sender_flags) as every layer states them.

CPU: on the grid of golden/sender_flags.json (every combination of ChunkStage.launch's options, with the word the stage
submitted for it before the rules were gathered into sender_flags, or null where it refused it), sender_flags,
ChunkStage.launch, ChunkStage.process and GatewayCompressHash accept and refuse the same cases and give the same words; a
refused or failed process() call gives its staging slot back.
GPU: sky_submit takes every word sender_flags accepts on the grid, and refuses the naive word of every refused case whose
rule the library's own flag check also states."""
import ctypes
import hashlib
import itertools
import json
import multiprocessing as mp
from pathlib import Path
from types import SimpleNamespace

import pytest

from skyplane_b200 import native, stage as stage_mod
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash
from skyplane_b200.stage import ChunkStage

TABLE = json.loads((Path(__file__).resolve().parent / "golden" / "sender_flags.json").read_text())
NAMES = [name for name, _ in TABLE["axes"]]
CASES = [(dict(zip(NAMES, values)), word) for values, word in zip(itertools.product(*(v for _, v in TABLE["axes"])), TABLE["words"])]
KEY = bytes((11 * i + 5) & 0xFF for i in range(32))
# the stage's keywords -> GatewayCompressHash's parameters
OPERATOR_NAMES = {"compress": "use_compression", "hc": "high_ratio", "level": "compression_level", "checksum": "content_checksum",
                  "block_checksum": "block_checksum", "verify": "verify_frames", "linked": "block_linked", "optimal": "optimal_parse",
                  "passthrough": "skip_incompressible"}


def test_the_table_covers_the_grid():
    assert len(CASES) == len(TABLE["words"]) == 2 ** 9 * 9
    accepted = [w for _, w in CASES if w is not None]
    assert len(set(accepted)) > 300 and all(w & native.F_MD5 for w in accepted)


class _Ctx:
    """A context that records the words submitted and completes every ticket as wait_ex does, with empty payloads."""

    def __init__(self, fail=None):
        self.flags, self.fail = [], fail

    def submit(self, src, lens, dst, caps, flags, nonces=None):
        if self.fail is not None:
            raise self.fail
        self.flags.append(flags)
        self.n = len(lens)
        return len(self.flags)

    def wait_ex(self, ticket):
        return [0] * self.n, [bytes(16)] * self.n, None, [True] * self.n, 0.0


def _recording_stage(ctx=None):
    stage = ChunkStage.__new__(ChunkStage)
    stage.ctx = ctx or _Ctx()
    return stage


def _slot():
    return SimpleNamespace(lens=[100], in_off=[0], out_off=[0], inp=SimpleNamespace(addr=1 << 20), out=SimpleNamespace(addr=2 << 20),
                           flags=0, ticket=None)


def _launch_word(**opts):
    stage = _recording_stage()
    try:
        stage.launch(_slot(), nonces=bytes(24), **opts)
    except ValueError:
        return None
    (word,) = stage.ctx.flags
    return word


def _sender_word(**opts):
    try:
        return native.sender_flags(**opts)
    except ValueError:
        return None


def test_sender_flags_and_launch_equal_the_table():
    assert [_sender_word(**opts) for opts, _ in CASES] == TABLE["words"]
    assert [_launch_word(**opts) for opts, _ in CASES] == TABLE["words"]


class _Buf:
    def __init__(self, addr, nbytes):
        self.addr, self.nbytes = addr, nbytes
        self.view = memoryview(bytearray(nbytes))


def _stage_with_one_slot(ctx):
    """A ChunkStage over a context double with one staging slot of plain memory (no device)."""
    stage = _recording_stage(ctx)
    stage.max_chunks = 4
    slot = object.__new__(stage_mod._Slot)
    slot.inp, slot.out = _Buf(1 << 20, 1 << 16), _Buf(2 << 20, 1 << 16)
    slot.reset()
    stage._slots = [slot]
    stage._free = [slot]
    return stage, slot


def test_process_refuses_exactly_the_refused_cases_without_taking_the_slot():
    ctx = _Ctx()
    stage, slot = _stage_with_one_slot(ctx)
    for opts, word in CASES:
        submitted = len(ctx.flags)
        if word is None:
            with pytest.raises(ValueError):
                stage.process([b"x" * 100], **opts)
            assert len(ctx.flags) == submitted, opts
        else:
            assert len(stage.process([b"x" * 100], **opts)) == 1
            assert ctx.flags[submitted:] == [word], opts
        assert stage._free == [slot], opts


def test_process_gives_the_slot_back_when_launch_refuses():
    stage, slot = _stage_with_one_slot(_Ctx())
    with pytest.raises(ValueError):
        stage.process([b"x" * 100], compress=False, hc=True)
    assert stage._free == [slot]


def test_process_gives_the_slot_back_when_submit_fails():
    stage, slot = _stage_with_one_slot(_Ctx(fail=native.SkyChunkError(native.SKY_E_NOKEY)))
    for _ in range(3):
        with pytest.raises(native.SkyChunkError) as e:
            stage.process([b"x" * 100], encrypt=True)
        assert e.value.code == native.SKY_E_NOKEY
        assert stage._free == [slot]


class _KeywordStage:
    """A stage that records the keywords GatewayCompressHash launches a batch with."""

    def launch(self, slot, **kw):
        self.kw = kw
        return slot


def test_operator_refuses_the_refused_cases_and_hands_the_stage_the_same_word(tmp_path):
    args = ("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), ChunkStore(tmp_path))
    for opts, word in CASES:
        params = {OPERATOR_NAMES[k]: v for k, v in opts.items() if k in OPERATOR_NAMES}
        params["e2ee_key_bytes"] = KEY if opts["encrypt"] else None
        if word is None:
            with pytest.raises(ValueError):
                GatewayCompressHash(*args, n_processes=0, **params)
            continue
        op = GatewayCompressHash(*args, n_processes=0, **params)
        op._stage = _KeywordStage()
        assert op._launch_staged(_slot(), []) is True
        kw = op._stage.kw
        # only the options that are set: a stage double may take compress, encrypt and nothing else
        assert all(v is True for k, v in kw.items() if k not in ("compress", "encrypt", "level")), (opts, kw)
        assert kw.get("level") == opts["level"], (opts, kw)
        assert _launch_word(**kw) == word, (opts, kw)


# ------------------------------------------------------------------ the library's own check, on the GPU
def _python_only(opts) -> bool:
    """A refusal the library's flag check cannot state: a level that is not an int, or one of the fast compressor's
    levels 0..2 together with hc=True or without compression (the word would simply not carry the level)."""
    level = opts["level"]
    if level is None:
        return False
    return isinstance(level, bool) or not isinstance(level, int) or (level < native.HC_MIN_LEVEL and (opts["hc"] or not opts["compress"]))


def _naive_word(opts) -> int:
    """Every option's bit OR-ed in with no rule applied; a level of 3 or more goes into the level field with F_HC."""
    level = opts["level"]
    bits = ((opts["compress"], native.F_LZ4), (opts["encrypt"], native.F_E2EE), (opts["hc"], native.F_HC),
            (opts["checksum"], native.F_CHECKSUM), (opts["block_checksum"], native.F_BLOCK_CHECKSUM), (opts["verify"], native.F_VERIFY),
            (opts["linked"], native.F_LINKED), (opts["optimal"], native.F_OPTIMAL), (opts["passthrough"], native.F_PASSTHROUGH))
    word = native.F_MD5
    for on, bit in bits:
        word |= bit if on else 0
    if level is not None and level >= native.HC_MIN_LEVEL:
        word |= native.F_HC | level << native.HC_LEVEL_SHIFT
    return word


def test_naive_words_of_refused_cases_break_a_library_rule():
    """What the GPU test below submits: every refused case that is not Python-only has a naive word, and none of those is
    a word sender_flags accepts."""
    naive = {_naive_word(o) for o, w in CASES if w is None and not _python_only(o)}
    assert len(naive) > 1000 and not naive & {w for _, w in CASES if w is not None}


@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_library_takes_the_accepted_words_and_refuses_the_naive_refused_ones():
    data = bytes(range(100))
    accepted = sorted({w for _, w in CASES if w is not None})
    refused = sorted({_naive_word(o) for o, w in CASES if w is None and not _python_only(o)})
    ctx = native.Context(0, 1 << 20, 4, 1)
    src, dst = native.PinnedBuffer(4096), native.PinnedBuffer(4096)
    try:
        ctx.set_e2ee_key(KEY)
        src.view[: len(data)] = data
        for word in accepted:  # (the chunk is 100 distinct bytes: no frame makes it smaller, so pass-through sends it as itself)
            t = ctx.submit([src.addr], [len(data)], [dst.addr], [dst.nbytes], word, bytes(24) if word & native.F_E2EE else None)
            out_lens, digests, verify, compressed, _ = ctx.wait_ex(t)
            framed = bool(word & native.F_LZ4) and not word & native.F_PASSTHROUGH
            assert digests == [hashlib.md5(data).digest()] and compressed == [framed], hex(word)
            assert (out_lens[0] > 0) == (framed or bool(word & native.F_E2EE)), hex(word)
            assert verify == ([0] if word & native.F_VERIFY else None), hex(word)
        L = native.lib()
        A, U = ctypes.c_void_p * 1, ctypes.c_uint64 * 1
        t = ctypes.c_uint64()
        for word in refused:
            rc = L.sky_submit(ctx._h, 1, A(src.addr), U(len(data)), A(dst.addr), U(dst.nbytes), word, bytes(24), ctypes.byref(t))
            assert rc == native.SKY_E_INVALID, hex(word)
    finally:
        src.close()
        dst.close()
        ctx.close()
