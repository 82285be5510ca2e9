"""CPU tests of the frame check's switches (SKY_F_VERIFY, ChunkStage's verify, GatewayCompressHash's verify_frames) that
need no GPU: the header's flag and status code against native, and the argument rules of ChunkStage, GatewayCompressHash
and the program loader."""
import multiprocessing as mp
import subprocess
from pathlib import Path
from types import SimpleNamespace

import pytest

from skyplane_b200 import native
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash
from skyplane_b200.stage import ChunkStage

ROOT = Path(__file__).resolve().parent.parent


def test_header_flag_and_code_equal_native(tmp_path):
    src = tmp_path / "verify.c"
    src.write_text('#include <stdio.h>\n#include "skychunk.h"\n'
                   'int main(void) { printf("%u %d\\n", (unsigned)SKY_F_VERIFY, SKY_D_MISMATCH); return 0; }\n')
    exe = tmp_path / "verify"
    subprocess.check_call(["gcc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    flag, code = subprocess.check_output([str(exe)], text=True).split()
    assert int(flag) == native.F_VERIFY == 1 << 12 and int(code) == native.D_MISMATCH == -9
    # outside the level field and every other flag
    assert native.F_VERIFY & (native.HC_LEVEL_MASK | native.F_LZ4 | native.F_MD5 | native.F_E2EE | native.F_HC | native.F_CHECKSUM
                              | native.F_BLOCK_CHECKSUM) == 0
    assert native.D_NAMES[native.D_MISMATCH] and native.D_MISMATCH not in (native.D_OK, native.D_CHECKSUM, native.D_AUTH)


class _Ctx:
    def __init__(self):
        self.flags = []

    def submit(self, src, lens, dst, caps, flags, nonces):
        self.flags.append(flags)
        return len(self.flags)


def test_chunkstage_launch_verify_flags():
    stage = ChunkStage.__new__(ChunkStage)  # a stage whose context only records what launch() submits (no device)
    stage.ctx = _Ctx()
    slot = SimpleNamespace(lens=[1000], in_off=[0], out_off=[0], inp=SimpleNamespace(addr=1 << 20), out=SimpleNamespace(addr=2 << 20),
                           flags=0, ticket=None)
    base = native.F_MD5 | native.F_LZ4
    stage.launch(slot, verify=True)
    assert slot.flags == base | native.F_VERIFY
    stage.launch(slot, verify=True, level=9, checksum=True, block_checksum=True)
    stage.launch(slot)
    assert stage.ctx.flags == [base | native.F_VERIFY,
                               base | native.F_VERIFY | native.hc_level_flag(9) | native.F_CHECKSUM | native.F_BLOCK_CHECKSUM, base]
    with pytest.raises(ValueError, match="verify"):
        stage.launch(slot, compress=False, verify=True)
    with pytest.raises(ValueError, match="verify"):
        stage.process([b"x" * 100], compress=False, verify=True)
    assert len(stage.ctx.flags) == 3


def _operator(tmp_path, **kw):
    return GatewayCompressHash("ch", "test:r", GatewayQueue(), None, mp.Event(), mp.Queue(), ChunkStore(tmp_path), **kw)


def test_gateway_compress_hash_verify_frames(tmp_path):
    assert not _operator(tmp_path).verify_frames
    assert _operator(tmp_path, verify_frames=True).verify_frames
    assert _operator(tmp_path, verify_frames=True, compression_level=5, e2ee_key_bytes=bytes(32)).verify_frames
    with pytest.raises(ValueError, match="verify_frames"):
        _operator(tmp_path, verify_frames=True, use_compression=False)


def test_program_json_verify_frames(tmp_path):
    from skyplane_b200.program import build_operator_graph

    def graph(**fields):
        prog = [{"partitions": ["0"], "value": [{"op_type": "compress_hash", "handle": "a", "num_gpus": 1, "children": [], **fields}]}]
        return build_operator_graph(prog, ChunkStore(tmp_path), "r", mp.Event(), mp.Queue()).operators["compress_hash_a"]

    assert not graph().verify_frames
    assert graph(verify_frames=True).verify_frames
    with pytest.raises(ValueError, match="verify_frames"):
        graph(verify_frames=True, compress=False)
