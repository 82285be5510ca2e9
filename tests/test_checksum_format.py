"""CPU tests of SKY_F_CHECKSUM (LZ4's content checksum, XXH32) that need no GPU: the frame bytes the checksum epilogue
writes, against liblz4's own frames for the same preferences, and the static schedule of the sender kernel that computes
the XXH32 beside MD5 (tools/md5_schedule.py reads it from the SASS)."""
import sys
from pathlib import Path

import pytest

import oracle
import oracle.reflib as ref

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import hc_model  # noqa: E402
import md5_schedule  # noqa: E402

pytestmark = pytest.mark.skipif(not ref.available(), reason="liblz4.so.1 not found")


def with_content_checksum(frame: bytes, data: bytes) -> bytes:
    """The stage's SKY_F_CHECKSUM frame from the same frame without the flag (FLG 0x68 / 0x60): C.Checksum set and the
    header checksum byte over that descriptor (the compressor writes this header), u32le XXH32(chunk) behind the EndMark
    (sky_checksum_kernel appends it)."""
    dlen = 10 if data else 2
    f = bytearray(frame)
    f[4] |= 0x04
    f[4 + dlen] = (oracle.xxh32(bytes(f[4 : 4 + dlen])) >> 8) & 0xFF
    return bytes(f) + oracle.xxh32(data).to_bytes(4, "little")


def liblz4_checksummed(data: bytes) -> bytes:
    return hc_model.liblz4_frame(data, 0, content_checksum=True)


def test_empty_chunk_frame_equals_liblz4():
    want = liblz4_checksummed(b"")
    assert len(want) == 15 and want[4] == 0x64 and want[5] == 0x40
    assert want == with_content_checksum(oracle.lz4f_compress_indep(b""), b"")
    assert want[-4:] == oracle.xxh32(b"").to_bytes(4, "little") == bytes.fromhex("055dcc02")
    assert ref.lz4f_decompress(want, 0) == b""


@pytest.mark.parametrize("n", [1, 15, 16, 17, 63, 64, 65, 65535, 65536, 65537, 300000])
def test_header_and_trailer_equal_liblz4(n):
    """FLG 0x6C and its header checksum byte, and the trailer, equal liblz4's with contentChecksumFlag = 1 and independent
    blocks; with random (stored) blocks the whole frame is liblz4's byte for byte."""
    data = bytes((i * 2654435761 >> 13) & 0xFF for i in range(n))
    want = liblz4_checksummed(data)
    ours = with_content_checksum(oracle.lz4f_compress_indep(data), data)
    assert want[4] == 0x6C and ours[:15] == want[:15]
    assert ours[-4:] == want[-4:] == oracle.xxh32(data).to_bytes(4, "little")
    assert ref.lz4f_decompress(ours, n) == data  # liblz4 verifies the content checksum


def test_liblz4_rejects_a_wrong_content_checksum():
    data = b"skyplane " * 1000
    f = bytearray(with_content_checksum(oracle.lz4f_compress_indep(data), data))
    f[-1] ^= 1
    with pytest.raises(ValueError):
        ref.lz4f_decompress(bytes(f), len(data))


@pytest.mark.skipif(md5_schedule.cuobjdump_path() is None, reason="cuobjdump not found")
def test_sender_xxh_kernel_keeps_the_md5_chain():
    """The XXH32 stripes sit between the MD5 rounds of sky_fused_xxh_kernel's steady-state loop without touching the
    chain: still 12-cycle ALU-only steps, within 0.8 cycles per step of the bare kernel."""
    from skyplane_b200 import build

    r = md5_schedule.report(build.build())["fused_xxh"]
    assert r["lea_hi"] == 256, "the steady-state loop hashes four blocks of 64 steps"
    assert r["shape"]["BRA"] == 1 and r["shape"]["BSSY"] == 0 and r["shape"]["BSYNC"] == 0, r["shape"]
    assert r["cycles_per_step"] <= 12.8, r
    main = r["chains"][0]
    assert main["ops"] == ["LEA.HI(alu)", "LOP3(alu)", "IADD3(alu)", "LEA.HI(alu)"], main
    assert main["distances"] == [4, 4, 4], main
    assert main["steps"] >= 3 * r["lea_hi"] // 4, r["chains"]
