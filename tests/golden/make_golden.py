"""Generates the committed golden fixtures (needs a checkout of the reference, skyplane @ 4602d9c).

  wire_headers.json  WireProtocolHeader.to_bytes() produced by the REFERENCE's own skyplane/chunk.py
                     (imported by file path -- it is stdlib-only) for a handful of field values,
                     plus Chunk.as_dict() of a reference Chunk.
  md5_kat.json       RFC 1321 appendix A.5 suite + padding-boundary lengths, digests from hashlib
                     (the call the reference makes, s3_interface.py:181-192).
  lz4_frames.json    small inputs and the exact frames liblz4 1.9.4 LZ4F_compressFrame emits for them with
                     python-lz4's default preferences (what lz4.frame.compress(data) returns,
                     gateway_operator.py:359), via oracle/reflib.py.
Usage: python tests/golden/make_golden.py <path of the skyplane checkout>
"""
import hashlib
import importlib.util
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

import oracle.reflib as ref  # noqa: E402


def load_reference_chunk():
    spec = importlib.util.spec_from_file_location("ref_chunk", Path(sys.argv[1]) / "skyplane" / "chunk.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_chunk"] = mod
    spec.loader.exec_module(mod)
    return mod


def wire_headers():
    rc = load_reference_chunk()
    cases = [
        dict(chunk_id="00000000000000000000000000000000", data_len=0, raw_data_len=0, is_compressed=False, n_chunks_left_on_socket=0),
        dict(chunk_id="0123456789abcdef0123456789abcdef", data_len=8389139, raw_data_len=8388608, is_compressed=True, n_chunks_left_on_socket=0),
        dict(chunk_id="ffffffffffffffffffffffffffffffff", data_len=2**40 + 5, raw_data_len=2**41 + 7, is_compressed=True, n_chunks_left_on_socket=12799),
        dict(chunk_id="deadbeefdeadbeefdeadbeefdeadbeef", data_len=34580, raw_data_len=8388608, is_compressed=True, n_chunks_left_on_socket=3),
    ]
    out = []
    for c in cases:
        h = rc.WireProtocolHeader(**c)
        out.append({"fields": c, "bytes_hex": h.to_bytes().hex()})
    chunk = rc.Chunk(src_key="a/b", dest_key="c/d", chunk_id="0123456789abcdef0123456789abcdef", chunk_length_bytes=8388608,
                     partition_id="0", file_offset_bytes=16777216, part_number=3, multi_part=True, upload_id="u1")
    req = rc.ChunkRequest(chunk=chunk, src_region="aws:us-east-1", dst_region="gcp:us-west1")
    hdr = chunk.to_wire_header(n_chunks_left_on_socket=5, wire_length=100, raw_wire_length=200, is_compressed=True)
    return {
        "length_bytes": rc.WireProtocolHeader.length_bytes(),
        "magic": rc.WireProtocolHeader.magic_hex(),
        "version": rc.WireProtocolHeader.protocol_version(),
        "headers": out,
        "chunk_as_dict": chunk.as_dict(),
        "chunk_request_as_dict": req.as_dict(),
        "to_wire_header_hex": hdr.to_bytes().hex(),
        "chunk_states": [s.name for s in rc.ChunkState],
    }


def md5_kat():
    rfc = [b"", b"a", b"abc", b"message digest", b"abcdefghijklmnopqrstuvwxyz",
           b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789", b"1234567890" * 8]
    out = {"rfc1321": [{"msg_hex": m.hex(), "md5": hashlib.md5(m).hexdigest()} for m in rfc]}
    out["zeros"] = [{"len": n, "md5": hashlib.md5(bytes(n)).hexdigest()}
                    for n in (55, 56, 57, 63, 64, 65, 119, 120, 121, 127, 128, 129, 65535, 65536, 65537, 1 << 20, 8 << 20)]
    rng = np.random.default_rng(1321)
    out["seeded"] = []
    for n in (1, 2, 3, 31, 100, 1000, 4097, 65536 + 13):
        m = rng.bytes(n)
        out["seeded"].append({"seed": 1321, "len": n, "msg_hex": m.hex() if n <= 1000 else None, "md5": hashlib.md5(m).hexdigest()})
    return out


def lz4_frames():
    rng = np.random.default_rng(42)
    text = (b"the quick brown fox jumps over the lazy dog. " * 40)
    inputs = {
        "empty": b"",
        "one": b"x",
        "twelve": b"abcdefghijkl",
        "thirteen_a": b"a" * 13,
        "zeros_100": bytes(100),
        "zeros_4096": bytes(4096),
        "text_1800": text,
        "period7_300": (b"abcdefg" * 50)[:300],
        "random_64": rng.bytes(64),
        "random_1000": rng.bytes(1000),
        "mixed_3000": text[:1500] + rng.bytes(500) + bytes(1000),
    }
    out = {"liblz4": ref.version(), "cases": []}
    for name, data in inputs.items():
        out["cases"].append({"name": name, "input_hex": data.hex(), "frame_hex": ref.lz4f_compress(data).hex(),
                             "md5": hashlib.md5(data).hexdigest()})
    # larger cases: keep only sizes + digests of the frame (inputs are regenerated from the seed)
    big = []
    for name, n, seed in (("zeros_8MiB", 8 << 20, None), ("random_1MiB", 1 << 20, 43), ("random_8MiB", 8 << 20, 44)):
        data = bytes(n) if seed is None else np.random.default_rng(seed).bytes(n)
        fr = ref.lz4f_compress(data)
        big.append({"name": name, "len": n, "seed": seed, "frame_len": len(fr), "frame_md5": hashlib.md5(fr).hexdigest(),
                    "frame_head_hex": fr[:19].hex(), "md5": hashlib.md5(data).hexdigest()})
    out["big"] = big
    return out


if __name__ == "__main__":
    (HERE / "wire_headers.json").write_text(json.dumps(wire_headers(), indent=1) + "\n")
    (HERE / "md5_kat.json").write_text(json.dumps(md5_kat(), indent=1) + "\n")
    (HERE / "lz4_frames.json").write_text(json.dumps(lz4_frames(), indent=1) + "\n")
    print("wrote", [p.name for p in HERE.glob("*.json")])
