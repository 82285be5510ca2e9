"""tools/lz4hc_model.c (the sequential twin of the high-ratio SKY_F_HC parse) must emit valid LZ4 frames in the stage's
format and buy the ratio the mode exists for: every frame is decoded with the strict oracle decoder, liblz4 and pyarrow."""
import re
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import oracle.reflib as ref
from skyplane_b200 import native, synth

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools import hc_model as hm  # noqa: E402


def _datas():  # the edge lengths and data kinds of test_tools_model.py
    rng = np.random.default_rng(3)
    return [rng.bytes(n) for n in (1, 12, 13, 100, 65536)] + [bytes(70000), (b"abcdefg" * 20000)[:131073], b"",
                                                             synth.silesia_like_chunk(11, 300000), b"x" * 13 + rng.bytes(40) + b"x" * 200,
                                                             rng.bytes(40000) + synth.silesia_like_chunk(3, 90000)]


@pytest.mark.parametrize("opts", [hm.kernel_opts(), hm.Opts(1, 12, 4), hm.Opts(64, 16, 252)])
def test_hc_twin_emits_valid_lz4(opts):
    pa = pytest.importorskip("pyarrow")
    for d in _datas():
        fr = hm.frame(d, opts)
        assert oracle.lz4f_decode(fr, len(d)) == d
        assert ref.lz4f_decompress(fr, len(d)) == d
        if d:
            assert pa.decompress(fr, decompressed_size=len(d), codec="lz4").to_pybytes() == d
        assert len(fr) <= 15 + len(d) + 4 * ((len(d) + 65535) // 65536) + 4


def test_hc_twin_long_matches_are_extended():
    """Matches that reach the search's stop length are extended to their real end: zeros take one sequence per block."""
    d = bytes(3 * 65536)
    fr = hm.frame(d)
    assert oracle.lz4f_decode(fr, len(d)) == d and len(fr) < 15 + 3 * (4 + 300) + 4


def test_hc_twin_ratio_on_study_set():
    """2 x 4 MiB Silesia-like: >= 1.12 x the reference's ratio (linked blocks, liblz4 level 0) and >= 0.95 x liblz4 level 9
    with independent 64 KiB blocks (the frame format both this parse and the stage are held to)."""
    datas = [synth.silesia_like_chunk(i, 4 << 20) for i in range(2)]
    raw = sum(map(len, datas))
    ours = sum(len(hm.frame(d)) for d in datas)
    reference = sum(len(ref.lz4f_compress(d)) for d in datas)
    l9 = sum(len(hm.liblz4_frame(d, 9)) for d in datas)
    assert raw / ours >= 1.12 * raw / reference, (raw / ours, raw / reference)
    assert raw / ours >= 0.95 * raw / l9, (raw / ours, raw / l9)


def test_hc_flag_in_header_equals_native():
    hdr = (ROOT / "include" / "skychunk.h").read_text()
    assert int(re.search(r"#define SKY_F_HC (\d+)u", hdr).group(1)) == native.F_HC == 32
    assert native.F_HC not in (native.F_LZ4, native.F_MD5, native.F_E2EE)
