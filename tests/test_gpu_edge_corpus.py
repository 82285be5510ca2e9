"""The edge corpus (edge_corpus.py: chunks built for the edges of the parses, whose reach test_edge_corpus.py checks on
the twins) through every compressor kernel, in one batch each: the four fused fast kernels (plain, content checksum,
block checksum, both) against tools/lz4_tile_model.c, and the 56 high-ratio kernels against tools/lz4hc_model.c, byte for
byte; MD5 against hashlib; every frame decodes with liblz4 and sky_decode; SKY_F_VERIFY passes every frame unchanged."""
import hashlib
import sys
from pathlib import Path

import pytest

import oracle.reflib as ref
from edge_corpus import corpus
from skyplane_b200 import native
from test_checksum_format import with_content_checksum
from test_gpu_hc_levels import HC_KERNELS, assert_frames_equal_twin, run_device
from test_gpu_hc_levels import ctx, stage  # noqa: F401  (module fixtures)

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools import tile_model as tm  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]


@pytest.fixture(scope="module")
def cases():
    return corpus()


@pytest.mark.parametrize("xxh,bc", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["plain", "checksum", "bc", "checksum-bc"])
def test_fast_kernels_equal_the_twin_on_the_edge_corpus(ctx, stage, cases, xxh, bc):  # noqa: F811
    k = native.kernel_config()
    o = tm.kernel_opts(k["lz4_entries"], k["seg_slots"], k["max_step_log"])
    datas = [c.data for c in cases]
    flags = native.F_LZ4 | native.F_MD5 | (native.F_CHECKSUM if xxh else 0) | (native.F_BLOCK_CHECKSUM if bc else 0)
    extra = (native.CHECKSUM_BYTES if xxh else 0) + (4 * -(-max(map(len, datas)) // 65536) if bc else 0)
    frames, digests, lens = run_device(ctx, datas, flags, extra)
    for c, f, dg, ln in zip(cases, frames, digests, lens):
        want = tm.frame(c.data, o, block_checksum=bc)
        if xxh:
            want = with_content_checksum(want, c.data)
        assert f == want, f"{c.tag}: GPU frame {len(f)} B != twin {len(want)} B (flags {flags:#x})"
        assert ln == len(f) and dg == hashlib.md5(c.data).digest(), c.tag
        assert ref.lz4f_decompress(f, len(c.data)) == c.data, c.tag
    for c, (data, dg, st) in zip(cases, stage.decode(frames, [len(d) for d in datas])):
        assert st == 0 and data == c.data and dg == hashlib.md5(c.data).digest(), c.tag
    for c, f, r in zip(cases, frames, stage.process(datas, checksum=xxh, block_checksum=bc, verify=True)):
        assert r.verify_status == 0 and bytes(r.frame) == f, f"verify: {c.tag}"


@pytest.mark.parametrize("level,bc,linked,optimal", HC_KERNELS)
def test_high_ratio_kernels_equal_the_twin_on_the_edge_corpus(ctx, stage, cases, level, bc, linked, optimal):  # noqa: F811
    assert_frames_equal_twin(ctx, stage, [c.data for c in cases], level, bc, linked, optimal, [c.tag for c in cases])
