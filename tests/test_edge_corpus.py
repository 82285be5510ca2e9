"""The edge corpus (edge_corpus.py) reaches what it targets: each chunk's expectations hold on the sequential twins of the
compressors (tools/lz4_tile_model.c, tools/lz4hc_model.c), read from their output -- the fast twin's probe counters, the
matches of its blocks, and the high-ratio twin's blocks at the levels and modes a target names -- and every twin frame
decodes with liblz4.  This keeps the corpus honest when a kernel constant changes: a chunk that no longer reaches its edge
fails here, on the CPU, before the GPU tests would quietly pass on it."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle.reflib as ref
from edge_corpus import BLOCK, K1, K2, M32, corpus, geometry
from lz4_craft import walk_block
from skyplane_b200 import native

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools import hc_model as hm  # noqa: E402
from tools import tile_model as tm  # noqa: E402


@pytest.fixture(scope="module")
def cases():
    return corpus()


@pytest.fixture(scope="module")
def g():
    return geometry()


def fast_opts(g, near_mask=None):
    o = tm.kernel_opts(g["lz4_entries"], g["seg_slots"], g["max_step_log"])
    if near_mask is not None:
        o.near_mask = near_mask
    return o


def hc_opts(g, level):
    return hm.Opts(g["depth"][level], g["hc_hash_bits"], g["hc_nice"])


def matches(blocks):
    """{(block, pos, off, len)} of a twin's compressed blocks."""
    return {(j, pos, off, ln) for j, (c, b) in enumerate(blocks) if c for pos, off, ln in walk_block(b)[0]}


def hc_blocks(g, data, level, linked, optimal):
    return hm.blocks(data, hc_opts(g, level), linked, optimal, g["hc_opt_seg"])


def test_the_corpus_is_small_and_every_target_is_checked(cases):
    assert sum(len(c.data) for c in cases) < 4 << 20 and max(len(c.data) for c in cases) <= 200 << 10
    assert len({c.tag for c in cases}) == len(cases)
    for family in ("F1", "F2", "F3", "F4", "F5", "H1", "H2", "H3", "H4"):
        assert any(c.tag.startswith(family) for c in cases), family
    assert all(c.expect for c in cases), [c.tag for c in cases if not c.expect]


def test_the_pad_period_fits_the_strides(g):
    from edge_corpus import PAD_PERIOD

    assert PAD_PERIOD % (1 << g["max_step_log"]) == 0 and PAD_PERIOD > 8 << g["max_step_log"]


def test_three_agreeing_bytes_cannot_be_a_table_false_hit():
    """Why F1 stops at two agreeing bytes: two 5-byte strings that agree on their first three bytes differ in le32 by
    da << 24 and in the fifth byte by db, and no (da, db) != 0 keeps hash bits 8..31 (the index and the tag) equal -- so
    the parse's `mlen < 4` rejection only ever sees 0, 1 or 2 agreeing bytes."""
    da, db = np.meshgrid(np.arange(-255, 256, dtype=np.int64), np.arange(-255, 256, dtype=np.int64))
    diff = (da * ((K1 << 24) & M32) + db * K2) & M32
    same = (diff >> 8) == 0
    assert same.sum() == 1 and same[255, 255]  # only da = db = 0


def test_fast_targets_on_the_twin(cases, g):
    L = tm.lib()
    st = tm.Stats()
    o = fast_opts(g)
    for c in cases:
        e = c.expect
        L.tile_model_stats(ctypes.byref(st), 1)
        blocks = tm.blocks(c.data, o)
        L.tile_model_stats(ctypes.byref(st), 1)
        if "fast_rejects" in e:
            n, breaks = e["fast_rejects"]
            broken = bytearray(c.data)
            for q in breaks:
                broken[q] ^= 0xA5
            tm.blocks(bytes(broken), o)
            ctl = tm.Stats()
            L.tile_model_stats(ctypes.byref(ctl), 1)
            assert (st.hits - st.accepted) - (ctl.hits - ctl.accepted) == n, (c.tag, st.hits, st.accepted, ctl.hits, ctl.accepted)
        if "fast_matches" in e:
            missing = set(e["fast_matches"]) - matches(blocks)
            assert not missing, (c.tag, sorted(missing))
        if "fast_absent" in e:
            assert not set(e["fast_absent"]) & matches(blocks), c.tag
        if "near_mask" in e:
            assert tm.frame(c.data, fast_opts(g, e["near_mask"])) != tm.assemble(len(c.data), blocks), c.tag
        if "last_block" in e:
            assert len(c.data) - (len(blocks) - 1) * BLOCK == e["last_block"], c.tag


def test_high_ratio_targets_on_the_twin(cases, g):
    for c in cases:
        e = c.expect
        for key, want in e.get("hc_matches", {}).items():
            missing = set(want) - matches(hc_blocks(g, c.data, *key))
            assert not missing, (c.tag, key, sorted(missing))
        for key, absent in e.get("hc_absent", {}).items():
            assert not set(absent) & matches(hc_blocks(g, c.data, *key)), (c.tag, key)
        for a, b in e.get("levels_differ", []):
            assert hm.frame(c.data, hc_opts(g, a)) != hm.frame(c.data, hc_opts(g, b)), (c.tag, a, b)
        if "linked_offsets" in e or "linked_raw" in e:
            blocks = hc_blocks(g, c.data, 5, True, False)
            ms = matches(blocks)
            assert all(off <= 65535 for _, _, off, _ in ms)
            for j, off in e.get("linked_offsets", []):
                assert any(m[0] == j and m[2] == off for m in ms), (c.tag, off)
            if "linked_raw" in e:
                assert blocks[e["linked_raw"]][0] == 0, c.tag


def test_x_then_x_shifted_is_matched_only_at_the_window_limit(cases, g):
    """Every match of X + X[1:]'s second block lies exactly 65535 bytes back, and X + X has none there: the window's
    two limits, on the twin, at every level and with the optimal parse."""
    x1 = next(c.data for c in cases if c.tag.startswith("H3 X + X[1:]"))
    xx = next(c.data for c in cases if c.tag.startswith("H3 X + X:"))
    for level, optimal in ((3, False), (5, True), (9, False)):
        offs = {off for j, _, off, _ in matches(hc_blocks(g, x1, level, True, optimal)) if j == 1}
        assert offs == {65535}, (level, optimal, offs)
        assert hc_blocks(g, xx, level, True, optimal)[1][0] == 0


@pytest.mark.parametrize("mode", ["fast", "hc3", "hc9", "hc5-linked", "hc5-optimal", "hc5-linked-optimal"])
def test_every_twin_frame_decodes_with_liblz4(cases, g, mode):
    for c in cases:
        if mode == "fast":
            fr = tm.frame(c.data, fast_opts(g))
        else:
            level = int(mode[2])
            fr = hm.frame(c.data, hc_opts(g, level), linked="linked" in mode, optimal="optimal" in mode, seg=g["hc_opt_seg"])
        assert ref.lz4f_decompress(fr, len(c.data)) == c.data, (mode, c.tag)
