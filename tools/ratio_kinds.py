#!/usr/bin/env python
"""Compression ratio of the kernel's parse (its sequential CPU twin, tools/lz4_tile_model.c) on data kinds beyond the bench's
Silesia-like set, next to liblz4's: linked blocks (what the reference emits) and independent blocks (what any block-parallel
compressor is limited to), plus the twin's linked-block mode (blocks after a chunk's first match into the previous 64 KiB
window), the high-ratio parse (SKY_F_HC, its twin tools/lz4hc_model.c), its linked blocks (SKY_F_LINKED) and its optimal parse
(SKY_F_OPTIMAL, independent and linked).  Development tool: CPU only, reads files that happen to be installed in the build container."""
import glob
import json
import os
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import oracle  # noqa: E402
import oracle.reflib as ref  # noqa: E402
from skyplane_b200 import synth  # noqa: E402
from tools import hc_model as hm  # noqa: E402
from tools import tile_model as tm  # noqa: E402


def cat(pattern, limit):
    out = bytearray()
    for f in sorted(glob.glob(pattern, recursive=True)):
        if os.path.isfile(f) and not os.path.islink(f):
            try:
                out += open(f, "rb").read()
            except OSError:
                pass
        if len(out) >= limit:
            break
    return bytes(out[:limit])


def kinds():
    r = np.random.default_rng(1)
    walk = np.cumsum(r.integers(-3, 4, size=1 << 19))
    py = cat("/usr/lib/python3*/**/*.py", 8 << 20)
    return {
        "silesia-like 4 x 4 MiB (bench set)": b"".join(synth.silesia_like_chunk(i, 4 << 20) for i in range(4)),
        "shared objects 8 MiB": cat("/usr/lib/x86_64-linux-gnu/*.so*", 8 << 20),
        "python sources 8 MiB": py,
        "c headers 8 MiB": cat("/usr/local/cuda/include/**/*.h", 8 << 20),
        "utf-16 text 4 MiB": py[: 2 << 20].decode("latin1").encode("utf-16-le"),
        "float64 walk 4 MiB": (walk * 0.25).astype("<f8").tobytes(),
        "int64 ids 4 MiB": (np.arange(1 << 19, dtype="<i8") * 7 + 1000).tobytes(),
        "int32 walk 4 MiB": synth._numeric(np.random.default_rng(7), 4 << 20),
        "rgb runs 3 MiB": np.repeat(r.integers(0, 255, size=(1 << 12, 3), dtype=np.uint8), 256, axis=0).tobytes(),
        "int16 audio-like 4 MiB": (np.sin(np.arange(1 << 21) / 50) * 3000 + r.integers(-2, 3, size=1 << 21)).astype("<i2").tobytes(),
    }


if __name__ == "__main__":
    for name, d in kinds().items():
        if not d:
            continue
        raw = len(d)
        ours = len(tm.frame(d))
        ours_linked = len(tm.frame(d, linked=True))
        hc = len(hm.frame(d))
        hc_linked = len(hm.frame(d, linked=True))
        hc_opt = len(hm.frame(d, optimal=True))
        hc_linked_opt = len(hm.frame(d, linked=True, optimal=True))
        linked = len(ref.lz4f_compress(d))
        indep = len(oracle.lz4f_compress_indep(d)) if hasattr(oracle, "lz4f_compress_indep") else None
        row = {"data": name, "bytes": raw, "kernel_parse_ratio": round(raw / ours, 4), "liblz4_linked_ratio": round(raw / linked, 4),
               "vs_reference": round(linked / ours, 4), "linked_parse_ratio": round(raw / ours_linked, 4),
               "linked_vs_reference": round(linked / ours_linked, 4), "hc_parse_ratio": round(raw / hc, 4), "hc_vs_reference": round(linked / hc, 4),
               "hc_linked_ratio": round(raw / hc_linked, 4), "hc_linked_vs_hc": round(hc / hc_linked, 4),
               "hc_linked_vs_reference": round(linked / hc_linked, 4), "hc_opt_ratio": round(raw / hc_opt, 4),
               "hc_opt_vs_hc": round(hc / hc_opt, 4), "hc_linked_opt_ratio": round(raw / hc_linked_opt, 4),
               "hc_linked_opt_vs_hc_linked": round(hc_linked / hc_linked_opt, 4)}
        if indep:
            row["liblz4_independent_blocks_ratio"] = round(raw / indep, 4)
            row["vs_liblz4_independent"] = round(indep / ours, 4)
            row["linked_vs_liblz4_independent"] = round(indep / ours_linked, 4)
            row["hc_vs_liblz4_independent"] = round(indep / hc, 4)
        print(json.dumps(row), flush=True)
