#!/usr/bin/env python
"""Segment-size study of the high-ratio mode's optimal parse (SKY_F_OPTIMAL) on its CPU twin (tools/lz4hc_model.c,
hc_compress_block_opt): the frame-size ratio of the lazy parse and of the optimal parse with parse segments of 1, 2, 4
and 8 KiB and of one segment per block, independent and linked, at the given levels, on the Silesia-like study set
(synth.silesia_like_chunk(10..13, 4 MiB)).  A segment is what one warp of the kernel parses; every frame is decoded with
liblz4.  Development tool: CPU only."""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import oracle.reflib as ref  # noqa: E402
from skyplane_b200 import synth  # noqa: E402

from tools import hc_model as hm  # noqa: E402

SEGS = [1024, 2048, 4096, 8192, 0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", default="5,9")
    ap.add_argument("--chunks", type=int, default=4)
    a = ap.parse_args()
    data = [synth.silesia_like_chunk(10 + i, 4 << 20) for i in range(a.chunks)]
    raw = sum(map(len, data))
    for level in map(int, a.levels.split(",")):
        o = hm.kernel_opts(level=level)
        for linked in (False, True):
            lazy = sum(len(hm.frame(d, o, linked=linked)) for d in data)
            row = {"level": level, "linked": linked, "lazy_ratio": round(raw / lazy, 4)}
            for seg in SEGS:
                total = 0
                for d in data:
                    f = hm.frame(d, o, linked=linked, optimal=True, seg=seg)
                    assert ref.lz4f_decompress(f, len(d)) == d
                    total += len(f)
                key = f"opt_{seg // 1024}k" if seg else "opt_block"
                row[key + "_ratio"] = round(raw / total, 4)
                row[key + "_vs_lazy"] = round(lazy / total, 4)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
