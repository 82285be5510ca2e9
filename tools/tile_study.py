#!/usr/bin/env python
"""Compression-ratio study on the CPU twin of the round-2 GPU block compressor (tools/lz4_tile_model.c).
Prints frame-size ratios for design variants next to liblz4's (linked blocks = what the reference emits), and for the
twin's linked-block mode with the previous window's last 64 / 16 / 4 KiB of positions seeding the table.
Every model output is decoded with liblz4 to prove the variant emits valid LZ4."""
import ctypes
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from skyplane_b200 import synth  # noqa: E402

from tools import tile_model as tm  # noqa: E402

M = tm.lib()
Opts, Stats = tm.Opts, tm.Stats
LZ4 = ctypes.CDLL("liblz4.so.1")
LZ4.LZ4_decompress_safe.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
LZ4.LZ4_decompress_safe_usingDict.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]


def model_size(data: bytes, o: Opts, check: bool = True, seed: int = 0) -> int:
    """seed > 0: the linked-block mode, the table of block j >= 1 seeded with that many of block j-1's last positions."""
    total, pos = 15 + 4, 0
    back = ctypes.create_string_buffer(65536)
    for c, b in tm.blocks(data, o, linked=seed > 0, seed=seed):
        n = min(65536, len(data) - pos)
        if c and check:
            if seed and pos:
                r = LZ4.LZ4_decompress_safe_usingDict(b, back, c, 65536, data[pos - 65536:pos], 65536)
            else:
                r = LZ4.LZ4_decompress_safe(b, back, c, 65536)
            assert r == n and back.raw[:r] == data[pos:pos + n], "model emitted an invalid block"
        pos += n
        total += 4 + len(b)
    return total


def liblz4_linked_size(data: bytes) -> int:
    import oracle.reflib as ref  # dev tool: only used to print the reference's ratio next to ours

    return len(ref.lz4f_compress(data))


VARIANTS = {
    "kernel: 4096e seg1024 step16 near{3,4,8}": tm.kernel_opts(),
    "no segment clipping": Opts(4096, 1024, 4, 1, 0, 1, 0x8C),
    "seg512": tm.kernel_opts(4096, 512),
    "seg2048": tm.kernel_opts(4096, 2048),
    "3072e": tm.kernel_opts(3072),
    "2048e": tm.kernel_opts(2048),
    "no back ext": Opts(4096, 1024, 4, 0, 1, 1, 0x8C),
    "step1": tm.kernel_opts(4096, 1024, 0),
    "sequential probe (every slot sees the one before)": Opts(4096, 1024, 4, 1, 1, 0, 0),
    "no in-group candidates": Opts(4096, 1024, 4, 1, 1, 1, 0),
    "near {4}": Opts(4096, 1024, 4, 1, 1, 1, 0x8),
    "near {1,2,3,4,8}": Opts(4096, 1024, 4, 1, 1, 1, 0x8F),
    "near {1..31}": Opts(4096, 1024, 4, 1, 1, 1, 0x7FFFFFFF),
}
LINKED = {  # name: (options, positions of the previous window that seed the table)
    "linked, seed 64 KiB": (tm.kernel_opts(), 65536),
    "linked, seed 16 KiB": (tm.kernel_opts(), 16384),
    "linked, seed 4 KiB": (tm.kernel_opts(), 4096),
    "linked, seed 64 KiB, no segment clipping": (Opts(4096, 1024, 4, 1, 0, 1, 0x8C), 65536),
}

if __name__ == "__main__":
    sets = {"silesia-like 4 x 4 MiB": [synth.silesia_like_chunk(i, 4 << 20) for i in range(4)],
            "text-only 4 MiB": [synth._text(np.random.default_rng(5), 4 << 20)],
            "records 4 MiB": [synth._records(np.random.default_rng(6), 4 << 20)],
            "numeric 4 MiB": [synth._numeric(np.random.default_rng(7), 4 << 20)],
            "random 1 MiB": [synth.random_chunk(0, 1 << 20)]}
    for sname, datas in sets.items():
        raw = sum(map(len, datas))
        refsz = sum(liblz4_linked_size(d) for d in datas)
        row = {"set": sname, "reference (liblz4 linked)": round(raw / refsz, 4)}
        for vname, o in VARIANTS.items():
            st = Stats()
            M.tile_model_stats(ctypes.byref(st), 1)
            row[vname] = round(raw / sum(model_size(d, o) for d in datas), 4)
            M.tile_model_stats(ctypes.byref(st), 1)
            if vname.startswith("kernel:"):
                row["stats"] = {"probes/B": round(st.probes / raw, 3), "hits/B": round(st.hits / raw, 3), "B/seq": round(raw / max(1, st.accepted), 1)}
        for vname, (o, seed) in LINKED.items():
            row[vname] = round(raw / sum(model_size(d, o, seed=seed) for d in datas), 4)
        print(json.dumps(row), flush=True)
