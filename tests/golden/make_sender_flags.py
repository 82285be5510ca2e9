"""Generates sender_flags.json: the flag word ChunkStage.launch submits for every combination of the sender's options on
a grid, or null where launch refuses the combination with ValueError.  tests/test_sender_options.py holds the stage, the
operator and native.sender_flags to this table.

The table was made by the ChunkStage.launch of the commit before native.sender_flags existed, which wrote each rule out
where it was used; regenerating it with a later launch only proves that launch agrees with itself.  The words are read
from a recording context, so no GPU is needed; launch loads libskychunk.so for kernel_config().
Usage: python tests/golden/make_sender_flags.py
"""
import itertools
import json
import sys
from pathlib import Path
from types import SimpleNamespace

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from skyplane_b200.stage import ChunkStage  # noqa: E402

# ChunkStage.launch's keywords and the values each takes on the grid; "5" and True are levels launch must refuse
AXES = [("compress", [False, True]), ("encrypt", [False, True]), ("hc", [False, True]),
        ("level", [None, 0, 2, 3, 5, 9, 10, True, "5"]), ("checksum", [False, True]), ("block_checksum", [False, True]),
        ("verify", [False, True]), ("linked", [False, True]), ("optimal", [False, True]), ("passthrough", [False, True])]


class _Ctx:
    def submit(self, src, lens, dst, caps, flags, nonces):
        self.flags = flags
        return 1


def word(**opts):
    """The word ChunkStage.launch submits for a one-chunk batch with `opts`, or None when it raises ValueError."""
    stage = ChunkStage.__new__(ChunkStage)
    stage.ctx = _Ctx()
    slot = SimpleNamespace(lens=[100], in_off=[0], out_off=[0], inp=SimpleNamespace(addr=1 << 20), out=SimpleNamespace(addr=2 << 20),
                           flags=0, ticket=None)
    try:
        stage.launch(slot, nonces=bytes(24), **opts)
    except ValueError:
        return None
    return stage.ctx.flags


def main():
    names = [n for n, _ in AXES]
    words = [word(**dict(zip(names, values))) for values in itertools.product(*(v for _, v in AXES))]
    table = {"axes": AXES, "words": words}
    (HERE / "sender_flags.json").write_text(json.dumps(table, separators=(",", ":")) + "\n")
    print(f"{len(words)} cases, {sum(w is not None for w in words)} accepted, {len(set(words) - {None})} distinct words")


if __name__ == "__main__":
    main()
