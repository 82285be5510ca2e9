"""Static schedule of the MD5 steady-state loop, read from the SASS of the built libskychunk.so (no GPU needed).

On sm_90a the integer ops of the MD5 chain have fixed latency, so ptxas schedules them by the stall count it writes into
each instruction's control bits (bits 41-44 of the high 64-bit word).  With no variable-latency op on the chain, the sum
of the stall counts over the loop is the loop's time in cycles.  For `sky_fused_kernel`, `sky_fused_xxh_kernel` and
`sky_decode_kernel` this tool finds the innermost loop that holds the most `LEA.HI` (one per MD5 step: `b + rotl(t, s)`),
sums its stalls and follows each step's dependent chain back from its `LEA.HI` to the previous step's, through the source
written last.

    python tools/md5_schedule.py [--lib path/to/libskychunk.so] [--json]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

LIB = Path(__file__).resolve().parent.parent / "skyplane_b200" / "libskychunk.so"
KERNELS = {
    "fused": "_ZN3sky16sky_fused_kernelENS_6ParamsE",
    "fused_xxh": "_ZN3sky20sky_fused_xxh_kernelENS_6ParamsE",  # SKY_F_CHECKSUM: XXH32 stripes between the MD5 rounds
    "decode": "_ZN3sky17sky_decode_kernelENS_9DecParamsE",
}
# Execution pipe of the opcodes that can sit on the chain (sm_90: ALU = integer logic/add/shift, FMA = IMAD forms).
PIPES = {"LOP3": "alu", "IADD3": "alu", "LEA": "alu", "SHF": "alu", "SEL": "alu", "IMAD": "fma"}

_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;\s*/\*\s*0x([0-9a-f]{16})\s*\*/")
_HIGH = re.compile(r"^\s*/\*\s*0x([0-9a-f]{16})\s*\*/\s*$")
_REG = re.compile(r"\bR(\d+)\b")


class Insn:
    def __init__(self, addr: int, text: str, hi: int):
        self.addr, self.text = addr, text
        self.stall = (hi >> 41) & 0xF
        body = re.sub(r"^@!?U?P\w+\s+", "", text)  # guard predicate
        self.op, _, ops = body.partition(" ")
        self.args = ops
        self.base = self.op.split(".")[0]
        operands = [o.strip() for o in ops.split(",")]
        # destination: the first register operand, unless the op writes none (stores, branches, barriers)
        writes = not self.base.startswith(("ST", "BRA", "BAR", "RED", "ATOM", "LDGSTS", "DEPBAR", "EXIT", "NOP"))
        width = 4 if ".128" in self.op else 2 if (".64" in self.op or ".WIDE" in self.op) else 1
        self.dst: set[int] = set()
        self.src: set[int] = set()
        for i, o in enumerate(operands):
            regs = {int(r) for r in _REG.findall(o)}
            if i == 0 and writes and regs:
                r = min(regs)
                self.dst = set(range(r, r + width))
            else:
                self.src |= regs

    @property
    def pipe(self) -> str:
        return PIPES.get(self.base, "other")

    @property
    def name(self) -> str:
        return self.op.replace(".LUT", "")


def cuobjdump_path() -> str | None:
    """cuobjdump from $CUOBJDUMP, $PATH or the default CUDA install (where skyplane_b200/build.py finds nvcc)."""
    for cand in (os.environ.get("CUOBJDUMP"), shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and Path(cand).exists():
            return cand
    return None


def sass(lib: Path, func: str) -> list[Insn]:
    tool = cuobjdump_path()
    if tool is None:
        raise RuntimeError("cuobjdump not found")
    out = subprocess.run([tool, "-sass", "-fun", func, str(lib)], capture_output=True, text=True, check=True).stdout
    insns: list[Insn] = []
    lines = out.splitlines()
    in_func = False
    for i, line in enumerate(lines):
        if "Function :" in line:
            in_func = line.split("Function :")[1].strip() == func
            continue
        m = _INSN.search(line) if in_func else None
        if m and i + 1 < len(lines) and (h := _HIGH.match(lines[i + 1])):
            insns.append(Insn(int(m.group(1), 16), m.group(2), int(h.group(1), 16)))
    if not insns:
        raise RuntimeError(f"{func}: no SASS found in {lib}")
    return insns


def md5_loop(insns: list[Insn]) -> list[Insn]:
    """The body of the innermost backward branch that closes the most LEA.HI.

    Loops that enclose another loop with LEA.HI in it (the per-group loop around md5_warp, the receiver's row loop) are
    skipped, so the tail blocks and the set-up outside the steady-state loop are not counted."""
    index = {x.addr: k for k, x in enumerate(insns)}
    loops = []
    for k, x in enumerate(insns):
        m = re.fullmatch(r"(?:!?U?P\w+, )?(0x[0-9a-f]+)", x.args) if x.base == "BRA" else None
        if m and (t := int(m.group(1), 16)) <= x.addr and t in index:
            lea = sum(y.op == "LEA.HI" for y in insns[index[t]:k + 1])
            if lea:
                loops.append((index[t], k, lea))
    inner = [(s, e, n) for s, e, n in loops if not any(s <= s2 and e2 <= e and (s2, e2) != (s, e) for s2, e2, _ in loops)]
    if not inner:
        raise RuntimeError("no loop with LEA.HI found")
    s, e, _ = max(inner, key=lambda l: l[2])
    return insns[s:e + 1]


def analyse(body: list[Insn]) -> dict:
    total = sum(x.stall for x in body)
    n = len(body)
    # two back-to-back iterations, so the chain of the first steps can be followed into the previous iteration
    seq = body + body
    issue = [0] * (2 * n)
    for k in range(1, 2 * n):
        issue[k] = issue[k - 1] + seq[k - 1].stall
    last_def: dict[int, int] = {}
    producers: list[list[int]] = []
    for k, x in enumerate(seq):
        producers.append([last_def[r] for r in x.src if r in last_def])
        for r in x.dst:
            last_def[r] = k
    steps = [k for k in range(n, 2 * n) if seq[k].op == "LEA.HI"]
    patterns: collections.Counter = collections.Counter()
    for k in steps:
        chain = [k]
        while True:  # back through the source written last, to the previous step's LEA.HI
            p = producers[chain[-1]]
            if not p:
                break
            j = max(p)
            chain.append(j)
            if seq[j].op == "LEA.HI" or len(chain) > 8:
                break
        chain.reverse()
        ops = tuple(f"{seq[j].name}({seq[j].pipe})" for j in chain)
        dist = tuple(issue[b] - issue[a] for a, b in zip(chain, chain[1:]))
        patterns[(ops, dist)] += 1
    nsteps = len(steps)
    return {
        "instructions": n,
        "lea_hi": nsteps,
        "stall_cycles": total,
        "cycles_per_step": round(total / nsteps, 3),
        # the loop is one branch-free body: the back edge is its only BRA, with no reconvergence (BSSY/BSYNC) or moves
        "shape": {op: sum(x.op.startswith(op) for x in body) for op in ("BRA", "BSSY", "BSYNC", "IMAD.MOV")},
        "chains": [{"ops": list(o), "distances": list(d), "steps": c} for (o, d), c in patterns.most_common()],
    }


def report(lib: Path) -> dict:
    return {k: analyse(md5_loop(sass(lib, f))) for k, f in KERNELS.items()}


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--lib", type=Path, default=LIB)
    ap.add_argument("--json", action="store_true", help="one JSON line instead of the text report")
    a = ap.parse_args()
    if cuobjdump_path() is None:
        print("cuobjdump not found", file=sys.stderr)
        return 2
    rep = report(a.lib)
    if a.json:
        print(json.dumps(rep))
        return 0
    for k, r in rep.items():
        print(f"{k}: {r['instructions']} instructions, {r['lea_hi']} LEA.HI, {r['stall_cycles']} stall cycles, "
              f"{r['cycles_per_step']:.2f} cycles/step; " + ", ".join(f"{op} {n}" for op, n in r["shape"].items()))
        for c in r["chains"]:
            hops = " ".join(f"{op} -{d}->" for op, d in zip(c["ops"], c["distances"])) + " " + c["ops"][-1]
            print(f"  {c['steps']:4d} steps: {hops}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
