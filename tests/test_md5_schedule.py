"""CPU test of the MD5 loop's static schedule in the built libskychunk.so (tools/md5_schedule.py reads it from the SASS).

The MD5 pass is a serial chain per chunk, so its cycles per step are the flagship workload's time: a compiler or source
change that puts the chain back across the ALU and FMA pipes (14 cycles per step) fails here, without a GPU."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

import md5_schedule  # noqa: E402

pytestmark = pytest.mark.skipif(md5_schedule.cuobjdump_path() is None, reason="cuobjdump not found")


@pytest.fixture(scope="module")
def schedule():
    from skyplane_b200 import build

    return md5_schedule.report(build.build())


@pytest.mark.parametrize("kernel", ["fused", "decode"])
def test_md5_chain_is_alu_only_at_12_cycles_per_step(schedule, kernel):
    r = schedule[kernel]
    assert r["lea_hi"] == 256, "the steady-state loop hashes four blocks of 64 steps"
    assert r["shape"]["BRA"] == 1 and r["shape"]["BSSY"] == 0 and r["shape"]["BSYNC"] == 0, r["shape"]
    assert r["cycles_per_step"] <= 12.5, r
    main = r["chains"][0]
    assert main["ops"] == ["LEA.HI(alu)", "LOP3(alu)", "IADD3(alu)", "LEA.HI(alu)"], main
    assert main["distances"] == [4, 4, 4], main
    assert main["steps"] >= 3 * r["lea_hi"] // 4, r["chains"]
