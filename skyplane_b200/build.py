"""Builds libskychunk.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libskychunk.so"
SOURCES = [CSRC / "skychunk.cu"]


def _deps():
    # build.py itself: a change of NVCC_FLAGS (e.g. the target architecture) must rebuild the library
    return sorted(CSRC.glob("*.cu*")) + sorted((PKG.parent / "include").glob("*.h")) + [Path(__file__).resolve()]


NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-cudart", "static",
]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libskychunk.so cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    return any(d.stat().st_mtime > t for d in _deps())


def build_variant(out: Path, defines: dict, verbose: bool = False) -> Path:
    """Tuning builds for tools/ (same ABI, different kernel constants), e.g. {"SKY_WARPS": 24, "SKY_HASHLOG": 11}."""
    cmd = [nvcc_path(), *NVCC_FLAGS, *[f"-D{k}={v}" for k, v in defines.items()], *(["-Xptxas", "-v"] if verbose else []),
           "-o", str(out), *map(str, SOURCES)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(r.stderr, file=sys.stderr)
    return out


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    # build next to the target and rename into place: concurrent builders (forked workers) never load a partial file
    tmp = LIB.with_name(f".{LIB.name}.{os.getpid()}.tmp")
    cmd = [nvcc_path(), *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-o", str(tmp), *map(str, SOURCES)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    if verbose:
        print(r.stderr, file=sys.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
