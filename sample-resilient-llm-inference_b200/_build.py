"""Build librr_b200.so in-tree with nvcc for sm_90a (Hopper H100; no torch extension machinery, no JIT cache).

Objects go to <repo>/build/, the shared library next to this file so the package imports from the
source tree.  Only stale objects are rebuilt (mtime of the .cu and of every header in csrc/ and
include/).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
REPO = PKG.parent
CSRC = PKG / "csrc"
OBJ = REPO / "build" / "obj"
LIB = PKG / "librr_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
    "-I", str(REPO / "include"),
    "-I", str(CSRC),
]


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _headers_mtime() -> float:
    hs = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + list((REPO / "include").glob("*.h"))
    return max((h.stat().st_mtime for h in hs), default=0.0)


def _compile(src: Path, verbose: bool) -> Path:
    obj = OBJ / (src.stem + ".o")
    cmd = [NVCC, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link librr_b200.so. Returns the library path."""
    OBJ.mkdir(parents=True, exist_ok=True)
    hdr_m = _headers_mtime()
    srcs = _sources()
    stale = []
    for s in srcs:
        o = OBJ / (s.stem + ".o")
        if force or not o.exists() or o.stat().st_mtime < max(s.stat().st_mtime, hdr_m):
            stale.append(s)
    if stale:
        with ThreadPoolExecutor(max_workers=min(8, len(stale))) as ex:
            list(ex.map(lambda s: _compile(s, verbose), stale))
    objs = [OBJ / (s.stem + ".o") for s in srcs]
    need_link = force or bool(stale) or not LIB.exists() or any(
        o.stat().st_mtime > LIB.stat().st_mtime for o in objs)
    if need_link:
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
               "-o", str(LIB), *map(str, objs), "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
