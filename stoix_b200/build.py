"""In-tree build of libstoixb200.so (sm_90a, H100) with nvcc.

`python -m stoix_b200.build` or `__graft_entry__.build()`.  Objects go to stoix_b200/lib/obj, the
shared library to stoix_b200/lib/libstoixb200.so (git-ignored build products).
nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIBDIR = ROOT / "lib"
OBJDIR = LIBDIR / "obj"
LIB = LIBDIR / "libstoixb200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libstoixb200.so cannot be built")


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "stx.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_library(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ for sm_90a and link the C-ABI shared library."""
    OBJDIR.mkdir(parents=True, exist_ok=True)
    stamp = LIBDIR / "build.stamp"
    digest = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJDIR / (src.stem + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [nvcc] + ARCH + ["-shared", "-o", str(LIB)] + [str(o) for o in objs] + []
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
