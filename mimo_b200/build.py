"""Build the sm_90a C-ABI library in-tree (mimo_b200/libmimo_b200.so) with nvcc.

No torch types cross the boundary, so this is a plain `nvcc -shared` of the .cu files under csrc/; cudart is
linked statically and the driver (for cuTensorMapEncodeTiled) is resolved at run time, so the library loads
and exports its symbols on a machine without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libmimo_b200.so"
OBJ = PKG / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xptxas=-v",
]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; cannot build mimo_b200")
    return exe


def _sources():
    return sorted(CSRC.glob("*.cu"))


GEN_WGMMA = PKG.parent / "scripts" / "gen_wgmma.py"  # writes wgmma.cuh (one wrapper per wgmma shape) into OBJ


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
                    + [PKG.parent / "include" / "mimo_b200.h", GEN_WGMMA]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    stamp = OBJ / "stamp.txt"
    dig = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == dig:
        return LIB
    OBJ.mkdir(exist_ok=True)
    r = subprocess.run([sys.executable, str(GEN_WGMMA), str(OBJ / "wgmma.cuh")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"gen_wgmma.py failed:\n{r.stdout}\n{r.stderr}")
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJ / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(OBJ), "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        (OBJ / (src.stem + ".ptxas.txt")).write_text(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-cudart", "static", "-Xlinker", "--no-undefined"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(dig)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
