"""Build the C-ABI shared library (bagel_b200/libbagel_b200.so) in-tree with nvcc for sm_90a (H100).

No JIT cache, no torch.utils.cpp_extension: the library has no torch types in its interface, so it is a
plain `nvcc -shared`. The built .so is git-ignored but travels with the tree to the GPU box.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libbagel_b200.so"
STAMP = PKG_DIR / ".libbagel_b200.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; bagel_b200 needs the CUDA toolkit to build its sm_90a kernels")
    return cand


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
                    + [PKG_DIR.parent / "include" / "bagel_b200.h"]):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    return LIB_PATH.exists() and STAMP.exists() and STAMP.read_text().strip() == _digest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu and link libbagel_b200.so. Idempotent (content-hash stamp)."""
    if not force and is_fresh():
        return LIB_PATH
    nvcc = _nvcc()
    objdir = PKG_DIR / "build"
    objdir.mkdir(exist_ok=True)
    objs = []
    procs = []
    for src in _sources():
        obj = objdir / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"nvcc failed on {src.name}:\n{out}\n")
        elif verbose and out:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("bagel_b200: CUDA build failed")
    tmp = objdir / (LIB_PATH.name + ".tmp")   # link beside the objects, then rename: a reader never sees a partial library
    link = [nvcc, "-shared", "-o", str(tmp), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"bagel_b200: link failed:\n{r.stdout}")
    os.replace(tmp, LIB_PATH)
    STAMP.write_text(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
