"""SASS check (no GPU): the wide GEMM kernel makes no function calls. Its epilogue code runs right after the MMA loop,
and a call anywhere in it (such as the slow-path subroutine the compiler emits for an IEEE fp32 division) costs a
branch per element and keeps the epilogue code from being scheduled freely; silu_f divides without one."""
import os
import re
import shutil
import subprocess

import pytest

from bagel_b200 import build as bb


def test_gemm_kernels_make_no_calls():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found (CUDA toolkit binaries are not on PATH or in /usr/local/cuda/bin)")
    lib = bb.build()   # no-op when the library is up to date with csrc/
    sass = subprocess.run([tool, "-sass", str(lib)], check=True, capture_output=True, text=True).stdout
    calls, name, kernels = {}, None, 0
    for line in sass.splitlines():
        m = re.match(r"\s*Function\s*:\s*(\S+)", line)
        if m:
            name = m.group(1) if "gemm_bf16_kernel" in m.group(1) else None
            kernels += name is not None
            continue
        if name is not None and re.search(r"\bCALL\b", line):
            calls[name] = calls.get(name, 0) + 1
    assert kernels, "no gemm_bf16_kernel instantiation found in the library"
    assert not calls, f"{len(calls)} of {kernels} GEMM kernels contain CALL instructions, e.g. {sorted(calls)[:3]}"
