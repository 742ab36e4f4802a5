"""SASS check (no GPU): no tensor-core kernel of the library runs its wgmma instructions one at a time.

When ptxas cannot keep a wgmma pipeline live (for example across a function call such as printf on a path reached
while a wgmma group is in flight) it serializes every wgmma of the kernel: each HGMMA then carries the `gsb0`
scoreboard and is followed by a wait for it to retire. A pipelined kernel has runs of HGMMAs in which only the last
one carries `gsb0`. A kernel whose every HGMMA carries `gsb0` is therefore reported as serialized."""
import os
import re
import shutil
import subprocess

import pytest

from bagel_b200 import build as bb


def _cuobjdump():
    cand = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return cand if os.path.exists(cand) else None


def _hgmma_per_kernel(sass: str):
    """{kernel name: (HGMMA count, HGMMAs carrying gsb0)} for every kernel that contains HGMMA."""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function\s*:\s*(\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "HGMMA." in line:
            n, g = out.get(name, (0, 0))
            out[name] = (n + 1, g + ("gsb0" in line))
    return out


def test_no_serialized_wgmma():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found (CUDA toolkit binaries are not on PATH or in /usr/local/cuda/bin)")
    lib = bb.build()   # no-op when the library is up to date with csrc/
    sass = subprocess.run([tool, "-sass", str(lib)], check=True, capture_output=True, text=True).stdout
    kernels = _hgmma_per_kernel(sass)
    assert kernels, "no HGMMA found in the library: the tensor-core kernels are missing"
    serialized = sorted(k for k, (n, g) in kernels.items() if n == g)
    assert not serialized, (f"{len(serialized)} of {len(kernels)} wgmma kernels issue every HGMMA serialized "
                            f"(each carries gsb0), e.g. {serialized[:3]}")
