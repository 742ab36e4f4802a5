"""-m gpu: silu_f (csrc/gemm_params.h) divides without the call into the compiler's division slow path, and must still give
exactly the IEEE quotient x / (1 + e^-x). Its argument in the GEMM epilogues is always a bf16 value, so every one of the
65 536 bf16 bit patterns (zeros, subnormals, infinities and NaNs included) is checked on the device against the plain
`x / y` compiled with the default IEEE division."""
import ctypes
import subprocess

import numpy as np
import pytest

from bagel_b200 import build as bb

pytestmark = pytest.mark.gpu

SRC = r"""
#include "gemm_params.h"
__global__ void silu_all_bf16(float* got, float* want) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 65536) return;
  const float x = __uint_as_float((uint32_t)i << 16);
  got[i] = bagel::silu_f(x);
  want[i] = x / (1.0f + __expf(-x));
}
extern "C" int run(float* got, float* want) {
  float *g = nullptr, *w = nullptr;
  if (cudaMalloc(&g, 65536 * 4) || cudaMalloc(&w, 65536 * 4)) return 1;
  silu_all_bf16<<<256, 256>>>(g, w);
  int rc = (int)cudaMemcpy(got, g, 65536 * 4, cudaMemcpyDeviceToHost);
  rc |= (int)cudaMemcpy(want, w, 65536 * 4, cudaMemcpyDeviceToHost);
  cudaFree(g);
  cudaFree(w);
  return rc;
}
"""


def test_silu_division_bit_identical_for_every_bf16(tmp_path):
    src = tmp_path / "silu_check.cu"
    src.write_text(SRC)
    lib = tmp_path / "libsilu_check.so"
    subprocess.run([bb._nvcc(), *bb.NVCC_FLAGS, "-shared", "-I", str(bb.CSRC), str(src), "-o", str(lib)], check=True)
    got = np.zeros(65536, np.float32)
    want = np.zeros(65536, np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    assert ctypes.CDLL(str(lib)).run(got.ctypes.data_as(fp), want.ctypes.data_as(fp)) == 0
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    bad = np.nonzero(~same)[0]
    assert bad.size == 0, [(hex(int(i) << 16), float(got[i]), float(want[i])) for i in bad[:8]]
