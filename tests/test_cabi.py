"""The C-ABI library loads, exports exactly what include/bagel_b200.h declares, and the Python layer refuses
to run without CUDA tensors (no CPU fallback anywhere in the product)."""
import ctypes

import pytest
import torch

from bagel_b200 import _cabi, build, ops


@pytest.fixture(scope="module")
def lib():
    build.build()  # no-op when fresh; cross-compiles sm_90a without a GPU
    return _cabi.lib()


def test_header_and_bindings_agree(lib):
    declared = set(_cabi.declared_symbols())
    assert declared == set(_cabi.SIGNATURES), declared ^ set(_cabi.SIGNATURES)
    for name in declared:
        assert isinstance(getattr(lib, name), ctypes._CFuncPtr)


def test_abi_version_and_counters(lib):
    assert lib.bagel_abi_version() == 3
    assert lib.bagel_launch_count() >= 0
    assert isinstance(lib.bagel_last_error(), bytes)


def test_no_cpu_fallback():
    a = torch.zeros(8, 64, dtype=torch.bfloat16)
    w = torch.zeros(16, 64, dtype=torch.bfloat16)
    with pytest.raises(_cabi.BagelB200Error):
        ops.gemm(a, w)
    with pytest.raises(_cabi.BagelB200Error):
        ops.rmsnorm(a, w[0])


def test_argument_validation_without_gpu(lib):
    # shape / alignment errors are reported before any CUDA call
    rc = lib.bagel_gemm_bf16(None, 64, None, 64, None, 64, 0, 16, 64, None, None, 0, None, 0, None)
    assert rc == -1 and b"M,N,K" in lib.bagel_last_error()
    rc = lib.bagel_gemm_bf16(None, 63, None, 64, None, 64, 8, 16, 64, None, None, 0, None, 0, None)
    assert rc == -2
    rc = lib.bagel_attn_varlen_fwd(None, None, None, None, None, None, 8, 8, 1, 4, 2, 96, 8, 8, 0, 1.0, 384, 192,
                                   192, 384, None, None)
    assert rc == -1 and b"head_dim" in lib.bagel_last_error()


def test_gate_up_interleave_layout():
    I, K = 256, 8
    g = torch.arange(I * K, dtype=torch.float32).reshape(I, K)
    u = -g
    w = ops.interleave_gate_up(g, u)
    assert w.shape == (2 * I, K)
    assert torch.equal(w[0:128], g[0:128]) and torch.equal(w[128:256], u[0:128])
    assert torch.equal(w[256:384], g[128:256]) and torch.equal(w[384:512], u[128:256])
