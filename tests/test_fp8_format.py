"""No GPU: the block-scaled FP8 format of `fp8_gen_mlp=True` as restated in tests/fp8_oracle.py, the argument checks of
its two C-ABI entry points, the refusals of the model flag, and the SASS of the fp8 GEMM kernels."""
import inspect
import os
import re
import shutil
import subprocess

import pytest
import torch

import fp8_oracle as fo
from bagel_b200 import _cabi, build, ops


def _bf16_exact(x: torch.Tensor) -> bool:
    return torch.equal(x.float(), x.float().to(torch.bfloat16).float())


def test_scales_are_powers_of_two_and_q_in_range():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(300, 512, generator=g) * torch.logspace(-30, 30, 300)[:, None]).to(torch.bfloat16)
    for block_rows in (1, 128):
        q, s = fo.quantize(x, block_rows)
        m, e = torch.frexp(s)
        assert torch.all(m == 0.5), "every scale is a power of two"
        assert torch.all(s >= 2.0 ** -126)
        assert q.float().abs().max() <= 448
        # smallest such power: half the scale would not fit the group maximum
        R = s.shape[0]
        pad = torch.zeros(R * block_rows, 512)
        pad[:300] = x.float()
        amax = pad.abs().reshape(R, block_rows, 4, 128).amax(dim=(1, 3))
        assert torch.all(amax <= 448 * s)
        assert torch.all((amax > 448 * s / 2) | (s == 2.0 ** -126) | (amax == 0))


def test_dequantized_values_are_bf16_exact():
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(130, 256, generator=g) * 3).to(torch.bfloat16)
    for block_rows in (1, 128):
        q, s = fo.quantize(x, block_rows)
        d = fo.dequantize(q, s, block_rows)
        assert _bf16_exact(d)
        # and the error is that of e4m3 rounding: at most half an e4m3 ulp (2^-4 relative for normals) of each value
        assert torch.all((d - x.float()).abs() <= x.float().abs() * 2.0 ** -4 + s.max() * 2.0 ** -10)


def test_ties_round_to_even():
    # scale 1 (amax 448 exactly). Between 1.0 and 1.125 (e4m3 spacing 1/8 at [1, 2)) the midpoint 1.0625 goes to 1.0
    # (even mantissa), the midpoint 1.1875 between 1.125 and 1.25 goes to 1.25; between 256 and 288 (spacing 32) 272 -> 256.
    x = torch.zeros(1, 128, dtype=torch.bfloat16)
    x[0, :5] = torch.tensor([448.0, 1.0625, 1.1875, 272.0, -1.0625])
    q, s = fo.quantize(x, 1)
    assert s.item() == 1.0
    assert q.float()[0, :5].tolist() == [448.0, 1.0, 1.25, 256.0, -1.0]


def test_zero_groups_get_scale_one():
    x = torch.zeros(3, 256, dtype=torch.bfloat16)
    x[1, 128:] = 2.0
    q, s = fo.quantize(x, 1)
    assert s.tolist() == [[1.0, 1.0], [1.0, 2.0 ** -7], [1.0, 1.0]]   # [rows, K / 128]
    assert torch.all(q.float()[0] == 0) and torch.all(q.float()[1, :128] == 0)
    q, s = fo.quantize(torch.zeros(200, 128, dtype=torch.bfloat16), 128)
    assert s.tolist() == [[1.0], [1.0]]


@pytest.mark.parametrize("e", [-20, -3, 0, 1, 7, 30])
def test_scale_boundaries(e):
    x = torch.zeros(2, 128, dtype=torch.bfloat16)
    at = 448.0 * 2.0 ** e                                          # exactly representable in bf16 (1.75 * 2^(8+e))
    above = torch.tensor(at, dtype=torch.bfloat16).view(torch.int16) + 1   # next bf16 above it
    x[0, 5] = at
    x[1, 9] = -above.view(torch.bfloat16)
    q, s = fo.quantize(x, 1)
    assert s[0, 0].item() == 2.0 ** e and q.float()[0, 5].item() == 448.0
    assert s[1, 0].item() == 2.0 ** (e + 1) and q.float()[1, 9].item() == -224.0   # 448.x / 2 rounds to 224
    assert fo.scales_of(torch.tensor([2.0 ** -140])).item() == 2.0 ** -126          # clamp


def test_fake_quantize_keeps_dtype_and_rows():
    x = torch.randn(5, 7, 256).to(torch.bfloat16)
    y = fo.fake_quantize_rows(x)
    assert y.dtype == x.dtype and y.shape == x.shape
    assert fo.fake_quantize_rows(x[:0]).shape[0] == 0


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _cabi.lib()


def test_fp8_argument_validation_without_gpu(lib):
    # bagel_gemm_fp8(A, lda, a_scales, ld_as, W, ldw, w_scales, C, ldc, M, N, K, resid, ldr, epilogue, stream)
    rc = lib.bagel_gemm_fp8(None, 256, None, 8, None, 256, None, None, 256, 8, 256, 200, None, 0, ops.EPI_SWIGLU, None)
    assert rc == -1 and b"multiples of 128" in lib.bagel_last_error()
    rc = lib.bagel_gemm_fp8(None, 256, None, 8, None, 256, None, None, 256, 8, 192, 256, None, 0, ops.EPI_SWIGLU, None)
    assert rc == -1
    for epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_F32, ops.EPI_RESID_F32, 6, 99):
        rc = lib.bagel_gemm_fp8(None, 256, None, 8, None, 256, None, None, 256, 8, 256, 256, None, 0, epi, None)
        assert rc == -5 and b"epilogue" in lib.bagel_last_error(), epi
    rc = lib.bagel_gemm_fp8(None, 200, None, 8, None, 256, None, None, 256, 8, 256, 256, None, 0, ops.EPI_SWIGLU, None)
    assert rc == -2
    rc = lib.bagel_gemm_fp8(None, 256, None, 8, None, 256, None, None, 256, 8, 256, 256, None, 0, ops.EPI_RESID, None)
    assert rc == -5 and b"resid" in lib.bagel_last_error()
    # bagel_quantize_fp8_bf16(X, ldx, Q, ldq, scales, lds, M, K, block_rows, stream)
    rc = lib.bagel_quantize_fp8_bf16(None, 200, None, 200, None, 8, 8, 200, 1, None)
    assert rc == -1 and b"multiple of 128" in lib.bagel_last_error()
    rc = lib.bagel_quantize_fp8_bf16(None, 256, None, 256, None, 8, 8, 256, 64, None)
    assert rc == -5 and b"block_rows" in lib.bagel_last_error()
    rc = lib.bagel_quantize_fp8_bf16(None, 256, None, 256, None, 4, 8, 256, 1, None)
    assert rc == -5 and b"lds" in lib.bagel_last_error()
    # leading dimensions shorter than a row would make rows overlap
    rc = lib.bagel_quantize_fp8_bf16(None, 128, None, 256, None, 8, 8, 256, 1, None)
    assert rc == -5 and b"ldx and ldq" in lib.bagel_last_error()
    rc = lib.bagel_quantize_fp8_bf16(None, 256, None, 128, None, 8, 8, 256, 1, None)
    assert rc == -5 and b"ldx and ldq" in lib.bagel_last_error()
    for lda, ldw, ldc, ldr, epi in ((128, 256, 256, 0, ops.EPI_SWIGLU), (256, 128, 256, 0, ops.EPI_SWIGLU),
                                    (256, 256, 64, 0, ops.EPI_SWIGLU), (256, 256, 128, 256, ops.EPI_RESID),
                                    (256, 256, 256, 128, ops.EPI_RESID)):
        resid = 256 if epi == ops.EPI_RESID else None   # a non-null, 16-byte-aligned address; no call reaches the GPU
        rc = lib.bagel_gemm_fp8(None, lda, None, 8, None, ldw, None, None, ldc, 8, 256, 256, resid, ldr, epi, None)
        assert rc == -5 and b"lda, ldw" in lib.bagel_last_error(), (lda, ldw, ldc, ldr, epi)


def test_fp8_ops_refuse_cpu_tensors():
    a = torch.zeros(8, 128, dtype=torch.bfloat16)
    with pytest.raises(_cabi.BagelB200Error):
        ops.quantize_fp8(a)


def _llm(layer_module="Qwen2MoTDecoderLayer", hidden=256, inter=512):
    from bagel_b200.config import Qwen2Config
    return Qwen2Config(vocab_size=1024, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=2,
                       num_attention_heads=2, num_key_value_heads=1, qk_norm=True, layer_module=layer_module)


def test_model_flag_refusals():
    from bagel_b200.qwen2_navit import Qwen2ForCausalLM
    assert "fp8_gen_mlp" in inspect.signature(Qwen2ForCausalLM).parameters
    assert Qwen2ForCausalLM(_llm(), device="cpu").model.fp8_gen_mlp is False
    assert Qwen2ForCausalLM(_llm("Qwen2MoEDecoderLayer"), device="cpu", fp8_gen_mlp=True).model.fp8_gen_mlp
    with pytest.raises(NotImplementedError, match="dtype_mode"):
        Qwen2ForCausalLM(_llm(), device="cpu", dtype_mode="B", fp8_gen_mlp=True)
    with pytest.raises(ValueError, match="generation expert"):
        Qwen2ForCausalLM(_llm("Qwen2DecoderLayer"), device="cpu", fp8_gen_mlp=True)
    with pytest.raises(ValueError, match="multiples of 128"):
        Qwen2ForCausalLM(_llm(inter=576), device="cpu", fp8_gen_mlp=True)
    with pytest.raises(ValueError, match="multiples of 128"):
        Qwen2ForCausalLM(_llm(hidden=320), device="cpu", fp8_gen_mlp=True)


def test_public_entry_points_take_the_flag():
    from bagel_b200 import loader, synthetic
    assert inspect.signature(loader.load_bagel).parameters["fp8_gen_mlp"].default is False
    assert inspect.signature(synthetic.build_random_bagel).parameters["fp8_gen_mlp"].default is False


def test_training_forward_refuses_fp8():
    from bagel_b200.bagel import Bagel
    from bagel_b200.config import AutoEncoderParams, BagelConfig
    from bagel_b200.qwen2_navit import Qwen2ForCausalLM
    llm = _llm()
    bcfg = BagelConfig(visual_gen=True, visual_und=False, llm_config=llm, vit_config=None,
                       vae_config=AutoEncoderParams(), latent_patch_size=2, max_latent_size=8)
    model = Bagel(Qwen2ForCausalLM(llm, device="cpu", fp8_gen_mlp=True), None, bcfg)
    assert model.fp8_gen_mlp
    with pytest.raises(NotImplementedError, match="fp8_gen_mlp"):
        model.forward(4, torch.zeros(4, dtype=torch.long), torch.arange(4), [4], torch.arange(4)[None],
                      split_lens=[4], attn_modes=["causal"])


def _cuobjdump():
    cand = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return cand if os.path.exists(cand) else None


def test_fp8_wgmma_kernels_are_pipelined():
    """The fp8 GEMM assembles to QGMMA (test_sass_wgmma.py only looks at HGMMA): it must be there, and no kernel may
    carry gsb0 on every QGMMA (ptxas serialising the wgmma pipeline)."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found (CUDA toolkit binaries are not on PATH or in /usr/local/cuda/bin)")
    lib = build.build()
    sass = subprocess.run([tool, "-sass", str(lib)], check=True, capture_output=True, text=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function\s*:\s*(\S+)", line)
        if m:
            name = m.group(1)
        elif name is not None and "QGMMA." in line:
            n, g = kernels.get(name, (0, 0))
            kernels[name] = (n + 1, g + ("gsb0" in line))
    assert kernels, "no QGMMA found in the library: the fp8 GEMM kernels are missing"
    assert all("gemm_fp8_kernel" in k for k in kernels), sorted(kernels)
    serialized = sorted(k for k, (n, g) in kernels.items() if n == g)
    assert not serialized, f"fp8 wgmma kernels issue every QGMMA serialized: {serialized}"
