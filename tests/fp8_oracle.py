"""TEST INFRASTRUCTURE — the block-scaled FP8 format of `fp8_gen_mlp=True`, restated in plain torch, independently of
bagel_b200 (nothing here calls the product's quantiser or its fp8 module).

  scale   s = the smallest power of two with amax <= 448 s, at least 2^-126; s = 1 for an all-zero group. Written here
          with frexp (amax = f 2^E, f in [0.5, 1); 448 = 0.875 2^9), not with the exponent-bit rule the CUDA kernel uses.
  value   q = e4m3(x / s), round to nearest even (torch's float8_e4m3fn cast); q s is exactly a bf16 value.
  groups  1 x 128 along K (activations) or 128 x 128 (weights).

Under `fp8_contract()` the oracle's SwiGLU MLP (oracle/qwen2_mot.py swiglu_mlp) runs the generation expert
(`mlp_moe_gen.`) on fake-quantised inputs: the MLP input and the down_proj input are replaced by q s, and its weights are
expected to be the dequantised ones (`reference_state_dict`). Any fp32-accumulating bf16 GEMM then computes the
contract's sum; only the order of the fp32 additions differs from the product's fp8 GEMM."""
from __future__ import annotations

import contextlib
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import gpu_leg
from oracle import qwen2_mot as om

E4M3 = torch.float8_e4m3fn
GEN_PREFIX = "mlp_moe_gen."


def scales_of(amax: torch.Tensor) -> torch.Tensor:
    """fp32 power-of-two scales for group maxima `amax` (>= 0)."""
    a = amax.float()
    f, e = torch.frexp(a)
    k = (e - 9 + (f > 0.875).to(e.dtype)).clamp(min=-126)
    s = torch.ldexp(torch.ones_like(a), k)
    return torch.where(a == 0, torch.ones_like(a), s)


def quantize(x: torch.Tensor, block_rows: int):
    """x [M, K] (K % 128 == 0) -> (q e4m3 [M, K], s fp32 [ceil(M / block_rows), K / 128])."""
    M, K = x.shape
    xf = x.float()
    R = (M + block_rows - 1) // block_rows
    pad = torch.zeros(R * block_rows, K, dtype=torch.float32, device=x.device)
    pad[:M] = xf
    amax = pad.abs().reshape(R, block_rows, K // 128, 128).amax(dim=(1, 3))
    s = scales_of(amax)
    s_full = s.repeat_interleave(block_rows, 0)[:M].repeat_interleave(128, 1)
    q = (xf / s_full).to(E4M3)
    return q, s


def dequantize(q: torch.Tensor, s: torch.Tensor, block_rows: int) -> torch.Tensor:
    M, K = q.shape
    return q.float() * s.repeat_interleave(block_rows, 0)[:M].repeat_interleave(128, 1)


def fake_quantize_rows(x: torch.Tensor) -> torch.Tensor:
    """x [..., K] -> q s per 1 x 128 group, in x's dtype (exact for bf16)."""
    shp = x.shape
    x2 = x.reshape(-1, shp[-1])
    if x2.shape[0] == 0:
        return x
    q, s = quantize(x2, 1)
    return dequantize(q, s, 1).to(x.dtype).reshape(shp)


def _swiglu_fp8(orig):
    def swiglu_mlp(x, sd, pfx):
        if not pfx.endswith(GEN_PREFIX):
            return orig(x, sd, pfx)
        xq = fake_quantize_rows(x.to(om._AUTOCAST[0]))
        g = om.linear(xq, sd[pfx + "gate_proj.weight"])
        u = om.linear(xq, sd[pfx + "up_proj.weight"])
        return om.linear(fake_quantize_rows(F.silu(g) * u), sd[pfx + "down_proj.weight"])
    return swiglu_mlp


@contextlib.contextmanager
def fp8_contract():
    """with fp8_contract(): the oracle's gen-expert MLP fake-quantises its two GEMM inputs."""
    orig = om.swiglu_mlp
    om.swiglu_mlp = _swiglu_fp8(orig)
    try:
        yield
    finally:
        om.swiglu_mlp = orig


def gen_mlp_weights(e) -> Dict[str, torch.Tensor]:
    """Reference-layout bf16 gate / up / down of a product expert holding fp8 weights, dequantised here from the raw
    e4m3 bytes and scales (layouts: include/bagel_b200.h, bagel_gemm_fp8)."""
    m = e.fp8
    I2, K = m.wgu.shape
    q = m.wgu.view(torch.uint8).reshape(I2 // 128, 2, 64, K)
    out = {}
    for j, name in ((0, "gate_proj.weight"), (1, "up_proj.weight")):
        qj = q[:, j].reshape(I2 // 2, K).view(E4M3)
        s64 = m.wgu_s[j::2]                       # one scale per 64 rows of this matrix and K block
        out[name] = dequantize(qj, s64, 64).to(torch.bfloat16)
    out["down_proj.weight"] = dequantize(m.wd, m.wd_s, 64).to(torch.bfloat16)
    return out


def reference_state_dict(model) -> Dict[str, torch.Tensor]:
    """gpu_leg.export_reference_state_dict for a model loaded with fp8_gen_mlp=True: the gen MLP weights are the exact
    dequantised bf16 matrices the product's fp8 GEMMs multiply by."""
    lm = model.language_model.model
    saved = []
    for li, layer in enumerate(lm.layers):
        e = layer.gen
        w = gen_mlp_weights(e)
        saved.append((e, e.wgu, e.wd))
        e.wgu = torch.stack((w["gate_proj.weight"].view(-1, 128, w["gate_proj.weight"].shape[1]),
                             w["up_proj.weight"].view(-1, 128, w["up_proj.weight"].shape[1])), dim=1)
        e.wgu = e.wgu.reshape(-1, w["gate_proj.weight"].shape[1])   # the bf16 path's 128-row gate | up interleave
        e.wd = w["down_proj.weight"]
    try:
        return gpu_leg.export_reference_state_dict(model)
    finally:
        for e, wgu, wd in saved:
            e.wgu, e.wd = wgu, wd
