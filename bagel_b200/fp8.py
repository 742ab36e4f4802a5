"""Block-scaled FP8 weights of the generation expert's MLP (`fp8_gen_mlp=True`, opt-in).

The format is defined once, in bagel_b200/csrc/gemm_fp8.cu (and include/bagel_b200.h): float8_e4m3fn values with one
power-of-two fp32 scale per 128 x 128 block of each reference weight matrix and per 1 x 128 group of each activation row.
This module owns the weight side: it quantises the reference `mlp_moe_gen` matrices at load with the same CUDA quantiser
the layer loop uses for activations, lays them out for bagel_gemm_fp8, and turns them back into reference-layout bf16
(`dequantize`), which is exact because every q * s is a bf16 value.

Layouts (bagel_gemm_fp8):
  wgu    e4m3 [2I, H]: gate and up rows interleaved in blocks of 64 (rows 128t..128t+63 = gate rows 64t.., the next 64 =
         up rows 64t..), so one 128-row tile of the GEMM holds 64 matching gate | up columns for the SwiGLU epilogue.
  wgu_s  fp32 [2I / 64, H / 128]: the scale of each 64-row half of the interleaved matrix, i.e. of the 128 x 128 gate or
         up block that half comes from.
  wd     e4m3 [H, I] (down_proj as in the reference); wd_s fp32 [H / 64, I / 128], each block scale repeated for its two
         64-row halves.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import ops

BF16 = torch.bfloat16
HALF = 64     # W rows per scale row of bagel_gemm_fp8 (half of its 128-row tile)


def _interleave(qg: torch.Tensor, qu: torch.Tensor) -> torch.Tensor:
    I, K = qg.shape
    g = qg.view(torch.uint8).reshape(I // HALF, HALF, K)
    u = qu.view(torch.uint8).reshape(I // HALF, HALF, K)
    return torch.stack((g, u), dim=1).reshape(2 * I, K).view(ops.FP8).contiguous()


def _dequant(q: torch.Tensor, s_half: torch.Tensor) -> torch.Tensor:
    """e4m3 [N, K] with per-(64 rows x 128 columns) scales [N / 64, K / 128] -> bf16 [N, K] (exact)."""
    N, K = q.shape
    x = q.float().reshape(N // HALF, HALF, K // 128, 128) * s_half[:, None, :, None]
    return x.reshape(N, K).to(BF16)


class GenMlpFp8:
    """The three quantised matrices of one layer's generation-expert MLP, in bagel_gemm_fp8 layouts."""
    __slots__ = ("wgu", "wgu_s", "wd", "wd_s")

    @classmethod
    def from_reference(cls, gate: torch.Tensor, up: torch.Tensor, down: torch.Tensor) -> "GenMlpFp8":
        """gate_proj / up_proj [I, H] and down_proj [H, I] bf16 CUDA tensors (reference layout)."""
        qg, sg = ops.quantize_fp8(gate.contiguous(), 128)
        qu, su = ops.quantize_fp8(up.contiguous(), 128)
        qd, sd = ops.quantize_fp8(down.contiguous(), 128)
        m = cls()
        m.wgu = _interleave(qg, qu)
        kb = sg.shape[1]
        m.wgu_s = torch.stack((sg.repeat_interleave(2, dim=0), su.repeat_interleave(2, dim=0)), dim=1).reshape(-1, kb)
        m.wgu_s = m.wgu_s.contiguous()
        m.wd = qd
        m.wd_s = sd.repeat_interleave(2, dim=0).contiguous()
        return m

    @classmethod
    def from_interleaved_bf16(cls, wgu: torch.Tensor, down: torch.Tensor) -> "GenMlpFp8":
        """From the bf16 gate|up layout of bagel_gemm_bf16 (blocks of 128, ops.interleave_gate_up) and down_proj."""
        I2, K = wgu.shape
        gu = wgu.view(I2 // 256, 2, 128, K)
        return cls.from_reference(gu[:, 0].reshape(I2 // 2, K), gu[:, 1].reshape(I2 // 2, K), down)

    def dequantize(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(gate_proj, up_proj, down_proj) as reference-layout bf16: exactly the weights the fp8 GEMMs multiply by."""
        I2, K = self.wgu.shape
        q = self.wgu.view(torch.uint8).reshape(I2 // (2 * HALF), 2, HALF, K)
        qg = q[:, 0].reshape(I2 // 2, K).view(ops.FP8)
        qu = q[:, 1].reshape(I2 // 2, K).view(ops.FP8)
        return _dequant(qg, self.wgu_s[0::2]), _dequant(qu, self.wgu_s[1::2]), _dequant(self.wd, self.wd_s)
