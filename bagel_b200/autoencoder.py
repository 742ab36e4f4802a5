"""FLUX VAE (AutoEncoder) — host side (reference: modeling/autoencoder.py:20-360).

Same surface as the reference: `AutoEncoderParams`, `AutoEncoder(params).encode(x) / .decode(z)`, `load_ae(path)`
returning `(ae, params)`; state-dict keys follow the reference's module names (SURVEY.md §8b).

Execution model (GPU-first): activations are NHWC bf16 and stay on the device; every convolution is the
implicit-GEMM wgmma kernel (bagel_conv2d_nhwc_bf16: no im2col buffer, the 3x3 taps are K-slices fetched by 4-D
TMA boxes whose out-of-image coordinates are the zero padding, stride-2 via TMA element strides, bias and the
ResnetBlock skip connection fused in the epilogue); GroupNorm(32)+swish is a deterministic two-stage reduction +
one fused normalise/activate pass; 1x1 convs of the attention block are plain GEMMs; the single-head d=512
attention is QK^T (fp32 logits) -> row softmax -> P V^T with the same GEMM kernel.

Numerics follow the reference under CUDA autocast (eval drivers, gen_images_mp.py:73,175): bf16 convolutions with
fp32 accumulation, GroupNorm + swish in fp32 on the bf16 conv output, fp32 GroupNorm parameters.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import ops
from .config import AutoEncoderParams

BF16 = torch.bfloat16


def _pad_to(n: int, m: int) -> int:
    return (n + m - 1) // m * m


class _Conv:
    """Conv2d weights in the kernel layout [Cout_pad8, k, k, Cin_pad64] bf16 (+ bf16 bias)."""

    def __init__(self, sd, name, device):
        w = sd[name + ".weight"].to(device, torch.float32)
        b = sd[name + ".bias"].to(device, torch.float32)
        co, ci, k, _ = w.shape
        self.cout, self.cin, self.k = co, ci, k
        cop, cip = _pad_to(co, 8), _pad_to(ci, 64)
        wk = torch.zeros((cop, k, k, cip), dtype=BF16, device=device)
        wk[:co, :, :, :ci] = w.permute(0, 2, 3, 1).to(BF16)
        bk = torch.zeros((cop,), dtype=BF16, device=device)
        bk[:co] = b.to(BF16)
        self.w, self.b = wk.contiguous(), bk.contiguous()

    def __call__(self, x, stride=1, pad=None, out_hw=None, resid=None):
        if pad is None:
            pad = self.k // 2
        return ops.conv2d_nhwc(x, self.w, self.b, stride=stride, pad=pad, out_hw=out_hw, resid=resid)


class _Norm:
    def __init__(self, sd, name, device):
        self.w = sd[name + ".weight"].to(device, torch.float32).contiguous()
        self.b = sd[name + ".bias"].to(device, torch.float32).contiguous()

    def __call__(self, x, swish=True):
        return ops.groupnorm_nhwc(x, self.w, self.b, 1e-6, swish)


class _ResBlock:
    def __init__(self, sd, name, device):
        self.norm1, self.conv1 = _Norm(sd, name + ".norm1", device), _Conv(sd, name + ".conv1", device)
        self.norm2, self.conv2 = _Norm(sd, name + ".norm2", device), _Conv(sd, name + ".conv2", device)
        self.shortcut = _Conv(sd, name + ".nin_shortcut", device) if (name + ".nin_shortcut.weight") in sd else None

    def __call__(self, x):
        h = self.conv1(self.norm1(x))
        skip = x if self.shortcut is None else self.shortcut(x)
        return self.conv2(self.norm2(h), resid=skip)       # x + h fused into conv2's epilogue


class _AttnBlock:
    def __init__(self, sd, name, device):
        self.norm = _Norm(sd, name + ".norm", device)
        self.q, self.k = _Conv(sd, name + ".q", device), _Conv(sd, name + ".k", device)
        self.v, self.proj = _Conv(sd, name + ".v", device), _Conv(sd, name + ".proj_out", device)

    def __call__(self, x):
        B, H, W, C = x.shape
        L = H * W
        h = self.norm(x, swish=False).view(B * L, C)
        lin = lambda conv, t: ops.gemm(t, conv.w.view(conv.w.shape[0], -1), bias=conv.b)  # 1x1 conv == GEMM
        q, k, v = lin(self.q, h), lin(self.k, h), lin(self.v, h)
        o = torch.empty((B * L, C), dtype=BF16, device=x.device)
        scale = float(C) ** -0.5
        for b in range(B):                                   # single head, d = C: per-image dense attention
            qb, kb, vb = q[b * L:(b + 1) * L], k[b * L:(b + 1) * L], v[b * L:(b + 1) * L]
            s = ops.gemm(qb, kb, epilogue=ops.EPI_F32)       # [L, L] fp32 logits
            p = ops.softmax_rows(s, scale)
            ops.gemm(p, ops.transpose(vb), out=o[b * L:(b + 1) * L])
        return ops.gemm(o, self.proj.w.view(C, -1), bias=self.proj.b, resid=x.view(B * L, C),
                        epilogue=ops.EPI_RESID).view(B, H, W, C)


class Encoder:
    def __init__(self, sd, p: AutoEncoderParams, device, pfx="encoder"):
        self.p = p
        self.conv_in = _Conv(sd, pfx + ".conv_in", device)
        self.down = []
        nres = len(p.ch_mult)
        for lvl in range(nres):
            blocks = [_ResBlock(sd, f"{pfx}.down.{lvl}.block.{i}", device) for i in range(p.num_res_blocks)]
            ds = _Conv(sd, f"{pfx}.down.{lvl}.downsample.conv", device) if lvl != nres - 1 else None
            self.down.append((blocks, ds))
        self.mid1 = _ResBlock(sd, pfx + ".mid.block_1", device)
        self.attn = _AttnBlock(sd, pfx + ".mid.attn_1", device)
        self.mid2 = _ResBlock(sd, pfx + ".mid.block_2", device)
        self.norm_out, self.conv_out = _Norm(sd, pfx + ".norm_out", device), _Conv(sd, pfx + ".conv_out", device)

    def __call__(self, x):
        h = self.conv_in(x)
        for blocks, ds in self.down:
            for blk in blocks:
                h = blk(h)
            if ds is not None:   # F.pad(x, (0,1,0,1)) + stride-2 valid conv (autoencoder.py:104-108)
                h = ds(h, stride=2, pad=0, out_hw=(h.shape[1] // 2, h.shape[2] // 2))
        h = self.mid2(self.attn(self.mid1(h)))
        return self.conv_out(self.norm_out(h))


class Decoder:
    def __init__(self, sd, p: AutoEncoderParams, device, pfx="decoder"):
        self.p = p
        self.conv_in = _Conv(sd, pfx + ".conv_in", device)
        self.mid1 = _ResBlock(sd, pfx + ".mid.block_1", device)
        self.attn = _AttnBlock(sd, pfx + ".mid.attn_1", device)
        self.mid2 = _ResBlock(sd, pfx + ".mid.block_2", device)
        self.up = {}
        nres = len(p.ch_mult)
        for lvl in range(nres):
            blocks = [_ResBlock(sd, f"{pfx}.up.{lvl}.block.{i}", device) for i in range(p.num_res_blocks + 1)]
            us = _Conv(sd, f"{pfx}.up.{lvl}.upsample.conv", device) if lvl != 0 else None
            self.up[lvl] = (blocks, us)
        self.norm_out, self.conv_out = _Norm(sd, pfx + ".norm_out", device), _Conv(sd, pfx + ".conv_out", device)

    def __call__(self, z):
        h = self.mid2(self.attn(self.mid1(self.conv_in(z))))
        for lvl in reversed(range(len(self.p.ch_mult))):
            blocks, us = self.up[lvl]
            for blk in blocks:
                h = blk(h)
            if us is not None:
                h = us(ops.upsample2x_nhwc(h))
        return self.conv_out(self.norm_out(h))


def _to_nhwc_padded(x: torch.Tensor, device) -> torch.Tensor:
    """[B,C,H,W] float -> [B,H,W,pad64(C)] bf16 (zero channels), the layout the conv kernel reads through TMA."""
    B, C, H, W = x.shape
    out = torch.zeros((B, H, W, _pad_to(C, 64)), dtype=BF16, device=device)
    out[..., :C] = x.to(device).permute(0, 2, 3, 1).to(BF16)
    return out


class AutoEncoder:
    def __init__(self, params: AutoEncoderParams, device="cuda"):
        self.params = params
        self.device = torch.device(device)
        self.scale_factor, self.shift_factor = params.scale_factor, params.shift_factor
        self.sample = True          # DiagonalGaussian(sample=True), autoencoder.py:276-287
        self.encoder: Optional[Encoder] = None
        self.decoder: Optional[Decoder] = None

    def eval(self):
        return self

    def to(self, device):
        assert self.encoder is None, "move before loading weights"
        self.device = torch.device(device)
        return self

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict=False, assign=False):
        self.encoder = Encoder(sd, self.params, self.device)
        self.decoder = Decoder(sd, self.params, self.device)
        return [], []

    @torch.no_grad()
    def encode(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B,3,H,W] in [-1,1] -> latent [B,z,H/f,W/f] (bf16). `noise` overrides the DiagonalGaussian draw
        (reference: torch.randn_like on the execution device, autoencoder.py:285)."""
        h = self.encoder(_to_nhwc_padded(x, self.device))                  # [B,h,w,2z]
        zc = self.params.z_channels
        moments = h[..., : 2 * zc].permute(0, 3, 1, 2)
        mean, logvar = moments[:, :zc], moments[:, zc:]
        if self.sample:
            std = torch.exp(0.5 * logvar)
            eps = torch.randn_like(mean) if noise is None else noise.to(mean.device, mean.dtype)
            z = mean + std * eps
        else:
            z = mean
        return self.scale_factor * (z - self.shift_factor)

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """latent [B,z,h,w] -> image [B,3,H,W] bf16 (autoencoder.py:320-322)."""
        z = z.to(self.device) / self.scale_factor + self.shift_factor
        img = self.decoder(_to_nhwc_padded(z, self.device))                # [B,H,W,8] (3 real channels)
        return img[..., : self.params.out_ch].permute(0, 3, 1, 2)

    def forward(self, x):
        return self.decode(self.encode(x))

    __call__ = forward


def load_ae(local_path: Optional[str], device="cuda") -> Tuple[AutoEncoder, AutoEncoderParams]:
    """Reference load_ae (autoencoder.py:339-360): fixed FLUX hyper-parameters, weights from ae.safetensors."""
    params = AutoEncoderParams(resolution=256, in_channels=3, downsample=8, ch=128, out_ch=3, ch_mult=[1, 2, 4, 4],
                               num_res_blocks=2, z_channels=16, scale_factor=0.3611, shift_factor=0.1159)
    ae = AutoEncoder(params, device)
    if local_path is not None:
        from safetensors.torch import load_file
        ae.load_state_dict(load_file(local_path))
    return ae, params
