"""TEST INFRASTRUCTURE — an fp64 reference of bagel_gemm_bf16 with its rounding points bracketed, and a plain-Python
restatement of the host dispatch (gemm.cu, gemm_skinny.cu, attn.cu / attn_decode.cu). Pure torch, CPU-importable.

Epilogues (include/bagel_b200.h): every value the kernel holds in an fp32 register or stores as bf16 is a rounding
point. The bracket check carries an interval [lo, hi] (float64) through the header's formula:

  accumulator   acc32 in [acc64 - delta, acc64 + delta], ends rounded outward to fp32, where acc64 is the exact product
                of the bf16 operands (float64: exact for every shape here) and delta is the accumulation model
                    delta = (ceil(K / 16) + 16) * 2^-23 * sum_k |a_k w_k|
                one fp32 rounding of a full ulp (truncation allowed) per 16-wide wgmma k-step, plus one per split-K partial
                summed by the skinny kernel (cluster size <= 16);
  fp32 / bf16   round-to-nearest-even applied to both ends (monotone, so the image of the interval is inside);
  silu / gelu   exact image of the interval in float64, including the minimum where the function is not monotone, then
                widened by the error of the fp32 __expf / tanhf evaluation (SLACK below) before the next rounding.

Where the fp64 value is not near a rounding boundary the bracket is one value: the kernel must be correctly rounded bit for
bit. With exact-sum operands (exact_operands) acc32 == acc64 in any summation order, delta = 0, and every rounding point is
pinned: a skipped or added rounding point fails."""
from __future__ import annotations

import json
import math
import os
import re
import subprocess
import sys
from dataclasses import dataclass
from typing import Optional

import torch

EPI_BIAS, EPI_RESID, EPI_SWIGLU, EPI_GELU, EPI_SILU, EPI_F32, EPI_RESID_F32 = 0, 1, 2, 3, 4, 5, 7
EPI_NAMES = {EPI_BIAS: "BIAS", EPI_RESID: "RESID", EPI_SWIGLU: "SWIGLU", EPI_GELU: "GELU", EPI_SILU: "SILU",
             EPI_F32: "F32", EPI_RESID_F32: "RESID_F32"}
F32_OUT = (EPI_F32, EPI_RESID_F32)
SKINNY_EPIS = (EPI_BIAS, EPI_RESID, EPI_SWIGLU, EPI_GELU, EPI_SILU)
WIDE_EPIS = (EPI_BIAS, EPI_RESID, EPI_GELU, EPI_SILU, EPI_F32, EPI_RESID_F32)   # + SWIGLU at BN = 256
U23 = 2.0 ** -23

# ------------------------------------------------------------------------------------------------------------------
# rounding of float64 tensors
# ------------------------------------------------------------------------------------------------------------------


def rn_f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).double()


def rn_bf16(x: torch.Tensor) -> torch.Tensor:
    """Round to nearest even bf16. x must hold fp32 values (every bracket end passes rn_f32 / rd_f32 / ru_f32 first:
    the kernel rounds to bf16 from an fp32 register), so the float -> bf16 cast is a single rounding."""
    return x.to(torch.float32).to(torch.bfloat16).double()


def rd_f32(x: torch.Tensor) -> torch.Tensor:
    f = x.to(torch.float32)
    f = torch.where(f.double() > x, torch.nextafter(f, torch.full_like(f, -math.inf)), f)
    return f.double()


def ru_f32(x: torch.Tensor) -> torch.Tensor:
    f = x.to(torch.float32)
    f = torch.where(f.double() < x, torch.nextafter(f, torch.full_like(f, math.inf)), f)
    return f.double()


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (normal range)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


# ------------------------------------------------------------------------------------------------------------------
# epilogue functions and their interval images
# ------------------------------------------------------------------------------------------------------------------


def silu64(x):
    return x * torch.sigmoid(x)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def _argmin(f, lo, hi):
    lo, hi = torch.tensor(lo, dtype=torch.float64), torch.tensor(hi, dtype=torch.float64)
    for _ in range(200):   # golden-section search of the single minimum
        a, b = lo + 0.382 * (hi - lo), hi - 0.382 * (hi - lo)
        if f(a) < f(b):
            hi = b
        else:
            lo = a
    return float((lo + hi) / 2)


SILU_XMIN = _argmin(silu64, -3.0, 0.0)   # -1.2785
GELU_XMIN = _argmin(gelu64, -3.0, 0.0)   # -0.7518


def _image(f, xmin, lo, hi):
    """[min, max] of f over [lo, hi] for f decreasing left of xmin and increasing right of it."""
    flo, fhi = f(lo), f(hi)
    inside = (lo <= xmin) & (hi >= xmin)
    mn = torch.where(inside, torch.full_like(lo, float(f(torch.tensor(xmin, dtype=torch.float64)))), torch.minimum(flo, fhi))
    return mn, torch.maximum(flo, fhi)


def silu_slack(x, y):
    """|silu_f(x) - silu(x)| for silu_f = x / (1 + __expf(-x)): __expf is within (2 + 1.2 |x|) fp32 ulps, the add and the
    IEEE division add one rounding each."""
    return y.abs() * (4.0 + 2.0 * x.abs()) * U23 + 2.0 ** -149


def gelu_slack(x, y):
    """|gelu_tanh_f(x) - gelu(x)|: tanhf and the fp32 cubic move 1 + tanh(.) by a few ulps of 1 (absolute), the products
    add relative roundings."""
    return 0.5 * x.abs() * 8.0 * U23 + y.abs() * 4.0 * U23 + 2.0 ** -149


def _fn_bracket(kind, lo, hi):
    f, xmin, slack = (silu64, SILU_XMIN, silu_slack) if kind == "silu" else (gelu64, GELU_XMIN, gelu_slack)
    mn, mx = _image(f, xmin, lo, hi)
    amax = torch.maximum(lo.abs(), hi.abs())
    return rd_f32(mn - slack(amax, mn)), ru_f32(mx + slack(amax, mx))


# ------------------------------------------------------------------------------------------------------------------
# reference + bracket
# ------------------------------------------------------------------------------------------------------------------


def exact_product(a: torch.Tensor, w: torch.Tensor):
    """(acc64, sum_k |a_k w_k|) in float64 on a's device."""
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def delta_of(abs_sum: torch.Tensor, K: int) -> torch.Tensor:
    return (math.ceil(K / 16) + 16) * U23 * abs_sum


@dataclass
class Bracket:
    lo: torch.Tensor    # [M, n_out] float64
    hi: torch.Tensor
    point: torch.Tensor  # the fp64 value rounded at the header's points (round-to-nearest at every point)


def interleaved_halves(t: torch.Tensor):
    """Columns of a SwiGLU accumulator [M, 2I] (W rows interleaved per 128: gate block, up block) -> (gate, up) [M, I]."""
    M, N = t.shape
    t = t.reshape(M, N // 256, 2, 128)
    return t[:, :, 0].reshape(M, N // 2), t[:, :, 1].reshape(M, N // 2)


def bracket(a, w, epi, bias=None, resid=None, row_map=None, exact=False) -> Bracket:
    """Bracket of bagel_gemm_bf16's output rows [M, n_out] in A-row order (resid is gathered through row_map).
    exact=True asserts the operands are an exact-sum family (delta = 0)."""
    acc64, abs_sum = exact_product(a, w)
    K = a.shape[1]
    delta = torch.zeros_like(acc64) if exact else delta_of(abs_sum, K)
    lo, hi, pt = rd_f32(acc64 - delta), ru_f32(acc64 + delta), rn_f32(acc64)
    if resid is not None:
        r = resid[row_map.long()] if row_map is not None else resid[: a.shape[0]]
        r = r.double()
    if epi == EPI_SWIGLU:
        (glo, ulo), (ghi, uhi), (gpt, upt) = interleaved_halves(lo), interleaved_halves(hi), interleaved_halves(pt)
        glo, ghi, gpt = rn_bf16(glo), rn_bf16(ghi), rn_bf16(gpt)
        ulo, uhi, upt = rn_bf16(ulo), rn_bf16(uhi), rn_bf16(upt)
        slo, shi = _fn_bracket("silu", glo, ghi)
        slo, shi, spt = rn_bf16(slo), rn_bf16(shi), rn_bf16(rn_f32(silu64(gpt)))
        corners = torch.stack([slo * ulo, slo * uhi, shi * ulo, shi * uhi])   # bf16 x bf16: exact in fp32 and fp64
        return Bracket(rn_bf16(corners.amin(0)), rn_bf16(corners.amax(0)), rn_bf16(spt * upt))
    if bias is not None:
        b = bias.double()[None, :]
        lo, hi, pt = rn_f32(lo + b), rn_f32(hi + b), rn_f32(pt + b)
    if epi == EPI_F32:
        return Bracket(lo, hi, pt)
    lo, hi, pt = rn_bf16(lo), rn_bf16(hi), rn_bf16(pt)
    if epi == EPI_BIAS:
        return Bracket(lo, hi, pt)
    if epi == EPI_RESID:
        return Bracket(rn_bf16(rn_f32(r + lo)), rn_bf16(rn_f32(r + hi)), rn_bf16(rn_f32(r + pt)))
    if epi == EPI_RESID_F32:
        return Bracket(rn_f32(r + lo), rn_f32(r + hi), rn_f32(r + pt))
    kind = "silu" if epi == EPI_SILU else "gelu"
    f = silu64 if epi == EPI_SILU else gelu64
    flo, fhi = _fn_bracket(kind, lo, hi)
    return Bracket(rn_bf16(flo), rn_bf16(fhi), rn_bf16(rn_f32(f(pt))))


def check(out_rows: torch.Tensor, br: Bracket, what: str = "") -> dict:
    """Assert out_rows (kernel output in A-row order) lies in the bracket element by element. Returns statistics."""
    o = out_rows.double()
    ok = (o >= br.lo) & (o <= br.hi)
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i, j = bad[0].tolist()
        raise AssertionError(
            f"{what}: {bad.shape[0]} of {o.numel()} outputs outside the rounding-point bracket; first at [{i}, {j}]: "
            f"got {o[i, j].item()!r}, bracket [{br.lo[i, j].item()!r}, {br.hi[i, j].item()!r}], "
            f"fp64 rounded at the header's points {br.point[i, j].item()!r}")
    return {"pinned": float((br.lo == br.hi).double().mean()), "equal_point": float((o == br.point).double().mean())}


def reference(a, w, bias=None, resid=None, epi=EPI_BIAS, row_map=None) -> torch.Tensor:
    """The fp64 product rounded at the header's points (round-to-nearest everywhere), in A-row order."""
    return bracket(a, w, epi, bias, resid, row_map, exact=True).point


# ------------------------------------------------------------------------------------------------------------------
# operand families
# ------------------------------------------------------------------------------------------------------------------


def exact_operands(M, N, K, gen, device="cpu"):
    """a = i * 2^-4, w = j * 2^-e with |i|, |j| <= m and m^2 K < 2^24: every product is an integer multiple of 2^-(4+e)
    and every partial sum up to K stays below 2^24 * 2^-(4+e), so fp32 accumulation is exact in any order. e is chosen so
    that the sums are O(1), the range of real activations."""
    m = min(31, math.isqrt((2 ** 24 - 1) // K))
    e = max(0, round(math.log2(math.sqrt(K) * m * m / 48)))
    a = torch.randint(-m, m + 1, (M, K), generator=gen, device=device).float() * 2.0 ** -4
    w = torch.randint(-m, m + 1, (N, K), generator=gen, device=device).float() * 2.0 ** -e
    return a.to(torch.bfloat16), w.to(torch.bfloat16)


def normal_operands(M, N, K, gen, device="cpu"):
    a = torch.randn(M, K, generator=gen, device=device).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=gen, device=device) / K ** 0.5).to(torch.bfloat16)
    return a, w


# ------------------------------------------------------------------------------------------------------------------
# dispatch (restated from the host code; a change there must be mirrored here, and the GPU route proof checks it)
# ------------------------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class Route:
    kernel: str           # "gemm_bf16_kernel", "gemm_skinny_kernel", "attn_decode_kernel", "attn_varlen_kernel"
    targs: tuple          # template arguments as they appear in the kernel name
    split: int = 1        # skinny split-K / decode key split (cluster size)
    grid: Optional[tuple] = None

    @property
    def name(self):
        return f"{self.kernel}<{', '.join(str(t).lower() if isinstance(t, bool) else str(t) for t in self.targs)}>"


def skinny_supported(M, N, K, epi):
    return M <= 64 and N >= 256 and K >= 64 and epi in SKINNY_EPIS


def route(M, N, K, epi, sm_count=132, skinny_on=True) -> Route:
    """Which kernel bagel_gemm_bf16 launches for (M, N, K, epilogue) on a device with sm_count SMs (default
    environment: no BAGEL_SKINNY_SPLIT override)."""
    if skinny_on and skinny_supported(M, N, K, epi):
        nw = 2 if epi == EPI_SWIGLU else 1
        mt = 16 if M <= 16 else (32 if M <= 32 else 64)
        num_k = -(-K // 64)
        tiles = -(-N // (nw * 128))
        split = 1
        if nw == 1:
            split = max(1, min((sm_count * 8 // 5) // tiles, num_k // 12, 8))
            split = min(split, num_k, 16)
        return Route("gemm_skinny_kernel", (nw, epi, mt), split, (tiles, split, 1))
    if epi == EPI_SWIGLU:
        bn = 256
    else:
        bn = 256 if (N % 256 == 0 or N >= 1024) else (128 if N > 64 else 64)
        if M <= 128 and N >= 1024:
            bn = 32 if N <= 8192 else 64
    cluster = 2 if -(-M // 128) >= 2 else 1
    return Route("gemm_bf16_kernel", (bn, epi, False, cluster), 1)


DECODE_GROUPS = (1, 2, 4, 7, 8)


def attn_route(batch, Hq, Hk, D, max_seqlen_q, max_seqlen_k, sm_count=132) -> Route:
    """bagel_attn_varlen_fwd: the split-KV decode kernel for one query per sample at D = 128 and a supported GQA group,
    the prefill kernel otherwise."""
    G = Hq // Hk
    if max_seqlen_q == 1 and D == 128 and Hq % Hk == 0 and G in DECODE_GROUPS:
        pairs = batch * Hk
        split = 1
        while split < 8 and pairs * split * 2 <= 2 * sm_count:
            split *= 2
        if max_seqlen_k > 0:
            while split > 1 and (max_seqlen_k + split - 1) // split < 64:
                split >>= 1
        return Route("attn_decode_kernel", (G,), split, (split, Hk, batch))
    return Route("attn_varlen_kernel", (D,), 1)


# ------------------------------------------------------------------------------------------------------------------
# route table
# ------------------------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class Case:
    M: int
    N: int
    K: int
    epi: int
    label: str          # the instantiation (and split class) the shape must reach on a 132-SM H100
    note: str = ""

    @property
    def id(self):
        return f"{self.label}-{self.M}x{self.N}x{self.K}"

    @property
    def n_out(self):
        return self.N // 2 if self.epi == EPI_SWIGLU else self.N


def label_of(r: Route) -> str:
    if r.kernel == "gemm_skinny_kernel":
        return f"{r.name}/split{'1' if r.split == 1 else '>1'}"
    return r.name


def _wide(bn, cl, shapes):
    """One case per epilogue of gemm_bf16_kernel<bn, EPI, false, cl>; shapes: epi -> (M, N, K, note)."""
    out = []
    for epi in ((EPI_SWIGLU,) + WIDE_EPIS if bn == 256 else WIDE_EPIS):
        M, N, K, note = shapes(epi)
        out.append(Case(M, N, K, epi, f"gemm_bf16_kernel<{bn}, {epi}, false, {cl}>", note))
    return out


# Edges: ragged M (not a multiple of 128), N ragged inside the last tile, a K tail shorter than one 64-wide block, K < 64,
# an odd M-tile count under CLUSTER 2 (rank 1 of the last pair has no rows), N < 64 under CLUSTER 2 (rank 1's W slice is
# wholly out of bounds). Model shapes: BAGEL-7B (H 3584, I 18944, qkv 4608, vocab 152064) and SigLIP-so400m (H 1152,
# I 4304).
ROUTES = (
    # BN 256, one M tile: N % 256 == 0 and N < 1024 (M <= 64 only where the skinny path cannot take it)
    _wide(256, 1, lambda e: {EPI_SWIGLU: (100, 512, 200, "K tail 8"), EPI_BIAS: (65, 768, 64, ""),
                             EPI_RESID: (128, 256, 3584, "7B K"), EPI_GELU: (77, 512, 40, "K < 64"),
                             EPI_SILU: (90, 256, 136, "K tail 8"), EPI_F32: (1, 512, 64, "M = 1, wide at M <= 64"),
                             EPI_RESID_F32: (33, 768, 72, "wide at M <= 64")}[e])
    # BN 256, CLUSTER 2: odd M-tile counts, SigLIP widths with a ragged last N tile
    + _wide(256, 2, lambda e: {EPI_SWIGLU: (300, 1024, 1152, "3 M tiles"), EPI_BIAS: (729, 1152, 1152, "so400m o_proj, N tail 128"),
                               EPI_RESID: (385, 1152, 4304, "so400m fc2, 4 M tiles"), EPI_GELU: (729, 4304, 1152, "so400m fc1, N tail 208"),
                               EPI_SILU: (257, 1040, 96, "N tail 16, 3 M tiles"), EPI_F32: (200, 1032, 520, "N tail 8, K tail 8"),
                               EPI_RESID_F32: (600, 3584, 3584, "7B o_proj, 5 M tiles")}[e])
    # BN 128: 64 < N < 1024, N % 256 != 0
    + _wide(128, 1, lambda e: {EPI_BIAS: (70, 264, 72, "N tail 8"), EPI_RESID: (128, 136, 512, "N tail 8"),
                               EPI_GELU: (100, 384, 48, "K < 64"), EPI_SILU: (127, 640, 264, "K tail 8"),
                               EPI_F32: (17, 200, 64, "wide at M <= 64 (N < 256)"),
                               EPI_RESID_F32: (64, 904, 200, "wide at M <= 64")}[e])
    + _wide(128, 2, lambda e: {EPI_BIAS: (300, 264, 4304, ""), EPI_RESID: (129, 72, 64, "N = 72, one row in tile 2"),
                               EPI_GELU: (257, 1000, 8, "K = 8"), EPI_SILU: (640, 384, 128, "5 M tiles"),
                               EPI_F32: (200, 264, 512, "VAE logits shape"), EPI_RESID_F32: (383, 136, 3584, "")}[e])
    # BN 64: N <= 64 (both cluster sizes), or M <= 128 with N > 8192
    + _wide(64, 1, lambda e: {EPI_BIAS: (100, 152064, 128, "lm_head width, N > 8192"), EPI_RESID: (65, 8200, 64, "N > 8192, N tail 8"),
                              EPI_GELU: (128, 40, 96, "N < 64"), EPI_SILU: (50, 64, 64, "wide: N < 256"),
                              EPI_F32: (3, 16, 16, "K < 64, N < 64"), EPI_RESID_F32: (120, 18944, 72, "7B I width")}[e])
    + _wide(64, 2, lambda e: {EPI_BIAS: (4096, 64, 3584, "llm2vae"), EPI_RESID: (300, 24, 64, "N < 32: rank 1 slice out of bounds"),
                              EPI_GELU: (257, 56, 136, "3 M tiles"), EPI_SILU: (129, 8, 8, "N = K = 8"),
                              EPI_F32: (1000, 64, 520, ""), EPI_RESID_F32: (400, 32, 200, "N = 32: rank 1 slice out of bounds")}[e])
    # BN 32: M <= 128, 1024 <= N <= 8192 (CLUSTER 1 only: gemm_bf16_kernel<32, *, false, 2> is compiled but unreachable)
    + _wide(32, 1, lambda e: {EPI_BIAS: (80, 3584, 3584, "7B o_proj at 80 samples"), EPI_RESID: (128, 3584, 18944, "7B down_proj"),
                              EPI_GELU: (65, 1024, 200, ""), EPI_SILU: (100, 8192, 64, "N = 8192"),
                              EPI_F32: (5, 1032, 48, "K < 64, N tail 8"), EPI_RESID_F32: (80, 4608, 3584, "7B qkv width")}[e])
    # skinny: MT in {16, 32, 64} x {split 1, split > 1} (SwiGLU never splits: two W slabs per CTA)
    + [Case(M, N, K, epi, f"gemm_skinny_kernel<{2 if epi == EPI_SWIGLU else 1}, {epi}, {mt}>/split{s}", note)
       for (epi, mt, s, M, N, K, note) in (
           (EPI_BIAS, 16, "1", 1, 1024, 320, "K tail 0, split 1 (K too short)"),
           (EPI_BIAS, 16, ">1", 7, 4608, 3584, "7B qkv decode"),
           (EPI_BIAS, 32, "1", 24, 152064, 512, "lm_head width"),
           (EPI_BIAS, 32, ">1", 32, 264, 3584, "N tail 8"),
           (EPI_BIAS, 64, "1", 64, 2048, 72, "K tail 8"),
           (EPI_BIAS, 64, ">1", 33, 3584, 3584, ""),
           (EPI_RESID, 16, "1", 16, 8192, 64, ""),
           (EPI_RESID, 16, ">1", 1, 3584, 18944, "7B down_proj decode"),
           (EPI_RESID, 32, "1", 17, 3584, 1000, ""),
           (EPI_RESID, 32, ">1", 32, 3584, 3584, "7B o_proj decode"),
           (EPI_RESID, 64, "1", 40, 1024, 200, "K tail 8"),
           (EPI_RESID, 64, ">1", 64, 1152, 4304, "so400m fc2"),
           (EPI_SWIGLU, 16, "1", 5, 37888, 3584, "7B gate|up decode"),
           (EPI_SWIGLU, 32, "1", 31, 512, 136, "K tail 8"),
           (EPI_SWIGLU, 64, "1", 64, 2048, 64, ""),
           (EPI_GELU, 16, "1", 9, 256, 64, ""),
           (EPI_GELU, 16, ">1", 2, 4304, 1536, "so400m fc1 width (34 tiles)"),
           (EPI_GELU, 32, "1", 20, 520, 1472, "num_k 23: split 1"),
           (EPI_GELU, 32, ">1", 30, 1024, 1536, "num_k 24: split 2"),
           (EPI_GELU, 64, "1", 50, 1152, 264, ""),
           (EPI_GELU, 64, ">1", 63, 1152, 4304, ""),
           (EPI_SILU, 16, "1", 3, 3584, 256, "timestep MLP width"),
           (EPI_SILU, 16, ">1", 1, 256, 3584, "one W slab"),
           (EPI_SILU, 32, "1", 32, 13568, 3584, "106 tiles: split 1"),
           (EPI_SILU, 32, ">1", 25, 13440, 3584, "105 tiles: split 2"),
           (EPI_SILU, 64, "1", 64, 256, 64, ""),
           (EPI_SILU, 64, ">1", 48, 2048, 8192, ""),
       )]
)

# gemm_bf16_kernel<32, EPI, false, 2> is instantiated (dispatch_epi<32> passes the cluster size through) but no shape
# reaches it: BN 32 needs M <= 128, i.e. one M tile.
UNREACHABLE = tuple(f"gemm_bf16_kernel<32, {e}, false, 2>" for e in WIDE_EPIS)


_KERNEL_RE = re.compile(r"(gemm_bf16_kernel|gemm_skinny_kernel|attn_decode_kernel|attn_varlen_kernel)<([^>]*)>")


def observe_kernels(fn, trace_path):
    """Run fn() once under torch.profiler (CUDA activities) -> (number of kernel events, [(bagel kernel name as
    Route.name spells it, launch grid or None)] in launch order)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(trace_path))
    with open(trace_path) as f:
        events = json.load(f).get("traceEvents", [])
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    seen = []
    for e in kernels:
        m = _KERNEL_RE.search(e.get("name", ""))
        if m:
            grid = e.get("args", {}).get("grid")
            seen.append((f"{m.group(1)}<{', '.join(p.strip() for p in m.group(2).split(','))}>",
                         tuple(grid) if grid else None))
    return len(kernels), seen


IN_CHILD = os.environ.get("BAGEL_TEST_CHILD") == "1"


def run_in_child(test_file, test_name, **env):
    """Run one GPU test in a fresh Python process and return its output; skip if it skipped. Used for the profiler route
    proofs (a torch.profiler session that follows earlier ones in the same process may record only part of the kernel
    events) and for the BAGEL_GEMM_SKINNY / BAGEL_PDL switches, which the library reads once per process. The child
    inherits BAGEL_TEST_LIB, which conftest honours."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    proc = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-rs", "-p", "no:cacheprovider", "-m", "gpu",
                           f"{test_file}::{test_name}"], env=dict(os.environ, BAGEL_TEST_CHILD="1", **env),
                          capture_output=True, text=True, timeout=1800, cwd=root)
    if re.search(r"\b1 skipped", proc.stdout):
        import pytest
        pytest.skip("child: " + proc.stdout[proc.stdout.rfind("SKIPPED"):][:400])
    assert proc.returncode == 0 and re.search(r"\b1 passed", proc.stdout), proc.stdout[-4000:] + proc.stderr[-2000:]
    return proc.stdout


def reachable_instantiations():
    """Every (kernel instantiation, split class) bagel_gemm_bf16 can launch on a 132-SM device."""
    out = set()
    for bn, epis, clusters in ((256, (EPI_SWIGLU,) + WIDE_EPIS, (1, 2)), (128, WIDE_EPIS, (1, 2)), (64, WIDE_EPIS, (1, 2)),
                               (32, WIDE_EPIS, (1,))):
        out |= {f"gemm_bf16_kernel<{bn}, {e}, false, {c}>" for e in epis for c in clusters}
    for epi in SKINNY_EPIS:
        for mt in (16, 32, 64):
            splits = ("1",) if epi == EPI_SWIGLU else ("1", ">1")
            out |= {f"gemm_skinny_kernel<{2 if epi == EPI_SWIGLU else 1}, {epi}, {mt}>/split{s}" for s in splits}
    return out
