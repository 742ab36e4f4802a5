"""-m gpu: C-ABI entry points that were reached only through whole-model runs, against fp64 / fp32 restatements of the
header's formulas: layernorm (every VPL bucket, large common offset, strided rows), rmsnorm (incl. the H > 3584 bucket that
loads the weights after the reduction), rmsnorm_f32, latent_embed_add_f32, copy_rows_f32, the decode bookkeeping kernels,
unrounded RoPE tables, and q/k-norm + RoPE flows 2 and 3 in the separate kernel and the fused QKV epilogue."""
import pytest
import torch

import gemm_oracle as go
from bagel_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
U24 = 2.0 ** -24


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _mul(lo, hi, c, rnd):
    """Bracket of rnd(t * c) for t in [lo, hi] (c a tensor of exact values, any sign)."""
    p, q = rnd(lo * c), rnd(hi * c)
    return torch.minimum(p, q), torch.maximum(p, q)


def _within(out, lo, hi, what):
    o = out.double()
    ok = (o >= lo) & (o <= hi)
    assert bool(ok.all()), f"{what}: {(~ok).sum().item()} outside the bracket; first {o[~ok][:3].tolist()} vs " \
                           f"[{lo[~ok][:3].tolist()}, {hi[~ok][:3].tolist()}]"


# ----------------------------------------------------------------------------------------------------------------- norms

@pytest.mark.parametrize("H", [64, 144, 256, 512, 1152, 2048, 4096])   # VPL buckets 1, 1, 1, 2, 5, 8, 16 and their edges
def test_layernorm_every_bucket_offset_rows_strided(H):
    g = _gen(H)
    N = 37
    x = torch.randn(N, H, device=DEV, generator=g)
    x[::3] += 50.0                                   # large common offset: a one-pass variance loses it
    x = x.to(BF)
    w = (1 + 0.2 * torch.randn(H, device=DEV, generator=g)).to(BF)
    b = (0.1 * torch.randn(H, device=DEV, generator=g)).to(BF)
    xbuf = torch.full((N, H + 24), float("nan"), device=DEV, dtype=BF)
    xbuf[:, :H] = x
    ybuf = torch.full((N, H + 40), 0x7FA5, dtype=torch.int16, device=DEV).view(BF)
    before = ybuf.view(torch.int16).clone()
    ops.layernorm(xbuf[:, :H], w, b, 1e-6, out=ybuf[:, :H])
    assert torch.equal(ybuf.view(torch.int16)[:, H:], before[:, H:]), "padding columns of y were written"
    y = ybuf[:, :H].double()
    x64 = x.double()
    mean = x64.mean(1, keepdim=True)
    xc = x64 - mean
    r = (xc.pow(2).mean(1, keepdim=True) + 1e-6).rsqrt()
    t = xc * r * w.double()
    ref = t + b.double()
    # one bf16 rounding of the fp64 value; fp32 evaluation error (two-pass mean / variance, rsqrtf) as slack
    slack = 64 * U24 * (t.abs() + b.double().abs()) + 64 * U24 * mean.abs() * r * w.double().abs()
    err = (y - ref).abs()
    assert bool((err <= go.bf16_ulp(ref) + slack).all()), f"H={H}: max err {err.max().item():.3e}"
    assert (y != go.rn_bf16(go.rn_f32(ref))).double().mean().item() < 0.01


def _rms_r(x64, H, eps=1e-6):
    r = (x64.pow(2).mean(1, keepdim=True) + eps).rsqrt()
    s = (H / 1024 + 16) * U24                        # fp32 sum of squares (short per-thread runs + tree) and rsqrtf
    return r * (1 - s), r * (1 + s)


@pytest.mark.parametrize("N,H", [(5, 8), (33, 4096), (17, 8192)])
def test_rmsnorm_bf16_routed_all_buckets(N, H):
    """y = bf16(w_e * bf16(x * r)); H = 8192 is the VPL = 32 bucket (weights loaded after the reduction)."""
    g = _gen(H + N)
    x = torch.randn(N, H, device=DEV, generator=g).to(BF)
    w0 = (1 + 0.1 * torch.randn(H, device=DEV, generator=g)).to(BF)
    w1 = (1 + 0.1 * torch.randn(H, device=DEV, generator=g)).to(BF)
    ex = (torch.rand(N, device=DEV, generator=g) > 0.5).to(torch.uint8)
    y = ops.rmsnorm(x, w0, w1, ex)
    rlo, rhi = _rms_r(x.double(), H)
    x64 = x.double()
    n_lo, n_hi = _mul(rlo, rhi, x64, lambda v: go.rn_bf16(go.rn_f32(v)))
    wsel = torch.where(ex.bool()[:, None], w1.double()[None], w0.double()[None])
    lo, hi = _mul(n_lo, n_hi, wsel, go.rn_bf16)     # bf16 x bf16 is exact in fp32: one rounding
    _within(y, lo, hi, f"rmsnorm H={H}")


@pytest.mark.parametrize("out_f32", [0, 1])
@pytest.mark.parametrize("H", [64, 3584])
def test_rmsnorm_f32_routed(out_f32, H):
    """y = w_e * (x * r), both products rounded to fp32; out_f32 = 0 stores bf16(y)."""
    g = _gen(H + out_f32)
    N = 23
    x = 3 * torch.randn(N, H, device=DEV, generator=g)
    w0 = 1 + 0.1 * torch.randn(H, device=DEV, generator=g)
    w1 = 1 + 0.1 * torch.randn(H, device=DEV, generator=g)
    ex = (torch.rand(N, device=DEV, generator=g) > 0.5).to(torch.uint8)
    y = ops.rmsnorm_f32(x, w0, w1, ex, out_dtype=torch.float32 if out_f32 else BF)
    rlo, rhi = _rms_r(x.double(), H)
    t_lo, t_hi = _mul(rlo, rhi, x.double(), go.rn_f32)
    wsel = torch.where(ex.bool()[:, None], w1.double()[None], w0.double()[None])
    lo, hi = _mul(t_lo, t_hi, wsel, go.rn_f32)
    if not out_f32:
        lo, hi = go.rn_bf16(lo), go.rn_bf16(hi)
    _within(y, lo, hi, f"rmsnorm_f32 H={H} out_f32={out_f32}")


# ------------------------------------------------------------------------------------------------------- bit-exact kernels

@pytest.mark.parametrize("with_temb", [True, False])
def test_latent_embed_add_f32_bit_exact(with_temb):
    g = _gen(11)
    M, H = 50, 264
    proj = torch.randn(M, H + 8, device=DEV, generator=g).to(BF)[:, :H]
    temb = torch.randn(H, device=DEV, generator=g).to(BF) if with_temb else None
    table = torch.randn(64, H, device=DEV, generator=g)
    pid = torch.randint(0, 64, (M,), device=DEV, generator=g)
    seq = torch.full((70, H + 16), -3.0, device=DEV)
    rows = torch.randperm(70, device=DEV, generator=g)[:M].to(torch.int32)
    ops.latent_embed_add_f32(proj, temb, table, pid, seq, rows)
    s = (proj.float() + temb.float()).to(BF).float() if with_temb else proj.float()
    assert torch.equal(seq[rows.long(), :H], s + table[pid])
    untouched = torch.ones(70, dtype=torch.bool, device=DEV)
    untouched[rows.long()] = False
    assert bool((seq[untouched] == -3.0).all()) and bool((seq[:, H:] == -3.0).all())


def test_copy_rows_f32_bit_exact():
    g = _gen(12)
    src = torch.randn(100, 3584, device=DEV, generator=g)
    src[0, :4] = torch.tensor([float("nan"), float("-inf"), -0.0, 1e-40])   # bytes, not values
    idx = torch.randint(0, 100, (40,), device=DEV, generator=g).to(torch.int32)
    dst = torch.zeros(40, 3584, device=DEV)
    ops.copy_rows_f32(src, dst, src_rows=idx)
    assert torch.equal(dst.view(torch.int32), src[idx.long()].view(torch.int32))
    dst2 = torch.full((130, 3584), 7.0, device=DEV)
    perm = torch.randperm(130, device=DEV, generator=g)[:100].to(torch.int32)
    ops.copy_rows_f32(src, dst2, dst_rows=perm)
    assert torch.equal(dst2[perm.long()].view(torch.int32), src.view(torch.int32))
    untouched = torch.ones(130, dtype=torch.bool, device=DEV)
    untouched[perm.long()] = False
    assert bool((dst2[untouched] == 7.0).all())


@pytest.mark.parametrize("B", [1, 5, 33, 1024])
def test_decode_prepare_and_advance_bit_exact(B):
    g = _gen(B)
    seq_len = torch.randint(0, 900, (B,), device=DEV, generator=g).to(torch.int32)
    k_begin = torch.cat([torch.zeros(1, device=DEV), (seq_len.double() + 40).cumsum(0)]).to(torch.int32)
    pos = torch.randint(0, 5000, (B,), device=DEV, generator=g)
    steps = 4
    history = torch.full((steps + 1, B), -1, dtype=torch.int64, device=DEV)
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    kv_rows = torch.empty(B, dtype=torch.int32, device=DEV)
    used = torch.empty(B, dtype=torch.int32, device=DEV)
    sl0, pos0 = seq_len.clone(), pos.clone()
    toks = []
    for s in range(steps):
        ops.decode_prepare(k_begin, seq_len, kv_rows, used)
        assert torch.equal(kv_rows, k_begin[:B] + seq_len) and torch.equal(used, seq_len + 1)
        tok = torch.randint(0, 152064, (B,), device=DEV, generator=g)
        toks.append(tok)
        ops.decode_advance(seq_len, pos, tok, history, step_dev)
        assert step_dev.item() == s + 1
        assert torch.equal(seq_len, sl0 + s + 1) and torch.equal(pos, pos0 + s + 1)
    assert torch.equal(history[:steps], torch.stack(toks)), "history is [step, sample]"
    assert bool((history[steps] == -1).all())


# ------------------------------------------------------------------------------------------------------------------ RoPE

def _inv_freq(D, theta=1e6):
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(DEV)


def test_rope_table_unrounded_matches_fp32():
    pos = torch.cat([torch.arange(0, 70, device=DEV), torch.tensor([4095, 32767, 65567, 1 << 20], device=DEV)])
    inv = _inv_freq(128)
    cos, sin = ops.rope_table(pos, inv, round_bf16=False)
    ang = pos.float()[:, None] * inv[None, :]
    for got, ref in ((cos, torch.cos(ang)), (sin, torch.sin(ang))):
        ulp = (torch.nextafter(ref.abs(), torch.full_like(ref, float("inf"))) - ref.abs()).clamp_min(2.0 ** -149)
        assert bool(((got - ref).abs() <= ulp).all()), f"max err {(got - ref).abs().max().item():.3e}"
    c16, s16 = ops.rope_table(pos, inv, round_bf16=True)
    assert torch.equal(c16, cos.to(BF).float()) and torch.equal(s16, sin.to(BF).float())


def _qk_inputs(N, Hq, Hk, D, flow, seed):
    g = _gen(seed)
    qkv = torch.randn(N, (Hq + 2 * Hk) * D, device=DEV, generator=g).to(BF)
    qw = [1 + 0.1 * torch.randn(D, device=DEV, generator=g) for _ in range(2)]
    kw = [1 + 0.1 * torch.randn(D, device=DEV, generator=g) for _ in range(2)]
    ex = (torch.rand(N, device=DEV, generator=g) > 0.3).to(torch.uint8)
    pos = torch.randint(0, 5000, (N,), device=DEV, dtype=torch.int64, generator=g)
    cos, sin = ops.rope_table(pos, _inv_freq(D), round_bf16=False)   # flows 2, 3: fp32 tables
    return qkv, qw, kw, ex, cos, sin


def _qk_ref(qkv, qw, kw, ex, cos, sin, Hq, Hk, D, flow, eps=1e-6):
    """The header's fp32 formulas in torch fp32: flow 2 = bf16(x * r) * w, flow 3 = (x * r) * w, then
    q cos + rotate_half(q) sin with every product rounded to fp32."""
    N = qkv.shape[0]
    x = qkv.float()

    def one(t, wu, wg):
        r = (t.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
        n = t * r
        if flow == 2:
            n = n.to(BF).float()
        w = torch.where(ex.bool()[:, None, None], wg[None, None], wu[None, None])
        y = w * n
        a, b = y[..., : D // 2], y[..., D // 2:]
        c, s = cos[:, None], sin[:, None]
        out = torch.cat([a * c + (-b) * s, b * c + a * s], -1).to(BF)
        # flow 2 rounds x * r to bf16: a 1-ulp difference of r (rsqrtf, sum order) may move that rounding by one bf16 ulp
        # of the normalised value, which reaches the output scaled by |cos| and |sin|
        mix = torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], -1) if flow == 2 else 0 * out.float()
        return out, mix * 2.0 ** -7

    q, qm = one(x[:, : Hq * D].reshape(N, Hq, D), qw[0], qw[1])
    k, km = one(x[:, Hq * D:(Hq + Hk) * D].reshape(N, Hk, D), kw[0], kw[1])
    return q.reshape(N, Hq * D), k.reshape(N, Hk * D), qm.reshape(N, Hq * D), km.reshape(N, Hk * D)


def _close_1ulp(got, ref, what, flip):
    g, r = got.double(), ref.double()
    err = (g - r).abs()
    # one bf16 ulp of the output (rsqrt / sum-order ulps), flow 2's intermediate rounding (`flip`), a tiny floor near 0
    tol = go.bf16_ulp(r) * 1.01 + flip.double() * 1.01 + 8e-3 * 2.0 ** -4
    assert bool((err <= tol).all()), f"{what}: max err {err.max().item():.3e}"
    assert (g != r).double().mean().item() < 5e-3, f"{what}: {(g != r).double().mean().item():.4f} differ"


@pytest.mark.parametrize("D,Hq,Hk", [(128, 28, 4), (64, 4, 2)])
@pytest.mark.parametrize("flow", [2, 3])
def test_qk_norm_rope_flows_2_3(D, Hq, Hk, flow):
    N = 300
    qkv, qw, kw, ex, cos, sin = _qk_inputs(N, Hq, Hk, D, flow, D + flow)
    q_out = torch.zeros(N, Hq * D, device=DEV, dtype=BF)
    kbuf = torch.zeros(N + 50, Hk * D, device=DEV, dtype=BF)
    vbuf = torch.zeros_like(kbuf)
    rows = torch.randperm(N + 50, device=DEV, generator=_gen(9))[:N].to(torch.int32)
    ops.qk_norm_rope(qkv, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q_out, kbuf, vbuf, rows, Hq, Hk, D, 1e-6, flow)
    q_ref, k_ref, q_flip, k_flip = _qk_ref(qkv, qw, kw, ex, cos, sin, Hq, Hk, D, flow)
    _close_1ulp(q_out, q_ref, f"flow {flow} q", q_flip)
    _close_1ulp(kbuf[rows.long()], k_ref, f"flow {flow} k", k_flip)
    assert torch.equal(vbuf[rows.long()], qkv[:, (Hq + Hk) * D:])


@pytest.mark.parametrize("flow", [2, 3])
def test_fused_qkv_epilogue_flows_2_3_match_two_kernel_path(flow):
    """bagel_gemm_qkv_norm_rope == bagel_gemm_bf16 + bagel_qk_norm_rope for the fp32-weight flows, incl. row_map."""
    g = _gen(77 + flow)
    N, K, Hq, Hk, D = 700, 512, 6, 2, 128
    a = torch.randn(N, K, device=DEV, generator=g).to(BF)
    w = (torch.randn((Hq + 2 * Hk) * D, K, device=DEV, generator=g) / K ** 0.5).to(BF)
    b = (0.1 * torch.randn((Hq + 2 * Hk) * D, device=DEV, generator=g)).to(BF)
    _, qw, kw, ex, cos, sin = _qk_inputs(N, Hq, Hk, D, flow, 5)
    rows = torch.randperm(N + 40, device=DEV, generator=g)[:N].to(torch.int32)

    def run(fused):
        q = torch.zeros(N, Hq * D, device=DEV, dtype=BF)
        kb = torch.zeros(N + 40, Hk * D, device=DEV, dtype=BF)
        vb = torch.zeros_like(kb)
        if fused:
            ops.gemm_qkv_norm_rope(a, w, b, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q, kb, vb, rows, Hq, Hk, 1e-6, flow)
        else:
            qkv = ops.gemm(a, w, bias=b)
            ops.qk_norm_rope(qkv, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q, kb, vb, rows, Hq, Hk, D, 1e-6, flow)
        return q, kb, vb

    q1, k1, v1 = run(True)
    q0, k0, v0 = run(False)
    assert torch.equal(v1, v0)
    _, _, q_flip, k_flip = _qk_ref(ops.gemm(a, w, bias=b), qw, kw, ex, cos, sin, Hq, Hk, D, flow)
    k_flip = torch.zeros(N + 40, Hk * D, device=DEV).index_copy_(0, rows.long(), k_flip)
    for got, ref, nm, flip in ((q1, q0, "q", q_flip), (k1, k0, "k", k_flip)):
        _close_1ulp(got, ref, f"fused flow {flow} {nm}", flip)
    sel = torch.tensor([0, 5, 699, 128, 129], device=DEV, dtype=torch.int32)
    q2, k2, v2 = q1.clone(), k1.clone(), v1.clone()
    q2[sel.long()] = 0
    ops.gemm_qkv_norm_rope(a[sel.long()].contiguous(), w, b, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q2, k2, v2, rows,
                           Hq, Hk, 1e-6, flow, row_map=sel)
    assert torch.equal(q2, q1) and torch.equal(k2, k1) and torch.equal(v2, v1)
