"""-m gpu: adversarial inputs for the attention kernel's LAZY RESCALING path (bagel_b200/csrc/attn.cu: scores are
exponentiated against a reference maximum carried over from earlier key blocks; a block is redone exactly only when its
row sum leaves [0, 2^30]) and the large / causal shapes of BASELINE configs[4] (L = 4k causal, 16k), which the N(0,1)
tests in test_gpu_kernels.py never stress: row maxima that grow with every key block, |logit| up to ~100 (what trained
q/k-norm weights produce), single outlier keys placed after the reference maximum was fixed, jumps sized just below /
above the redo trigger, all-equal scores, fully masked tiles in causal ragged batches.

Reference: exact fp32 softmax attention on the same bf16 inputs (the semantics of flash_attn_varlen_func as the
reference calls it, qwen2_navit.py:579-588), computed on the GPU in plain torch for a subset of query rows."""
import math

import pytest
import torch

from bagel_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)


def _ref_rows(q, k, v, lq, lk, causal, rows_per_sample=None):
    """Exact fp32 attention for (a subset of) query rows of each packed sample -> (row index tensor, [R, Hq, D] fp32)."""
    Hq, Hk, D = q.shape[1], k.shape[1], q.shape[2]
    rep = Hq // Hk
    scale = D ** -0.5
    idx, outs = [], []
    qs = ks = 0
    for b, (nq, nk) in enumerate(zip(lq, lk)):
        if nq:
            rows = torch.arange(nq, device=DEV) if rows_per_sample is None else rows_per_sample(b, nq).to(DEV)
            qb = q[qs + rows].float().transpose(0, 1)                                  # [Hq, R, D]
            kb = k[ks:ks + nk].float().transpose(0, 1).repeat_interleave(rep, dim=0)   # [Hq, nk, D]
            vb = v[ks:ks + nk].float().transpose(0, 1).repeat_interleave(rep, dim=0)
            s = torch.matmul(qb, kb.transpose(1, 2)) * scale
            if causal:
                vis = torch.arange(nk, device=DEV)[None, :] <= (rows[:, None] + (nk - nq))
                s = s.masked_fill(~vis[None], float("-inf"))
            p = torch.softmax(s, dim=-1)
            o = torch.nan_to_num(torch.matmul(p, vb), nan=0.0).transpose(0, 1)          # rows without keys -> 0
            idx.append(qs + rows)
            outs.append(o)
        qs += nq
        ks += nk
    return torch.cat(idx), torch.cat(outs)


def _check(q, k, v, lq, lk, causal, rows_per_sample=None, atol=2e-2, rtol=2e-2):
    out = ops.attn_varlen(q, k, v, _cu(lq), _cu(lk), max(lq), max(lk), causal).float()
    assert torch.isfinite(out).all(), "attention produced inf/NaN"
    idx, ref = _ref_rows(q, k, v, lq, lk, causal, rows_per_sample)
    torch.testing.assert_close(out[idx], ref, atol=atol, rtol=rtol)
    return out


def _unit(n, D, g):
    x = torch.randn(n, D, device=DEV, generator=g)
    return x / x.norm(dim=-1, keepdim=True)


def _mk(Lq, Lk, Hq, Hk, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(Lq, Hq, D, device=DEV, generator=g)
    k = torch.randn(Lk, Hk, D, device=DEV, generator=g)
    v = torch.randn(Lk, Hk, D, device=DEV, generator=g)
    return q, k, v, g


@pytest.mark.parametrize("direction", ["up", "down", "saw"])
@pytest.mark.parametrize("peak", [12.0, 45.0, 100.0])
def test_row_max_moves_every_key_block(direction, peak):
    """logit(q_i, k_j) = peak * f(j): the row maximum grows (or falls, or zig-zags) with every block of 128 keys, so the
    carried-over reference maximum is stale at every block; peak 100 => p would overflow fp32 without the exact redo."""
    Lq, Lk, Hq, Hk, D = 384, 1536, 4, 2, 128
    q, k, v, g = _mk(Lq, Lk, Hq, Hk, D, 11)
    u = _unit(1, D, g)[0]
    ramp = torch.arange(Lk, device=DEV, dtype=torch.float32) / (Lk - 1)
    if direction == "down":
        ramp = 1.0 - ramp
    elif direction == "saw":
        ramp = ((torch.arange(Lk, device=DEV) // 128) % 2).float() * 0.9 + 0.1 * ramp
    a = math.sqrt(peak * math.sqrt(D))
    q = 0.05 * q + a * u
    k = 0.05 * k + (a * ramp)[:, None, None] * u
    _check(q.to(BF), k.to(BF), v.to(BF), [Lq], [Lk], False)


@pytest.mark.parametrize("where", [5, 700, 1535])
@pytest.mark.parametrize("boost", [20.0, 20.8, 21.5, 60.0, -60.0])
def test_single_outlier_key(where, boost):
    """One key whose logit is `boost` nats above (below) a flat background, placed in the first, a middle or the last key
    block. 20.8 nats = 2^30: the values around it straddle the kernel's redo trigger (row sum of a block > 2^30)."""
    Lq, Lk, Hq, Hk, D = 256, 1536, 4, 4, 128
    q, k, v, g = _mk(Lq, Lk, Hq, Hk, D, 12)
    u = _unit(1, D, g)[0]
    a = math.sqrt(abs(boost) * math.sqrt(D))
    q = 0.02 * q + a * u
    k = 0.02 * k
    k[where] += math.copysign(a, boost) * u
    out = _check(q.to(BF), k.to(BF), v.to(BF), [Lq], [Lk], False)
    if boost >= 20.0:   # the outlier takes (almost) all the weight: out == v[where]
        torch.testing.assert_close(out, v[where].to(BF).float()[None].expand(Lq, -1, -1).repeat_interleave(Hq // Hk, 1),
                                   atol=2e-2, rtol=2e-2)


def test_all_equal_scores_is_the_mean_of_v():
    Lq, Lk, Hq, Hk, D = 300, 1000, 4, 2, 128
    q, k, v, g = _mk(Lq, Lk, Hq, Hk, D, 13)
    q = torch.zeros_like(q)
    out = _check(q.to(BF), k.to(BF), v.to(BF), [Lq], [Lk], False)
    mean_v = v.to(BF).float().mean(0).repeat_interleave(Hq // Hk, 0)
    torch.testing.assert_close(out, mean_v[None].expand(Lq, -1, -1), atol=5e-3, rtol=1e-2)
    # identical keys: the same, with a large common logit (softmax is shift invariant)
    k2 = (k[:1] * 6.0).expand(Lk, -1, -1).contiguous()
    q2 = (k[:1, :1] * 6.0).expand(Lq, Hq, -1).contiguous()
    _check(q2.to(BF), k2.to(BF), v.to(BF), [Lq], [Lk], False)


@pytest.mark.parametrize("sigma", [3.0, 6.0])
@pytest.mark.parametrize("causal", [False, True])
def test_heavy_tailed_logits(sigma, causal):
    """q, k ~ N(0, sigma^2): logits ~ N(0, (sigma^2)^2) -> |logit| up to ~40 (sigma 3) / ~150 (sigma 6), maxima move a lot."""
    lq, lk = [257, 640, 130], [900, 640, 1300]
    Hq, Hk, D = 8, 2, 128
    q, k, v, g = _mk(sum(lq), sum(lk), Hq, Hk, D, 14)
    _check((sigma * q).to(BF), (sigma * k).to(BF), v.to(BF), lq, lk, causal)


def test_causal_ragged_with_fully_masked_tiles():
    """Bottom-right aligned causal masks over a ragged batch: Lq > Lk (leading rows see no key at all -> zeros, whole
    leading 256-row CTAs idle), Lq == Lk, Lq < Lk, a one-row sample, an empty-query sample, lengths straddling the
    128/256 tile edges; large logits so the masked (-inf) entries meet a moving maximum."""
    lq = [700, 256, 129, 1, 0, 515, 384]
    lk = [200, 256, 1000, 300, 40, 140, 385]
    Hq, Hk, D = 4, 2, 128
    q, k, v, g = _mk(sum(lq), sum(lk), Hq, Hk, D, 15)
    _check((2.5 * q).to(BF), (2.5 * k).to(BF), v.to(BF), lq, lk, True)
    _check((2.5 * q).to(BF), (2.5 * k).to(BF), v.to(BF), lq, lk, False)


def test_growing_max_with_causal_mask_d64():
    Lq = Lk = 1100
    Hq, Hk, D = 4, 4, 64
    q, k, v, g = _mk(Lq, Lk, Hq, Hk, D, 16)
    u = _unit(1, D, g)[0]
    a = math.sqrt(70.0 * math.sqrt(D))
    ramp = torch.arange(Lk, device=DEV, dtype=torch.float32) / (Lk - 1)
    q = 0.05 * q + a * u
    k = 0.05 * k + (a * ramp)[:, None, None] * u
    _check(q.to(BF), k.to(BF), v.to(BF), [Lq], [Lk], True)


# ---------------------------------------------------------------------------------------------------------------------
# BASELINE configs[4] shapes (heads 32, d 128): L = 16384 and causal L = 4096, checked on a row subset per sample
# ---------------------------------------------------------------------------------------------------------------------
def _subset(step, extra):
    def f(b, n):
        r = torch.cat([torch.arange(0, n, step), torch.tensor([e for e in extra if 0 <= e < n], dtype=torch.long)])
        return torch.unique(r)
    return f


@pytest.mark.parametrize("Hk", [32, 4])
def test_L16384_noncausal(Hk):
    L, Hq, D = 16384, 32, 128
    q, k, v, g = _mk(L, L, Hq, Hk, D, 17)
    _check(q.to(BF), k.to(BF), v.to(BF), [L], [L], False, _subset(211, [127, 128, 255, 256, 16383]), atol=1e-2)


@pytest.mark.parametrize("Hk", [32, 4])
def test_L4096_causal_and_ragged(Hk):
    Hq, D = 32, 128
    lq = [4096, 4096, 2049, 3333]
    lk = [4096, 4096 + 66, 2049, 4000]
    q, k, v, g = _mk(sum(lq), sum(lk), Hq, Hk, D, 18)
    _check((1.5 * q).to(BF), (1.5 * k).to(BF), v.to(BF), lq, lk, True,
           _subset(97, [0, 1, 127, 128, 129, 255, 256, 2048, 4095]), atol=1e-2)


def test_L1024_causal_16_sequences():
    Hq, Hk, D = 32, 32, 128
    lq = lk = [1024] * 16
    q, k, v, g = _mk(sum(lq), sum(lk), Hq, Hk, D, 19)
    _check(q.to(BF), k.to(BF), v.to(BF), lq, lk, True, _subset(61, [0, 127, 128, 1023]), atol=1e-2)
