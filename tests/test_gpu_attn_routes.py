"""-m gpu: every route of bagel_attn_varlen_fwd's single-query path against fp64 attention on the same bf16 inputs:
the split-KV decode kernel (attn_decode.cu) for each GQA group G in {1, 2, 4, 7, 8} at each split the rule picks on this
device (1, 2, 4, 8), the benchmark's decode shape, ragged and empty caches, a large-logit cross-CTA merge, the fallbacks to
the prefill kernel (D = 64, G = 3, G = 16), and strided q/k/v/out views with NaN gaps (SigLIP's fused-QKV layout)."""
import pytest
import torch

import gemm_oracle as go
from bagel_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
ATOL, RTOL = 1e-2, 2e-2   # the tolerances of test_gpu_kernels.py's decode test


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)


def _ref(q, k, v, lq, k_begin, lk, causal):
    """fp64 softmax attention per packed sample; keys of sample b are rows [k_begin[b], k_begin[b] + lk[b])."""
    Hq, Hk, D = q.shape[1], k.shape[1], q.shape[2]
    out = torch.zeros(q.shape, dtype=torch.float64, device=DEV)
    qs = 0
    for nq, kb, nk in zip(lq, k_begin, lk):
        if nq and nk:
            qb = q[qs:qs + nq].double().transpose(0, 1)
            kk = k[kb:kb + nk].double().transpose(0, 1).repeat_interleave(Hq // Hk, dim=0)
            vv = v[kb:kb + nk].double().transpose(0, 1).repeat_interleave(Hq // Hk, dim=0)
            s = qb @ kk.transpose(1, 2) * D ** -0.5
            if causal:
                vis = torch.arange(nk, device=DEV)[None, :] <= torch.arange(nq, device=DEV)[:, None] + (nk - nq)
                s = s.masked_fill(~vis[None], float("-inf"))
            out[qs:qs + nq] = torch.nan_to_num(torch.softmax(s, -1) @ vv, nan=0.0).transpose(0, 1)
        qs += nq
    return out


def _decode_inputs(lk, Hq, Hk, spare, seed, D=128):
    g = torch.Generator(device=DEV).manual_seed(seed)
    B = len(lk)
    cap = [n + spare for n in lk]
    q = torch.randn(B, Hq, D, device=DEV, generator=g).to(BF)
    k = torch.randn(sum(cap), Hk, D, device=DEV, generator=g).to(BF)
    v = torch.randn(sum(cap), Hk, D, device=DEV, generator=g).to(BF)
    return q, k, v, cap


def _run_decode(q, k, v, lk, cap, out=None):
    used = torch.tensor(lk, dtype=torch.int32, device=DEV)
    return ops.attn_varlen(q, k, v, _cu([1] * len(lk)), _cu(cap), 1, max(lk), True, out=out, seqused_k=used)


def _lens(B, seed, longest=1300):
    """Ragged cache lengths with empty caches and one long one (>= 64 keys per CTA even at split 8)."""
    g = torch.Generator().manual_seed(seed)
    lk = torch.randint(1, 700, (B,), generator=g).tolist()
    lk[0] = longest
    if B > 2:
        lk[B // 2] = 0
    if B > 4:
        lk[-1] = 1
    return lk


def _batch_for_split(split, Hk, sms):
    """A batch size at which the decode rule picks `split` (pairs = batch * Hk, one wave of ~2 CTAs per SM)."""
    pairs = {1: sms + 1, 2: sms, 4: sms // 2, 8: sms // 8}[split]
    return max(1, -(-pairs // Hk) if split == 1 else pairs // Hk)


GROUPS = {1: (4, 4), 2: (8, 4), 4: (16, 4), 7: (28, 4), 8: (8, 1)}   # G -> (Hq, Hk)


def _decode_cases():
    sms = _sms()
    cases = []
    for G, (Hq, Hk) in GROUPS.items():
        for split in (1, 2, 4, 8):
            B = _batch_for_split(split, Hk, sms)
            cases.append((f"G{G}-split{split}", _lens(B, 10 * G + split), Hq, Hk, 3))
    cases.append(("bench-32x1245", [1245] * 32, 28, 4, 0))
    cases.append(("80-samples", _lens(80, 7, 1245), 28, 4, 2))
    return cases


@pytest.fixture(scope="module")
def decode_cases():
    return _decode_cases()


def test_decode_every_group_and_split(decode_cases):
    for name, lk, Hq, Hk, spare in decode_cases:
        q, k, v, cap = _decode_inputs(lk, Hq, Hk, spare, len(name) + sum(lk))
        out = _run_decode(q, k, v, lk, cap)
        ref = _ref(q, k, v, [1] * len(lk), _cu(cap).tolist()[:-1], lk, True)
        assert torch.isfinite(out).all(), name
        torch.testing.assert_close(out.double(), ref, atol=ATOL, rtol=RTOL, msg=lambda m: f"{name}: {m}")
        assert bool((out[torch.tensor(lk, device=DEV) == 0] == 0).all()), f"{name}: empty cache must give 0"
        assert torch.equal(out, _run_decode(q, k, v, lk, cap)), f"{name}: repeated call differs"


def test_decode_routes_and_splits_observed(decode_cases, tmp_path):
    if not go.IN_CHILD:   # a fresh process: see gemm_oracle.run_in_child
        out = go.run_in_child(__file__, "test_decode_routes_and_splits_observed")
        print(out[out.find("decode route proof"):].splitlines()[0])
        return
    sms = _sms()
    inputs = []
    for name, lk, Hq, Hk, spare in decode_cases:
        q, k, v, cap = _decode_inputs(lk, Hq, Hk, spare, 1)
        inputs.append((name, lk, cap, q, k, v, go.attn_route(len(lk), Hq, Hk, 128, 1, max(lk), sms)))

    def run():
        for _, lk, cap, q, k, v, _r in inputs:
            _run_decode(q, k, v, lk, cap)

    n_kernels, seen = go.observe_kernels(run, tmp_path / "decode_routes.json")
    if n_kernels == 0:
        pytest.skip("torch.profiler recorded no CUDA kernel events on this machine (numerics: test_decode_every_group_and_split)")
    seen = [s for s in seen if s[0].startswith("attn_")]
    assert len(seen) == len(inputs)
    for (name, lk, *_x, want), (kname, grid) in zip(inputs, seen):
        assert kname == want.name, f"route table out of date: {name} ran {kname}, attn_route() predicts {want.name}"
        if grid is not None:
            assert grid == want.grid, f"route table out of date: {name} launched grid {grid}, predicted {want.grid}"
    splits = {want.split for *_x, want in inputs}
    assert splits == {1, 2, 4, 8}, splits
    print(f"decode route proof: {len(seen)} launches, splits observed {sorted(splits)} ({sms} SMs)")


@pytest.mark.parametrize("G,split", [(1, 8), (7, 8), (7, 2)])
def test_decode_large_logit_outlier_in_last_split(G, split):
    """|logit| ~ 60 with one outlier key in the last CTA's key range: the cluster merge combines very different maxima."""
    Hq, Hk = GROUPS[G]
    sms = _sms()
    B = _batch_for_split(split, Hk, sms)
    lk = [1500] * B
    q, k, v, cap = _decode_inputs(lk, Hq, Hk, 0, 100 + G)
    s = (60.0 * 128 ** 0.5) ** 0.5
    qf = q.float()
    qf = qf / qf.norm(dim=-1, keepdim=True) * s
    kf = k.float()
    kf = kf / kf.norm(dim=-1, keepdim=True) * s
    r = go.attn_route(B, Hq, Hk, 128, 1, max(lk), sms)
    assert r.split == split
    chunk = ((-(-1500 // split)) + 15) // 16 * 16
    for b in range(B):
        j = b * 1500 + min(1499, (split - 1) * chunk + 37)        # inside the last split's range
        kf[j] = qf[b, ::G]                                          # logit 60 for the first q head of each group
    q, k = qf.to(BF), kf.to(BF)
    out = _run_decode(q, k, v, lk, cap)
    ref = _ref(q, k, v, [1] * B, _cu(cap).tolist()[:-1], lk, True)
    assert torch.isfinite(out).all()
    torch.testing.assert_close(out.double(), ref, atol=ATOL, rtol=RTOL)


@pytest.mark.parametrize("Hq,Hk,D", [(8, 2, 64), (12, 4, 128), (16, 1, 128)], ids=["D64", "G3", "G16"])
def test_single_query_fallback_to_prefill(Hq, Hk, D, tmp_path):
    lk = _lens(6, Hq + D, 700)
    q, k, v, cap = _decode_inputs(lk, Hq, Hk, 5, Hq * D, D)
    want = go.attn_route(len(lk), Hq, Hk, D, 1, max(lk), _sms())
    assert want.kernel == "attn_varlen_kernel"
    n_kernels, seen = go.observe_kernels(lambda: _run_decode(q, k, v, lk, cap), tmp_path / "fallback.json")
    names = [s[0] for s in seen if s[0].startswith("attn_")]
    if names:   # the profiler may record nothing after earlier sessions in this process
        assert names == [want.name], "route table out of date"
    out = _run_decode(q, k, v, lk, cap)
    ref = _ref(q, k, v, [1] * len(lk), _cu(cap).tolist()[:-1], lk, True)
    torch.testing.assert_close(out.double(), ref, atol=ATOL, rtol=RTOL)


def _fused(n, Hq, Hk, head=72, seed=0):
    """SigLIP layout: q/k/v views of one [n, (Hq + 2 Hk) 128 + 64] buffer, channels past `head` zero, NaN tail columns."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    width = (Hq + 2 * Hk) * 128
    buf = torch.full((n, width + 64), float("nan"), device=DEV, dtype=BF)
    x = torch.randn(n, Hq + 2 * Hk, 128, device=DEV, generator=g)
    x[:, :, head:] = 0
    buf[:, :width] = x.reshape(n, width).to(BF)
    q = buf[:, :Hq * 128].unflatten(1, (Hq, 128))
    k = buf[:, Hq * 128:(Hq + Hk) * 128].unflatten(1, (Hk, 128))
    v = buf[:, (Hq + Hk) * 128:width].unflatten(1, (Hk, 128))
    return q, k, v


def _strided_out(n, Hq):
    buf = torch.full((n, Hq * 128 + 40), 0x7FA5, dtype=torch.int16, device=DEV).view(BF)
    return buf, buf[:, :Hq * 128].unflatten(1, (Hq, 128))


@pytest.mark.parametrize("kind", ["prefill", "decode"])
def test_strided_views_with_nan_gaps(kind):
    if kind == "prefill":   # SigLIP: 16 heads of 72 channels padded to 128, non-causal, ragged images
        Hq = Hk = 16
        lq = lk = [100, 257, 33]
        q, k, v = _fused(sum(lq), Hq, Hk, seed=1)
        cap, begins, maxq = lk, _cu(lk).tolist()[:-1], max(lq)
        used, causal = None, False
    else:                   # one query per sample against a fused K/V buffer with spare rows
        Hq, Hk = 28, 4
        lk = _lens(8, 3)
        lq = [1] * len(lk)
        cap = [n + 4 for n in lk]
        q, _, _ = _fused(len(lk), Hq, Hk, seed=2)
        _, k, v = _fused(sum(cap), Hq, Hk, seed=3)
        begins, maxq, causal = _cu(cap).tolist()[:-1], 1, True
        used = torch.tensor(lk, dtype=torch.int32, device=DEV)
    assert q.stride(0) > Hq * 128 and k.stride(0) > Hk * 128
    obuf, out = _strided_out(sum(lq), Hq)
    before = obuf.view(torch.int16).clone()
    ops.attn_varlen(q, k, v, _cu(lq), _cu(cap), maxq, max(lk), causal, out=out, seqused_k=used)
    assert torch.equal(obuf.view(torch.int16)[:, Hq * 128:], before[:, Hq * 128:]), "out's gap columns were written"
    assert torch.isfinite(out).all(), "a NaN gap leaked into the output"
    assert bool((out[:, :, 72:] == 0).all()), "padded head channels must stay exactly 0"
    ref = _ref(q, k, v, lq, begins, lk, causal)
    torch.testing.assert_close(out.double(), ref, atol=ATOL, rtol=RTOL)
