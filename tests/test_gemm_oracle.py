"""CPU: self-tests of the GEMM rounding-point bracket (tests/gemm_oracle.py) on emulated kernel outputs, and coverage of
its route table. The mutations below are the subtle kernel bugs the GPU route tests must catch: each one is rejected."""
import pytest
import torch
import torch.nn.functional as F

import gemm_oracle as go

BF = torch.bfloat16


def _silu32(x):
    return x / (1.0 + torch.exp(-x))


def _gelu32(x):
    return F.gelu(x, approximate="tanh")


def _accumulate(a, w, order="kstep", drop_last_block=False):
    """fp32 accumulation of a @ w.T: one fp32 add per 16-wide k-step, in k order or reversed."""
    K = a.shape[1]
    if drop_last_block:
        K = (K - 1) // 64 * 64
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
    steps = list(range(0, K, 16))
    for s in (reversed(steps) if order == "reverse" else steps):
        e = min(s + 16, K)
        acc = acc + a[:, s:e].float() @ w[:, s:e].float().t()
    return acc


def emulate(a, w, epi, bias=None, resid=None, row_map=None, order="kstep", mutation=None):
    """The kernel's epilogue in fp32 / bf16 torch arithmetic; returns the output rows in A-row order (float64)."""
    acc = _accumulate(a, w, order, drop_last_block=mutation == "drop_last_k_block")
    skip = mutation == "skip_inner"
    r = None
    if resid is not None:
        rows = row_map.long() + (1 if mutation == "row_map_off_by_one" else 0) if row_map is not None else slice(0, a.shape[0])
        r = resid[rows].float()
    if epi == go.EPI_SWIGLU:
        g, u = go.interleaved_halves(acc)
        if mutation == "swap_gate_up_block":
            g, u = g.clone(), u.clone()
            g[:, :128], u[:, :128] = u[:, :128].clone(), g[:, :128].clone()
        s = _silu32(g.to(BF).float())
        s = s if skip else s.to(BF).float()
        return (s * u.to(BF).float()).to(BF).double()
    x = acc
    if bias is not None:
        b = bias.roll(1) if mutation == "bias_shift" else bias
        x = x + b.float()[None, :]
    if epi == go.EPI_F32:
        return x.double()
    xb = x if skip else x.to(BF).float()
    if epi == go.EPI_BIAS:
        return x.to(BF).double()
    if epi == go.EPI_RESID:
        return (r + xb).to(BF).double()
    if epi == go.EPI_RESID_F32:
        return (r + xb).double()
    f = _silu32 if epi == go.EPI_SILU else _gelu32
    return f(xb).to(BF).double()


def _operands(family, M, N, K, epi, seed):
    g = torch.Generator().manual_seed(seed)
    a, w = (go.exact_operands if family == "exact" else go.normal_operands)(M, N, K, g)
    bias = None if epi == go.EPI_SWIGLU else torch.randn(N, generator=g).to(BF)
    resid = None
    if epi == go.EPI_RESID:
        resid = torch.randn(M + 5, N, generator=g).to(BF)
    elif epi == go.EPI_RESID_F32:
        resid = torch.randn(M + 5, N, generator=g)
    return a, w, bias, resid


ALL_EPIS = (go.EPI_BIAS, go.EPI_RESID, go.EPI_SWIGLU, go.EPI_GELU, go.EPI_SILU, go.EPI_F32, go.EPI_RESID_F32)
SHAPE = (48, 512, 200)   # K tail of 8 past three 64-wide blocks


@pytest.mark.parametrize("family", ["exact", "normal"])
@pytest.mark.parametrize("epi", ALL_EPIS, ids=lambda e: go.EPI_NAMES[e])
def test_bracket_accepts_correct_rounding_and_any_order(epi, family):
    M, N, K = SHAPE
    a, w, bias, resid = _operands(family, M, N, K, epi, 1 + epi)
    br = go.bracket(a, w, epi, bias, resid, exact=family == "exact")
    go.check(br.point, br, "fp64 rounded at the header's points")
    go.check(emulate(a, w, epi, bias, resid), br, "fp32 k-step order")
    go.check(emulate(a, w, epi, bias, resid, order="reverse"), br, "fp32 reversed order")
    stats = go.check(emulate(a, w, epi, bias, resid), br)
    if family == "exact":
        # exact sums: apart from the transcendental slack every element is pinned to one value
        assert stats["pinned"] > (0.97 if epi in (go.EPI_GELU, go.EPI_SILU, go.EPI_SWIGLU) else 0.9999), stats
        assert torch.equal(emulate(a, w, epi, bias, resid, order="reverse"), emulate(a, w, epi, bias, resid))


def test_reference_is_the_pinned_value():
    a, w, bias, resid = _operands("exact", *SHAPE, go.EPI_RESID, 3)
    ref = go.reference(a, w, bias, resid, go.EPI_RESID)
    assert torch.equal(ref, emulate(a, w, go.EPI_RESID, bias, resid))


@pytest.mark.parametrize("epi", ALL_EPIS, ids=lambda e: go.EPI_NAMES[e])
def test_bracket_rejects_one_ulp(epi):
    a, w, bias, resid = _operands("exact", *SHAPE, epi, 4)
    br = go.bracket(a, w, epi, bias, resid, exact=True)
    out = emulate(a, w, epi, bias, resid)
    pinned = ((br.lo == br.hi) & (out.abs() > 1e-3)).nonzero()
    i, j = pinned[len(pinned) // 2].tolist()
    if epi in go.F32_OUT:
        step = torch.nextafter(out[i, j].float(), torch.tensor(float("inf"))).double() - out[i, j]
    else:
        step = go.bf16_ulp(out[i, j])
    bad = out.clone()
    bad[i, j] += step
    with pytest.raises(AssertionError, match="outside the rounding-point bracket"):
        go.check(bad, br)


@pytest.mark.parametrize("epi", [go.EPI_RESID, go.EPI_RESID_F32, go.EPI_GELU, go.EPI_SILU, go.EPI_SWIGLU],
                         ids=lambda e: go.EPI_NAMES[e])
def test_bracket_rejects_skipped_inner_rounding(epi):
    """E.g. bf16_round(x0) replaced by x0 in the RESID branch of gemm.cu: the old 2-4 ulp tolerance accepts it."""
    a, w, bias, resid = _operands("exact", *SHAPE, epi, 5)
    br = go.bracket(a, w, epi, bias, resid, exact=True)
    with pytest.raises(AssertionError, match="outside the rounding-point bracket"):
        go.check(emulate(a, w, epi, bias, resid, mutation="skip_inner"), br)


@pytest.mark.parametrize("family", ["exact", "normal"])
@pytest.mark.parametrize("mutation,epi", [("bias_shift", go.EPI_BIAS), ("drop_last_k_block", go.EPI_BIAS),
                                          ("drop_last_k_block", go.EPI_F32), ("swap_gate_up_block", go.EPI_SWIGLU),
                                          ("row_map_off_by_one", go.EPI_RESID)])
def test_bracket_rejects_wrong_kernel(mutation, epi, family):
    M, N, K = SHAPE
    a, w, bias, resid = _operands(family, M, N, K, epi, 6)
    row_map = None
    if mutation == "row_map_off_by_one":
        row_map = torch.randperm(M + 4, generator=torch.Generator().manual_seed(7))[:M].to(torch.int32)
    br = go.bracket(a, w, epi, bias, resid, row_map=row_map, exact=family == "exact")
    go.check(emulate(a, w, epi, bias, resid, row_map), br)
    with pytest.raises(AssertionError, match="outside the rounding-point bracket"):
        go.check(emulate(a, w, epi, bias, resid, row_map, mutation=mutation), br)


def test_exact_operands_sum_exactly_in_fp32():
    for K in (8, 200, 3584, 18944):
        a, w = go.exact_operands(4, 16, K, torch.Generator().manual_seed(K))
        acc64, abs_sum = go.exact_product(a, w)
        assert float(abs_sum.max()) * float(1 / (a.float().abs()[a != 0].min() * w.float().abs()[w != 0].min())) < 2 ** 24
        assert torch.equal(_accumulate(a, w).double(), acc64)
        assert torch.equal(_accumulate(a, w, "reverse").double(), acc64)


@pytest.mark.parametrize("case", go.ROUTES, ids=lambda c: c.id)
def test_route_table_case_routes_where_labelled(case):
    assert go.label_of(go.route(case.M, case.N, case.K, case.epi, sm_count=132)) == case.label
    assert case.K % 8 == 0 and case.N % 8 == 0 and (case.epi != go.EPI_SWIGLU or case.N % 256 == 0)


def test_route_table_covers_every_reachable_instantiation():
    labels = {c.label for c in go.ROUTES}
    assert labels == go.reachable_instantiations()
    wide = {lbl for lbl in labels if lbl.startswith("gemm_bf16_kernel")}
    skinny = {lbl for lbl in labels if lbl.startswith("gemm_skinny_kernel")}
    assert len(wide) == 44 and len(skinny) == 27
    assert not set(go.UNREACHABLE) & labels
    # the unreachable CLUSTER 2 BN 32 instantiations: no M gives BN 32 with two M tiles
    for M in (1, 64, 65, 128, 129, 4096):
        for N in (1024, 3584, 8192):
            r = go.route(M, N, 512, go.EPI_F32)
            assert not (r.targs[0] == 32 and r.targs[3] == 2)
    # the table includes the 7B and SigLIP-so400m projection widths
    dims = {(c.N, c.K) for c in go.ROUTES}
    for nk in ((3584, 3584), (4608, 3584), (3584, 18944), (37888, 3584), (1152, 1152), (4304, 1152), (1152, 4304)):
        assert nk in dims, nk


def test_skinny_switch_off_routes_wide():
    for c in go.ROUTES:
        r = go.route(c.M, c.N, c.K, c.epi, skinny_on=False)
        assert r.kernel == "gemm_bf16_kernel"


@pytest.mark.parametrize("batch,Hq,Hk,D,lk,want", [
    (32, 28, 4, 128, 1245, ("attn_decode_kernel<7>", 2)),     # the benchmark's decode step
    (80, 28, 4, 128, 1245, ("attn_decode_kernel<7>", 1)),
    (34, 28, 4, 128, 4000, ("attn_decode_kernel<7>", 1)),
    (33, 28, 4, 128, 4000, ("attn_decode_kernel<7>", 2)),
    (12, 8, 4, 128, 4000, ("attn_decode_kernel<2>", 4)),
    (4, 8, 8, 128, 4000, ("attn_decode_kernel<1>", 8)),
    (4, 8, 8, 128, 400, ("attn_decode_kernel<1>", 4)),        # >= 64 keys per CTA caps the split
    (3, 12, 4, 128, 100, ("attn_varlen_kernel<128>", 1)),      # G = 3
    (3, 16, 1, 128, 100, ("attn_varlen_kernel<128>", 1)),      # G = 16
    (3, 8, 2, 64, 100, ("attn_varlen_kernel<64>", 1)),         # D = 64
])
def test_attn_route(batch, Hq, Hk, D, lk, want):
    r = go.attn_route(batch, Hq, Hk, D, 1, lk, sm_count=132)
    assert (r.name, r.split) == want
