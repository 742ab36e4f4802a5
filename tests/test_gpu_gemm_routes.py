"""-m gpu: every dispatch route of bagel_gemm_bf16 (tests/gemm_oracle.py ROUTES: 44 wide and 27 skinny instantiation /
split classes) against the fp64 reference with its rounding points bracketed, on dense, strided (NaN gaps, sentinel
output padding) and row_map-scattered layouts; a profiler pass proves each case ran the kernel the table predicts."""
import os

import pytest
import torch

import gemm_oracle as go
from bagel_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
SENTINEL16 = 0x7FA5              # bf16 NaN payload: a stray store or a read-back of the gap shows
SENTINEL32 = 0x7FA5A5A5
SKINNY_ON = os.environ.get("BAGEL_GEMM_SKINNY", "1") != "0"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _out_dtype(epi):
    return torch.float32 if epi in go.F32_OUT else BF


def _sentinel(rows, cols, dtype):
    if dtype == torch.float32:
        return torch.full((rows, cols), SENTINEL32, dtype=torch.int32, device=DEV).view(torch.float32)
    return torch.full((rows, cols), SENTINEL16, dtype=torch.int16, device=DEV).view(BF)


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _in_gap(t, rows, cols, nan=True):
    """t [r, c] as the top-left view of a larger buffer [rows, cols] whose other elements are NaN (or random)."""
    buf = torch.full((rows, cols), float("nan"), dtype=t.dtype, device=DEV) if nan else \
        torch.randn(rows, cols, device=DEV).to(t.dtype)
    buf[: t.shape[0], : t.shape[1]] = t
    return buf[: t.shape[0], : t.shape[1]]


def _operands(case, family, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a, w = (go.exact_operands if family == "exact" else go.normal_operands)(case.M, case.N, case.K, g, DEV)
    bias = None if case.epi == go.EPI_SWIGLU else torch.randn(case.N, device=DEV, generator=g).to(BF)
    resid = None
    if case.epi == go.EPI_RESID:
        resid = torch.randn(case.M, case.N, device=DEV, generator=g).to(BF)
    elif case.epi == go.EPI_RESID_F32:
        resid = torch.randn(case.M, case.N, device=DEV, generator=g)
    return a, w, bias, resid


def _check_case(case, tag=""):
    """Dense (both operand families, repeat bit-identical), strided and row_map layouts of one route case."""
    epi, M, N, K, n_out = case.epi, case.M, case.N, case.K, case.n_out
    for fi, family in enumerate(("exact", "normal")):
        a, w, bias, resid = _operands(case, family, 1000 * fi + M + 7 * N + K)
        out = ops.gemm(a, w, bias=bias, resid=resid, epilogue=epi)
        br = go.bracket(a, w, epi, bias, resid, exact=family == "exact")
        go.check(out, br, f"{tag}{case.id} dense {family}")
        again = ops.gemm(a, w, bias=bias, resid=resid, epilogue=epi)
        assert torch.equal(_bits(out), _bits(again)), f"{case.id}: repeated call differs"

    # strided: lda > K, ldw > K (NaN gaps and NaN rows past M / N), ldc > n_out, ldr != ldc, each a multiple of 8
    a, w, bias, resid = _operands(case, "exact", 3 + M + N + K)
    br = go.bracket(a, w, epi, bias, resid, exact=True)
    a_s = _in_gap(a, M + 5, K + 24)
    w_s = _in_gap(w, N + 8, K + 40)
    r_s = None if resid is None else _in_gap(resid, M + 3, N + 56)
    cbuf = _sentinel(M + 4, n_out + 16, _out_dtype(epi))
    before = _bits(cbuf).clone()
    ops.gemm(a_s, w_s, bias=bias, resid=r_s, epilogue=epi, out=cbuf[:M, :n_out])
    go.check(cbuf[:M, :n_out], br, f"{tag}{case.id} strided")
    keep = torch.ones_like(before, dtype=torch.bool)
    keep[:M, :n_out] = False
    assert torch.equal(_bits(cbuf)[keep], before[keep]), f"{case.id}: strided call wrote outside C's [M, n_out] view"

    # row_map scatter, residual gathered through the map; every other row untouched
    R = M + 37
    rm = torch.randperm(R, device=DEV, generator=torch.Generator(device=DEV).manual_seed(M))[:M].to(torch.int32)
    rbig = None
    if resid is not None:
        rbig = _in_gap(torch.randn(R, N, device=DEV).to(resid.dtype), R, N + 24)
    br = go.bracket(a, w, epi, bias, rbig, row_map=rm, exact=True)
    cbig = _sentinel(R, n_out + 8, _out_dtype(epi))
    before = _bits(cbig).clone()
    ops.gemm(a_s, w_s, bias=bias, resid=rbig, row_map=rm, epilogue=epi, out=cbig[:, :n_out])
    go.check(cbig[rm.long(), :n_out], br, f"{tag}{case.id} row_map")
    keep = torch.ones_like(before, dtype=torch.bool)
    keep[rm.long(), :n_out] = False
    assert torch.equal(_bits(cbig)[keep], before[keep]), f"{case.id}: row_map call wrote outside the mapped rows"


@pytest.mark.parametrize("case", go.ROUTES, ids=lambda c: c.id)
def test_route_numerics(case):
    _check_case(case)


def _observe(cases, tmp_path, skinny_on):
    """Each case once in its own profiler session; the GEMM launch it records must be exactly the kernel (and skinny grid)
    route() predicts. A session that records no kernel event skips only that case's proof, with the reason."""
    sms = _sms()
    seen, unrecorded = [], []
    for i, c in enumerate(cases):
        a, w, bias, resid = _operands(c, "normal", 5)
        n_kernels, names = go.observe_kernels(lambda: ops.gemm(a, w, bias=bias, resid=resid, epilogue=c.epi),
                                              tmp_path / f"route{i}.json")
        gemm = [s for s in names if s[0].startswith("gemm_")]
        if not gemm:
            unrecorded.append(c.id)
            continue
        assert len(gemm) == 1, f"{c.id}: {len(gemm)} GEMM launches for one call"
        name, grid = gemm[0]
        want = go.route(c.M, c.N, c.K, c.epi, sms, skinny_on)
        assert name == want.name, f"route table out of date: {c.id} ran {name}, route() predicts {want.name}"
        if want.grid is not None and grid is not None:
            assert grid == want.grid, f"route table out of date: {c.id} launched grid {grid}, route() predicts {want.grid}"
        seen.append(name)
    if unrecorded:
        pytest.skip(f"torch.profiler recorded no kernel event for {len(unrecorded)} of {len(cases)} cases "
                    f"({', '.join(unrecorded[:5])}...); their numeric checks ran in test_route_numerics")
    return seen


def test_routes_observed(tmp_path):
    if not go.IN_CHILD:
        out = go.run_in_child(__file__, "test_routes_observed")
        print(out[out.find("route proof"):].splitlines()[0])
        return
    seen = _observe(go.ROUTES, tmp_path, SKINNY_ON)
    if SKINNY_ON and _sms() == 132:
        assert {go.label_of(go.route(c.M, c.N, c.K, c.epi)) for c in go.ROUTES} == go.reachable_instantiations()
    print(f"route proof: {len(seen)} GEMM launches matched route() ({_sms()} SMs)")


def test_f32_accumulator_within_delta():
    """EPI_F32 without bias stores the raw fp32 accumulator: |acc32 - acc64| <= delta on every F32 route."""
    worst = 0.0
    for c in [c for c in go.ROUTES if c.epi == go.EPI_F32] + [go.Case(300, 512, 18944, go.EPI_F32, "", "7B down K")]:
        g = torch.Generator(device=DEV).manual_seed(c.K)
        a, w = go.normal_operands(c.M, c.N, c.K, g, DEV)
        acc32 = ops.gemm(a, w, epilogue=go.EPI_F32).double()
        acc64, abs_sum = go.exact_product(a, w)
        ratio = ((acc32 - acc64).abs() / go.delta_of(abs_sum, c.K).clamp_min(1e-300)).max().item()
        assert ratio <= 1.0, f"{c.id}: |acc32 - acc64| / delta = {ratio}"
        worst = max(worst, ratio)
    print(f"largest |acc32 - acc64| / delta = {worst:.4f}")


SMALL_M = [c for c in go.ROUTES if c.M <= 64]


def test_skinny_switched_off(tmp_path):
    """BAGEL_GEMM_SKINNY=0 / BAGEL_PDL=0: the M <= 64 cases run in a child process, where they must land on the wide
    kernel and pass the same checks."""
    if not go.IN_CHILD:
        go.run_in_child(__file__, "test_skinny_switched_off", BAGEL_GEMM_SKINNY="0", BAGEL_PDL="0")
        return
    assert not SKINNY_ON
    for c in SMALL_M:
        _check_case(c, "skinny off: ")
    seen = _observe(SMALL_M, tmp_path, skinny_on=False)
    assert all(name.startswith("gemm_bf16_kernel") for name in seen)
