"""-m gpu: the CTA-pair GEMM (two or more M tiles: the two CTAs of a cluster share each W tile through TMA multicast)
against the single-CTA path. A 128-row call has one M tile and runs single-CTA with the same BN, K order, wgmma and
epilogue, so recomputing a big call slice by slice must give bit-identical outputs. Shapes keep every slice on the
wide kernel: N % 256 == 0 and N < 1024 (BN 256 at any M) and every slice longer than 64 rows (no skinny kernel)."""
import pytest
import torch

from bagel_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [  # (M, N, K) -> M tiles, cluster tiles = ceil(M tiles / 2) x N tiles
    (2048, 512, 320),    # 16 (even) -> 8 x 2 = 16 cluster tiles: fewer than the clusters resident at once
    (2140, 768, 200),    # 17 (odd, ragged, K tail) -> 27: the last pair's second CTA lies wholly past M
    (8320, 768, 512),    # 65 (odd) -> 99: several tiles per cluster in the persistent loop
    (10240, 512, 256),   # 80 (even) -> 80
]


def _by_slices(M, fn):
    return torch.cat([fn(r0, min(r0 + 128, M)) for r0 in range(0, M, 128)])


@pytest.mark.parametrize("M,N,K", CASES)
def test_gemm_cluster_pair_bit_identical_to_single_cta(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + 5 * N + K)
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    b = torch.randn(N, device=DEV, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, device=DEV, generator=g).to(torch.bfloat16)
    assert torch.equal(ops.gemm(a, w, bias=b), _by_slices(M, lambda r0, r1: ops.gemm(a[r0:r1], w, bias=b)))
    assert torch.equal(ops.gemm(a, w, bias=b, resid=res, epilogue=ops.EPI_RESID),
                       _by_slices(M, lambda r0, r1: ops.gemm(a[r0:r1], w, bias=b, resid=res[r0:r1],
                                                             epilogue=ops.EPI_RESID)))
    wi = ops.interleave_gate_up(w[: N // 2], w[N // 2:])
    assert torch.equal(ops.gemm(a, wi, epilogue=ops.EPI_SWIGLU),
                       _by_slices(M, lambda r0, r1: ops.gemm(a[r0:r1], wi, epilogue=ops.EPI_SWIGLU)))


@pytest.mark.parametrize("M,flow", [(2048, 0), (2140, 1)])
def test_fused_qkv_cluster_pair_bit_identical_to_single_cta(M, flow):
    g = torch.Generator(device=DEV).manual_seed(M + flow)
    K, Hq, Hk, D = 512, 6, 2, 128
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn((Hq + 2 * Hk) * D, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    b = (0.1 * torch.randn((Hq + 2 * Hk) * D, device=DEV, generator=g)).to(torch.bfloat16)
    qw = [(1 + 0.1 * torch.randn(D, device=DEV, generator=g)).to(torch.bfloat16) for _ in range(2)]
    kw = [(1 + 0.1 * torch.randn(D, device=DEV, generator=g)).to(torch.bfloat16) for _ in range(2)]
    ex = (torch.rand(M, device=DEV, generator=g) > 0.3).to(torch.uint8)
    pos = torch.randint(0, 5000, (M,), device=DEV, dtype=torch.int64, generator=g)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(DEV)
    cos, sin = ops.rope_table(pos, inv_freq, True)
    rows = torch.randperm(M + 40, device=DEV, generator=g)[:M].to(torch.int32)

    def buffers():
        kb = torch.zeros(M + 40, Hk * D, device=DEV, dtype=torch.bfloat16)
        return torch.zeros(M, Hq * D, device=DEV, dtype=torch.bfloat16), kb, torch.zeros_like(kb)

    q1, k1, v1 = buffers()
    ops.gemm_qkv_norm_rope(a, w, b, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q1, k1, v1, rows, Hq, Hk, 1e-6, bool(flow))
    q0, k0, v0 = buffers()
    for r0 in range(0, M, 128):   # one M tile per call; row_map puts each slice's rows at their places of the full call
        r1 = min(r0 + 128, M)
        ops.gemm_qkv_norm_rope(a[r0:r1], w, b, qw[0], kw[0], qw[1], kw[1], ex, cos, sin, q0, k0, v0, rows, Hq, Hk, 1e-6,
                               bool(flow), row_map=torch.arange(r0, r1, device=DEV, dtype=torch.int32))
    assert torch.equal(q1, q0) and torch.equal(k1, k0) and torch.equal(v1, v0)
