"""Small invocations of every kernel family for compute-sanitizer (memcheck / racecheck) on the GPU box."""
import sys, torch
sys.path.insert(0, ".")
from bagel_b200 import ops
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(0)
bf = torch.bfloat16
a = torch.randn(200, 192, device=dev, generator=g).to(bf); w = torch.randn(264, 192, device=dev, generator=g).to(bf)
b = torch.randn(264, device=dev, generator=g).to(bf)
out = ops.gemm(a, w, bias=b)
res = torch.randn(200, 264, device=dev, generator=g).to(bf)
out = ops.gemm(a, w, bias=b, resid=res, epilogue=ops.EPI_RESID)
gw = torch.randn(256, 192, device=dev, generator=g).to(bf)
out = ops.gemm(a, ops.interleave_gate_up(gw[:128], gw[128:]), epilogue=ops.EPI_SWIGLU)
s32 = ops.gemm(a, w, epilogue=ops.EPI_F32)
for (lq, lk, Hq, Hk, D, causal) in (([130], [300], 4, 2, 64, False), ([100, 257], [100, 300], 2, 1, 128, True)):
    q = torch.randn(sum(lq), Hq, D, device=dev, generator=g).to(bf); k = torch.randn(sum(lk), Hk, D, device=dev, generator=g).to(bf)
    v = torch.randn(sum(lk), Hk, D, device=dev, generator=g).to(bf)
    cq = torch.tensor([0] + torch.tensor(lq).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    ck = torch.tensor([0] + torch.tensor(lk).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    o = ops.attn_varlen(q, k, v, cq, ck, max(lq), max(lk), causal)
x = torch.randn(37, 256, device=dev, generator=g).to(bf); wn = torch.randn(256, device=dev, generator=g).to(bf)
ex = (torch.rand(37, device=dev, generator=g) > 0.5).to(torch.uint8)
y = ops.rmsnorm(x, wn, wn, ex); y = ops.layernorm(x, wn, wn)
N, Hq, Hk, D = 50, 2, 2, 128
qkv = torch.randn(N, (Hq + 2 * Hk) * D, device=dev, generator=g).to(bf)
pos = torch.arange(N, device=dev); inv = (1.0 / (1e6 ** (torch.arange(0, D, 2).float() / D))).to(dev)
cos, sin = ops.rope_table(pos, inv, True)
qo = torch.zeros(N, Hq * D, device=dev, dtype=bf); kb = torch.zeros(N, Hk * D, device=dev, dtype=bf); vb = torch.zeros_like(kb)
rows = torch.arange(N, device=dev, dtype=torch.int32)
ops.qk_norm_rope(qkv, wn[:D], wn[:D], wn[:D], wn[:D], ex.new_zeros(N), cos, sin, qo, kb, vb, rows, Hq, Hk, D, 1e-6, True)
ah = torch.randn(N, 256, device=dev, generator=g).to(bf); wq = torch.randn((Hq + 2 * Hk) * D, 256, device=dev, generator=g).to(bf)
bq = torch.randn((Hq + 2 * Hk) * D, device=dev, generator=g).to(bf)
ops.gemm_qkv_norm_rope(ah, wq, bq, wn[:D], wn[:D], wn[:D], wn[:D], ex.new_zeros(N), cos, sin, qo, kb, vb, rows, Hq, Hk, 1e-6, True)
xc = torch.randn(1, 8, 12, 128, device=dev, generator=g).to(bf); wc = torch.randn(128, 3, 3, 128, device=dev, generator=g).to(bf)
yc = ops.conv2d_nhwc(xc, wc, b[:128].contiguous(), pad=1)
yc2 = ops.conv2d_nhwc(xc, wc, b[:128].contiguous(), stride=2, pad=0, out_hw=(4, 6))
gnw = torch.ones(128, device=dev); yg = ops.groupnorm_nhwc(yc, gnw, gnw * 0)
yu = ops.upsample2x_nhwc(yg); P = ops.softmax_rows(s32, 0.1); T = ops.transpose(a)
xl = torch.randn(64, 64, device=dev, generator=g); vv = torch.randn(80, 64, device=dev, generator=g).to(bf)
ops.cfg_euler_step(vv, vv, None, torch.arange(64, device=dev, dtype=torch.int32), xl, torch.zeros(2, device=dev), 3.0, 1.0, 0.0, "global", 0.1)
# --- decode path: skinny GEMMs (cluster split-K over DSMEM), single-query attention (cp.async rings, cluster merge),
# argmax, TaylorSeer kernels ---
a2 = torch.randn(7, 832, device=dev, generator=g).to(bf); w2 = torch.randn(520, 832, device=dev, generator=g).to(bf)
b2 = torch.randn(520, device=dev, generator=g).to(bf); r2 = torch.randn(7, 520, device=dev, generator=g).to(bf)
o2 = ops.gemm(a2, w2, bias=b2); o2 = ops.gemm(a2, w2, bias=b2, resid=r2, epilogue=ops.EPI_RESID)
gw2 = torch.randn(512, 832, device=dev, generator=g).to(bf)
o3 = ops.gemm(a2, ops.interleave_gate_up(gw2[:256], gw2[256:]), epilogue=ops.EPI_SWIGLU)
for (lk, Hq, Hk) in (([300, 17, 0, 1100], 28, 4), ([33, 64], 8, 8), ([90], 4, 2)):
    B = len(lk); cap = [n + 3 for n in lk]
    q = torch.randn(B, Hq, 128, device=dev, generator=g).to(bf)
    k = torch.randn(sum(cap), Hk, 128, device=dev, generator=g).to(bf); v = torch.randn(sum(cap), Hk, 128, device=dev, generator=g).to(bf)
    cq = torch.arange(B + 1, dtype=torch.int32, device=dev)
    ck = torch.tensor([0] + torch.tensor(cap).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    od = ops.attn_varlen(q, k, v, cq, ck, 1, max(lk), True, seqused_k=torch.tensor(lk, dtype=torch.int32, device=dev))
lg = torch.randn(3, 1000, device=dev, generator=g).to(bf); tk = torch.empty(3, dtype=torch.int64, device=dev)
ops.argmax_rows(lg, tk, torch.empty(3, dtype=torch.int32, device=dev))
# per-request decode settings: mixed greedy / sampled rows (unaligned ld), per-row stop limits
lg2 = torch.randn(4, 1031, device=dev, generator=g).to(bf)[:, :1029]; tk2 = torch.empty(4, dtype=torch.int64, device=dev)
sd = torch.zeros(1, dtype=torch.int32, device=dev)
ops.sample_rows_mixed(lg2, torch.tensor([0.0, 2.0, 0.0, 1.0], device=dev), torch.arange(4, device=dev), sd, tk2,
                      torch.empty(4, dtype=torch.int32, device=dev))
i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device=dev)
# truncated sampling: top-k / top-p (its own high bin and top-k's) / min-p rows, unaligned ld
ops.sample_rows_filtered(lg2, torch.tensor([0.0, 2.0, 1.5, 1.0], device=dev), i32(3, 0, 40, 5),
                         torch.tensor([0.5, 0.9, 0.7, 1.0], device=dev), torch.tensor([0.0, 0.0, 0.1, 0.2], device=dev),
                         torch.arange(4, device=dev), sd, tk2, torch.empty(4, dtype=torch.int32, device=dev))
# penalties: one row off, a finished row, unaligned ld; the step adds each live row's fed token
ops.apply_penalties(lg2, torch.tensor([1.0, 1.05, 0.8, 1.0], device=dev), torch.tensor([0.0, 0.5, -1.0, 0.0], device=dev),
                    torch.tensor([0.0, 0.2, 0.0, 1.5], device=dev), tk2, i32(0, 0, 1, 0), i32(1),
                    ops.penalty_state(4, 3, dev))
ops.decode_advance_stop_limits(i32(3, 4, 5, 6), torch.arange(4, device=dev), tk2.clone(), tk2.to(torch.int32), tk2,
                               torch.zeros(3, 4, dtype=torch.int64, device=dev), sd, i32(0, 0, 1, 0), i32(4), 5,
                               i32(1, 3, 2, 5), -1)
fac = torch.zeros(7, 40, 256, device=dev, dtype=bf); ft = torch.randn(37, 256, device=dev, generator=g).to(bf)
ops.taylor_update(ft, fac[:, 2:39], 0, 1); ops.taylor_update(ft, fac[:, 2:39], 1, 3); ops.taylor_eval(fac[:, 2:39], 2, 2, ft)
torch.cuda.synchronize()
print("SANITIZE_SCRIPT_DONE finite:", bool(torch.isfinite(out.float()).all() and torch.isfinite(o.float()).all() and torch.isfinite(yc.float()).all() and torch.isfinite(od.float()).all() and torch.isfinite(o3.float()).all()))
