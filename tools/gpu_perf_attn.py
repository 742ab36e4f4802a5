"""Attention microbench (BASELINE configs[4]): packed varlen, d=128, bf16; ours vs flash_attn 2.8 (FA2 on the same GPU)."""
import sys, torch
sys.path.insert(0, ".")
import os
if os.environ.get("PERF_LIB"):      # same-box A/B against a variant build (tools/build_variant.py)
    from pathlib import Path
    from bagel_b200 import _cabi
    _cabi.LIB_PATH = Path(os.environ["PERF_LIB"]).resolve()
from bagel_b200 import ops
try:
    if os.environ.get("PERF_NO_FA2"):
        raise ImportError("PERF_NO_FA2 set")
    from flash_attn import flash_attn_varlen_func
except Exception as e:
    flash_attn_varlen_func = None
    print("flash_attn unavailable:", e)
dev = "cuda"
def bench(fn, iters=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters
torch.manual_seed(4)
for (Hq, Hk) in ((32, 32), (28, 4)):
    for L in (1024, 4096, 16384):
        for causal in (False, True):
            nseq = max(1, 16384 // L)
            lq = [L] * nseq
            S = sum(lq)
            q = torch.randn(S, Hq, 128, device=dev).to(torch.bfloat16); k = torch.randn(S, Hk, 128, device=dev).to(torch.bfloat16); v = torch.randn(S, Hk, 128, device=dev).to(torch.bfloat16)
            cu = torch.tensor([0] + list(torch.tensor(lq).cumsum(0)), dtype=torch.int32, device=dev)
            out = torch.empty_like(q)
            t = bench(lambda: ops.attn_varlen(q, k, v, cu, cu, L, L, causal, out=out))
            fl = 4.0 * nseq * L * L * Hq * 128 / (2 if causal else 1)
            line = f"[attn perf] H={Hq}/{Hk} L={L} nseq={nseq} causal={causal}: ours {t:.3f} ms = {fl/t/1e9:.0f} TFLOP/s"
            if flash_attn_varlen_func is not None:
                tf = bench(lambda: flash_attn_varlen_func(q, k, v, cu, cu, L, L, causal=causal))
                o2 = flash_attn_varlen_func(q, k, v, cu, cu, L, L, causal=causal)
                line += f" | FA2 {tf:.3f} ms = {fl/tf/1e9:.0f} TFLOP/s | max|ours-FA2|={(out.float()-o2.float()).abs().max().item():.3e}"
            print(line, flush=True)
# denoise-shaped: q=4098 vs kv=4098+66, B=16
lq = [4098] * 16; lk = [4164] * 16
q = torch.randn(sum(lq), 28, 128, device=dev).to(torch.bfloat16); k = torch.randn(sum(lk), 4, 128, device=dev).to(torch.bfloat16); v = torch.randn(sum(lk), 4, 128, device=dev).to(torch.bfloat16)
cq = torch.tensor([0] + list(torch.tensor(lq).cumsum(0)), dtype=torch.int32, device=dev); ck = torch.tensor([0] + list(torch.tensor(lk).cumsum(0)), dtype=torch.int32, device=dev)
out = torch.empty_like(q)
t = bench(lambda: ops.attn_varlen(q, k, v, cq, ck, 4098, 4164, False, out=out))
fl = 4.0 * 16 * 4098 * 4164 * 28 * 128
line = f"[attn perf] denoise B=16 q=4098 kv=4164 28/4: ours {t:.3f} ms = {fl/t/1e9:.0f} TFLOP/s"
if flash_attn_varlen_func is not None:
    tf = bench(lambda: flash_attn_varlen_func(q, k, v, cq, ck, 4098, 4164, causal=False))
    line += f" | FA2 {tf:.3f} ms = {fl/tf/1e9:.0f} TFLOP/s"
print(line, flush=True)
