"""The four dense GEMMs of one decoder layer at the denoising step's shape, with their real epilogues, next to
torch.matmul (cuBLAS) at the same M, N, K on the same card.

M = 16 x 4098 = 65 568 rows (8 images x 2 CFG branches packed into one LM call), BAGEL-7B: hidden 3584, intermediate
18944, 28 query / 4 KV heads of 128:
  qkv     gemm_qkv_norm_rope (bias, q/k RMSNorm with expert-routed weights, RoPE, K/V placement)   N 4608,  K 3584
  o_proj  EPI_RESID                                                                                N 3584,  K 3584
  gate|up EPI_SWIGLU (interleaved gate/up rows)                                                   N 37888, K 3584
  down    EPI_RESID                                                                                N 3584,  K 18944

--profile-step instead runs the benchmark's denoising workload (bench.py's synthetic model and inputs) and prints the
per-kernel split of ONE step from torch.profiler (kernels launched individually, no CUDA graph).

--root DIR imports bagel_b200 from another built checkout (e.g. a parent commit's tree) for same-card A/B runs.
Prints one JSON line last.

  python tools/gpu_perf_gemm_step.py [--root DIR] [--iters 10] [--profile-step]
"""
import argparse
import json
import os
import re
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=10, help="timed launches per call")
ap.add_argument("--profile-step", action="store_true")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from bagel_b200 import ops  # noqa: E402

assert os.path.abspath(ops.__file__).startswith(os.path.abspath(args.root)), ops.__file__
DEV = "cuda"
M, H, I, HQ, HK, D = 16 * 4098, 3584, 18944, 28, 4, 128


def timed(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gemm_step():
    g = torch.Generator(device=DEV).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device=DEV, generator=g) * scale).to(torch.bfloat16)

    x = rnd(M, H)
    h = rnd(M, H)                                     # residual stream
    out = torch.empty(M, H, device=DEV, dtype=torch.bfloat16)
    # qkv
    w_qkv, b_qkv = rnd((HQ + 2 * HK) * D, H, scale=H ** -0.5), rnd((HQ + 2 * HK) * D, scale=0.1)
    nw = [(1 + 0.1 * torch.randn(D, device=DEV, generator=g)).to(torch.bfloat16) for _ in range(4)]
    expert = torch.ones(M, device=DEV, dtype=torch.uint8)    # 1 = gen-expert norm weights
    pos = (torch.arange(M, device=DEV) % 4098).to(torch.int64)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(DEV)
    cos, sin = ops.rope_table(pos, inv_freq, True)
    q = torch.empty(M, HQ * D, device=DEV, dtype=torch.bfloat16)
    kbuf = torch.empty(M, HK * D, device=DEV, dtype=torch.bfloat16)
    vbuf = torch.empty_like(kbuf)
    kv_rows = torch.arange(M, device=DEV, dtype=torch.int32)
    # o_proj, gate|up, down
    w_o = rnd(H, H, scale=H ** -0.5)
    w_gu = ops.interleave_gate_up(rnd(I, H, scale=H ** -0.5), rnd(I, H, scale=H ** -0.5))
    act = torch.empty(M, I, device=DEV, dtype=torch.bfloat16)
    w_d = rnd(H, I, scale=I ** -0.5)
    calls = [
        ("qkv", 4608, H, w_qkv, x, lambda: ops.gemm_qkv_norm_rope(x, w_qkv, b_qkv, nw[0], nw[1], nw[2], nw[3], expert, cos,
                                                                   sin, q, kbuf, vbuf, kv_rows, HQ, HK, 1e-6, False)),
        ("o_proj", H, H, w_o, x, lambda: ops.gemm(x, w_o, resid=h, epilogue=ops.EPI_RESID, out=out)),
        ("gate_up", 2 * I, H, w_gu, x, lambda: ops.gemm(x, w_gu, epilogue=ops.EPI_SWIGLU, out=act)),
        ("down", H, I, w_d, act, lambda: ops.gemm(act, w_d, resid=h, epilogue=ops.EPI_RESID, out=out)),
    ]
    res = {}
    for name, n, k, w, a, fn in calls:
        flop = 2.0 * M * n * k
        t = timed(fn, args.iters)
        scratch = torch.empty(M, n, device=DEV, dtype=torch.bfloat16)
        tc = timed(lambda: torch.matmul(a, w.t(), out=scratch), args.iters)
        del scratch
        res[name] = {"ms": t, "tflops": flop / t / 1e9, "cublas_ms": tc, "cublas_tflops": flop / tc / 1e9}
        print(f"{name:8s} M={M} N={n:5d} K={k:5d}: {t:8.3f} ms {flop / t / 1e9:6.1f} TFLOP/s | "
              f"torch.matmul {tc:8.3f} ms {flop / tc / 1e9:6.1f} TFLOP/s", flush=True)
    total = sum(r["ms"] for r in res.values())
    print(f"one layer: {total:.3f} ms, x 28 layers = {28 * total:.1f} ms", flush=True)
    return {"gemms": res, "layer_ms": total}


def profile_step():
    from bagel_b200 import synthetic
    model = synthetic.build_random_bagel(device=DEV, seed=0)
    gen_input, cfg_text, ctxs = synthetic.t2i_inputs(model, 8, (1024, 1024), seed=1, noise_seed=2)
    gen_kwargs = dict(
        num_timesteps=50, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type="global",
        cfg_interval=[0.0, 1.0], cfg_text_scale=2.0, cfg_img_scale=1.0,
        cfg_text_packed_position_ids=cfg_text["cfg_packed_position_ids"],
        cfg_text_packed_query_indexes=cfg_text["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=cfg_text["cfg_key_values_lens"],
        cfg_text_packed_key_value_indexes=cfg_text["cfg_packed_key_value_indexes"],
        cfg_text_past_key_values=ctxs["cfg_text"])
    model.use_cuda_graph = False
    runner = model.make_flow_runner(past_key_values=ctxs["main"], **gen_input, **gen_kwargs)
    for i in range(2):
        runner.step(i)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        runner.step(2)
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m = re.search(r"(\w+<[^>]*>|\w+)\(", e.name)
        key = m.group(1) if m else e.name[:80]
        a = agg.setdefault(key, [0, 0.0])
        a[0] += 1
        a[1] += e.time_range.elapsed_us() / 1e3
    tot = sum(a[1] for a in agg.values())
    print(f"sum of kernel time in one step: {tot:.1f} ms")
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:20]:
        print(f"  {t:9.2f} ms {100 * t / tot:5.1f} %  {n:5d} x  {k}")
    return {"step_kernel_ms": tot, "kernels": {k: {"launches": n, "ms": t} for k, (n, t) in agg.items()}}


if __name__ == "__main__":
    r = profile_step() if args.profile_step else gemm_step()
    r["root"] = args.root
    r["device"] = torch.cuda.get_device_name()
    print(json.dumps(r))
