"""Measurement blocks bench.py adds to its JSON line so that EVERY BASELINE.json config is driver-measured, not only
configs[1]:

  attn                  configs[4]  packed varlen attention microbench (ours vs flash-attn on the same box)
  und_prefill           configs[2]  image-understanding prefill in the Bagel.chat call order, batch 32
  edit                  configs[3]  image edit through InterleaveInferencer, 2 samples per GPU (16 over 8 GPUs)
  decode                SURVEY §8 a15: greedy text decode step time
  gpu_library_baseline  the reference-equivalent GPU path (oracle = plain torch ops -> cuBLASLt + ATen eager + real
                        flash_attn_varlen_func) timed on one denoising step of the headline workload on this box
  parity                one Euler step of the headline workload: product vs that path, next to the reference's own
                        noise floor (flash-attn vs fp32-SDPA execution of the same reference code)
  strong_scaling        configs[1] with the GLOBAL batch fixed at 8 (8/N images per GPU)

Nothing here is on the product path; the two baseline/parity blocks are the only users of oracle/ (as the checker and
as the timed library baseline, never as the thing reported in `value`)."""
from __future__ import annotations

import os
import statistics
import time
from typing import Dict, List

import torch

EVALS = 49


def _ev_ms(fn, iters: int, warm: int = 3) -> float:
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


# ----------------------------------------------------------------------------------------------------------------
# configs[4]: attention microbench
# ----------------------------------------------------------------------------------------------------------------
def attn_block(peaks: Dict, dev, iters: int = 10) -> Dict:
    """SURVEY.md §8d cfg 5: bf16, d=128, Hq=32 (MHA 32:32 as written, and the model's 28:4 GQA); L in {1k,4k,16k} x
    {uniform non-causal, causal, ragged (lengths randint(L/2, L), seed 5)}; plus the denoise shapes q=4098 vs
    kv=4098+{66, 9066}. 16384 packed query tokens per call -> q/k/v/out are 134 MB each (> the 50 MB L2, so successive
    iterations do not find their inputs cached). FLOPs = 4*sum(Lq*Lk)*Hq*d (/2 causal)."""
    from bagel_b200 import ops
    try:
        from flash_attn import flash_attn_varlen_func
    except Exception:
        flash_attn_varlen_func = None
    burst = float(peaks.get("bf16_tflops", 989.0))
    hbm = float(peaks.get("hbm_gbs", 3350.0))
    g = torch.Generator(device=dev).manual_seed(4)
    rows: List[Dict] = []

    def cu(lens):
        return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)

    def one(name, Hq, Hk, lq, lk, causal):
        D = 128
        q = torch.randn(sum(lq), Hq, D, device=dev, generator=g).to(torch.bfloat16)
        k = torch.randn(sum(lk), Hk, D, device=dev, generator=g).to(torch.bfloat16)
        v = torch.randn(sum(lk), Hk, D, device=dev, generator=g).to(torch.bfloat16)
        cq, ck = cu(lq), cu(lk)
        out = torch.empty_like(q)
        mq, mk = max(lq), max(lk)
        ms = _ev_ms(lambda: ops.attn_varlen(q, k, v, cq, ck, mq, mk, causal, out=out), iters)
        if causal:   # bottom-right aligned: row i of an (a, b) = (Lq, Lk) sample sees min(b, b - a + i + 1) keys
            pairs = sum(a * (b - a) + a * (a + 1) // 2 if a <= b else b * (b + 1) // 2 for a, b in zip(lq, lk))
        else:
            pairs = sum(a * b for a, b in zip(lq, lk))
        flops = 4.0 * pairs * Hq * D
        byts = 2.0 * (2 * sum(lq) * Hq + 2 * sum(lk) * Hk) * D
        r = {"shape": name, "Hq": Hq, "Hk": Hk, "causal": bool(causal), "n_seq": len(lq), "tokens_q": sum(lq),
             "ms": ms, "tflops": flops / ms / 1e9, "frac_of_burst_peak": flops / ms / 1e9 / burst,
             "hbm_gbs": byts / ms / 1e6, "frac_of_hbm_peak": byts / ms / 1e6 / hbm}
        if flash_attn_varlen_func is not None:
            msf = _ev_ms(lambda: flash_attn_varlen_func(q, k, v, cq, ck, mq, mk, causal=causal), iters)
            r["fa2_ms"], r["fa2_tflops"], r["speedup_vs_fa2"] = msf, flops / msf / 1e9, msf / ms
        rows.append(r)

    rg = torch.Generator().manual_seed(5)
    for Hq, Hk in ((32, 32), (28, 4)):
        for L in (1024, 4096, 16384):
            n = max(1, 16384 // L)
            one(f"uniform L={L}", Hq, Hk, [L] * n, [L] * n, False)
            one(f"causal L={L}", Hq, Hk, [L] * n, [L] * n, True)
            rag = torch.randint(L // 2, L + 1, (n,), generator=rg).tolist()
            one(f"ragged L<={L}", Hq, Hk, rag, rag, False)
    one("denoise q=4098 kv=4164 B=4", 28, 4, [4098] * 4, [4164] * 4, False)
    one("denoise q=4098 kv=13164 B=4 (edit ctx)", 28, 4, [4098] * 4, [13164] * 4, False)
    best = max(rows, key=lambda r: r["tflops"])
    return {"peak_tflops_burst": burst, "peak_source": "bench.py measured_peaks() bf16_tflops",
            "l2": "inputs > 50 MB L2 (16384 packed query tokens per call)", "iters": iters, "shapes": rows,
            "best_tflops": best["tflops"], "best_shape": best["shape"]}


# ----------------------------------------------------------------------------------------------------------------
# configs[2]: understanding prefill, Bagel.chat call order, batch 32; and the decode step on top of that context
# ----------------------------------------------------------------------------------------------------------------
def und_prefill_and_decode_block(model, dev, batch: int = 32, text_tokens: int = 512, decode: bool = True,
                                 hbm_gbs: float = 3350.0) -> Dict:
    """32 synthetic 378x378 PIL images -> VLM transform ImageTransform(980, 378, 14, max_pixels=2_007_040)
    (data/configs/example.yaml:32-36: 378^2 stays 378^2 = 729 patches) -> prepare_vit_images -> forward_cache_update_vit
    -> prepare_prompts (512 random ids + bos/eos) -> forward_cache_update_text: the order of Bagel.chat
    (bagel.py:1030-1056), batched. Timed end to end from PIL images / token ids on the host to a complete KV cache on
    the device; `host_pack_s` is the part spent in the prepare_* packers + image transform (PIL, CPU)."""
    import numpy as np
    from PIL import Image
    from bagel_b200 import synthetic
    from bagel_b200.qwen2_navit import NaiveCache
    from bagel_b200.transforms import ImageTransform
    L = model.config.llm_config.num_hidden_layers
    rs = np.random.RandomState(3)
    imgs = [Image.fromarray(rs.randint(0, 255, (378, 378, 3)).astype(np.uint8)) for _ in range(batch)]
    tf = ImageTransform(980, 378, 14, max_pixels=2_007_040)
    tok = synthetic.RandomIdTokenizer(1)

    def run():
        t_host = 0.0
        cache = NaiveCache(L)
        t0 = time.perf_counter()
        gi, kv, rp = model.prepare_vit_images([0] * batch, [0] * batch, imgs, tf, synthetic.NEW_TOKEN_IDS)
        t_host += time.perf_counter() - t0
        cache = model.forward_cache_update_vit(cache, **gi)
        t0 = time.perf_counter()
        gt, kv, rp = model.prepare_prompts(kv, rp, [str(text_tokens)] * batch, tok, synthetic.NEW_TOKEN_IDS)
        t_host += time.perf_counter() - t0
        cache = model.forward_cache_update_text(cache, **gt)
        return cache, kv, rp, t_host

    run()
    torch.cuda.synchronize()
    times, hosts = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cache, kv, rp, th = run()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        hosts.append(th)
    dt, th = statistics.median(times), statistics.median(hosts)
    ntok = int(sum(kv))
    out = {"und_prefill": {
        "workload": f"BASELINE configs[2]: {batch} x (SigLIP 378^2 = 729 patches + soi/eoi + {text_tokens}+2 text tokens), "
                    "Bagel.chat call order, PIL images on the host -> KV cache on the device",
        "tokens": ntok, "tokens_per_sample": ntok // batch, "seconds": dt, "tokens_per_s": ntok / dt,
        "host_pack_s": th, "device_and_copies_s": dt - th, "runs": len(times)}}
    if decode:
        gs = model.prepare_start_tokens(kv, rp, synthetic.NEW_TOKEN_IDS)
        from copy import deepcopy
        calls = []
        for steps in (4, 16, 144, 16, 144):     # the 4-step call is a warm-up (lazy kernel loading, allocator growth)
            c = deepcopy(cache)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.generate_text(past_key_values=c, max_length=steps, do_sample=False, **gs)
            torch.cuda.synchronize()
            calls.append((steps, time.perf_counter() - t0))
            del c
        t16 = min(t for s_, t in calls if s_ == 16)
        t144 = min(t for s_, t in calls if s_ == 144)
        ms = (t144 - t16) / 128 * 1e3
        cfg = model.config.llm_config
        wbytes = 2.0 * cfg.num_hidden_layers * cfg.hidden_size * ((cfg.num_attention_heads * 2 + cfg.num_key_value_heads * 2)
                                                                  * cfg.head_dim + 3 * cfg.intermediate_size) \
            + 2.0 * cfg.vocab_size * cfg.hidden_size
        kvbytes = 2.0 * 2 * cfg.num_hidden_layers * cfg.num_key_value_heads * cfg.head_dim * float(sum(kv))
        out["decode"] = {"workload": f"greedy generate_text, batch {batch}, {ntok // batch}-token context, CUDA-graph replay; "
                                     "steady state = (min t[144 steps] - min t[16 steps]) / 128 over two rounds after a warm-up call",
                         "calls_s": [[s_, round(t, 4)] for s_, t in calls],
                         "ms_per_step": ms, "tokens_per_s": batch / ms * 1e3,
                         "hbm_bytes_per_step": wbytes + kvbytes, "hbm_roofline_ms": (wbytes + kvbytes) / (hbm_gbs * 1e6),
                         "frac_of_hbm_roofline": (wbytes + kvbytes) / (hbm_gbs * 1e6) / ms}
    return out


# ----------------------------------------------------------------------------------------------------------------
# configs[3]: image edit through the orchestrator
# ----------------------------------------------------------------------------------------------------------------
def edit_block(model, vae, dev, samples: int = 2) -> Dict:
    """BASELINE configs[3] / SURVEY §8d cfg 4: per sample VAE encode 1024^2 + SigLIP at 980^2 (4900 patches) + 64-token
    prompt, 50 timesteps with THREE CFG branches (text 4, image 2, renorm "text_channel"), VAE decode; through
    InterleaveInferencer.__call__ (single-sample API, as the reference), `samples` images one after another per GPU
    (2 per GPU x 8 GPUs = the batch of 16 the config names; no collective: samples are independent)."""
    import numpy as np
    from PIL import Image
    from bagel_b200 import synthetic
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    inf = InterleaveInferencer(model, vae, synthetic.RandomIdTokenizer(1), ImageTransform(1024, 512, 16),
                               ImageTransform(980, 224, 14), synthetic.NEW_TOKEN_IDS)
    rs = np.random.RandomState(0)
    kw = dict(cfg_text_scale=4.0, cfg_img_scale=2.0, cfg_interval=[0.0, 1.0], timestep_shift=3.0, num_timesteps=50,
              cfg_renorm_min=0.0, cfg_renorm_type="text_channel")
    imgs = [Image.fromarray(rs.randint(0, 255, (1024, 1024, 3)).astype(np.uint8)) for _ in range(samples)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i, im in enumerate(imgs):
        torch.manual_seed(i)
        out = inf(image=im, text="64", **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert out["image"].size == (1024, 1024)
    return {"samples_per_gpu": samples, "seconds": dt, "s_per_image": dt / samples}


# ----------------------------------------------------------------------------------------------------------------
# reference-equivalent GPU path: timed baseline + one-step parity probe at the headline workload
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def library_baseline_and_parity(model, gen_input, cfg_text_input, ctx_main, gen_kwargs: Dict, prompt_ids, dev,
                                ms_per_step_ours: float, batch: int) -> Dict:
    from bagel_b200 import synthetic
    from oracle import bagel_flow as obf, gpu_leg
    sd = gpu_leg.export_reference_state_dict(model)
    fc = gpu_leg.flow_config(model)
    gi, cache, br = gpu_leg.reference_contexts(sd, fc, prompt_ids, synthetic.NEW_TOKEN_IDS, gen_input, cfg_text_input, dev)
    ts = torch.linspace(1, 0, gen_kwargs["num_timesteps"])
    shift = gen_kwargs["timestep_shift"]
    ts = shift * ts / (1 + (shift - 1) * ts)
    dt0 = (ts[0] - ts[1]).to(dev)
    x0 = gi["packed_init_noises"]
    tvec = torch.full((x0.shape[0],), float(ts[0]), device=dev)

    def ref_v():
        return obf.forward_flow(sd, fc, x0, tvec, gi["packed_vae_token_indexes"], gi["packed_vae_position_ids"],
                                gi["packed_text_ids"], gi["packed_text_indexes"], gi["packed_indexes"],
                                gi["packed_position_ids"], gi["packed_seqlens"], gi["key_values_lens"], cache,
                                gi["packed_key_value_indexes"], gen_kwargs["cfg_renorm_min"], gen_kwargs["cfg_renorm_type"],
                                gen_kwargs["cfg_text_scale"], br)

    with gpu_leg.fa2():
        v_fa2 = ref_v()                                    # warm-up (cuBLAS heuristics, flash-attn) + parity sample
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(2):
            ref_v()
        e1.record()
        torch.cuda.synchronize()
        ms_lib = e0.elapsed_time(e1) / 2
    v_sdpa = ref_v()
    x1_fa2 = x0 - v_fa2 * dt0
    x1_sdpa = x0 - v_sdpa * dt0
    # product: one step of the planned run from the same x0
    runner = model.make_flow_runner(past_key_values=ctx_main, **gen_input, **gen_kwargs)
    runner.step(0)
    x1 = runner.st["x"].clone()
    torch.cuda.synchronize()
    del runner

    def rel(a, b):
        d = (a.double() - b.double())
        return {"rel_l2": float(d.norm() / b.double().norm()), "max_abs": float(d.abs().max()), "mean_abs": float(d.abs().mean())}

    dv = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    floor = rel(x1_sdpa, x1_fa2)
    got = rel(x1, x1_fa2)
    lib = {"what": "oracle (plain torch ops: cuBLASLt bf16 GEMMs + ATen elementwise, eager) + real flash_attn_varlen_func on "
                   "cuda — kernel for kernel the reference's own GPU path — one velocity evaluation (2 CFG branches run "
                   "back to back as the reference does) of the headline workload, same weights, same box",
           "ms_per_step": ms_lib, "images_per_s": batch / (EVALS * ms_lib / 1e3),
           "ours_ms_per_step": ms_per_step_ours, "speedup": ms_lib / ms_per_step_ours}
    par = {"what": "x_t after ONE Euler step of the headline workload (28 layers, batch as benchmarked, text CFG) from the same "
                   "init noise: product vs the reference-equivalent GPU path (flash-attn leg); `noise_floor` is the same "
                   "distance between two executions of the reference itself (flash-attn vs fp32-SDPA attention)",
           "product_vs_reference": got, "noise_floor": floor,
           "ratio_to_noise_floor": got["rel_l2"] / max(floor["rel_l2"], 1e-30),
           "velocity_rel_l2": {"product_vs_reference": dv((x0 - x1) / dt0, v_fa2.float()),
                               "noise_floor": dv(v_sdpa.float(), v_fa2.float())},
           "full_run_drift": "tests/test_gpu_drift_7b.py (28 layers x 49 steps incl. fp32 truth)"}
    return {"gpu_library_baseline": lib, "parity": par}
