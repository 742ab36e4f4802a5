"""Shared by tests/test_gpu_drift_7b.py and tools/gpu_drift_7b.py: run the SAME text->image denoising job through

  product  bagel_b200 (C ABI -> sm_90a kernels)
  fa2      the oracle on cuda with flash_attn_varlen_func  = the reference as it executes on a GPU
  sdpa     the oracle on cuda with its fp32 per-sample SDPA = the reference as pinned on the CPU (attention shim)
  truth    the oracle in fp32 end to end on the same bf16-valued weights (optional, first `truth_steps` steps)

on identical weights / prompts / init noise, recording x_t after every Euler step. `fa2` vs `sdpa` differ only in the
attention kernel's internal rounding — two equally valid executions of the reference — so their distance IS the
reference's own noise floor at that model size and step count; the product is judged against that measured number
(and against the truth), not against a tolerance picked by the builder."""
from __future__ import annotations

import time
from typing import Dict, List, Optional

import torch


def _stat(a: torch.Tensor, b: torch.Tensor) -> Dict[str, float]:
    d = (a.double() - b.double())
    return {"max": d.abs().max().item(), "mean": d.abs().mean().item(),
            "rel_l2": (d.norm() / b.double().norm().clamp_min(1e-30)).item()}


def series(xs: List[torch.Tensor], ys: List[torch.Tensor]) -> List[Dict[str, float]]:
    return [_stat(a, b) for a, b in zip(xs, ys)]


@torch.no_grad()
def run(layers: int = 28, evals: int = 49, truth_steps: int = 0, batch: int = 1, image_size: int = 1024,
        cfg_text_scale: float = 2.0, seed: int = 0, device: str = "cuda", legs=("fa2", "sdpa"), llm_kwargs=None,
        log=print) -> Dict:
    """Returns {"x": {leg: [x_t after step k]}, "t": {leg: seconds}, "scale": per-step max|x| of fa2}."""
    from bagel_b200 import synthetic
    from oracle import gpu_leg, qwen2_mot as om

    dev = torch.device(device)
    model = synthetic.build_random_bagel(llm_kwargs=llm_kwargs, device=dev, seed=seed, num_layers=layers)
    gi, ct, ctx = synthetic.t2i_inputs(model, batch, (image_size, image_size), prompt_tokens=64, seed=1, noise_seed=2)
    kw = dict(num_timesteps=evals + 1, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type="global",
              cfg_interval=[0.0, 1.0], cfg_text_scale=cfg_text_scale)
    out: Dict = {"x": {}, "t": {}}

    # ---- product ----
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    runner = model.make_flow_runner(
        past_key_values=ctx["main"], **gi, **kw,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
        cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=ct["cfg_key_values_lens"],
        cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
        cfg_text_past_key_values=ctx["cfg_text"])
    xs = []
    for i in range(runner.num_steps):
        runner.step(i)
        xs.append(runner.st["x"].clone())
    torch.cuda.synchronize()
    out["t"]["product"] = time.perf_counter() - t0
    out["x"]["product"] = xs
    del runner, ctx
    log(f"product: {len(xs)} steps in {out['t']['product']:.1f} s")

    # ---- reference legs on the same weights ----
    # The legs own the weights from here on: the product's activation workspaces go before the export, its interleaved
    # gate|up weights (de-interleaved copies are in `sd`) right after it, so the 7B job holds one copy of the weights.
    lm = model.language_model.model
    lm._ws.clear()
    torch.cuda.empty_cache()
    sd = gpu_leg.export_reference_state_dict(model)
    for layer in lm.layers:
        for e in (layer.und, layer.gen):
            if e is not None:
                e.wgu = None
    torch.cuda.empty_cache()
    fc = gpu_leg.flow_config(model)
    tok = synthetic.RandomIdTokenizer(1)
    prompt_ids = [tok.encode("64") for _ in range(batch)]

    def leg(name, steps=None, sd=sd):
        tr: List[torch.Tensor] = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gpu_leg.t2i_reference_run(sd, fc, prompt_ids, synthetic.NEW_TOKEN_IDS, gi, ct, dev, x_trace=tr,
                                  max_steps=steps, **kw)
        torch.cuda.synchronize()
        out["t"][name] = time.perf_counter() - t0
        out["x"][name] = tr
        log(f"{name}: {len(tr)} steps in {out['t'][name]:.1f} s")

    if "fa2" in legs:
        with gpu_leg.fa2():
            leg("fa2")
    if "sdpa" in legs:
        leg("sdpa")
    if truth_steps > 0:
        torch.backends.cuda.matmul.allow_tf32 = False
        with om.high_precision():
            leg("truth", truth_steps, om.LazyF32(sd))
    return out


def report(res: Dict, every: int = 1) -> str:
    """Text table of the per-step distances."""
    x = res["x"]
    lines = []
    pairs = [("product", "fa2"), ("sdpa", "fa2"), ("product", "sdpa")]
    if "truth" in x:
        pairs += [("product", "truth"), ("fa2", "truth"), ("sdpa", "truth")]
    pairs = [(a, b) for a, b in pairs if a in x and b in x]
    ser = {p: series(x[p[0]], x[p[1]]) for p in pairs}
    hdr = "step  |x|max   " + "  ".join(f"{a}-{b}: max     mean    rel_l2 " for a, b in pairs)
    lines.append(hdr)
    ref = x.get("fa2") or x.get("sdpa") or x["product"]
    n = max(len(s) for s in ser.values())
    for k in range(n):
        if k % every and k != n - 1:
            continue
        row = f"{k + 1:4d}  {ref[k].abs().max().item():6.3f}   "
        for p in pairs:
            if k < len(ser[p]):
                s = ser[p][k]
                row += f"{' ' * (len(p[0]) + len(p[1]) + 2)}{s['max']:.2e} {s['mean']:.2e} {s['rel_l2']:.2e}   "
            else:
                row += " " * (len(p[0]) + len(p[1]) + 2 + 30)
        lines.append(row)
    return "\n".join(lines)
