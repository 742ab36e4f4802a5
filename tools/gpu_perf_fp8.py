"""The opt-in FP8 generation-expert MLP (`fp8_gen_mlp=True`) against the bf16 one, on one GPU.

1. The MLP block at the denoising step's shape: M = 16 x 4098 = 65 568 rows (8 images x 2 CFG branches), BAGEL-7B
   hidden 3584, intermediate 18944, random weights:
     bf16  gate|up EPI_SWIGLU + down EPI_RESID                                   (bagel_gemm_bf16 x 2)
     fp8   quantise h + gate|up EPI_SWIGLU + quantise act + down EPI_RESID       (bagel_quantize_fp8_bf16 / bagel_gemm_fp8)
   CUDA events around each launch and around the whole sequence.
2. The full denoising step of bench.py's workload (synthetic BAGEL-7B, batch 8, 1024 x 1024, 2 CFG branches, kernels
   launched individually as in bench.py's timed region): `--warmup` + `--steps` steps with the flag off and on,
   alternating `--rounds` times; device memory after load for each.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_fp8.py [--iters 5] [--steps 12] [--warmup 3] [--rounds 2] [--no-step]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bagel_b200 import fp8, ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=5, help="timed repetitions of each MLP sequence")
ap.add_argument("--steps", type=int, default=12)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=2, help="off/on alternations of the step measurement")
ap.add_argument("--no-step", action="store_true", help="only the MLP sequences")
args = ap.parse_args()

DEV = "cuda"
M, H, I = 16 * 4098, 3584, 18944
EVALS_PER_IMAGE = 49


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fns, iters):
    """fns: [(name, fn)] run in order as one sequence; returns {name: [ms]} and the sequence times."""
    for _, f in fns:
        f()
    torch.cuda.synchronize()
    per = {n: [] for n, _ in fns}
    seq = []
    for _ in range(iters):
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)]
        evs[0].record()
        for i, (_, f) in enumerate(fns):
            f()
            evs[i + 1].record()
        torch.cuda.synchronize()
        for i, (n, _) in enumerate(fns):
            per[n].append(evs[i].elapsed_time(evs[i + 1]))
        seq.append(evs[0].elapsed_time(evs[-1]))
    return per, seq


def mlp_sequences():
    g = torch.Generator(device=DEV).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=DEV) * scale).to(torch.bfloat16)

    h = rnd(M, H)
    xb = rnd(M, H)
    gate, up, down = rnd(I, H, scale=0.02), rnd(I, H, scale=0.02), rnd(H, I, scale=0.02)
    wgu = ops.interleave_gate_up(gate, up)
    w8 = fp8.GenMlpFp8.from_reference(gate, up, down)
    del gate, up
    act = torch.empty(M, I, dtype=torch.bfloat16, device=DEV)
    xa = torch.empty(M, H, dtype=torch.bfloat16, device=DEV)
    hq = torch.empty(M, H, dtype=ops.FP8, device=DEV)
    hs = torch.empty(H // 128, M, dtype=torch.float32, device=DEV)
    aq = torch.empty(M, I, dtype=ops.FP8, device=DEV)
    as_ = torch.empty(I // 128, M, dtype=torch.float32, device=DEV)
    bf16 = [("gate_up", lambda: ops.gemm(h, wgu, epilogue=ops.EPI_SWIGLU, out=act)),
            ("down", lambda: ops.gemm(act, down, resid=xb, epilogue=ops.EPI_RESID, out=xa))]
    f8 = [("quant_h", lambda: ops.quantize_fp8(h, 1, q=hq, scales=hs)),
          ("gate_up", lambda: ops.gemm_fp8(hq, hs, w8.wgu, w8.wgu_s, epilogue=ops.EPI_SWIGLU, out=act)),
          ("quant_act", lambda: ops.quantize_fp8(act, 1, q=aq, scales=as_)),
          ("down", lambda: ops.gemm_fp8(aq, as_, w8.wd, w8.wd_s, resid=xb, epilogue=ops.EPI_RESID, out=xa))]
    out = {}
    for rnd_i in range(2):      # alternate: bf16, fp8, bf16, fp8
        for name, fns in (("bf16", bf16), ("fp8", f8)):
            per, seq = timed(fns, args.iters)
            o = out.setdefault(name, {"seq_ms": [], "kernels_ms": {}})
            o["seq_ms"] += seq
            for k, v in per.items():
                o["kernels_ms"].setdefault(k, []).extend(v)
    flops = {"gate_up": 2.0 * M * 2 * I * H, "down": 2.0 * M * H * I}
    for name, o in out.items():
        o["seq_ms_median"] = statistics.median(o["seq_ms"])
        o["kernels_ms_median"] = {k: statistics.median(v) for k, v in o["kernels_ms"].items()}
        o["tflops"] = {k: flops[k] / (o["kernels_ms_median"][k] * 1e-3) / 1e12 for k in flops}
        del o["kernels_ms"]
    return out


def denoising_steps():
    from bagel_b200 import synthetic
    res = {"off": [], "on": []}
    mem = {}
    for _ in range(args.rounds):
        for flag in (False, True):
            torch.cuda.empty_cache()
            model = synthetic.build_random_bagel(device=DEV, seed=0, fp8_gen_mlp=flag)
            torch.cuda.synchronize()
            mem["on" if flag else "off"] = torch.cuda.memory_allocated() / 1e9
            gen_input, cfg_text, ctxs = synthetic.t2i_inputs(model, 8, (1024, 1024), seed=1, noise_seed=2)
            kw = dict(num_timesteps=EVALS_PER_IMAGE + 1, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type="global",
                      cfg_interval=[0.0, 1.0], cfg_text_scale=2.0, cfg_img_scale=1.0,
                      cfg_text_packed_position_ids=cfg_text["cfg_packed_position_ids"],
                      cfg_text_packed_query_indexes=cfg_text["cfg_packed_query_indexes"],
                      cfg_text_key_values_lens=cfg_text["cfg_key_values_lens"],
                      cfg_text_packed_key_value_indexes=cfg_text["cfg_packed_key_value_indexes"],
                      cfg_text_past_key_values=ctxs["cfg_text"])
            model.use_cuda_graph = False
            runner = model.make_flow_runner(past_key_values=ctxs["main"], **gen_input, **kw)
            for i in range(args.warmup):
                runner.step(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.steps):
                runner.step(args.warmup + i)
            e1.record()
            torch.cuda.synchronize()
            res["on" if flag else "off"].append(e0.elapsed_time(e1) / args.steps)
            print(f"step fp8_gen_mlp={flag}: {res['on' if flag else 'off'][-1]:.1f} ms", flush=True)
            del runner, model, gen_input, cfg_text, ctxs
    return {"ms_per_step": res, "mem_after_load_gb": mem}


if __name__ == "__main__":
    assert torch.cuda.is_available(), "gpu_perf_fp8 needs a CUDA device"
    name = card()
    print(f"card: {name}", flush=True)
    r = {"card": name, "M": M, "H": H, "I": I, "mlp": mlp_sequences()}
    print(json.dumps(r["mlp"]), flush=True)
    torch.cuda.empty_cache()
    if not args.no_step:
        r["step"] = denoising_steps()
    r["card_after"] = card()
    print(json.dumps(r))
