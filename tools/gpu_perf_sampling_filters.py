"""Cost of truncated sampling (top-k / top-p / min-p, `bagel_sample_rows_filtered_bf16`) on one GPU.

1. Kernel time, CUDA events around `--launches` back-to-back launches after a warm-up, at B in {1, 32, 128} rows of
   V = 152064 bf16 logits (random normal * 3, the spread of a language model's logits): `sample_rows_mixed` (every
   row sampled at T = 0.7) against the filtered kernel with top-k alone (k = 50), top-p alone (p = 0.9), min-p alone
   (0.05) and all three. The four variants alternate `--rounds` times; the minimum per variant is reported.
2. Decode step inside the captured graph of synthetic BAGEL-7B (random init), at batch 1 and 32 on a `--prompt`-token
   context, sampled at T = 0.7 without and with all three filters: `generate_text_batch` for `--tokens` + 16 and for
   16 steps, alternating the two settings `--step-rounds` times. The step time is (min long - min short) / `--tokens`.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_sampling_filters.py [--launches 200] [--rounds 5] [--tokens 128] [--step-rounds 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bagel_b200 import ops, synthetic  # noqa: E402
from bagel_b200.qwen2_navit import NaiveCache  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=200)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--step-rounds", type=int, default=4)
ap.add_argument("--prompt", type=int, default=64)
args = ap.parse_args()

V = 152064
FILTERS = {"top_k": dict(top_k=50), "top_p": dict(top_p=0.9), "min_p": dict(min_p=0.05),
           "all": dict(top_k=50, top_p=0.9, min_p=0.05)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_times():
    out = {}
    for B in (1, 32, 128):
        g = torch.Generator().manual_seed(B)
        logits = (torch.randn(B, V, generator=g) * 3).to(torch.bfloat16).cuda()
        inv_t = torch.full((B,), float(np.float32(1.0) / np.float32(0.7)), device="cuda")
        keys = torch.arange(B, dtype=torch.int64, device="cuda") + (5 << 32)
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        tok = torch.empty(B, dtype=torch.int64, device="cuda")

        def filtered(top_k=0, top_p=1.0, min_p=0.0):
            k = torch.full((B,), top_k, dtype=torch.int32, device="cuda")
            p, m = (torch.full((B,), v, dtype=torch.float32, device="cuda") for v in (top_p, min_p))
            return lambda: ops.sample_rows_filtered(logits, inv_t, k, p, m, keys, step, tok)

        variants = {"mixed": lambda: ops.sample_rows_mixed(logits, inv_t, keys, step, tok),
                    **{name: filtered(**f) for name, f in FILTERS.items()}}
        best = {name: float("inf") for name in variants}
        for fn in variants.values():
            for _ in range(10):
                fn()
        for _ in range(args.rounds):
            for name, fn in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    fn()
                e1.record()
                e1.synchronize()
                best[name] = min(best[name], e0.elapsed_time(e1) * 1e3 / args.launches)
        for name, us in best.items():
            out[f"kernel_us_b{B}_{name}"] = us
        print(f"B {B:3d}: " + ", ".join(f"{n} {us:7.1f} us" for n, us in best.items()), flush=True)
    return out


def step_times():
    model = synthetic.build_random_bagel()
    tok = synthetic.RandomIdTokenizer(seed=1)
    NT = synthetic.NEW_TOKEN_IDS
    out = {}
    for B in (1, 32):
        gp, kv, rp = model.prepare_prompts([0] * B, [0] * B, [str(args.prompt)] * B, tok, NT)
        cache = model.forward_cache_update_text(NaiveCache(model.config.llm_config.num_hidden_layers), **gp)
        gs = model.prepare_start_tokens(kv, rp, NT)
        settings = {"plain": {}, "filtered": FILTERS["all"]}

        def run(n, s):
            return model.generate_text_batch(cache, max_length=n, do_sample=True, temperature=0.7, seeds=[7] * B,
                                             **settings[s], **gs)
        for s in settings:
            run(16, s)
        longs = {s: [] for s in settings}
        shorts = {s: [] for s in settings}
        for _ in range(args.step_rounds):
            for s in settings:
                longs[s].append(wall(lambda: run(16 + args.tokens, s)))
                shorts[s].append(wall(lambda: run(16, s)))
        for s in settings:
            out[f"step_ms_b{B}_{s}"] = (min(longs[s]) - min(shorts[s])) / args.tokens * 1e3
        d = out[f"step_ms_b{B}_filtered"] - out[f"step_ms_b{B}_plain"]
        print(f"decode step, batch {B:3d}: sampled {out[f'step_ms_b{B}_plain']:.3f} ms, with top-k/top-p/min-p "
              f"{out[f'step_ms_b{B}_filtered']:.3f} ms ({d * 1e3:+.1f} us); {16 + args.tokens} steps "
              f"{longs}, 16 steps {shorts}", flush=True)
    return out


def main():
    assert torch.cuda.is_available(), "gpu_perf_sampling_filters needs a CUDA device"
    name = card()
    print(f"card: {name}", flush=True)
    res = {"card": name, **kernel_times(), **step_times()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
