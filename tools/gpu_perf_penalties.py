"""Cost of the decode-step penalties (repetition, presence, frequency; `bagel_apply_penalties_bf16`) on one GPU.

1. Kernel time, CUDA events around one replay of a graph of `--launches` back-to-back launches, at B in {1, 32, 128}
   rows of V = 152064 bf16 logits, every row with all three penalties set, after 128 and 1024 generated tokens: a
   repetitive stream (16 distinct tokens) and a non-repetitive one (every token distinct). Each timed launch adds a
   token the row already holds, so only its count grows. The minimum over `--rounds` replays is reported.
2. Decode step inside the captured graph of synthetic BAGEL-7B (random init), at batch 1 and 32 on a `--prompt`-token
   context, sampled at T = 0.7 with top-k 20 and top-p 0.8, without and with repetition_penalty = 1.05,
   presence_penalty = 0.5 and frequency_penalty = 0.5: `generate_text_batch` for `--tokens` + 16 and for 16 steps,
   alternating the two settings `--step-rounds` times. The step time is (min long - min short) / `--tokens`.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_penalties.py [--launches 500] [--rounds 5] [--tokens 128] [--step-rounds 4]
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
ap.add_argument("--launches", type=int, default=500)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--step-rounds", type=int, default=4)
ap.add_argument("--prompt", type=int, default=64)
args = ap.parse_args()

V = 152064
PENALTIES = dict(repetition_penalty=1.05, presence_penalty=0.5, frequency_penalty=0.5)


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


def state(B, generated, distinct, cap, rng):
    """penalty_state after `generated` tokens drawn from `distinct` different ones (each appears at least once)."""
    seen = np.zeros((B, 1 + 2 * cap), dtype=np.int32)
    for b in range(B):
        toks = rng.choice(V, distinct, replace=False)
        counts = np.bincount(np.concatenate([np.arange(distinct), rng.integers(0, distinct, generated - distinct)]),
                             minlength=distinct)
        seen[b, 0] = distinct
        seen[b, 1:1 + distinct] = toks
        seen[b, 1 + cap:1 + cap + distinct] = counts
    return torch.from_numpy(seen).cuda()


def kernel_times():
    out = {}
    rng = np.random.default_rng(0)
    for B in (1, 32, 128):
        g = torch.Generator().manual_seed(B)
        logits = (torch.randn(B, V, generator=g) * 3).to(torch.bfloat16).cuda()
        rp, fp, pp = (torch.full((B,), v, dtype=torch.float32, device="cuda") for v in (1.05, 0.5, 0.5))
        finished = torch.zeros(B, dtype=torch.int32, device="cuda")
        step = torch.full((1,), 5, dtype=torch.int32, device="cuda")
        for n in (128, 1024):
            for kind, distinct in (("repetitive", 16), ("distinct", n)):
                cap = n + 64
                seen = state(B, n, distinct, cap, rng)
                tokens = torch.tensor(seen[:, 1].tolist(), dtype=torch.int64, device="cuda")   # one each row holds

                def launch():
                    ops.apply_penalties(logits, rp, fp, pp, tokens, finished, step, seen)
                for _ in range(10):
                    launch()
                # the launches run from one captured graph, as in the decode step: an eager loop would time the host
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    for _ in range(args.launches):
                        launch()
                graph.replay()
                best = float("inf")
                for _ in range(args.rounds):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    graph.replay()
                    e1.record()
                    e1.synchronize()
                    best = min(best, e0.elapsed_time(e1) * 1e3 / args.launches)
                out[f"kernel_us_b{B}_n{n}_{kind}"] = best
                print(f"B {B:3d}, {n:4d} generated, {kind:10s} ({distinct:4d} distinct): {best:6.2f} us", flush=True)
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
        settings = {"plain": {}, "penalised": PENALTIES}

        def run(n, s):
            return model.generate_text_batch(cache, max_length=n, do_sample=True, temperature=0.7, top_k=20, top_p=0.8,
                                             seeds=[7] * B, **settings[s], **gs)
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
        d = out[f"step_ms_b{B}_penalised"] - out[f"step_ms_b{B}_plain"]
        print(f"decode step, batch {B:3d}: top-k/top-p {out[f'step_ms_b{B}_plain']:.3f} ms, with penalties "
              f"{out[f'step_ms_b{B}_penalised']:.3f} ms ({d * 1e3:+.1f} us); {16 + args.tokens} steps "
              f"{longs}, 16 steps {shorts}", flush=True)
    return out


def main():
    assert torch.cuda.is_available(), "gpu_perf_penalties needs a CUDA device"
    name = card()
    print(f"card: {name}", flush=True)
    res = {"card": name, **kernel_times(), **step_times()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
