"""Batched image understanding (`Bagel.chat_batch`) against sequential `Bagel.chat`, on one GPU.

Synthetic BAGEL-7B (random init, SigLIP-so400m tower attached), 32 requests of one 378 x 378 image and a 64-token
prompt, `--tokens` decode steps each (random weights practically never emit the end token; the decoded counts are
reported as they came out).

1. End to end, alternating `--rounds` times: the 32 requests through sequential `chat`, then through one `chat_batch`.
   Total time (host clock around work that ends in a device synchronise) and decode tokens per second over that time.
2. Decode step time inside the captured graph, at batch 1 and batch 32, greedy and sampled: `generate_text_batch` on the
   same context for `--tokens` + 16 and for 16 steps, each `--step-rounds` times, alternating. The step time is
   (min long - min short) / `--tokens`: the difference removes setup and capture, and the minima drop runs in which the
   host-side setup (buffer allocation, graph capture) happened to be slow.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_chat_batch.py [--requests 32] [--tokens 128] [--rounds 2] [--step-rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bagel_b200 import synthetic  # noqa: E402
from bagel_b200.qwen2_navit import NaiveCache  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=32)
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--rounds", type=int, default=2, help="sequential / batched alternations")
ap.add_argument("--step-rounds", type=int, default=5, help="long / short decode alternations per step figure")
ap.add_argument("--image", type=int, default=378)
ap.add_argument("--prompt", type=int, default=64)
args = ap.parse_args()

NT = synthetic.NEW_TOKEN_IDS


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class CountingTokenizer(synthetic.RandomIdTokenizer):
    """RandomIdTokenizer whose decode counts the decoded ids (start token excluded) and renders them as numbers."""

    def __init__(self):
        super().__init__(seed=1)
        self.decoded = 0

    def decode(self, ids):
        ids = [int(i) for i in ids]
        self.decoded += len(ids) - 1
        return "<|im_start|>" + " ".join(map(str, ids[1:]))


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    assert torch.cuda.is_available(), "gpu_perf_chat_batch needs a CUDA device"
    name = card()
    print(f"card: {name}", flush=True)
    model = synthetic.build_random_bagel()
    synthetic.attach_random_vit(model)
    g = torch.Generator().manual_seed(3)
    images = [torch.rand(3, args.image, args.image, generator=g) * 2 - 1 for _ in range(args.requests)]
    prompts = [str(args.prompt)] * args.requests
    tok = CountingTokenizer()
    reqs = [([im], p) for im, p in zip(images, prompts)]
    ident = lambda x: x  # noqa: E731  (images are already transformed)

    def sequential():
        return [model.chat(tok, NT, ident, im, p, max_length=args.tokens + 1) for im, p in reqs]

    def batched():
        return model.chat_batch(tok, NT, ident, reqs, max_length=args.tokens + 1)

    # warm-up: every shape both paths use
    model.chat(tok, NT, ident, *reqs[0], max_length=4)
    model.chat_batch(tok, NT, ident, reqs, max_length=4)
    res = {"seq_s": [], "batch_s": [], "seq_tokens": [], "batch_tokens": []}
    for r in range(args.rounds):
        for key, fn in (("seq", sequential), ("batch", batched)):
            tok.decoded = 0
            t, _ = wall(fn)
            res[key + "_s"].append(t)
            res[key + "_tokens"].append(tok.decoded)
            print(f"round {r} {key:5s}: {t:8.3f} s, {tok.decoded} decode tokens, {tok.decoded / t:9.1f} tok/s", flush=True)

    # decode step inside the graph, on the batched context of the first B requests
    steps = {}
    for B in (1, args.requests):
        kv, rp = [0] * B, [0] * B
        gi, kv, rp = model.prepare_vit_image_round(kv, rp, images[:B], ident, NT)
        cache = model.forward_cache_update_vit(NaiveCache(model.config.llm_config.num_hidden_layers), **gi)
        gp, kv, rp = model.prepare_prompts(kv, rp, prompts[:B], tok, NT)
        cache = model.forward_cache_update_text(cache, **gp)
        gs = model.prepare_start_tokens(kv, rp, NT)
        for sample in (False, True):
            run = lambda n: model.generate_text_batch(cache, max_length=n, do_sample=sample, seeds=[7] * B, **gs)  # noqa: E731
            run(16)
            longs, shorts = [], []
            for _ in range(args.step_rounds):
                longs.append(wall(lambda: run(16 + args.tokens))[0])
                shorts.append(wall(lambda: run(16))[0])
            key = f"step_ms_b{B}_{'sampled' if sample else 'greedy'}"
            steps[key] = (min(longs) - min(shorts)) / args.tokens * 1e3
            print(f"decode step, batch {B:3d}, {'sampled' if sample else 'greedy '}: {steps[key]:7.3f} ms; "
                  f"{16 + args.tokens} steps {', '.join(f'{x:.3f}' for x in longs)} s, "
                  f"16 steps {', '.join(f'{x:.3f}' for x in shorts)} s; context {kv[0]} tokens", flush=True)

    seq_tps = statistics.median(a / b for a, b in zip(res["seq_tokens"], res["seq_s"]))
    bat_tps = statistics.median(a / b for a, b in zip(res["batch_tokens"], res["batch_s"]))
    out = {"card": name, "requests": args.requests, "tokens": args.tokens, "image": args.image, "prompt": args.prompt,
           "seq_s": res["seq_s"], "batch_s": res["batch_s"], "seq_tok_s": seq_tps, "batch_tok_s": bat_tps,
           "speedup_tok_s": bat_tps / seq_tps, **steps}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
