"""n samples per request (`num_samples`) against the same request listed n times, on one GPU.

Synthetic BAGEL-7B (random init, SigLIP-so400m tower attached). Two contexts: "short" is one 378 x 378 image and a
64-token prompt (the README's chat workload); "long" is `--long-images` such images and the prompt (about 3.7k tokens).

1. End to end, short context, n in `--ns`, alternating `--rounds` times: `chat_batch([req], num_samples=n)` against
   `chat_batch([req] * n)`, `--tokens` decode steps (host clock around work that ends in a device synchronise).
2. Decode step inside the captured graph, `generate_text_batch(num_samples=[n])` ("samples": the shared layout from
   SHARED_MIN_SAMPLES samples on, the context replicated per row below) against the context copied n times and
   `generate_text_batch` over n requests ("repeated"), for both contexts and n in `--step-ns` (n = 2 falls on the
   replicated side of the rule, 8 and 32 on the shared side): the long-minus-short method of gpu_perf_chat_batch.py,
   (min over `--step-rounds` of a `--tokens` + 16 step run - min of a 16 step run) / `--tokens`, alternating.
3. Attention kernel time per launch (one layer, Hq 28, Hk 4, each row 64 generated keys): the shared kernel against
   attn_decode_kernel on the replicated layout, CUDA events around a captured graph of `--graph-launches` launches.
   Bytes: the K/V rows each kernel has to read (shared: the prefix once per pass of up to 4 rows plus each row's
   suffix; replicated: each row's whole cache), over kernel time.
4. KV slab bytes at `--tokens` new tokens per row for all 28 layers, from the plan's row count.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_parallel_sampling.py [--ns 8 32] [--tokens 128] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bagel_b200 import ops, synthetic  # noqa: E402
from bagel_b200.qwen2_navit import ForwardPlan, NaiveCache, gather_requests  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ns", type=int, nargs="+", default=[8, 32])
ap.add_argument("--step-ns", type=int, nargs="+", default=[2, 8, 32])
ap.add_argument("--kernel-ns", type=int, nargs="+", default=[1, 2, 4, 8, 32])
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--step-rounds", type=int, default=3)
ap.add_argument("--graph-launches", type=int, default=200)
ap.add_argument("--image", type=int, default=378)
ap.add_argument("--long-images", type=int, default=5)
ap.add_argument("--prompt", type=int, default=64)
ap.add_argument("--layers", type=int, default=None, help="decoder layers of the synthetic model (default: all 28)")
args = ap.parse_args()

NT = synthetic.NEW_TOKEN_IDS
HQ, HK, D = 28, 4, 128
KV_ROW_BYTES = 28 * HK * D * 2 * 2       # K + V of one token over BAGEL-7B's 28 layers (57 344 B)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Tokenizer(synthetic.RandomIdTokenizer):
    """RandomIdTokenizer with a decode that renders the ids (start token excluded) as numbers."""

    def decode(self, ids):
        return "<|im_start|>" + " ".join(str(int(i)) for i in list(ids)[1:])


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def context(model, images, tok):
    """One request's cache and start-token inputs: its images in rounds, then the prompt, as chat_batch builds it."""
    kv, rp = [0], [0]
    cache = NaiveCache(model.config.llm_config.num_hidden_layers)
    for im in images:
        gi, kv, rp = model.prepare_vit_image_round(kv, rp, [im], lambda x: x, NT)
        cache = model.forward_cache_update_vit(cache, **gi)
    gp, kv, rp = model.prepare_prompts(kv, rp, [str(args.prompt)], tok, NT)
    cache = model.forward_cache_update_text(cache, **gp)
    return cache, model.prepare_start_tokens(kv, rp, NT), kv[0]


def replicate(cache, gs, n):
    kv = torch.as_tensor(gs["key_values_lens"]).cpu()
    rc = gather_requests(cache, kv, [0] * n)
    rep = lambda x: torch.as_tensor(x).cpu().repeat(n)  # noqa: E731
    return rc, dict(key_values_lens=rep(kv), packed_key_value_indexes=torch.arange(int(kv[0]) * n),
                    packed_start_tokens=rep(gs["packed_start_tokens"]),
                    packed_query_position_ids=rep(gs["packed_query_position_ids"]))


def kernel_times(ctx, n, used=64):
    """Per-launch time (ms) of the shared kernel and of attn_decode_kernel on the replicated layout, and their bytes."""
    g = torch.Generator(device="cuda").manual_seed(n + ctx)
    q = torch.randn(n, HQ, D, device="cuda", generator=g).to(torch.bfloat16)
    cap = ctx + n * used
    k = torch.randn(cap, HK, D, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(cap, HK, D, device="cuda", generator=g).to(torch.bfloat16)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    cu_rows, pb, pl = i32([0, n]), i32([0]), i32([ctx])
    sb, su = i32([ctx + r * used for r in range(n)]), i32([ctx + used] * n)
    rk = torch.randn(n * (ctx + used), HK, D, device="cuda", generator=g).to(torch.bfloat16)
    rv = torch.randn(n * (ctx + used), HK, D, device="cuda", generator=g).to(torch.bfloat16)
    cu_q = torch.arange(n + 1, dtype=torch.int32, device="cuda")
    cu_k = i32([r * (ctx + used) for r in range(n + 1)])
    out = torch.empty_like(q)
    shared = lambda: ops.attn_decode_shared(q, k, v, cu_rows, pb, pl, sb, su, n, ctx + used, out=out)  # noqa: E731
    repl = lambda: ops.attn_varlen(q, rk, rv, cu_q, cu_k, 1, ctx + used, True, out=out, seqused_k=su)  # noqa: E731
    res = {}
    for name, fn in (("shared", shared), ("replicated", repl)):
        fn()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.graph_launches):
                fn()
        graph.replay()
        best = float("inf")
        for _ in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            b.synchronize()
            best = min(best, a.elapsed_time(b) / args.graph_launches)
        res[name] = best
    row = HK * D * 2 * 2
    passes = -(-n // 4)
    res["shared_bytes"] = (passes * ctx + n * used) * row
    res["replicated_bytes"] = n * (ctx + used) * row
    return res


def main():
    assert torch.cuda.is_available(), "gpu_perf_parallel_sampling needs a CUDA device"
    name = card()
    print(f"card: {name}", flush=True)
    model = synthetic.build_random_bagel(num_layers=args.layers)
    synthetic.attach_random_vit(model)
    tok = Tokenizer(seed=1)
    g = torch.Generator().manual_seed(3)
    images = [torch.rand(3, args.image, args.image, generator=g) * 2 - 1 for _ in range(args.long_images)]
    ident = lambda x: x  # noqa: E731
    out = {"card": name, "tokens": args.tokens}

    # 1. end to end, short context
    req = ([images[0]], str(args.prompt))
    model.chat_batch(tok, NT, ident, [req] * 2, max_length=4)
    model.chat_batch(tok, NT, ident, [req], max_length=4, num_samples=2)
    for n in args.ns:
        ts = {"samples": [], "repeated": []}
        for r in range(args.rounds):
            for key, fn in (("repeated", lambda: model.chat_batch(tok, NT, ident, [req] * n, max_length=args.tokens + 1)),
                            ("samples", lambda: model.chat_batch(tok, NT, ident, [req], max_length=args.tokens + 1,
                                                                 num_samples=n))):
                t, _ = wall(fn)
                ts[key].append(t)
                print(f"e2e n={n:3d} round {r} {key:10s}: {t:7.3f} s", flush=True)
        out[f"e2e_s_n{n}"] = ts

    # 2. decode step inside the graph, 4. slab bytes
    lm = model.language_model.model
    for cname, imgs in (("short", images[:1]), ("long", images)):
        cache, gs, ctx = context(model, imgs, tok)
        out[f"ctx_{cname}"] = ctx
        print(f"context {cname}: {ctx} tokens", flush=True)
        for n in sorted(set(args.step_ns) | set(args.ns)):
            rc, rgs = replicate(cache, gs, n)
            runs = {"samples": lambda m: model.generate_text_batch(cache, max_length=m, seeds=[7], num_samples=[n], **gs),
                    "repeated": lambda m: model.generate_text_batch(rc, max_length=m, seeds=[7] * n, **rgs)}
            for fn in runs.values():
                fn(16)
            best = {k: [float("inf"), float("inf")] for k in runs}
            for _ in range(args.step_rounds):
                for key, fn in runs.items():
                    best[key][0] = min(best[key][0], wall(lambda: fn(16 + args.tokens))[0])
                    best[key][1] = min(best[key][1], wall(lambda: fn(16))[0])
            layout = "shared" if ForwardPlan.decode_shared(lm, [ctx], [n], 1).shared is not None else "replicated"
            out[f"layout_{cname}_n{n}"] = layout
            for key in runs:
                ms = (best[key][0] - best[key][1]) / args.tokens * 1e3
                out[f"step_ms_{cname}_n{n}_{key}"] = ms
                print(f"decode step {cname} n={n:3d} {key:8s}: {ms:7.3f} ms" + (f" ({layout} layout)" if key == "samples"
                                                                               else ""), flush=True)
            # the shared layout's rows, whichever layout the rule picks for this n
            sh = (ctx + n * args.tokens) * KV_ROW_BYTES
            rp = ForwardPlan.decode(lm, [ctx] * n, args.tokens).total_kv * KV_ROW_BYTES
            out[f"slab_bytes_{cname}_n{n}"] = {"shared": sh, "replicated": rp}
            print(f"KV slab {cname} n={n:3d}: shared {sh / 1e9:.3f} GB, replicated {rp / 1e9:.3f} GB", flush=True)
            del rc
        del cache
        torch.cuda.empty_cache()

    # 3. kernel time
    for cname in ("short", "long"):
        ctx = out[f"ctx_{cname}"]
        for n in args.kernel_ns:
            r = kernel_times(ctx, n)
            for key in ("shared", "replicated"):
                gbs = r[f"{key}_bytes"] / (r[key] * 1e-3) / 1e9
                out[f"kernel_us_{cname}_n{n}_{key}"] = r[key] * 1e3
                out[f"kernel_gbs_{cname}_n{n}_{key}"] = gbs
                print(f"kernel {cname} ctx={ctx} n={n:3d} {key:10s}: {r[key] * 1e3:8.2f} us, "
                      f"{r[f'{key}_bytes'] / 1e6:8.2f} MB, {gbs:7.1f} GB/s", flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
