"""Batched interleaved requests (`InterleaveInferencer.call_batch`) against sequential `InterleaveInferencer` calls, on
one GPU.

Synthetic BAGEL-7B (random init, SigLIP-so400m tower and FLUX VAE attached), 50 timesteps, timestep_shift 3, a 64-token
prompt per request, the inferencer's CFG defaults. Workloads:
  think512s   8 think text-to-image requests at 512 x 512, max_think_token_n=256, do_sample=True, temperature 0.3 (the
              setting of the reference's WISE / KRIS / RISE / ImgEdit think drivers);
  think1024s  the same at 1024 x 1024;
  think512g, think1024g   the same with greedy thoughts;
  mixed16     8 understanding requests (one 378 x 378 image + prompt, 128-token budget, greedy), 4 think text-to-image
              requests at 512 x 512 (sampled at 0.3, 256-token budget) and 4 edits of a 512 x 512 image.
Each workload runs both paths once with 3 timesteps to warm up, then `--rounds` alternations of sequential calls (one
`torch.manual_seed(i); inferencer(...)` per request) and one `call_batch`. Time is a host clock around work that ends in a
device synchronise, image encode and decode included. Decode time is the same clock around every Bagel.generate_text /
generate_text_batch call of the timed window. A random-init model rarely emits its end token, so most thoughts and
answers run to their budget; the real lengths are printed.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_think_batch.py [--rounds 1] [--workloads think512s,...] [--timesteps 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bagel_b200 import synthetic  # noqa: E402
from bagel_b200.bagel import Bagel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=1, help="sequential / batched alternations per workload")
ap.add_argument("--workloads", default="think512s,think512g,mixed16,think1024s,think1024g")
ap.add_argument("--timesteps", type=int, default=50)
args = ap.parse_args()

NT = synthetic.NEW_TOKEN_IDS
VOCAB = 151643


class Tokenizer:
    """Offline stand-in: the word "#n" -> n fixed pseudo-random ids, an integer word -> that id, any other word -> a
    stable id; decode writes ids back as such words (bos / eos as the strings the inferencer splits on)."""
    SPECIAL = {NT["bos_token_id"]: "<|im_start|>", NT["eos_token_id"]: "<|im_end|>"}

    def encode(self, text):
        ids = []
        for w in text.split():
            if w.startswith("#"):
                ids += torch.randint(0, VOCAB, (int(w[1:]),), generator=torch.Generator().manual_seed(len(ids))).tolist()
            elif w.isdigit():
                ids.append(int(w))
            else:
                ids.append(zlib.crc32(w.encode()) % VOCAB)
        return ids

    def decode(self, ids):
        return " ".join(self.SPECIAL.get(int(i), str(int(i))) for i in ids)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


DECODE = {"s": 0.0}


def _timed(fn):
    def wrapped(*a, **k):
        t, out = wall(lambda: fn(*a, **k))
        DECODE["s"] += t
        return out
    return wrapped


Bagel.generate_text = _timed(Bagel.generate_text)
Bagel.generate_text_batch = _timed(Bagel.generate_text_batch)


def workload(name):
    from PIL import Image
    rs = np.random.RandomState(0)

    def img(n):
        return Image.fromarray(rs.randint(0, 255, (n, n, 3)).astype(np.uint8))

    think = dict(think=True, max_think_token_n=256, do_sample=True, text_temperature=0.3)
    if name in ("think512s", "think1024s", "think512g", "think1024g"):
        n = 512 if "512" in name else 1024
        kw = dict(think, do_sample=name.endswith("s"))
        return [dict(text="#64", image_shapes=(n, n), seed=i, **kw) for i in range(8)]
    if name == "mixed16":
        und = [dict(text="#64", image=img(378), understanding_output=True, max_think_token_n=128, seed=i)
               for i in range(8)]
        t2i = [dict(text="#64", image_shapes=(512, 512), seed=8 + i, **think) for i in range(4)]
        edit = [dict(text="#64", image=img(512), seed=12 + i) for i in range(4)]
        return und + t2i + edit
    raise ValueError(name)


def main():
    assert torch.cuda.is_available(), "gpu_perf_think_batch needs a CUDA device"
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    name = card()
    print(f"card: {name}", flush=True)
    model = synthetic.build_random_bagel()
    synthetic.attach_random_vit(model)
    vae = synthetic.build_random_vae()
    tok = Tokenizer()
    inf = InterleaveInferencer(model, vae, tok, ImageTransform(1024, 512, 16), ImageTransform(980, 224, 14), NT)
    steps = dict(num_timesteps=args.timesteps, timestep_shift=3.0)

    def sequential(reqs, st=steps):
        out = []
        for r in reqs:
            r = dict(r)
            torch.manual_seed(r.pop("seed"))
            out.append(inf(image=r.pop("image", None), text=r.pop("text", None), **r, **st))
        return out

    def batched(reqs, st=steps):
        return inf.call_batch(reqs, **st)

    results = {}
    for wl in args.workloads.split(","):
        reqs = workload(wl)
        warm = dict(steps, num_timesteps=3)   # warm-up: every shape both paths use (the step count changes none)
        sequential(reqs[:1], warm)
        batched(reqs, warm)
        res = {"seq_s": [], "batch_s": [], "seq_decode_s": [], "batch_decode_s": []}
        for r in range(args.rounds):
            for key, fn in (("seq", sequential), ("batch", batched)):
                DECODE["s"] = 0.0
                t, outs = wall(lambda: fn(reqs))
                assert len(outs) == len(reqs)
                lens = [len(tok.encode(o["text"])) for o in outs if o["text"] is not None]
                n_img = sum(o["image"] is not None for o in outs)
                res[key + "_s"].append(t)
                res[key + "_decode_s"].append(DECODE["s"])
                res[key + "_text_tokens"] = lens
                print(f"{wl} round {r} {key:5s}: {t:8.3f} s per batch of {len(reqs)}, {len(reqs) / t:6.3f} requests/s, "
                      f"{n_img / t:6.3f} images/s, decode {DECODE['s']:7.3f} s = {sum(lens) / DECODE['s']:8.1f} tokens/s; "
                      f"text lengths {lens}", flush=True)
        seq, bat = statistics.median(res["seq_s"]), statistics.median(res["batch_s"])
        sd, bd = statistics.median(res["seq_decode_s"]), statistics.median(res["batch_decode_s"])
        n_img = sum(1 for r in reqs if not r.get("understanding_output"))
        ntok = sum(res["batch_text_tokens"])
        results[wl] = {"requests": len(reqs), "images": n_img, **res,
                       "seq_requests_s": len(reqs) / seq, "batch_requests_s": len(reqs) / bat,
                       "seq_images_s": n_img / seq, "batch_images_s": n_img / bat,
                       "seq_decode_tokens_s": sum(res["seq_text_tokens"]) / sd, "batch_decode_tokens_s": ntok / bd,
                       "speedup": seq / bat}
        print(f"{wl}: sequential {seq:.3f} s, batched {bat:.3f} s, {seq / bat:.2f}x; decode {sd:.3f} -> {bd:.3f} s",
              flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"card": name, "timesteps": args.timesteps, **results}))


if __name__ == "__main__":
    main()
