"""Batched image generation (`InterleaveInferencer.gen_image_batch`) against sequential `InterleaveInferencer` calls,
on one GPU.

Synthetic BAGEL-7B (random init, SigLIP-so400m tower and FLUX VAE attached), 50 timesteps, timestep_shift 3, a 64-token
prompt per request. Workloads:
  t2i512   8 text-to-image requests at 512 x 512, the inferencer defaults (text CFG 3, image CFG 1.5 -> 3 branches,
           interval (0.4, 1], "global" renorm);
  t2i1024  the same at 1024 x 1024;
  edit1024 2 edits of a 1024 x 1024 image with tools/bench_blocks.py::edit_block's settings (text CFG 4, image CFG 2,
           interval [0, 1], "text_channel").
Each workload runs both paths once with 3 timesteps to warm up, then `--rounds` alternations of sequential calls (one
`torch.manual_seed(i); inferencer(...)` per request, as edit_block does) and one `gen_image_batch`. Time is a host clock
around work that ends in a device synchronise, VAE encode / decode included; images/s = requests / time.

Prints the card name and power limit read in the same process, and one JSON line last.
  python tools/gpu_perf_gen_batch.py [--rounds 2] [--workloads t2i512,t2i1024,edit1024] [--timesteps 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bagel_b200 import synthetic  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=2, help="sequential / batched alternations per workload")
ap.add_argument("--workloads", default="t2i512,t2i1024,edit1024")
ap.add_argument("--timesteps", type=int, default=50)
args = ap.parse_args()

DEFAULTS = dict(cfg_text_scale=3.0, cfg_img_scale=1.5, cfg_interval=(0.4, 1.0), cfg_renorm_min=0.0,
                cfg_renorm_type="global")
EDIT = dict(cfg_text_scale=4.0, cfg_img_scale=2.0, cfg_interval=(0.0, 1.0), cfg_renorm_min=0.0,
            cfg_renorm_type="text_channel")


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


def workload(name):
    from PIL import Image
    rs = np.random.RandomState(0)
    if name == "t2i512":
        return [dict(text="64", image_shapes=(512, 512), seed=i, **DEFAULTS) for i in range(8)]
    if name == "t2i1024":
        return [dict(text="64", image_shapes=(1024, 1024), seed=i, **DEFAULTS) for i in range(8)]
    if name == "edit1024":
        return [dict(text="64", image=Image.fromarray(rs.randint(0, 255, (1024, 1024, 3)).astype(np.uint8)), seed=i,
                     **EDIT) for i in range(2)]
    raise ValueError(name)


def main():
    assert torch.cuda.is_available(), "gpu_perf_gen_batch needs a CUDA device"
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    name = card()
    print(f"card: {name}", flush=True)
    model = synthetic.build_random_bagel()
    synthetic.attach_random_vit(model)
    vae = synthetic.build_random_vae()
    inf = InterleaveInferencer(model, vae, synthetic.RandomIdTokenizer(1), ImageTransform(1024, 512, 16),
                               ImageTransform(980, 224, 14), synthetic.NEW_TOKEN_IDS)
    steps = dict(num_timesteps=args.timesteps, timestep_shift=3.0)

    def sequential(reqs):
        out = []
        for r in reqs:
            r = dict(r)
            torch.manual_seed(r.pop("seed"))
            out.append(inf(image=r.pop("image", None), text=r.pop("text"), **r, **steps)["image"])
        return out

    def batched(reqs):
        return inf.gen_image_batch(reqs, **steps)

    results = {}
    for wl in args.workloads.split(","):
        reqs = workload(wl)
        warm = dict(steps, num_timesteps=3)   # warm-up: every shape both paths use (the step count changes none)
        r0 = dict(reqs[0])
        torch.manual_seed(r0.pop("seed"))
        inf(image=r0.pop("image", None), text=r0.pop("text"), **r0, **warm)
        inf.gen_image_batch(reqs, **warm)
        res = {"seq_s": [], "batch_s": []}
        for r in range(args.rounds):
            for key, fn in (("seq", sequential), ("batch", batched)):
                t, imgs = wall(lambda: fn(reqs))
                assert len(imgs) == len(reqs)
                res[key + "_s"].append(t)
                print(f"{wl} round {r} {key:5s}: {t:8.3f} s per batch of {len(reqs)}, {len(reqs) / t:7.3f} images/s",
                      flush=True)
        seq, bat = statistics.median(res["seq_s"]), statistics.median(res["batch_s"])
        results[wl] = {"requests": len(reqs), **res, "seq_images_s": len(reqs) / seq, "batch_images_s": len(reqs) / bat,
                       "speedup": seq / bat}
        print(f"{wl}: sequential {seq:.3f} s, batched {bat:.3f} s, {seq / bat:.2f}x", flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"card": name, "timesteps": args.timesteps, **results}))


if __name__ == "__main__":
    main()
