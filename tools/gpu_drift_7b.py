"""Drift of the full BAGEL-7B-MoT sampler (28 layers x 49 evaluations, text CFG 2, 1024^2) on one GPU:
product vs the reference-equivalent GPU legs (oracle + flash-attn / oracle + fp32 SDPA shim) vs the fp32 truth,
per Euler step. Prints the table.

  python tools/gpu_drift_7b.py [--batch 1] [--truth-steps 49] [--layers 28] [--evals 49]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import drift  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--evals", type=int, default=49)
    ap.add_argument("--truth-steps", type=int, default=49)
    ap.add_argument("--image-size", type=int, default=1024)
    ap.add_argument("--out", default="drift_7b.txt")
    a = ap.parse_args()
    res = drift.run(layers=a.layers, evals=a.evals, truth_steps=a.truth_steps, batch=a.batch, image_size=a.image_size)
    txt = [f"# BAGEL-7B-MoT dims, {a.layers} layers, {a.evals} evaluations, text CFG scale 2 (2 branches), batch {a.batch}, "
           f"{a.image_size}^2, random init (bagel_b200.synthetic seed 0), {torch.cuda.get_device_name(0)}",
           "# product = bagel_b200; fa2 = oracle on cuda + flash_attn_varlen_func (the reference as it runs on a GPU);",
           "# sdpa = oracle on cuda + fp32 per-sample SDPA (the reference as pinned on the CPU); truth = oracle fp32 end to end",
           "# distances of x_t (fp32 latents [B*4096, 64]) after each Euler step: max|d|, mean|d|, ||d||2/||ref||2",
           "# seconds: " + ", ".join(f"{k} {v:.1f}" for k, v in res["t"].items()), ""]
    txt.append(drift.report(res))
    x = res["x"]
    last = len(x["product"]) - 1
    fl = drift._stat(x["sdpa"][last], x["fa2"][last])
    pr = drift._stat(x["product"][last], x["fa2"][last])
    txt += ["", f"final step: noise floor (sdpa vs fa2) rel_l2 {fl['rel_l2']:.3e} max {fl['max']:.3e} mean {fl['mean']:.3e}",
            f"final step: product vs fa2            rel_l2 {pr['rel_l2']:.3e} max {pr['max']:.3e} mean {pr['mean']:.3e}",
            f"ratio product/floor (rel_l2): {pr['rel_l2'] / max(fl['rel_l2'], 1e-30):.2f}"]
    if "truth" in x:
        k = len(x["truth"]) - 1
        for leg in ("product", "fa2", "sdpa"):
            s = drift._stat(x[leg][k], x["truth"][k])
            txt.append(f"step {k + 1}: {leg:8s} vs truth rel_l2 {s['rel_l2']:.3e} max {s['max']:.3e} mean {s['mean']:.3e}")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        f.write("\n".join(txt) + "\n")
    print("\n".join(txt))


if __name__ == "__main__":
    main()
