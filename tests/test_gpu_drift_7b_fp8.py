"""-m gpu: the opt-in FP8 generation-expert MLP (`fp8_gen_mlp=True`) at the benchmarked configuration — BAGEL-7B-MoT
dimensions, 28 layers, 49 velocity evaluations, text CFG scale 2, one 1024^2 sample — judged the way
tests/test_gpu_drift_7b.py judges the bf16 product (tests/drift.py, oracle/gpu_leg.py), with the oracle legs run under
the fp8 contract (tests/fp8_oracle.py: gen MLP weights = the exact dequantised e4m3 weights, its two GEMM inputs
fake-quantised):

  product vs reference  <= 3 x the contract's own fa2-vs-sdpa noise floor at the same step
  product vs truth      <= 1.5 x reference vs truth (fp32 oracle under the same contract, first two steps)
  device memory         the flag saves at least 5.5 GB after load (the gen MLP: 11.4 GB in bf16, 5.7 GB in e4m3)

It also runs the bf16 product and the bf16 reference (fa2 leg, no contract) on the same weights and prints, without a
threshold, what FP8 costs: the fp8 product's distance from the bf16 reference at every reported step next to the bf16
product's."""
import gc
import time

import pytest
import torch

import drift
import fp8_oracle as fo

pytestmark = pytest.mark.gpu

FLOOR_FACTOR = 3.0        # as tests/test_gpu_drift_7b.py
TRUTH_FACTOR = 1.5
LAYERS, EVALS, TRUTH_STEPS = 28, 49, 2


def _free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()


@torch.no_grad()
def _run(fp8_gen_mlp: bool, legs, log):
    """Product (all steps) then the oracle legs on the product's exact weights. Returns x traces, memory after load."""
    from bagel_b200 import synthetic
    from oracle import gpu_leg, qwen2_mot as om

    _free()
    m0 = torch.cuda.memory_allocated()
    model = synthetic.build_random_bagel(device="cuda", seed=0, num_layers=LAYERS, fp8_gen_mlp=fp8_gen_mlp)
    torch.cuda.synchronize()
    mem = torch.cuda.memory_allocated() - m0
    gi, ct, ctx = synthetic.t2i_inputs(model, 1, (1024, 1024), prompt_tokens=64, seed=1, noise_seed=2)
    kw = dict(num_timesteps=EVALS + 1, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type="global",
              cfg_interval=[0.0, 1.0], cfg_text_scale=2.0)
    runner = model.make_flow_runner(
        past_key_values=ctx["main"], **gi, **kw,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
        cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=ct["cfg_key_values_lens"],
        cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
        cfg_text_past_key_values=ctx["cfg_text"])
    xs = {"product": []}
    for i in range(runner.num_steps):
        runner.step(i)
        xs["product"].append(runner.st["x"].clone())
    del runner, ctx
    lm = model.language_model.model
    lm._ws.clear()
    _free()
    # the legs own the weights from here on (one copy on the device, as in tests/drift.py)
    sd = fo.reference_state_dict(model) if fp8_gen_mlp else gpu_leg.export_reference_state_dict(model)
    for layer in lm.layers:
        for e in (layer.und, layer.gen):
            e.wgu = e.wd = None
            e.fp8 = None
    _free()
    fc = gpu_leg.flow_config(model)
    tok = synthetic.RandomIdTokenizer(1)
    prompt_ids = [tok.encode("64")]

    def leg(name, steps=None, weights=sd):
        tr = []
        t0 = time.perf_counter()
        gpu_leg.t2i_reference_run(weights, fc, prompt_ids, synthetic.NEW_TOKEN_IDS, gi, ct, "cuda", x_trace=tr,
                                  max_steps=steps, **kw)
        torch.cuda.synchronize()
        xs[name] = tr
        log(f"fp8={fp8_gen_mlp} {name}: {len(tr)} steps in {time.perf_counter() - t0:.1f} s")

    contract = fo.fp8_contract() if fp8_gen_mlp else _Null()
    with contract:
        if "fa2" in legs:
            with gpu_leg.fa2():
                leg("fa2")
        if "sdpa" in legs:
            leg("sdpa")
        if "truth" in legs:
            tf32 = torch.backends.cuda.matmul.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            try:
                with om.high_precision():
                    leg("truth", TRUTH_STEPS, om.LazyF32(sd))
            finally:
                torch.backends.cuda.matmul.allow_tf32 = tf32
    del model, sd
    _free()
    return xs, mem


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@pytest.fixture(scope="module")
def res():
    if torch.cuda.get_device_properties(0).total_memory < 64e9:
        pytest.skip("needs about 48 GB of device memory")
    log = lambda *a: print(*a, flush=True)   # noqa: E731
    bf16, mem_bf16 = _run(False, ("fa2",), log)
    fp8, mem_fp8 = _run(True, ("fa2", "sdpa", "truth"), log)
    return {"bf16": bf16, "fp8": fp8, "mem_bf16": mem_bf16, "mem_fp8": mem_fp8}


def test_fp8_product_tracks_the_fp8_reference_within_its_noise_floor(res):
    x = res["fp8"]
    assert len(x["product"]) == len(x["fa2"]) == len(x["sdpa"]) == EVALS
    for k in (0, 9, 24, 48):
        floor = drift._stat(x["sdpa"][k], x["fa2"][k])
        got = drift._stat(x["product"][k], x["fa2"][k])
        got2 = drift._stat(x["product"][k], x["sdpa"][k])
        assert torch.isfinite(x["product"][k]).all()
        rel = min(got["rel_l2"], got2["rel_l2"])
        mean = min(got["mean"], got2["mean"])
        print(f"step {k + 1}: product-vs-reference rel_l2 {rel:.3e} mean {mean:.3e}; floor rel_l2 "
              f"{floor['rel_l2']:.3e} mean {floor['mean']:.3e}; ratio {rel / floor['rel_l2']:.2f}", flush=True)
        assert rel <= FLOOR_FACTOR * floor["rel_l2"] + 1e-4, (k, got, got2, floor)
        assert mean <= FLOOR_FACTOR * floor["mean"] + 1e-4, (k, got, got2, floor)


def test_fp8_product_no_further_from_fp32_truth_than_the_reference(res):
    x = res["fp8"]
    assert len(x["truth"]) == TRUTH_STEPS
    for k in range(TRUTH_STEPS):
        p = drift._stat(x["product"][k], x["truth"][k])
        r = max(drift._stat(x["fa2"][k], x["truth"][k])["rel_l2"], drift._stat(x["sdpa"][k], x["truth"][k])["rel_l2"])
        print(f"step {k + 1}: product-vs-truth rel_l2 {p['rel_l2']:.3e}; reference-vs-truth {r:.3e}; "
              f"ratio {p['rel_l2'] / r:.2f}", flush=True)
        assert p["rel_l2"] <= TRUTH_FACTOR * r + 1e-4, (k, p, r)


def test_fp8_saves_device_memory(res):
    saved = res["mem_bf16"] - res["mem_fp8"]
    print(f"device memory after load: bf16 {res['mem_bf16'] / 1e9:.2f} GB, fp8 {res['mem_fp8'] / 1e9:.2f} GB, "
          f"saved {saved / 1e9:.2f} GB", flush=True)
    assert saved >= 5.5e9, saved


def test_report_what_fp8_costs(res):
    """No threshold: the fp8 product's distance from the bf16 reference next to the bf16 product's."""
    ref = res["bf16"]["fa2"]
    for k in (0, 9, 24, 48):
        a = drift._stat(res["fp8"]["product"][k], ref[k])
        b = drift._stat(res["bf16"]["product"][k], ref[k])
        print(f"step {k + 1}: vs bf16 reference rel_l2 / max: fp8 product {a['rel_l2']:.3e} / {a['max']:.3e}, "
              f"bf16 product {b['rel_l2']:.3e} / {b['max']:.3e}", flush=True)
        assert torch.isfinite(res["fp8"]["product"][k]).all()
