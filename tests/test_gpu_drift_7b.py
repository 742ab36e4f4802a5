"""-m gpu: parity AT THE BENCHMARKED CONFIGURATION — BAGEL-7B-MoT dimensions, all 28 layers, all 49 velocity
evaluations, text CFG scale 2, one 1024^2 sample — product vs the reference-equivalent GPU legs (tests/drift.py,
oracle/gpu_leg.py). The tolerance is derived from the MEASURED noise floor of the reference itself (oracle+flash-attn
vs oracle+fp32-SDPA on identical inputs: two valid executions of the reference that differ only in the attention
kernel's internal rounding), not chosen by the builder; tools/gpu_drift_7b.py prints the per-step table of the
same run including the fp32 truth for all 49 steps. north_star's "1e-3 rtol" is compared against that floor in DESIGN.md §4."""
import pytest
import torch

import drift

pytestmark = pytest.mark.gpu

# product-vs-reference distance allowed, in units of the reference's own fa2-vs-sdpa distance at the same step. The
# product differs from either leg in MORE places than the legs differ from each other (GEMM accumulation order and
# fused-epilogue rounding on top of the attention kernel), so a factor somewhat above 1 is the expectation for "just
# another bf16 execution of the same network".
FLOOR_FACTOR = 3.0


@pytest.fixture(scope="module")
def res():
    if torch.cuda.get_device_properties(0).total_memory < 64e9:
        # peak 44 GB allocated (48 GB reserved) on an H100 80GB: 7B weights + the reference layout of gate/up + activations
        pytest.skip("needs about 48 GB of device memory")
    return drift.run(layers=28, evals=49, truth_steps=2, batch=1, image_size=1024, log=lambda *a: None)


def test_product_tracks_reference_within_its_noise_floor(res):
    x = res["x"]
    assert len(x["product"]) == len(x["fa2"]) == len(x["sdpa"]) == 49
    for k in (0, 9, 24, 48):
        floor = drift._stat(x["sdpa"][k], x["fa2"][k])
        got = drift._stat(x["product"][k], x["fa2"][k])
        got2 = drift._stat(x["product"][k], x["sdpa"][k])
        assert torch.isfinite(x["product"][k]).all()
        # against whichever execution of the reference is closer (both are "the reference")
        rel = min(got["rel_l2"], got2["rel_l2"])
        mean = min(got["mean"], got2["mean"])
        assert rel <= FLOOR_FACTOR * floor["rel_l2"] + 1e-4, (k, got, got2, floor)
        assert mean <= FLOOR_FACTOR * floor["mean"] + 1e-4, (k, got, got2, floor)


def test_product_no_further_from_fp32_truth_than_the_reference(res):
    x = res["x"]
    for k in range(len(x["truth"])):
        p = drift._stat(x["product"][k], x["truth"][k])
        r = max(drift._stat(x["fa2"][k], x["truth"][k])["rel_l2"], drift._stat(x["sdpa"][k], x["truth"][k])["rel_l2"])
        assert p["rel_l2"] <= 1.5 * r + 1e-4, (k, p, r)
