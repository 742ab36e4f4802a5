"""-m gpu: the extra measurement blocks of bench.py (tools/bench_blocks.py) run end to end on a SMALL random model, so a
broken block shows up in the GPU test tier and not only as an `error` field in the round-end bench line."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

SMALL_LLM = dict(vocab_size=152064, hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                 num_key_value_heads=2, max_position_embeddings=32768, rms_norm_eps=1e-6, rope_theta=1000000.0, qk_norm=True,
                 tie_word_embeddings=False, layer_module="Qwen2MoTDecoderLayer")
SMALL_VIT = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, num_channels=3,
                 image_size=980, patch_size=14)


@pytest.fixture(scope="module")
def model():
    from bagel_b200 import synthetic
    return synthetic.build_random_bagel(llm_kwargs=SMALL_LLM, device="cuda", seed=0)


def test_library_baseline_and_parity_block(model):
    from bagel_b200 import synthetic
    from tools import bench_blocks as bb
    B = 2
    gi, ct, ctx = synthetic.t2i_inputs(model, B, (256, 256), seed=1, noise_seed=2)
    kw = dict(num_timesteps=50, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type="global", cfg_interval=[0.0, 1.0],
              cfg_text_scale=2.0, cfg_img_scale=1.0, cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
              cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"], cfg_text_key_values_lens=ct["cfg_key_values_lens"],
              cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"], cfg_text_past_key_values=ctx["cfg_text"])
    tok = synthetic.RandomIdTokenizer(1)
    r = bb.library_baseline_and_parity(model, gi, ct, ctx["main"], kw, [tok.encode("64") for _ in range(B)], torch.device("cuda"),
                                       1.0, B)
    par = r["parity"]
    assert r["gpu_library_baseline"]["ms_per_step"] > 0
    assert par["noise_floor"]["rel_l2"] > 0 and par["ratio_to_noise_floor"] < 3.0, par


def test_attn_block_runs():
    from tools import bench_blocks as bb
    r = bb.attn_block({"bf16_tflops": 989.0, "hbm_gbs": 3350.0}, torch.device("cuda"), iters=2)
    assert len(r["shapes"]) == 20 and all(s["tflops"] > 50 for s in r["shapes"])
    assert all(s.get("speedup_vs_fa2", 2.0) > 1.0 for s in r["shapes"])


def test_und_prefill_decode_and_edit_blocks(model):
    from bagel_b200 import synthetic
    from tools import bench_blocks as bb
    synthetic.attach_random_vit(model, seed=5, vit_kwargs=SMALL_VIT)
    r = bb.und_prefill_and_decode_block(model, torch.device("cuda"), batch=2, text_tokens=32)
    assert r["und_prefill"]["tokens"] == 2 * (729 + 2 + 34) and r["und_prefill"]["tokens_per_s"] > 0
    assert "ms_per_step" in r["decode"] and r["decode"]["hbm_bytes_per_step"] > 0   # (the steady-state estimate of a TINY model is timing noise)
    vae = synthetic.build_random_vae("cuda")
    e = bb.edit_block(model, vae, torch.device("cuda"), samples=1)
    assert e["s_per_image"] > 0
