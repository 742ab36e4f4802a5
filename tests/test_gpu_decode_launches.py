"""-m gpu: the C-ABI entry points a text-decode step and a short causal prefill issue, in order. Which QKV path runs
depends on head_dim and, for decode, on the batch: the weight-streaming skinny GEMM + q/k-norm/RoPE kernel up to 64
samples, the fused QKV epilogue above that; a prefill at head_dim 128 always takes the fused epilogue."""
import pytest

import helpers
from oracle import fixtures

pytestmark = pytest.mark.gpu

CFG = fixtures.TINY128_LM     # head_dim 128, like BAGEL-7B


class _Recorder:
    """Stands in for the loaded library: records the name of every bagel_* entry point called, then forwards it."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("bagel_"):
            return fn

        def call(*args):
            self.calls.append(name)
            return fn(*args)
        return call


def _record(monkeypatch) -> _Recorder:
    from bagel_b200 import _cabi
    rec = _Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    return rec


def _layer(qkv):
    return ["bagel_rmsnorm_bf16", *qkv, "bagel_attn_varlen_fwd", "bagel_gemm_bf16",
            "bagel_rmsnorm_bf16", "bagel_gemm_bf16", "bagel_gemm_bf16"]


FUSED = ["bagel_gemm_qkv_norm_rope"]
TWO_KERNEL = ["bagel_gemm_bf16", "bagel_qk_norm_rope"]


@pytest.mark.parametrize("batch,qkv", [(2, TWO_KERNEL), (66, FUSED)])
def test_decode_step_launch_sequence(monkeypatch, batch, qkv):
    from bagel_b200.qwen2_navit import NaiveCache
    model = helpers.build_product_bagel(CFG, "cuda")
    model.use_cuda_graph = False
    L = CFG.num_hidden_layers
    prompts = (helpers.PROMPTS * batch)[:batch]
    gi, kv, rp = model.prepare_prompts([0] * batch, [0] * batch, prompts, helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS)
    cache = model.forward_cache_update_text(NaiveCache(L), **gi)
    gs = model.prepare_start_tokens(kv, rp, helpers.NEW_TOKEN_IDS)
    rec = _record(monkeypatch)
    toks = model.generate_text(past_key_values=cache, max_length=2, do_sample=False, **gs)
    assert tuple(toks.shape) == (2, batch)
    step = (["bagel_copy_rows_bf16", "bagel_rope_table", "bagel_decode_prepare"]      # embedding gather, RoPE, slots
            + _layer(qkv) * L
            + ["bagel_rmsnorm_bf16", "bagel_gemm_bf16"]                                   # final norm, lm_head
            + ["bagel_decode_advance", "bagel_argmax_rows_bf16"])
    context = ["bagel_copy_rows_bf16"] * (2 * L)                                          # K and V rows, once per call
    assert rec.calls == context + step * 2


def test_short_causal_prefill_uses_fused_qkv(monkeypatch):
    from bagel_b200.qwen2_navit import NaiveCache
    model = helpers.build_product_bagel(CFG, "cuda")
    gi, kv, _ = model.prepare_prompts([0, 0], [0, 0], helpers.PROMPTS, helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS)
    assert sum(kv) < 64
    rec = _record(monkeypatch)
    model.forward_cache_update_text(NaiveCache(CFG.num_hidden_layers), **gi)
    assert rec.calls == (["bagel_copy_rows_bf16", "bagel_rope_table"]                   # embedding gather, RoPE table
                         + _layer(FUSED) * CFG.num_hidden_layers + ["bagel_rmsnorm_bf16"])
