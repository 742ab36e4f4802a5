"""Synthetic (random-init) BAGEL-7B-MoT for benchmarks and smoke tests: there is no network for checkpoints, so
weights are drawn on the device with the reference's init recipe (normal, std = initializer_range;
modeling/qwen2/modeling_qwen2.py:563-572), llm2vae given non-zero weights (the reference zero-inits it,
bagel.py:96-99, which would make the velocity constant — SURVEY.md A.10), prompts are random token ids.
Shapes are the public BAGEL-7B-MoT llm_config.json (Qwen2.5-7B): SURVEY.md §8.
"""
from __future__ import annotations

from typing import Dict, List

import torch

from .bagel import Bagel
from .config import AutoEncoderParams, BagelConfig, Qwen2Config
from .fp8 import GenMlpFp8
from .qwen2_navit import Qwen2ForCausalLM, _Embedding, _ExpertWeights, _Linear

BF16 = torch.bfloat16

BAGEL_7B_LLM = dict(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                    num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=32768,
                    rms_norm_eps=1e-6, rope_theta=1000000.0, qk_norm=True, tie_word_embeddings=False,
                    layer_module="Qwen2MoTDecoderLayer")

NEW_TOKEN_IDS = dict(bos_token_id=151644, eos_token_id=151645, start_of_image=151652, end_of_image=151653)


class RandomIdTokenizer:
    """encode("<n>") -> n deterministic pseudo-random ids in [0, 151643) (no vocab files offline)."""

    def __init__(self, seed: int = 1, vocab: int = 151643):
        self.gen = torch.Generator().manual_seed(seed)
        self.vocab = vocab

    def encode(self, prompt: str) -> List[int]:
        n = int(prompt)
        return torch.randint(0, self.vocab, (n,), generator=self.gen).tolist()


def _randn(shape, std, gen, device):
    return (torch.randn(shape, generator=gen, device=device, dtype=torch.float32) * std).to(BF16)


def build_random_bagel(llm_kwargs: Dict = None, device="cuda", seed: int = 0, max_latent_size: int = 64,
                       num_layers: int = None, fp8_gen_mlp: bool = False) -> Bagel:
    """Random-init MoT model directly in the kernels' fused layouts (no intermediate fp32 state dict: the 7B
    model is 28 GB in bf16). fp8_gen_mlp=True draws the same weights and quantises the gen expert's MLP layer by
    layer (bagel_b200/fp8.py), so only its e4m3 copy stays on the device."""
    kw = dict(BAGEL_7B_LLM if llm_kwargs is None else llm_kwargs)
    if num_layers is not None:
        kw["num_hidden_layers"] = num_layers
    llm = Qwen2Config(**kw)
    bcfg = BagelConfig(visual_gen=True, visual_und=False, llm_config=llm, vit_config=None,
                       vae_config=AutoEncoderParams(), latent_patch_size=2, max_latent_size=max_latent_size)
    lm = Qwen2ForCausalLM(llm, device=device, fp8_gen_mlp=fp8_gen_mlp)
    dev = lm.device
    g = torch.Generator(device=dev).manual_seed(seed)
    std = llm.initializer_range
    H, I, d = llm.hidden_size, llm.intermediate_size, llm.head_dim
    Hq, Hk = llm.num_attention_heads, llm.num_key_value_heads
    lm.model.embed_tokens = _Embedding(_randn((llm.vocab_size, H), std, g, dev))
    for layer in lm.model.layers:
        for tgt in ("und", "gen"):
            e = _ExpertWeights()
            e.wqkv = _randn(((Hq + 2 * Hk) * d, H), std, g, dev)
            e.bqkv = _randn(((Hq + 2 * Hk) * d,), std, g, dev)
            e.wo = _randn((H, Hq * d), std, g, dev)
            e.wgu = _randn((2 * I, H), std, g, dev)       # already in the interleaved gate|up layout
            e.wd = _randn((H, I), std, g, dev)
            e.ln_in = (1.0 + _randn((H,), 0.02, g, dev).float()).to(BF16)
            e.ln_post = (1.0 + _randn((H,), 0.02, g, dev).float()).to(BF16)
            e.q_norm = (1.0 + _randn((d,), 0.02, g, dev).float()).to(BF16)
            e.k_norm = (1.0 + _randn((d,), 0.02, g, dev).float()).to(BF16)
            e.fp8 = None
            if tgt == "gen" and fp8_gen_mlp:
                e.fp8 = GenMlpFp8.from_interleaved_bf16(e.wgu, e.wd)
                e.wgu = e.wd = None
            setattr(layer, tgt, e)
    lm.model.norm = (1.0 + _randn((H,), 0.02, g, dev).float()).to(BF16)
    lm.model.norm_moe_gen = (1.0 + _randn((H,), 0.02, g, dev).float()).to(BF16)
    lm.lm_head = _Linear(_randn((llm.vocab_size, H), std, g, dev))
    model = Bagel(lm, None, bcfg)
    sd = {
        "time_embedder.mlp.0.weight": _randn((H, 256), std, g, dev), "time_embedder.mlp.0.bias": _randn((H,), std, g, dev),
        "time_embedder.mlp.2.weight": _randn((H, H), std, g, dev), "time_embedder.mlp.2.bias": _randn((H,), std, g, dev),
        "vae2llm.weight": _randn((H, model.patch_latent_dim), std, g, dev), "vae2llm.bias": _randn((H,), std, g, dev),
        "llm2vae.weight": _randn((model.patch_latent_dim, H), std, g, dev),
        "llm2vae.bias": _randn((model.patch_latent_dim,), std, g, dev),
    }
    model.time_embedder.load(sd, "time_embedder.", dev)
    model.vae2llm.load(sd, "vae2llm.", dev)
    model.llm2vae.load(sd, "llm2vae.", dev)
    return model


def t2i_inputs(model: Bagel, batch: int, image_size=(1024, 1024), prompt_tokens: int = 64, seed: int = 1,
               noise_seed: int = 2):
    """BASELINE configs[1] inputs (SURVEY.md §8d cfg 2): per sample 64 random ids + bos/eos as context, prefilled
    through forward_cache_update_text; returns (gen_input, cfg_text_input, contexts)."""
    from .qwen2_navit import NaiveCache
    L = model.config.llm_config.num_hidden_layers
    tok = RandomIdTokenizer(seed)
    kv0, rp0 = [0] * batch, [0] * batch
    gi, kv, rp = model.prepare_prompts(kv0, rp0, [str(prompt_tokens)] * batch, tok, NEW_TOKEN_IDS)
    cache = model.forward_cache_update_text(NaiveCache(L), **gi)
    torch.manual_seed(noise_seed)
    gen_input = model.prepare_vae_latent(kv, rp, [image_size] * batch, NEW_TOKEN_IDS)
    cfg_text = model.prepare_vae_latent_cfg(kv0, rp0, [image_size] * batch)
    return gen_input, cfg_text, dict(main=cache, cfg_text=NaiveCache(L), kv_lens=kv, ropes=rp)


# --------------------------------------------------------------------------------------------------------------
# random SigLIP-so400m tower + connector, and random FLUX VAE (BASELINE configs[2] and [3] need them; no checkpoints
# offline). Weights are drawn on the device with the reference's key names and go through the normal loaders.
# --------------------------------------------------------------------------------------------------------------
SIGLIP_SO400M = dict(hidden_size=1152, intermediate_size=4304, num_hidden_layers=26, num_attention_heads=16,
                     num_channels=3, image_size=980, patch_size=14)


def random_vit_state_dict(vcfg, llm_hidden: int, max_side: int, device, seed: int = 5) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device=device).manual_seed(seed)
    H, I = vcfg.hidden_size, vcfg.intermediate_size
    pd = vcfg.num_channels * vcfg.patch_size ** 2
    p = "vit_model.vision_model."
    sd = {p + "embeddings.patch_embedding.weight": _randn((H, pd), 0.05, g, device),
          p + "embeddings.patch_embedding.bias": _randn((H,), 0.1, g, device),
          p + "embeddings.position_embedding.weight": _randn((max_side * max_side, H), 0.5, g, device),
          p + "post_layernorm.weight": (1.0 + _randn((H,), 0.1, g, device).float()).to(BF16),
          p + "post_layernorm.bias": _randn((H,), 0.1, g, device)}
    for li in range(vcfg.num_hidden_layers):
        q = p + f"encoder.layers.{li}."
        for n in ("q", "k", "v", "out"):
            sd[q + f"self_attn.{n}_proj.weight"] = _randn((H, H), 0.03, g, device)
            sd[q + f"self_attn.{n}_proj.bias"] = _randn((H,), 0.1, g, device)
        for n in ("layer_norm1", "layer_norm2"):
            sd[q + n + ".weight"] = (1.0 + _randn((H,), 0.1, g, device).float()).to(BF16)
            sd[q + n + ".bias"] = _randn((H,), 0.1, g, device)
        sd[q + "mlp.fc1.weight"], sd[q + "mlp.fc1.bias"] = _randn((I, H), 0.03, g, device), _randn((I,), 0.1, g, device)
        sd[q + "mlp.fc2.weight"], sd[q + "mlp.fc2.bias"] = _randn((H, I), 0.03, g, device), _randn((H,), 0.1, g, device)
    sd["connector.fc1.weight"], sd["connector.fc1.bias"] = _randn((llm_hidden, H), 0.03, g, device), _randn((llm_hidden,), 0.1, g, device)
    sd["connector.fc2.weight"] = _randn((llm_hidden, llm_hidden), 0.02, g, device)
    sd["connector.fc2.bias"] = _randn((llm_hidden,), 0.1, g, device)
    return sd


def attach_random_vit(model: Bagel, seed: int = 5, max_side: int = 70, vit_kwargs: Dict = None) -> Bagel:
    """Give a visual_gen-only synthetic model the understanding branch (SigLIP tower + connector + ViT position table)."""
    from .config import SiglipVisionConfig
    from .modeling_utils import MLPconnector, PositionEmbedding
    from .siglip_navit import SiglipVisionModel
    dev = model.device
    vcfg = SiglipVisionConfig(**dict(SIGLIP_SO400M if vit_kwargs is None else vit_kwargs), rope=False)
    sd = random_vit_state_dict(vcfg, model.hidden_size, max_side, dev, seed)
    vit = SiglipVisionModel(vcfg, dev)
    vit.load_state_dict({k[len("vit_model."):]: v for k, v in sd.items() if k.startswith("vit_model.")})
    model.vit_model, model.config.vit_config, model.config.visual_und = vit, vcfg, True
    model.vit_patch_size, model.vit_max_num_patch_per_side = vcfg.patch_size, max_side
    model.vit_hidden_size = vcfg.hidden_size
    model.connector = MLPconnector(vcfg.hidden_size, model.hidden_size)
    model.connector.load(sd, "connector.", dev)
    model.vit_pos_embed = PositionEmbedding(max_side, model.hidden_size, dev)
    return model


def random_vae_state_dict(params: AutoEncoderParams, device, seed: int = 7) -> Dict[str, torch.Tensor]:
    """Random FLUX-VAE weights, reference key names (modeling/autoencoder.py module tree), fp32 like ae.safetensors."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def rn(shape, std):
        return torch.randn(shape, generator=g, device=device, dtype=torch.float32) * std

    def conv(name, co, ci, k):
        sd[name + ".weight"], sd[name + ".bias"] = rn((co, ci, k, k), (1.0 / (ci * k * k)) ** 0.5), rn((co,), 0.05)

    def norm(name, c):
        sd[name + ".weight"], sd[name + ".bias"] = 1.0 + rn((c,), 0.1), rn((c,), 0.1)

    def res(name, ci, co):
        norm(name + ".norm1", ci); conv(name + ".conv1", co, ci, 3)
        norm(name + ".norm2", co); conv(name + ".conv2", co, co, 3)
        if ci != co:
            conv(name + ".nin_shortcut", co, ci, 1)

    def attn(name, c):
        norm(name + ".norm", c)
        for n in ("q", "k", "v", "proj_out"):
            conv(f"{name}.{n}", c, c, 1)

    ch, mult, nrb, z = params.ch, list(params.ch_mult), params.num_res_blocks, params.z_channels
    n = len(mult)
    in_mult = [1] + mult
    conv("encoder.conv_in", ch, params.in_channels, 3)
    bi = ch
    for lvl in range(n):
        bi, bo = ch * in_mult[lvl], ch * mult[lvl]
        for i in range(nrb):
            res(f"encoder.down.{lvl}.block.{i}", bi, bo)
            bi = bo
        if lvl != n - 1:
            conv(f"encoder.down.{lvl}.downsample.conv", bi, bi, 3)
    res("encoder.mid.block_1", bi, bi); attn("encoder.mid.attn_1", bi); res("encoder.mid.block_2", bi, bi)
    norm("encoder.norm_out", bi); conv("encoder.conv_out", 2 * z, bi, 3)
    bi = ch * mult[-1]
    conv("decoder.conv_in", bi, z, 3)
    res("decoder.mid.block_1", bi, bi); attn("decoder.mid.attn_1", bi); res("decoder.mid.block_2", bi, bi)
    for lvl in reversed(range(n)):
        bo = ch * mult[lvl]
        for i in range(nrb + 1):
            res(f"decoder.up.{lvl}.block.{i}", bi, bo)
            bi = bo
        if lvl != 0:
            conv(f"decoder.up.{lvl}.upsample.conv", bi, bi, 3)
    norm("decoder.norm_out", bi); conv("decoder.conv_out", params.out_ch, bi, 3)
    return sd


def build_random_vae(device="cuda", seed: int = 7):
    from .autoencoder import load_ae
    vae, params = load_ae(None, device=device)
    vae.load_state_dict(random_vae_state_dict(params, device, seed))
    vae.sample = False
    return vae
