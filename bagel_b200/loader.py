"""HF-style checkpoint loader for BAGEL-7B-MoT (reference: app.py:39-133, eval/gen/gen_images_mp.py:137-175).

Directory layout expected (same files the reference reads): llm_config.json, vit_config.json, ema.safetensors,
ae.safetensors (+ tokenizer files, handled by the caller). The same post-load overrides as every shipped loader are
applied: qk_norm=True, tie_word_embeddings=False, layer_module="Qwen2MoTDecoderLayer", vit rope=False, one ViT layer
dropped (app.py:40-46). Weights are streamed tensor-by-tensor from safetensors into the kernels' fused bf16 layouts.
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Tuple

import torch

from .autoencoder import AutoEncoder, load_ae
from .bagel import Bagel
from .config import AutoEncoderParams, BagelConfig, Qwen2Config, SiglipVisionConfig
from .qwen2_navit import Qwen2ForCausalLM
from .siglip_navit import SiglipVisionModel


def load_configs(model_path: str, max_latent_size: int = 64) -> BagelConfig:
    llm = Qwen2Config.from_json_file(os.path.join(model_path, "llm_config.json"))
    llm.qk_norm = True
    llm.tie_word_embeddings = False
    llm.layer_module = "Qwen2MoTDecoderLayer"
    vit = SiglipVisionConfig.from_json_file(os.path.join(model_path, "vit_config.json"))
    vit.rope = False
    vit.num_hidden_layers = vit.num_hidden_layers - 1
    return BagelConfig(visual_gen=True, visual_und=True, llm_config=llm, vit_config=vit,
                       vae_config=AutoEncoderParams(), vit_max_num_patch_per_side=70,
                       connector_act="gelu_pytorch_tanh", latent_patch_size=2, max_latent_size=max_latent_size)


def read_safetensors(path: str) -> Dict[str, torch.Tensor]:
    from safetensors import safe_open
    out = {}
    with safe_open(path, framework="pt", device="cpu") as f:
        for k in f.keys():
            out[k] = f.get_tensor(k)
    return out


def load_bagel(model_path: str, device="cuda", max_latent_size: int = 64,
               state_dict: Optional[Dict[str, torch.Tensor]] = None, dtype_mode: str = "A",
               fp8_gen_mlp: bool = False) -> Tuple[Bagel, AutoEncoder, BagelConfig]:
    """Returns (model, vae_model, config) ready for InterleaveInferencer(model, vae_model, tokenizer, ...).
    dtype_mode "A": checkpoint cast to bf16 (app.py:111); "B": fp32 master weights + autocast numerics (eval drivers).
    fp8_gen_mlp=True: the generation expert's gate/up/down_proj are quantised to block-scaled FP8 at load (bagel_b200/fp8.py)."""
    cfg = load_configs(model_path, max_latent_size)
    lm = Qwen2ForCausalLM(cfg.llm_config, device=device, dtype_mode=dtype_mode, fp8_gen_mlp=fp8_gen_mlp)
    vit = SiglipVisionModel(cfg.vit_config, device=device)
    model = Bagel(lm, vit, cfg)
    sd = state_dict if state_dict is not None else read_safetensors(os.path.join(model_path, "ema.safetensors"))
    model.load_state_dict(sd)
    ae_path = os.path.join(model_path, "ae.safetensors")
    vae, _ = load_ae(ae_path if os.path.exists(ae_path) else None, device=device)
    return model, vae, cfg
