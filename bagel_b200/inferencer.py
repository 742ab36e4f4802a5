"""InterleaveInferencer — orchestration of interleaved text / image inputs into text or image outputs.

Same class, methods, keyword arguments and defaults as the reference's inferencer.py:23-313. Three contexts are
maintained (main / cfg_text / cfg_img), each a dict {kv_lens, ropes, past_key_values}; contexts are deep-copied at
the same points as the reference so the CFG branches see the same prefixes.

Scope (SURVEY.md §8): the text->image and text-decode paths run on the H100 kernels. Image *inputs* need the
SigLIP encoder / VAE encoder (`update_context_image`) and decoded image *outputs* need the VAE decoder
(`decode_image`); both delegate to the `vit_model` / `vae_model` objects handed to the constructor and raise if
those are absent.
"""
from __future__ import annotations

from copy import deepcopy
from typing import Any, Dict, List, Optional, Sequence, Union

import torch

from .qwen2_navit import NaiveCache

VLM_THINK_SYSTEM_PROMPT = '''You should first think about the reasoning process in the mind and then provide the user with the answer. 
The reasoning process is enclosed within <think> </think> tags, i.e. <think> reasoning process here </think> answer here'''

GEN_THINK_SYSTEM_PROMPT = '''You should first think about the planning process in the mind and then generate the image. 
The planning process is enclosed within <think> </think> tags, i.e. <think> planning process here </think> image here'''


def _is_image(x) -> bool:
    return hasattr(x, "size") and hasattr(x, "mode") and not isinstance(x, str)


class InterleaveInferencer:
    def __init__(self, model, vae_model, tokenizer, vae_transform, vit_transform, new_token_ids):
        self.model = model
        self.vae_model = vae_model
        self.tokenizer = tokenizer
        self.vae_transform = vae_transform
        self.vit_transform = vit_transform
        self.new_token_ids = new_token_ids

    # ---- contexts ---------------------------------------------------------------------------------
    def init_gen_context(self) -> Dict[str, Any]:
        return {"kv_lens": [0], "ropes": [0],
                "past_key_values": NaiveCache(self.model.config.llm_config.num_hidden_layers)}

    @torch.no_grad()
    def update_context_text(self, text: str, gen_context: Dict[str, Any]) -> Dict[str, Any]:
        gi, kv_lens, ropes = self.model.prepare_prompts(
            curr_kvlens=gen_context["kv_lens"], curr_rope=gen_context["ropes"], prompts=[text],
            tokenizer=self.tokenizer, new_token_ids=self.new_token_ids)
        cache = self.model.forward_cache_update_text(gen_context["past_key_values"], **gi)
        gen_context.update(kv_lens=kv_lens, ropes=ropes, past_key_values=cache)
        return gen_context

    @torch.no_grad()
    def update_context_image(self, image, gen_context, vae: bool = True, vit: bool = True):
        assert vae or vit
        cache, kv_lens, ropes = gen_context["past_key_values"], gen_context["kv_lens"], gen_context["ropes"]
        if vae:
            if not hasattr(self.model, "prepare_vae_images"):
                raise NotImplementedError("VAE image context needs the VAE encoder path (SURVEY.md §8 a14)")
            gi, kv_lens, ropes = self.model.prepare_vae_images(
                curr_kvlens=kv_lens, curr_rope=ropes, images=[image], transforms=self.vae_transform,
                new_token_ids=self.new_token_ids)
            cache = self.model.forward_cache_update_vae(self.vae_model, cache, **gi)
        if vit:
            if not hasattr(self.model, "prepare_vit_images"):
                raise NotImplementedError("ViT image context needs the SigLIP encoder path (SURVEY.md §8 a13)")
            gi, kv_lens, ropes = self.model.prepare_vit_images(
                curr_kvlens=kv_lens, curr_rope=ropes, images=[image], transforms=self.vit_transform,
                new_token_ids=self.new_token_ids)
            cache = self.model.forward_cache_update_vit(cache, **gi)
        gen_context.update(kv_lens=kv_lens, ropes=ropes, past_key_values=cache)
        return gen_context

    # ---- generation -------------------------------------------------------------------------------
    @torch.no_grad()
    def gen_latent(self, image_shape, gen_context, cfg_text_scale=4.0, cfg_img_scale=1.5, cfg_text_precontext=None,
                   cfg_img_precontext=None, cfg_interval=(0.4, 1.0), cfg_renorm_min=0.0, cfg_renorm_type="global",
                   num_timesteps=50, timestep_shift=3.0, enable_taylorseer=False):
        """The denoising part of gen_image: returns the [h*w, 64] fp32 latent of the generated image."""
        m = self.model
        gi = m.prepare_vae_latent(curr_kvlens=gen_context["kv_lens"], curr_rope=gen_context["ropes"],
                                  image_sizes=[image_shape], new_token_ids=self.new_token_ids)
        ct = m.prepare_vae_latent_cfg(curr_kvlens=cfg_text_precontext["kv_lens"],
                                      curr_rope=cfg_text_precontext["ropes"], image_sizes=[image_shape])
        ci = m.prepare_vae_latent_cfg(curr_kvlens=cfg_img_precontext["kv_lens"],
                                      curr_rope=cfg_img_precontext["ropes"], image_sizes=[image_shape])
        latents = m.generate_image(
            past_key_values=gen_context["past_key_values"],
            cfg_text_past_key_values=cfg_text_precontext["past_key_values"],
            cfg_img_past_key_values=cfg_img_precontext["past_key_values"],
            num_timesteps=num_timesteps, cfg_text_scale=cfg_text_scale, cfg_img_scale=cfg_img_scale,
            cfg_interval=cfg_interval, cfg_renorm_min=cfg_renorm_min, cfg_renorm_type=cfg_renorm_type,
            timestep_shift=timestep_shift, **gi,
            cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
            cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
            cfg_text_key_values_lens=ct["cfg_key_values_lens"],
            cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
            cfg_img_packed_position_ids=ci["cfg_packed_position_ids"],
            cfg_img_packed_query_indexes=ci["cfg_packed_query_indexes"],
            cfg_img_key_values_lens=ci["cfg_key_values_lens"],
            cfg_img_packed_key_value_indexes=ci["cfg_packed_key_value_indexes"],
            enable_taylorseer=enable_taylorseer)
        return latents[0]

    @torch.no_grad()
    def gen_image(self, image_shape, gen_context, **kwargs):
        return self.decode_image(self.gen_latent(image_shape, gen_context, **kwargs), image_shape)

    def decode_image(self, latent: torch.Tensor, image_shape):
        """Un-patchify [h*w, p*p*c] -> [1, c, h*p, w*p] and run the VAE decoder (reference :174-186)."""
        if self.vae_model is None:
            raise NotImplementedError("decode_image needs a VAE decoder (SURVEY.md §8 a14)")
        m = self.model
        H, W = image_shape
        h, w = H // m.latent_downsample, W // m.latent_downsample
        p, c = m.latent_patch_size, m.latent_channel
        z = latent.reshape(1, h, w, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(1, c, h * p, w * p)
        image = self.vae_model.decode(z)
        image = ((image * 0.5 + 0.5).clamp(0, 1)[0].permute(1, 2, 0) * 255).to(torch.uint8).cpu().numpy()
        from PIL import Image
        return Image.fromarray(image)

    @torch.no_grad()
    def gen_text(self, gen_context, max_length: int = 500, do_sample: bool = True, temperature: float = 1.0):
        gen_context = deepcopy(gen_context)
        gi = self.model.prepare_start_tokens(gen_context["kv_lens"], gen_context["ropes"], self.new_token_ids)
        toks = self.model.generate_text(past_key_values=gen_context["past_key_values"], max_length=max_length,
                                        do_sample=do_sample, temperature=temperature,
                                        end_token_id=self.new_token_ids["eos_token_id"], **gi)
        output = self.tokenizer.decode(toks[:, 0])
        return output.split("<|im_end|>")[0].split("<|im_start|>")[1]

    @torch.no_grad()
    def interleave_inference(self, input_lists: List[Union[str, Any]], think=False, understanding_output=False,
                             max_think_token_n=1000, do_sample=False, text_temperature=0.3, cfg_text_scale=3.0,
                             cfg_img_scale=1.5, cfg_interval=(0.4, 1.0), timestep_shift=3.0, num_timesteps=50,
                             cfg_renorm_min=0.0, cfg_renorm_type="global", image_shapes=(1024, 1024),
                             enable_taylorseer=False) -> List[Union[str, Any]]:
        outputs: List[Union[str, Any]] = []
        ctx = self.init_gen_context()
        ctx_cfg_text = deepcopy(ctx)
        ctx_cfg_img = deepcopy(ctx)
        if think:
            system_prompt = VLM_THINK_SYSTEM_PROMPT if understanding_output else GEN_THINK_SYSTEM_PROMPT
            ctx = self.update_context_text(system_prompt, ctx)
            ctx_cfg_img = self.update_context_text(system_prompt, ctx_cfg_img)
        for item in input_lists:
            if isinstance(item, str):
                ctx_cfg_text = deepcopy(ctx)          # text-dropped branch = everything before this text
                ctx = self.update_context_text(item, ctx)
                ctx_cfg_img = self.update_context_text(item, ctx_cfg_img)
            elif _is_image(item):
                from .transforms import pil_img2rgb
                item = self.vae_transform.resize_transform(pil_img2rgb(item))
                ctx = self.update_context_image(item, ctx, vae=not understanding_output)
                image_shapes = item.size[::-1]
                ctx_cfg_text = deepcopy(ctx)
            else:
                raise ValueError(f"Unsupported input type: {type(item)}")
        if understanding_output:
            outputs.append(self.gen_text(ctx, do_sample=do_sample, temperature=text_temperature,
                                         max_length=max_think_token_n))
            return outputs
        if think:
            thought = self.gen_text(ctx, do_sample=do_sample, temperature=text_temperature, max_length=max_think_token_n)
            ctx = self.update_context_text(thought, ctx)
            outputs.append(thought)
        outputs.append(self.gen_image(
            image_shapes, ctx, cfg_text_precontext=ctx_cfg_text, cfg_img_precontext=ctx_cfg_img,
            cfg_text_scale=cfg_text_scale, cfg_img_scale=cfg_img_scale, cfg_interval=cfg_interval,
            timestep_shift=timestep_shift, num_timesteps=num_timesteps, cfg_renorm_min=cfg_renorm_min,
            cfg_renorm_type=cfg_renorm_type, enable_taylorseer=enable_taylorseer))
        return outputs

    # per-request defaults of gen_image_batch: those of interleave_inference
    GEN_BATCH_DEFAULTS = dict(cfg_text_scale=3.0, cfg_img_scale=1.5, cfg_interval=(0.4, 1.0), cfg_renorm_min=0.0,
                              cfg_renorm_type="global", image_shapes=(1024, 1024))

    @torch.no_grad()
    def gen_image_batch(self, requests: Sequence[Dict[str, Any]], num_timesteps: int = 50,
                        timestep_shift: float = 3.0) -> List[Any]:
        """Text-to-image and edit requests in one packed denoising run; returns one PIL image per request.

        Each request is a dict: `text` (required), `image` (optional PIL image: an edit, whose output takes the resized
        input's shape), `image_shapes` (T2I only), `cfg_text_scale`, `cfg_img_scale`, `cfg_interval`, `cfg_renorm_min`,
        `cfg_renorm_type` (defaults of interleave_inference) and `seed`. Request i with seed s gets what
        `torch.manual_seed(s); inferencer(image=..., text=..., **its settings)` gives it alone (think=False): its VAE-encode
        noise comes from the CUDA generator seeded with s in its own latent shape, its init noise from a CPU generator
        seeded with s. `seed=None` draws one from torch.default_generator.

        The contexts are those interleave_inference builds per request (T2I: main [text], cfg_text empty, cfg_img
        [text]; edit: main [VAE + ViT image, text], cfg_text [VAE + ViT image], cfg_img [text]), built for all requests
        at once: one VAE image round (each image encoded on its own, so that its latents do not depend on the padding
        a batch would add), one SigLIP call and one ViT round, one text prefill for the main contexts and one for the
        cfg_img contexts; cfg_text is a copy of the main caches after the image rounds. One Bagel.generate_image_batch
        denoises every request; the VAE decodes each image on its own."""
        from .transforms import pil_img2rgb
        m = self.model
        R = len(requests)
        if R == 0:
            return []
        unknown = [k for r in requests for k in r if k not in ("text", "image", "seed", *self.GEN_BATCH_DEFAULTS)]
        if unknown:
            raise ValueError(f"gen_image_batch: unknown request keys {sorted(set(unknown))}")
        reqs = [{**self.GEN_BATCH_DEFAULTS, **r} for r in requests]
        seeds = [int(r["seed"]) if r.get("seed") is not None else int(torch.randint(0, 2 ** 32, (1,), dtype=torch.int64))
                 for r in reqs]
        images = [None if r.get("image") is None else self.vae_transform.resize_transform(pil_img2rgb(r["image"]))
                  for r in reqs]
        shapes = [tuple(im.size[::-1]) if im is not None else tuple(r["image_shapes"]) for im, r in zip(images, reqs)]
        L = m.config.llm_config.num_hidden_layers
        kv, rope = [0] * R, [0] * R
        cache = NaiveCache(L)
        if any(im is not None for im in images):
            if self.vae_model is None:
                raise NotImplementedError("edit requests need the VAE encoder")
            gi, kv, rope, tensors = m.prepare_vae_image_round(kv, rope, images, self.vae_transform, self.new_token_ids,
                                                              return_tensors=True)
            gi.pop("padded_images")
            lat_shapes = gi.pop("patchified_vae_latent_shapes")
            present = [q for q in range(R) if images[q] is not None]
            latents = [self._encode_image(t, seeds[q]) for t, q in zip(tensors, present)]
            cache = m._prefill_vae_latents(cache, m._patchify_latents(latents, lat_shapes), **gi)
            gi, kv, rope = m.prepare_vit_image_round(kv, rope, images, self.vit_transform, self.new_token_ids)
            cache = m.forward_cache_update_vit(cache, **gi)
        text_ctx = (deepcopy(cache), kv, rope)       # text-dropped branch = everything before the text
        texts = [r["text"] for r in reqs]
        gi, kv, rope = m.prepare_prompts(kv, rope, texts, self.tokenizer, self.new_token_ids)
        cache = m.forward_cache_update_text(cache, **gi)
        gi, kv_i, rope_i = m.prepare_prompts([0] * R, [0] * R, texts, self.tokenizer, self.new_token_ids)
        cache_img = m.forward_cache_update_text(NaiveCache(L), **gi)
        gi = m.prepare_vae_latent(kv, rope, shapes, self.new_token_ids,
                                  generators=[torch.Generator().manual_seed(s) for s in seeds])
        ct = m.prepare_vae_latent_cfg(text_ctx[1], text_ctx[2], shapes)
        ci = m.prepare_vae_latent_cfg(kv_i, rope_i, shapes)
        latents = m.generate_image_batch(
            past_key_values=cache, cfg_text_past_key_values=text_ctx[0], cfg_img_past_key_values=cache_img,
            num_timesteps=num_timesteps, timestep_shift=timestep_shift,
            **{k: [r[k] for r in reqs] for k in ("cfg_text_scale", "cfg_img_scale", "cfg_interval", "cfg_renorm_min",
                                                 "cfg_renorm_type")},
            **gi,
            cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
            cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
            cfg_text_key_values_lens=ct["cfg_key_values_lens"],
            cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
            cfg_img_packed_position_ids=ci["cfg_packed_position_ids"],
            cfg_img_packed_query_indexes=ci["cfg_packed_query_indexes"],
            cfg_img_key_values_lens=ci["cfg_key_values_lens"],
            cfg_img_packed_key_value_indexes=ci["cfg_packed_key_value_indexes"])
        return [self.decode_image(lat, hw) for lat, hw in zip(latents, shapes)]

    def _encode_image(self, image: torch.Tensor, seed: int) -> torch.Tensor:
        """VAE-encode one transformed image [C, H, W] on its own, with its DiagonalGaussian noise drawn as a single
        request seeded with `seed` draws it: from the default CUDA generator of the VAE's device, seeded with `seed`,
        in the image's own latent shape. The caller's CUDA RNG state is restored. Returns its latent [z, h, w]."""
        dev = torch.device(getattr(self.vae_model, "device", self.model.device))
        with torch.random.fork_rng(devices=[dev]):
            with torch.cuda.device(dev):
                torch.cuda.manual_seed(seed)
            return self.vae_model.encode(image[None].to(torch.float32))[0]    # the fp32 canvas prepare_vae_images builds

    def __call__(self, image=None, text: Optional[str] = None, **kargs) -> Dict[str, Any]:
        result = {"image": None, "text": None}
        if image is None and text is None:
            print("Please provide at least one input: either an image or text.")
            return result
        inputs = ([image] if image is not None else []) + ([text] if text is not None else [])
        for o in self.interleave_inference(inputs, **kargs):
            result["text" if isinstance(o, str) else "image"] = o
        return result
