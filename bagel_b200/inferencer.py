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

from .bagel import _penalties, _sampling_filters
from .qwen2_navit import NaiveCache, gather_requests

VLM_THINK_SYSTEM_PROMPT = '''You should first think about the reasoning process in the mind and then provide the user with the answer. 
The reasoning process is enclosed within <think> </think> tags, i.e. <think> reasoning process here </think> answer here'''

GEN_THINK_SYSTEM_PROMPT = '''You should first think about the planning process in the mind and then generate the image. 
The planning process is enclosed within <think> </think> tags, i.e. <think> planning process here </think> image here'''


def _is_image(x) -> bool:
    return hasattr(x, "size") and hasattr(x, "mode") and not isinstance(x, str)


def call_batch_schedule(requests: Sequence[Dict[str, Any]]) -> Dict[str, List[int]]:
    """Which requests of InterleaveInferencer.call_batch take part in each of its rounds, in interleave_inference's
    order (a pure function of the requests' inputs and flags). A request with neither text nor image takes part in
    none. Understanding requests (understanding_output=True) build only the main context, take the ViT image round
    only, and decode their answer; every other request generates an image, and its cfg_img context gets the system
    prompt and the prompt."""
    def has(r, k):
        return r.get(k) is not None

    live = [q for q, r in enumerate(requests) if has(r, "text") or has(r, "image")]
    gen = [q for q in live if not requests[q].get("understanding_output", False)]
    think = [q for q in live if requests[q].get("think", False)]
    return {
        "system": think,                                            # 1. think system prompt (main)
        "system_cfg_img": [q for q in think if q in gen],           #    and cfg_img
        "vae": [q for q in gen if has(requests[q], "image")],       # 2. VAE image round
        "vit": [q for q in live if has(requests[q], "image")],      # 3. ViT image round
        "prompt": [q for q in live if has(requests[q], "text")],    # 5. prompt (main)
        "prompt_cfg_img": [q for q in gen if has(requests[q], "text")],   # and cfg_img
        "decode": [q for q in live if q not in gen or q in think],  # 6. understanding answers and thoughts
        "thought": [q for q in gen if q in think],                  # 7. thought into main
        "generate": gen,                                            # 8. denoising + VAE decode
    }


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
        seeds = self._request_seeds(reqs)
        images = [None if r.get("image") is None else self.vae_transform.resize_transform(pil_img2rgb(r["image"]))
                  for r in reqs]
        shapes = [tuple(im.size[::-1]) if im is not None else tuple(r["image_shapes"]) for im, r in zip(images, reqs)]
        L = m.config.llm_config.num_hidden_layers
        kv, rope = [0] * R, [0] * R
        cache = NaiveCache(L)
        if any(im is not None for im in images):
            cache, kv, rope = self._vae_image_round(cache, kv, rope, images, seeds)
            gi, kv, rope = m.prepare_vit_image_round(kv, rope, images, self.vit_transform, self.new_token_ids)
            cache = m.forward_cache_update_vit(cache, **gi)
        text_ctx = (deepcopy(cache), kv, rope)       # text-dropped branch = everything before the text
        texts = [r["text"] for r in reqs]
        gi, kv, rope = m.prepare_prompts(kv, rope, texts, self.tokenizer, self.new_token_ids)
        cache = m.forward_cache_update_text(cache, **gi)
        gi, kv_i, rope_i = m.prepare_prompts([0] * R, [0] * R, texts, self.tokenizer, self.new_token_ids)
        cache_img = m.forward_cache_update_text(NaiveCache(L), **gi)
        latents = self._denoise_batch(reqs, shapes, seeds, (cache, kv, rope), text_ctx, (cache_img, kv_i, rope_i),
                                      num_timesteps, timestep_shift)
        return [self.decode_image(lat, hw) for lat, hw in zip(latents, shapes)]

    @staticmethod
    def _request_seeds(reqs) -> List[int]:
        """Each request's seed; `seed=None` draws one from torch.default_generator."""
        return [int(r["seed"]) if r.get("seed") is not None else int(torch.randint(0, 2 ** 32, (1,), dtype=torch.int64))
                for r in reqs]

    def _vae_image_round(self, cache, kv, rope, images, seeds):
        """One VAE image round: images[q] is request q's resized input image or None. Each image is encoded on its own
        with request q's encode noise (_encode_image), then one LM prefill holds every present image."""
        if self.vae_model is None:
            raise NotImplementedError("edit requests need the VAE encoder")
        m = self.model
        gi, kv, rope, tensors = m.prepare_vae_image_round(kv, rope, images, self.vae_transform, self.new_token_ids,
                                                          return_tensors=True)
        gi.pop("padded_images")
        lat_shapes = gi.pop("patchified_vae_latent_shapes")
        present = [q for q in range(len(images)) if images[q] is not None]
        latents = [self._encode_image(t, seeds[q]) for t, q in zip(tensors, present)]
        return m._prefill_vae_latents(cache, m._patchify_latents(latents, lat_shapes), **gi), kv, rope

    def _denoise_batch(self, reqs, shapes, seeds, main, text_ctx, img_ctx, num_timesteps, timestep_shift):
        """One Bagel.generate_image_batch over requests `reqs` (their CFG settings), each context a (packed cache,
        kv lens, rope positions) triple over exactly these requests; init noise from a CPU generator per seed."""
        m = self.model
        cache, kv, rope = main
        gi = m.prepare_vae_latent(kv, rope, shapes, self.new_token_ids,
                                  generators=[torch.Generator().manual_seed(s) for s in seeds])
        ct = m.prepare_vae_latent_cfg(text_ctx[1], text_ctx[2], shapes)
        ci = m.prepare_vae_latent_cfg(img_ctx[1], img_ctx[2], shapes)
        return m.generate_image_batch(
            past_key_values=cache, cfg_text_past_key_values=text_ctx[0], cfg_img_past_key_values=img_ctx[0],
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

    # per-request defaults of call_batch: those of interleave_inference
    CALL_BATCH_DEFAULTS = dict(think=False, understanding_output=False, max_think_token_n=1000, do_sample=False,
                               text_temperature=0.3, **GEN_BATCH_DEFAULTS)
    # high word of the Philox key of call_batch's sampled text (the low word is the request's seed): a fixed stream
    # id, so a request's draws do not depend on its position in the batch
    TEXT_KEY_STREAM = 0x74657874
    # optional truncation of a request's sampled thought or answer (Bagel.generate_text_batch); absent or None: off
    TEXT_FILTERS = ("top_k", "top_p", "min_p")
    # optional penalties on the tokens a request's thought or answer has generated (Bagel.generate_text_batch);
    # absent or None: off
    TEXT_PENALTIES = ("repetition_penalty", "presence_penalty", "frequency_penalty")

    def _call_batch_requests(self, requests: Sequence[Dict[str, Any]]) -> List[Dict[str, Any]]:
        """call_batch's requests with their defaults filled in; refuses unknown keys, TaylorSeer and inputs that are
        neither a string nor an image."""
        allowed = ("text", "image", "seed", "enable_taylorseer", *self.TEXT_FILTERS, *self.TEXT_PENALTIES,
                   *self.CALL_BATCH_DEFAULTS)
        unknown = [k for r in requests for k in r if k not in allowed]
        if unknown:
            raise ValueError(f"call_batch: unknown request keys {sorted(set(unknown))}")
        if any(r.get("enable_taylorseer") for r in requests):
            raise NotImplementedError("call_batch: TaylorSeer is not implemented for batched requests; use "
                                      "inferencer(..., enable_taylorseer=True) per request")
        for r in requests:
            _sampling_filters(1, True, *(r.get(f) for f in self.TEXT_FILTERS), who="call_batch")
            _penalties(1, *(r.get(f) for f in self.TEXT_PENALTIES), who="call_batch")
            if r.get("text") is not None and not isinstance(r["text"], str):
                raise ValueError(f"call_batch: text must be a string, got {type(r['text'])}")
            if r.get("image") is not None and not _is_image(r["image"]):
                raise ValueError(f"Unsupported input type: {type(r['image'])}")
        return [{**self.CALL_BATCH_DEFAULTS, **{k: v for k, v in r.items() if k != "enable_taylorseer"}}
                for r in requests]

    @torch.no_grad()
    def call_batch(self, requests: Sequence[Dict[str, Any]], num_timesteps: int = 50,
                   timestep_shift: float = 3.0) -> List[Dict[str, Any]]:
        """`__call__` for a batch of independent requests; returns one {"image": ..., "text": ...} per request.

        Each request is a dict: `text` and / or `image` (a PIL image; the input is the image, then the text, as in
        __call__; a request with neither gets {"image": None, "text": None}), `think`, `understanding_output`,
        `max_think_token_n`, `do_sample`, `text_temperature`, the image settings of gen_image_batch (`cfg_text_scale`,
        `cfg_img_scale`, `cfg_interval`, `cfg_renorm_min`, `cfg_renorm_type`, `image_shapes`) with the defaults of
        interleave_inference, `top_k` / `top_p` / `min_p` (truncated sampling of its sampled thought or answer, see
        Bagel.generate_text_batch; off when absent or None), `repetition_penalty` / `presence_penalty` /
        `frequency_penalty` (penalties on the tokens its thought or answer has generated, greedy or sampled, see
        Bagel.generate_text_batch; off when absent or None; __call__ has no penalties) and `seed` (None: drawn from
        torch.default_generator).
        `enable_taylorseer=True` is refused; num_timesteps and timestep_shift are shared.

        Request q with seed s gets what `torch.manual_seed(s); inferencer(image=..., text=..., **its settings)` gives it
        alone: greedy text (do_sample=False) the same tokens up to bf16 ties; an image the same image whenever the
        thought feeding it is the same. Sampled text is drawn on the device (Gumbel-max over Philox4x32-10, as
        Bagel.chat_batch) with the key (low 32 bits of s, TEXT_KEY_STREAM), so it depends on nothing but the request's
        own inputs, settings and seed (not on its position in the batch or on other requests); it does not reproduce
        torch.multinomial's stream, which the single-request path draws from.

        Every request's contexts are built in interleave_inference's order, each step one packed round over the
        requests call_batch_schedule lists for it: the think system prompt (main and cfg_img), the VAE image round,
        the ViT image round, cfg_text := main, the prompt (main and cfg_img), one Bagel.generate_text_batch over every
        understanding answer and thought (each with its own budget, sampling and temperature), the re-tokenized
        thoughts into main, then one Bagel.generate_image_batch over the generation requests and one VAE decode per
        image. Images are resized by vae_transform first, as interleave_inference does."""
        from .transforms import pil_img2rgb
        m = self.model
        reqs = self._call_batch_requests(requests)
        R = len(reqs)
        results: List[Dict[str, Any]] = [{"image": None, "text": None} for _ in range(R)]
        sched = call_batch_schedule(reqs)
        if not any(sched.values()):
            return results
        seeds = self._request_seeds(reqs)
        images = [None if r.get("image") is None else self.vae_transform.resize_transform(pil_img2rgb(r["image"]))
                  for r in reqs]
        L = m.config.llm_config.num_hidden_layers

        def only(members, value):
            return [value(q) if q in members else None for q in range(R)]

        def text_round(ctx, texts):
            if all(t is None for t in texts):
                return ctx
            gi, kv, rope = m.prepare_prompts_round(ctx[1], ctx[2], texts, self.tokenizer, self.new_token_ids)
            return m.forward_cache_update_text(ctx[0], **gi), kv, rope

        def subset(ctx, members):
            return gather_requests(ctx[0], ctx[1], members), [ctx[1][q] for q in members], [ctx[2][q] for q in members]

        def system(q):
            return VLM_THINK_SYSTEM_PROMPT if reqs[q]["understanding_output"] else GEN_THINK_SYSTEM_PROMPT

        main = (NaiveCache(L), [0] * R, [0] * R)
        img = (NaiveCache(L), [0] * R, [0] * R)
        main = text_round(main, only(sched["system"], system))
        img = text_round(img, only(sched["system_cfg_img"], system))
        if sched["vae"]:
            main = self._vae_image_round(*main, only(sched["vae"], images.__getitem__), seeds)
        if sched["vit"]:
            gi, kv, rope = m.prepare_vit_image_round(main[1], main[2], only(sched["vit"], images.__getitem__),
                                                     self.vit_transform, self.new_token_ids)
            main = (m.forward_cache_update_vit(main[0], **gi), kv, rope)
        gen = sched["generate"]
        text_ctx = subset(main, gen)             # text-dropped branch = everything before the text
        main = text_round(main, only(sched["prompt"], lambda q: reqs[q]["text"]))
        img = text_round(img, only(sched["prompt_cfg_img"], lambda q: reqs[q]["text"]))
        dec = sched["decode"]
        if dec:
            cache, kv, rope = subset(main, dec)
            gi = m.prepare_start_tokens(kv, rope, self.new_token_ids)
            toks = m.generate_text_batch(
                past_key_values=cache, max_length=[int(reqs[q]["max_think_token_n"]) for q in dec],
                do_sample=[bool(reqs[q]["do_sample"]) for q in dec],
                temperature=[float(reqs[q]["text_temperature"]) for q in dec],
                end_token_id=self.new_token_ids["eos_token_id"],
                keys=[(seeds[q] & 0xFFFFFFFF) | (self.TEXT_KEY_STREAM << 32) for q in dec],
                **{f: [reqs[q].get(f) for q in dec] for f in self.TEXT_FILTERS + self.TEXT_PENALTIES}, **gi)
            for q, t in zip(dec, toks):
                results[q]["text"] = self.tokenizer.decode(t.tolist()).split("<|im_end|>")[0].split("<|im_start|>")[1]
        main = text_round(main, only(sched["thought"], lambda q: results[q]["text"]))
        if gen:
            shapes = [tuple(images[q].size[::-1]) if images[q] is not None else tuple(reqs[q]["image_shapes"])
                      for q in gen]
            latents = self._denoise_batch([reqs[q] for q in gen], shapes, [seeds[q] for q in gen], subset(main, gen),
                                          text_ctx, subset(img, gen), num_timesteps, timestep_shift)
            for q, lat, hw in zip(gen, latents, shapes):
                results[q]["image"] = self.decode_image(lat, hw)
        return results

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
