"""-m gpu: the product path (bagel_b200 host code -> C ABI -> sm_90a kernels) against the committed reference
outputs (tests/golden) and the oracle.

Tolerance model. The reference is a bf16 pipeline (autocast): its own outputs carry bf16 rounding noise, and any
implementation with a different fp32 accumulation order (tensor-core tiles, flash softmax) differs from it at that
level. Two checks per tensor:
  (1) |gpu - reference| bounded by a few bf16 ulps of the tensor's scale (stated per test), and
  (2) the GPU result is no further from the exact (fp32, same bf16-valued weights) answer than ~1.5x the
      reference's own distance from it.
BASELINE.json's "1e-3 rtol on fp32 latents" is not reachable by ANY re-ordered bf16 implementation — flash_attn vs
the reference's CPU SDPA shim already differ by more — which is why (2) is the operative definition; DESIGN.md."""
import os

import pytest
import torch
from safetensors.torch import load_file

import helpers
from oracle import bagel_flow as obf
from oracle import fixtures, qwen2_mot as om

pytestmark = pytest.mark.gpu


def _stats(a, b):
    d = (a.float().cpu() - b.float().cpu()).abs()
    return d.max().item(), d.mean().item()


def _check(name, gpu, ref, truth, max_ulps_of_scale=8.0):
    scale = ref.float().abs().max().item()
    gmax, gmean = _stats(gpu, ref)
    assert torch.isfinite(gpu.float()).all()
    assert gmax <= max_ulps_of_scale * scale * 2 ** -8, f"{name}: |gpu-ref| max {gmax:.4e} vs scale {scale:.3f}"
    if truth is not None:
        tg_max, tg_mean = _stats(gpu, truth)
        tr_max, tr_mean = _stats(ref, truth)
        assert tg_mean <= 1.5 * tr_mean + 1e-4, f"{name}: mean err to truth gpu {tg_mean:.3e} vs ref {tr_mean:.3e}"
        assert tg_max <= 2.5 * tr_max + 1e-3, f"{name}: max err to truth gpu {tg_max:.3e} vs ref {tr_max:.3e}"


@pytest.fixture(scope="module")
def g_lm(golden_dir):
    return load_file(os.path.join(golden_dir, "lm_config1.safetensors"))


@pytest.fixture(scope="module")
def g_flow(golden_dir):
    return load_file(os.path.join(golden_dir, "flow_tiny.safetensors"))


def _f32(sd):
    return {k: v.float() for k, v in sd.items()}


@pytest.mark.parametrize("tag,cfg", [("d64", fixtures.TINY_LM), ("d128", fixtures.TINY128_LM)])
def test_lm_forward_config1(g_lm, tag, cfg):
    """BASELINE configs[0] on the GPU: und prefill (causal, cache update) then gen forward on top of the cache."""
    from bagel_b200.qwen2_navit import NaiveCache
    model = helpers.build_product_bagel(cfg, "cuda")
    lm = model.language_model
    inp = fixtures.config1_inputs(cfg)
    cache = NaiveCache(cfg.num_hidden_layers)
    kw_und = dict(query_lens=inp["query_lens"], packed_query_position_ids=inp["und_position_ids"],
                  packed_query_indexes=inp["query_indexes"], key_values_lens=torch.tensor([0], dtype=torch.int32),
                  packed_key_value_indexes=torch.zeros(0, dtype=torch.long), update_past_key_values=True,
                  is_causal=True, mode="und")
    und = lm.forward_inference(packed_query_sequence=inp["x"], past_key_values=cache, **kw_und)
    n = 130
    xg = torch.randn(n, cfg.hidden_size, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    kw_gen = dict(query_lens=torch.tensor([n], dtype=torch.int32),
                  packed_query_position_ids=torch.full((n,), 512, dtype=torch.long),
                  packed_query_indexes=torch.arange(512, 512 + n), key_values_lens=torch.tensor([512], dtype=torch.int32),
                  packed_key_value_indexes=torch.arange(512), update_past_key_values=False, is_causal=False, mode="gen",
                  packed_vae_token_indexes=torch.arange(1, n - 1), packed_text_indexes=torch.tensor([0, n - 1]))
    gen = lm.forward_inference(packed_query_sequence=xg, past_key_values=cache, **kw_gen)
    torch.cuda.synchronize()
    # exact answer: same bf16-valued weights, fp32 everywhere
    sd32 = _f32(fixtures.lm_state_dict(cfg, seed=0))
    with torch.no_grad(), om.high_precision():
        oc = om.KVCache(cfg.num_hidden_layers)
        t_und, oc = om.lm_forward_inference(sd32, cfg, inp["x"].float(), past_key_values=oc, **kw_und)
        t_gen, _ = om.lm_forward_inference(sd32, cfg, xg.float(), past_key_values=oc, **kw_gen)
    last = cfg.num_hidden_layers - 1
    pre = f"{tag}.A."
    _check("und hidden", und.packed_query_sequence, g_lm[pre + "und_hidden"], t_und)
    _check("k cache", cache.key_cache[last], g_lm[pre + "k_cache_last"], oc.key_cache[last])
    _check("v cache", cache.value_cache[last], g_lm[pre + "v_cache_last"], oc.value_cache[last])
    _check("gen hidden", gen.packed_query_sequence, g_lm[pre + "gen_hidden"], t_gen)
    assert cache.key_cache[last].shape == g_lm[pre + "k_cache_last"].shape


def _contexts(model, cfg):
    from bagel_b200.qwen2_navit import NaiveCache
    tok = helpers.IntTokenizer()

    def ctx(with_text):
        c, kv, rp = NaiveCache(cfg.num_hidden_layers), [0, 0], [0, 0]
        if with_text:
            gi, kv, rp = model.prepare_prompts(kv, rp, helpers.PROMPTS, tok, helpers.NEW_TOKEN_IDS)
            c = model.forward_cache_update_text(c, **gi)
        return c, kv, rp

    return ctx


VARIANTS = [("nocfg", 1.0, 1.0, "global"), ("global", 4.0, 1.0, "global"), ("channel", 4.0, 1.0, "channel"),
            ("global_img", 4.0, 1.5, "global"), ("text_channel_img", 4.0, 1.5, "text_channel"),
            # enable_taylorseer=True: 13 evaluations, 7 computed + 6 extrapolated (Taylor orders up to 3)
            ("taylor_nocfg", 1.0, 1.0, "global"), ("taylor_global_img", 4.0, 1.5, "global"),
            ("taylor_text_channel", 4.0, 1.0, "text_channel")]


@pytest.mark.parametrize("name,sT,sI,rt", VARIANTS)
def test_generate_image_tiny(g_flow, name, sT, sI, rt):
    """Packers -> text prefill -> 3-evaluation rectified-flow run, B=2 ragged images, every CFG/renorm variant."""
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    ctx = _contexts(model, cfg)
    c_main, kv_m, rp_m = ctx(True)
    c_txt, kv_t, rp_t = ctx(False)
    c_img, kv_i, rp_i = ctx(True)
    _check("prefill k", c_main.key_cache[cfg.num_hidden_layers - 1], g_flow["prefill.k_cache_last"], None)
    torch.manual_seed(2)
    gi = model.prepare_vae_latent(kv_m, rp_m, helpers.IMAGE_SIZES, helpers.NEW_TOKEN_IDS)
    for k in gi:
        assert torch.equal(gi[k], g_flow["latent." + k]), k
    ct = model.prepare_vae_latent_cfg(kv_t, rp_t, helpers.IMAGE_SIZES)
    ci = model.prepare_vae_latent_cfg(kv_i, rp_i, helpers.IMAGE_SIZES)
    taylor = name.startswith("taylor_")
    kw = dict(num_timesteps=14 if taylor else 4, timestep_shift=3.0, cfg_renorm_min=0.0, cfg_renorm_type=rt,
              cfg_interval=[0.4, 1.0], cfg_text_scale=sT, cfg_img_scale=sI, enable_taylorseer=taylor)
    lat = model.generate_image(
        past_key_values=c_main, **gi, **kw,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"], cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=ct["cfg_key_values_lens"], cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
        cfg_text_past_key_values=c_txt,
        cfg_img_packed_position_ids=ci["cfg_packed_position_ids"], cfg_img_packed_query_indexes=ci["cfg_packed_query_indexes"],
        cfg_img_key_values_lens=ci["cfg_key_values_lens"], cfg_img_packed_key_value_indexes=ci["cfg_packed_key_value_indexes"],
        cfg_img_past_key_values=c_img)
    torch.cuda.synchronize()
    assert [tuple(x.shape) for x in lat] == [(16, 64), (24, 64)] and lat[0].dtype == torch.float32
    got = torch.cat(lat, 0).cpu()
    ref = (load_file(os.path.join(os.path.dirname(__file__), "golden", "flow_taylor_tiny.safetensors")) if taylor
           else g_flow)[f"gen.{name}.latents"]

    # exact answer on the host: fp32 everywhere, same bf16-valued weights and the same init noise
    sd32 = _f32(helpers.flow_state_dict(cfg))
    fc = obf.FlowConfig(lm=cfg, max_latent_size=8)
    tok = helpers.IntTokenizer()
    with torch.no_grad(), om.high_precision():
        def octx(with_text):
            c, kvv, rpp = om.KVCache(cfg.num_hidden_layers), [0, 0], [0, 0]
            if with_text:
                g, kvv, rpp = obf.prepare_prompts(kvv, rpp, [tok.encode(p) for p in helpers.PROMPTS], 1000, 1001)
                c = obf.forward_cache_update_text(sd32, fc, c, **g)
            return c
        def br(d, cache):
            return dict(packed_position_ids=d["cfg_packed_position_ids"], packed_query_indexes=d["cfg_packed_query_indexes"],
                        key_values_lens=d["cfg_key_values_lens"], past_key_values=cache,
                        packed_key_value_indexes=d["cfg_packed_key_value_indexes"])
        truth = obf.generate_image(sd32, fc, gi, octx(True), cfg_text=br(ct, octx(False)), cfg_img=br(ci, octx(True)), **kw)
    truth = torch.cat(truth, 0)
    # CFG scale 4 amplifies branch differences 4x (and the image CFG again 1.5x)
    amp = 1.0 if sT <= 1 else (4.0 if sI <= 1 else 6.0)
    if taylor:   # 13 evaluations instead of 3, and finite differences of bf16 features extrapolated 1-2 steps ahead
        amp *= 3.0
    _check(f"latents[{name}]", got, ref, truth, max_ulps_of_scale=2.0 * amp)


def test_forward_flow_api(g_flow):
    """_forward_flow returns the CFG-combined velocity for given x_t / timestep (reference bagel.py:757-907)."""
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    ctx = _contexts(model, cfg)
    c_main, kv_m, rp_m = ctx(True)
    c_txt, kv_t, rp_t = ctx(False)
    torch.manual_seed(2)
    gi = model.prepare_vae_latent(kv_m, rp_m, helpers.IMAGE_SIZES, helpers.NEW_TOKEN_IDS)
    ct = model.prepare_vae_latent_cfg(kv_t, rp_t, helpers.IMAGE_SIZES)
    x = gi["packed_init_noises"]
    t = torch.full((x.shape[0],), 0.7)
    v = model._forward_flow(
        x_t=x, timestep=t, packed_vae_token_indexes=gi["packed_vae_token_indexes"],
        packed_vae_position_ids=gi["packed_vae_position_ids"], packed_text_ids=gi["packed_text_ids"],
        packed_text_indexes=gi["packed_text_indexes"], packed_indexes=gi["packed_indexes"],
        packed_position_ids=gi["packed_position_ids"], packed_seqlens=gi["packed_seqlens"],
        key_values_lens=gi["key_values_lens"], past_key_values=c_main,
        packed_key_value_indexes=gi["packed_key_value_indexes"], cfg_renorm_type="channel", cfg_text_scale=3.0,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"], cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=ct["cfg_key_values_lens"], cfg_text_past_key_values=c_txt,
        cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"])
    sd = helpers.flow_state_dict(cfg)
    fc = obf.FlowConfig(lm=cfg, max_latent_size=8)
    tok = helpers.IntTokenizer()
    with torch.no_grad():
        g, kvv, rpp = obf.prepare_prompts([0, 0], [0, 0], [tok.encode(p) for p in helpers.PROMPTS], 1000, 1001)
        oc = obf.forward_cache_update_text(sd, fc, om.KVCache(cfg.num_hidden_layers), **g)
        ref = obf.forward_flow(
            sd, fc, x, t, gi["packed_vae_token_indexes"], gi["packed_vae_position_ids"], gi["packed_text_ids"],
            gi["packed_text_indexes"], gi["packed_indexes"], gi["packed_position_ids"], gi["packed_seqlens"],
            gi["key_values_lens"], oc, gi["packed_key_value_indexes"], 0.0, "channel", 3.0,
            dict(packed_position_ids=ct["cfg_packed_position_ids"], packed_query_indexes=ct["cfg_packed_query_indexes"],
                 key_values_lens=ct["cfg_key_values_lens"], past_key_values=om.KVCache(cfg.num_hidden_layers),
                 packed_key_value_indexes=ct["cfg_packed_key_value_indexes"]))
    assert v.dtype == torch.bfloat16 and v.shape == ref.shape
    _check("forward_flow", v, ref, None, max_ulps_of_scale=8.0)


def test_kv_cache_survives_deepcopy_and_context_is_not_mutated():
    """inferencer.py:230-253 deep-copies whole contexts; generate_image must leave the cached context untouched
    (update_past_key_values=False, bagel.py:828)."""
    import copy
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    c_main, kv_m, rp_m = _contexts(model, cfg)(True)
    snap = copy.deepcopy(c_main)
    torch.manual_seed(2)
    gi = model.prepare_vae_latent(kv_m, rp_m, helpers.IMAGE_SIZES, helpers.NEW_TOKEN_IDS)
    model.generate_image(past_key_values=c_main, **gi, num_timesteps=3)
    torch.cuda.synchronize()
    for li in range(cfg.num_hidden_layers):
        assert torch.equal(snap.key_cache[li], c_main.key_cache[li])
        assert torch.equal(snap.value_cache[li], c_main.value_cache[li])


def test_smoke_entry():
    import __graft_entry__
    __graft_entry__.smoke()


def test_generate_text_greedy(g_flow):
    """Text decode (bagel.py:930-1000). Token ids must be bit-exact wherever the reference's own top-1/top-2 logit
    margin exceeds bf16 noise; the fixture holds the reference's logits so the first divergence (if any) is
    attributed: a random-init model has near-uniform logits (min margin in the fixture: 1 bf16 ulp)."""
    from copy import deepcopy
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    c_main, kv_m, rp_m = _contexts(model, cfg)(True)
    gs = model.prepare_start_tokens(kv_m, rp_m, helpers.NEW_TOKEN_IDS)
    for k in gs:
        assert torch.equal(gs[k], g_flow["start." + k]), k
    toks = model.generate_text(past_key_values=deepcopy(c_main), max_length=12, do_sample=False, **gs).cpu()
    ref = g_flow["text.tokens"]
    ref_logits = g_flow["text.logits"].float()               # [steps, B, V]
    assert toks.shape == ref.shape and toks.dtype == torch.int64
    assert torch.equal(toks[0], ref[0])
    top2 = ref_logits.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]                      # [steps, B]
    for b in range(ref.shape[1]):
        for s in range(1, ref.shape[0]):
            if toks[s, b] != ref[s, b]:
                # tokens diverge only where the reference's decision at step s-1 was within bf16 noise
                assert margin[s - 1, b] <= 0.07, f"sample {b} diverged at step {s} with margin {margin[s-1, b]:.4f}"
                break
    # teacher-forced: with the reference's token prefix, logits must agree to bf16 accuracy at every step
    from bagel_b200.bagel import _ranges
    cache = deepcopy(c_main)
    kv = torch.tensor(kv_m, dtype=torch.int64)
    pos = torch.tensor(rp_m, dtype=torch.int64)
    for s in range(ref.shape[0]):
        emb = model.language_model.model.embed_tokens(ref[s])
        starts = torch.cumsum(kv + 1, 0) - (kv + 1)
        out = model.language_model.forward_inference(
            packed_query_sequence=emb, query_lens=torch.ones(2, dtype=torch.int32), packed_query_position_ids=pos,
            packed_query_indexes=starts + kv, past_key_values=cache, key_values_lens=kv.to(torch.int32),
            packed_key_value_indexes=_ranges(starts, kv), update_past_key_values=True, is_causal=True, mode="und")
        logits = model.language_model.lm_head(out.packed_query_sequence).float().cpu()
        torch.testing.assert_close(logits, ref_logits[s], atol=0.06, rtol=0.02)
        kv, pos = kv + 1, pos + 1


def test_vit_tower_and_image_understanding_prefill(golden_dir):
    """SigLIP NaViT tower (head_dim 72 -> padded heads on the d=128 attention path), connector, ViT-context prefill
    (non-causal image block) and a causal text prefill on top of it (BASELINE configs[2] shape, tiny model)."""
    from bagel_b200.qwen2_navit import NaiveCache
    from oracle import siglip as osl
    g = load_file(os.path.join(golden_dir, "vit_tiny.safetensors"))
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel_with_vit(cfg, "cuda")
    gi, kv, rp = model.prepare_vit_images([0, 0], [0, 0], fixtures.vit_images(), lambda im: im, helpers.NEW_TOKEN_IDS)
    for k in gi:
        assert torch.equal(gi[k], g["vit_in." + k]), k
    vl = gi["vit_token_seqlens"]
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), vl.to(torch.int64).cumsum(0)]).to(torch.int32)
    feats = model.vit_model(packed_pixel_values=gi["packed_vit_tokens"],
                            packed_flattened_position_ids=gi["packed_vit_position_ids"], cu_seqlens=cu,
                            max_seqlen=int(vl.max()))
    # exact fp32 answer for the tower
    tv = fixtures.TINY_VIT
    vc = osl.VitConfig(hidden_size=tv["hidden"], intermediate_size=tv["inter"], num_hidden_layers=tv["layers"],
                       num_attention_heads=tv["heads"])
    sd32 = _f32(helpers.vit_flow_state_dict(cfg))
    with torch.no_grad(), om.high_precision():
        truth = osl.vit_forward(sd32, vc, gi["packed_vit_tokens"], gi["packed_vit_position_ids"], vl)
    _check("vit features", feats, g["vit.features"], truth, max_ulps_of_scale=8.0)
    cache = model.forward_cache_update_vit(NaiveCache(cfg.num_hidden_layers), **gi)
    gt, kv2, rp2 = model.prepare_prompts(kv, rp, ["5 17 900", "8 8 100 4"], helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS)
    cache = model.forward_cache_update_text(cache, **gt)
    torch.cuda.synchronize()
    last = cfg.num_hidden_layers - 1
    assert cache.key_cache[last].shape == g["vit.k_cache_last"].shape
    _check("vit ctx k", cache.key_cache[last], g["vit.k_cache_last"], None)
    _check("vit ctx v", cache.value_cache[last], g["vit.v_cache_last"], None)


def test_cuda_graph_replay_is_bit_identical_to_eager(g_flow):
    """generate_image captures the step's launch sequence once per branch set and replays it; results must equal the
    eager launch sequence bit for bit (cfg_interval makes the run use both the 2-branch and the 1-branch graph)."""
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    ctx = _contexts(model, cfg)
    c_main, kv_m, rp_m = ctx(True)
    c_txt, kv_t, rp_t = ctx(False)
    ct = model.prepare_vae_latent_cfg(kv_t, rp_t, helpers.IMAGE_SIZES)
    outs = []
    for use_graph in (False, True):
        model.use_cuda_graph = use_graph
        torch.manual_seed(2)
        gi = model.prepare_vae_latent(kv_m, rp_m, helpers.IMAGE_SIZES, helpers.NEW_TOKEN_IDS)
        lat = model.generate_image(
            past_key_values=c_main, **gi, num_timesteps=9, timestep_shift=3.0, cfg_renorm_type="global",
            cfg_interval=[0.4, 1.0], cfg_text_scale=3.0,
            cfg_text_packed_position_ids=ct["cfg_packed_position_ids"], cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
            cfg_text_key_values_lens=ct["cfg_key_values_lens"], cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
            cfg_text_past_key_values=c_txt)
        torch.cuda.synchronize()
        outs.append(torch.cat(lat, 0).clone())
    assert torch.equal(outs[0], outs[1])


def test_generate_text_graph_vs_eager_and_eos(g_flow):
    """The decode step replayed as a CUDA graph must produce the same ids as the eager launch sequence; generation
    stops when sample 0 emits end_token_id and the stopping token is not returned (reference bagel.py:996)."""
    from copy import deepcopy
    cfg = fixtures.TINY_LM
    model = helpers.build_product_bagel(cfg, "cuda")
    c_main, kv_m, rp_m = _contexts(model, cfg)(True)
    gs = model.prepare_start_tokens(kv_m, rp_m, helpers.NEW_TOKEN_IDS)
    outs = []
    for use_graph in (False, True):
        model.use_cuda_graph = use_graph
        outs.append(model.generate_text(past_key_values=deepcopy(c_main), max_length=10, do_sample=False, **gs).cpu())
    assert torch.equal(outs[0], outs[1]) and outs[0].shape == (10, 2)
    # stop on the token sample 0 produces at step 3 (history rows 0..3 are returned, the EOS itself is not)
    eos = int(outs[0][4, 0])
    first = next(i for i in range(1, 10) if int(outs[0][i, 0]) == eos)
    short = model.generate_text(past_key_values=deepcopy(c_main), max_length=10, do_sample=False, end_token_id=eos, **gs).cpu()
    assert short.shape[0] == first and torch.equal(short, outs[0][:first])
    # the context handed in is not modified (gen_text deep-copies it anyway, inferencer.py:189)
    snap = deepcopy(c_main)
    model.generate_text(past_key_values=c_main, max_length=3, do_sample=True, temperature=0.7, **gs)
    for li in range(cfg.num_hidden_layers):
        assert torch.equal(snap.key_cache[li], c_main.key_cache[li])


def test_hf_style_loader_equals_direct_construction(tmp_path):
    """loader.load_bagel on a checkpoint directory laid out like the reference's (llm_config.json, vit_config.json,
    ema.safetensors; app.py:39-133) must build the same model as loading the state dict directly: identical K cache of
    a text + ViT prefill (same kernels, same fused layouts -> bit-identical)."""
    import json
    from safetensors.torch import save_file
    from bagel_b200.loader import load_bagel
    cfg, tv = fixtures.TINY_LM, fixtures.TINY_VIT
    sd = helpers.flow_state_dict(cfg, max_latent_size=64)                  # the loader fixes 64 latent / 70 ViT positions
    sd.update(fixtures.vit_state_dict(tv["hidden"], tv["inter"], tv["layers"], tv["heads"], cfg.hidden_size, max_side=70))
    sd["vit_pos_embed.pos_embed"] = obf.sincos_2d_table(cfg.hidden_size, 70).to(torch.bfloat16)
    save_file({k: v.contiguous() for k, v in sd.items()}, str(tmp_path / "ema.safetensors"))
    (tmp_path / "llm_config.json").write_text(json.dumps(dict(
        model_type="qwen2", vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
        num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
        num_key_value_heads=cfg.num_key_value_heads, rope_theta=cfg.rope_theta, rms_norm_eps=cfg.rms_norm_eps,
        tie_word_embeddings=True)))
    (tmp_path / "vit_config.json").write_text(json.dumps(dict(
        model_type="siglip_vision_model", hidden_size=tv["hidden"], intermediate_size=tv["inter"],
        num_hidden_layers=tv["layers"] + 1, num_attention_heads=tv["heads"], num_channels=3, image_size=980, patch_size=14)))
    model, vae, bcfg = load_bagel(str(tmp_path), device="cuda")
    assert bcfg.vit_config.num_hidden_layers == tv["layers"] and bcfg.llm_config.layer_module == "Qwen2MoTDecoderLayer"
    assert vae is not None and model.vit_model is not None

    from bagel_b200.bagel import Bagel
    from bagel_b200.config import AutoEncoderParams, BagelConfig, Qwen2Config, SiglipVisionConfig
    from bagel_b200.qwen2_navit import NaiveCache, Qwen2ForCausalLM
    from bagel_b200.siglip_navit import SiglipVisionModel
    llm = Qwen2Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                      num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                      num_key_value_heads=cfg.num_key_value_heads, rope_theta=cfg.rope_theta, rms_norm_eps=cfg.rms_norm_eps,
                      qk_norm=True, layer_module="Qwen2MoTDecoderLayer")
    vcfg = SiglipVisionConfig(hidden_size=tv["hidden"], intermediate_size=tv["inter"], num_hidden_layers=tv["layers"],
                              num_attention_heads=tv["heads"], num_channels=3, image_size=980, patch_size=14, rope=False)
    direct = Bagel(Qwen2ForCausalLM(llm, device="cuda"), SiglipVisionModel(vcfg, device="cuda"),
                   BagelConfig(visual_gen=True, visual_und=True, llm_config=llm, vit_config=vcfg,
                               vae_config=AutoEncoderParams(), latent_patch_size=2, max_latent_size=64,
                               vit_max_num_patch_per_side=70))
    direct.load_state_dict(sd)

    def prefill(m):
        tok = helpers.IntTokenizer()
        c, kv, rp = NaiveCache(cfg.num_hidden_layers), [0, 0], [0, 0]
        gi, kv, rp = m.prepare_vit_images(kv, rp, fixtures.vit_images(), lambda im: im, helpers.NEW_TOKEN_IDS)
        c = m.forward_cache_update_vit(c, **gi)
        gi, kv, rp = m.prepare_prompts(kv, rp, helpers.PROMPTS, tok, helpers.NEW_TOKEN_IDS)
        c = m.forward_cache_update_text(c, **gi)
        return c, kv, rp

    ca, kva, rpa = prefill(model)
    cb, kvb, rpb = prefill(direct)
    assert kva == kvb and rpa == rpb
    for li in range(cfg.num_hidden_layers):
        assert torch.equal(ca.key_cache[li], cb.key_cache[li]) and torch.equal(ca.value_cache[li], cb.value_cache[li])
