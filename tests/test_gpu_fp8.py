"""-m gpu: the opt-in block-scaled FP8 generation-expert MLP (`fp8_gen_mlp=True`).

  quantiser  bit-exact (e4m3 bytes and scales) against tests/fp8_oracle.py, both block shapes;
  GEMM       against the dequantised operands multiplied in fp64 and passed through the same bf16 epilogue, within
             2 bf16 ulps of the output's scale, for 1- and 2-CTA launches (odd / even M-tile counts, a past-the-end peer)
             and pair-tile counts below and above the number of resident clusters;
  models     TINY_LM / TINY128_LM / TINY_MOE_LM with the flag on against the oracle under the fp8 contract
             (hidden states and KV: tests/test_gpu_model.py's criterion; a CFG image run: bounded by the distance
             between the contract's own bf16 and fp32 legs), and und-mode calls unchanged by the flag."""
import pytest
import torch

import fp8_oracle as fo
import helpers
from bagel_b200 import fp8, ops
from oracle import bagel_flow as obf
from oracle import fixtures, qwen2_mot as om

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _x(M, K, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(M, K, generator=g, device="cuda") * scale).to(BF16)


@pytest.mark.parametrize("block_rows", [1, 128])
@pytest.mark.parametrize("M,K", [(1, 128), (63, 256), (129, 384), (300, 1024), (4097, 3584)])
def test_quantizer_bit_exact(block_rows, M, K):
    x = _x(M, K, M + K, scale=3.0)
    x[M // 2] = 0                                           # an all-zero row (and, for M >= 2, a zero group)
    if M > 2:
        x[1, :128] = 448.0 * 2.0 ** -5                      # group maximum exactly at a scale boundary
        x[2, :128] = 0.25
        x[2, 7] = -torch.tensor(448.0 * 2.0 ** -5, dtype=BF16).view(torch.int16).add(1).view(BF16)   # just above it
        x[2, 8] = 2.0 ** -130                               # a bf16 denormal next to it
    if M >= 300:
        x[200:] *= torch.logspace(-20, 20, M - 200, device="cuda")[:, None].to(BF16)
    q, s = ops.quantize_fp8(x, block_rows)
    rq, rs = fo.quantize(x.cpu(), block_rows)
    if block_rows == 1:
        rs = rs.t()                                         # the product's activation scales are K-block major
    assert torch.equal(s.cpu(), rs)
    assert torch.equal(q.view(torch.uint8).cpu(), rq.view(torch.uint8))


def _ref_gemm(A, As, W_deq, epilogue, resid):
    """fp64 product of the dequantised operands, then the product's bf16 epilogue rounding points."""
    a = fo.dequantize(A.cpu(), As.t().cpu(), 1).double()
    y = a @ W_deq.cpu().double().t()
    if epilogue == ops.EPI_SWIGLU:
        I = y.shape[1] // 2
        g = y[:, :I].float().to(BF16).float()
        u = y[:, I:].float().to(BF16).float()
        return (torch.nn.functional.silu(g).to(BF16).float() * u).to(BF16)
    return (resid.cpu().float() + y.float().to(BF16).float()).to(BF16)


# M: 1 and 63 (one tile, no cluster), 128 (one full tile), 129 (a pair), 384 (odd tile count: the last pair's second CTA
# lies past M), 65 568 (the denoising shape; 513 M tiles). N tiles x pair tiles go from 1 to ~1000 (above the ~66
# resident clusters) between the small and the large cases.
@pytest.mark.parametrize("M", [1, 63, 128, 129, 384, 65568])
@pytest.mark.parametrize("epilogue", [ops.EPI_SWIGLU, ops.EPI_RESID])
def test_gemm_fp8_against_fp64(M, epilogue):
    H, I = 512, 384
    g = torch.Generator(device="cuda").manual_seed(M)

    def blocky(rows, cols, rb):
        """randn * 0.02 with every rb x 128 block scaled by its own 2^[-3, 3]: each block gets a different scale, so a
        wrong scale index (gate vs up half, tile row, K block) shows."""
        e = torch.randint(-3, 4, (rows // rb, cols // 128), generator=g, device="cuda").float()
        f = torch.exp2(e).repeat_interleave(rb, 0).repeat_interleave(128, 1)
        return (torch.randn(rows, cols, generator=g, device="cuda") * 0.02 * f).to(BF16)

    gate, up, down = blocky(I, H, 128), blocky(I, H, 128), blocky(H, I, 128)
    w = fp8.GenMlpFp8.from_reference(gate, up, down)

    class _E:
        pass
    e = _E()
    e.fp8 = w
    deq = fo.gen_mlp_weights(e)                             # reference-layout bf16, from the raw bytes and scales
    # the layout round trip: the dequantised weights are the fp8 images of the originals
    for name, orig in (("gate_proj.weight", gate), ("up_proj.weight", up), ("down_proj.weight", down)):
        rq, rs = fo.quantize(orig.cpu(), 128)
        assert torch.equal(deq[name].cpu(), fo.dequantize(rq, rs, 128).to(BF16)), name
    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(w.dequantize(), deq.values()))

    for name, t in (("gate", gate), ("up", up), ("down", down)):
        assert fo.quantize(t.cpu(), 128)[1].unique().numel() >= 4, name   # the blocks' scales do differ
    if epilogue == ops.EPI_SWIGLU:
        x = blocky(M, H, 1) * 50
        xq, xs = ops.quantize_fp8(x)
        out = ops.gemm_fp8(xq, xs, w.wgu, w.wgu_s, epilogue=epilogue)
        ref = _ref_gemm(xq, xs, torch.cat([deq["gate_proj.weight"], deq["up_proj.weight"]]), epilogue, None)
    else:
        x = blocky(M, I, 1) * 50
        resid = _x(M, H, 17 + M)
        xq, xs = ops.quantize_fp8(x)
        out = ops.gemm_fp8(xq, xs, w.wd, w.wd_s, resid=resid, epilogue=epilogue)
        ref = _ref_gemm(xq, xs, deq["down_proj.weight"], epilogue, resid)
    torch.cuda.synchronize()
    out = out.cpu().float()
    ref = ref.float()
    scale = ref.abs().max().item()
    err = (out - ref).abs().max().item()
    assert torch.isfinite(out).all()
    assert err <= 2 * scale * 2 ** -8, f"M={M} epi={epilogue}: max err {err:.3e} vs scale {scale:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# tiny models against the oracle under the fp8 contract
# ------------------------------------------------------------------------------------------------------------------
def _check(name, gpu, ref, truth, max_ulps_of_scale=8.0):
    """tests/test_gpu_model.py's criterion."""
    gpu, ref, truth = gpu.float().cpu(), ref.float().cpu(), truth.float().cpu()
    scale = ref.abs().max().item()
    d = (gpu - ref).abs()
    assert torch.isfinite(gpu).all()
    assert d.max().item() <= max_ulps_of_scale * scale * 2 ** -8, f"{name}: |gpu-ref| max {d.max().item():.4e} vs {scale:.3f}"
    tg, tr = (gpu - truth).abs(), (ref - truth).abs()
    assert tg.mean() <= 1.5 * tr.mean() + 1e-4, f"{name}: mean err to truth gpu {tg.mean():.3e} vs ref {tr.mean():.3e}"
    assert tg.max() <= 2.5 * tr.max() + 1e-3, f"{name}: max err to truth gpu {tg.max():.3e} vs ref {tr.max():.3e}"


def _lm(cfg, fp8_gen_mlp):
    from bagel_b200.config import Qwen2Config
    from bagel_b200.qwen2_navit import Qwen2ForCausalLM
    llm = Qwen2Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                      num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                      num_key_value_heads=cfg.num_key_value_heads, rope_theta=cfg.rope_theta,
                      rms_norm_eps=cfg.rms_norm_eps, qk_norm=True, layer_module=cfg.layer_module)
    lm = Qwen2ForCausalLM(llm, device="cuda", fp8_gen_mlp=fp8_gen_mlp)
    lm.load_state_dict(fixtures.lm_state_dict(cfg, seed=0))
    return lm


def _fp8_sd(lm, cfg):
    """The reference state dict with the gen MLP weights replaced by the dequantised ones."""
    sd = fixtures.lm_state_dict(cfg, seed=0)
    for li, layer in enumerate(lm.model.layers):
        for k, v in fo.gen_mlp_weights(layer.gen).items():
            sd[f"model.layers.{li}.mlp_moe_gen.{k}"] = v.cpu()
    return sd


def _kw(cfg):
    inp = fixtures.config1_inputs(cfg)
    kw_und = dict(query_lens=inp["query_lens"], packed_query_position_ids=inp["und_position_ids"],
                  packed_query_indexes=inp["query_indexes"], key_values_lens=torch.tensor([0], dtype=torch.int32),
                  packed_key_value_indexes=torch.zeros(0, dtype=torch.long), update_past_key_values=True,
                  is_causal=True, mode="und")
    n = 130
    xg = torch.randn(n, cfg.hidden_size, generator=torch.Generator().manual_seed(5)).to(BF16)
    kw_gen = dict(query_lens=torch.tensor([n], dtype=torch.int32),
                  packed_query_position_ids=torch.full((n,), 512, dtype=torch.long),
                  packed_query_indexes=torch.arange(512, 512 + n), key_values_lens=torch.tensor([512], dtype=torch.int32),
                  packed_key_value_indexes=torch.arange(512), update_past_key_values=True, is_causal=False, mode="gen",
                  packed_vae_token_indexes=torch.arange(1, n - 1), packed_text_indexes=torch.tensor([0, n - 1]))
    return inp["x"], kw_und, xg, kw_gen


def _dev(kw, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()}


@pytest.mark.parametrize("tag,cfg", [("d64", fixtures.TINY_LM), ("d128", fixtures.TINY128_LM),
                                     ("moe", fixtures.TINY_MOE_LM)])
def test_lm_gen_forward_fp8(tag, cfg):
    """und prefill (unchanged by the flag) then a gen-mode forward through the fp8 gen MLP: hidden states and KV."""
    from bagel_b200.qwen2_navit import NaiveCache
    lm = _lm(cfg, True)
    x, kw_und, xg, kw_gen = _kw(cfg)
    cache = NaiveCache(cfg.num_hidden_layers)
    lm.forward_inference(packed_query_sequence=x, past_key_values=cache, **kw_und)
    gen = lm.forward_inference(packed_query_sequence=xg, past_key_values=cache, **kw_gen).packed_query_sequence
    torch.cuda.synchronize()
    last = cfg.num_hidden_layers - 1
    sd = _fp8_sd(lm, cfg)
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    sd32 = {k: v.float().cuda() for k, v in sd.items()}
    outs = {}
    with torch.no_grad(), fo.fp8_contract():
        for leg, s, cast in (("ref", sd_cuda, BF16), ("truth", sd32, torch.float32)):
            ctx = om.high_precision() if leg == "truth" else _Null()
            with ctx:
                oc = om.KVCache(cfg.num_hidden_layers)
                _, oc = om.lm_forward_inference(s, cfg, x.to("cuda", cast), past_key_values=oc, **_dev(kw_und, "cuda"))
                h, oc = om.lm_forward_inference(s, cfg, xg.to("cuda", cast), past_key_values=oc, **_dev(kw_gen, "cuda"))
            outs[leg] = (h, oc)
    (ref, rc), (truth, tc) = outs["ref"], outs["truth"]
    _check(f"{tag} gen hidden", gen, ref, truth)
    _check(f"{tag} k cache", cache.key_cache[last], rc.key_cache[last], tc.key_cache[last])
    _check(f"{tag} v cache", cache.value_cache[last], rc.value_cache[last], tc.value_cache[last])


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@pytest.mark.parametrize("cfg", [fixtures.TINY_LM, fixtures.TINY_MOE_LM])
def test_und_calls_unchanged_by_the_flag(cfg):
    """Text prefill and a one-token und step never reach the gen expert: bit-identical with the flag on and off."""
    from bagel_b200.qwen2_navit import NaiveCache
    x, kw_und, _, _ = _kw(cfg)
    res = []
    for flag in (False, True):
        lm = _lm(cfg, flag)
        cache = NaiveCache(cfg.num_hidden_layers)
        a = lm.forward_inference(packed_query_sequence=x, past_key_values=cache, **kw_und).packed_query_sequence
        n0 = x.shape[0]
        b = lm.forward_inference(packed_query_sequence=x[:1], query_lens=torch.tensor([1], dtype=torch.int32),
                                 packed_query_position_ids=torch.tensor([n0]), packed_query_indexes=torch.tensor([n0]),
                                 past_key_values=cache, key_values_lens=torch.tensor([n0], dtype=torch.int32),
                                 packed_key_value_indexes=torch.arange(n0), update_past_key_values=True,
                                 is_causal=True, mode="und").packed_query_sequence
        res.append((a.cpu(), b.cpu(), cache.key_cache[cfg.num_hidden_layers - 1].cpu()))
    for u, v in zip(*res):
        assert torch.equal(u, v)


def test_generate_image_fp8_tiny():
    """Packers -> text prefill -> a 4-step text-CFG rectified-flow run with the fp8 gen MLP (CUDA-graph replay of the
    step), against the oracle under the fp8 contract: bf16 on the host, and fp32 for the exact answer."""
    from bagel_b200.bagel import Bagel
    from bagel_b200.qwen2_navit import NaiveCache, Qwen2ForCausalLM
    cfg = fixtures.TINY_LM
    base = helpers.build_product_bagel(cfg, "cuda", load=False)
    model = Bagel(Qwen2ForCausalLM(base.language_model.config, device="cuda", fp8_gen_mlp=True), None, base.config)
    sd = helpers.flow_state_dict(cfg)
    model.load_state_dict(sd)
    tok = helpers.IntTokenizer()
    gi_p, kv, rp = model.prepare_prompts([0, 0], [0, 0], helpers.PROMPTS, tok, helpers.NEW_TOKEN_IDS)
    cache = model.forward_cache_update_text(NaiveCache(cfg.num_hidden_layers), **gi_p)
    torch.manual_seed(2)
    gi = model.prepare_vae_latent(kv, rp, helpers.IMAGE_SIZES, helpers.NEW_TOKEN_IDS)
    ct = model.prepare_vae_latent_cfg([0, 0], [0, 0], helpers.IMAGE_SIZES)
    kw = dict(num_timesteps=4, timestep_shift=3.0, cfg_renorm_type="global", cfg_interval=[0.4, 1.0], cfg_text_scale=4.0)
    lat = model.generate_image(
        past_key_values=cache, **gi, **kw,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"], cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"],
        cfg_text_key_values_lens=ct["cfg_key_values_lens"], cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"],
        cfg_text_past_key_values=NaiveCache(cfg.num_hidden_layers))
    torch.cuda.synchronize()
    got = torch.cat(lat, 0).cpu()

    lm = model.language_model
    for li, layer in enumerate(lm.model.layers):
        for k, v in fo.gen_mlp_weights(layer.gen).items():
            sd[f"language_model.model.layers.{li}.mlp_moe_gen.{k}"] = v.cpu()
    fc = obf.FlowConfig(lm=cfg, max_latent_size=8)
    outs = []
    with torch.no_grad(), fo.fp8_contract():
        for s, hp in ((sd, False), ({k: v.float() for k, v in sd.items()}, True)):
            ctx = om.high_precision() if hp else _Null()
            with ctx:
                g, _, _ = obf.prepare_prompts([0, 0], [0, 0], [tok.encode(p) for p in helpers.PROMPTS], 1000, 1001)
                c = obf.forward_cache_update_text(s, fc, om.KVCache(cfg.num_hidden_layers), **g)
                br = dict(packed_position_ids=ct["cfg_packed_position_ids"], packed_query_indexes=ct["cfg_packed_query_indexes"],
                          key_values_lens=ct["cfg_key_values_lens"], past_key_values=om.KVCache(cfg.num_hidden_layers),
                          packed_key_value_indexes=ct["cfg_packed_key_value_indexes"])
                outs.append(torch.cat(obf.generate_image(s, fc, gi, c, cfg_text=br, **kw), 0))
    # Over several steps with CFG 4 the e4m3 rounding of h and act is discontinuous: a last-bit difference of the fp32
    # sums can move a value to the neighbouring e4m3 step (1/16 relative), and the contract's own two legs (bf16 oracle,
    # fp32 oracle) already differ by such flips. So the bound is relative to that noise floor instead of a fixed number of
    # bf16 ulps: the product may be no further from the bf16 leg than the two legs are from each other (x2), and no
    # further from the fp32 leg than the bf16 leg is (test_gpu_model.py's truth criterion).
    gpu, ref, truth = got.float(), outs[0].float().cpu(), outs[1].float().cpu()
    assert torch.isfinite(gpu).all()
    floor = (ref - truth).abs()
    d = (gpu - ref).abs()
    assert d.max() <= 2.0 * floor.max(), f"|gpu-ref| max {d.max():.3e} vs |ref-truth| max {floor.max():.3e}"
    tg = (gpu - truth).abs()
    assert tg.mean() <= 1.5 * floor.mean() + 1e-4, f"mean err to truth gpu {tg.mean():.3e} vs ref {floor.mean():.3e}"
    assert tg.max() <= 2.5 * floor.max() + 1e-3, f"max err to truth gpu {tg.max():.3e} vs ref {floor.max():.3e}"
    print(f"fp8 latents: |gpu-ref| max {d.max():.3e} mean {d.mean():.3e}; |ref-truth| max {floor.max():.3e} "
          f"mean {floor.mean():.3e}; |gpu-truth| max {tg.max():.3e} mean {tg.mean():.3e}")
