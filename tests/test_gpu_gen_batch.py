"""-m gpu: batched image generation of independent requests. bagel_cfg_euler_step_batch against a per-request host
restatement and against bagel_cfg_euler_step, its determinism and graph replay; Bagel.generate_image_batch's
independence between requests, graph against eager and launches per step; InterleaveInferencer.gen_image_batch
against the reference's inferencer golden and against sequential single-request calls."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

import helpers
from oracle import fixtures
from test_gpu_inferencer import KW, TEXT, _check_image

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from bagel_b200 import ops
    return ops


# ------------------------------------------------------------------------------------------------------------ kernel

def _i32(x):
    return torch.tensor(x, dtype=torch.int32, device=DEV)


def _f32(x):
    return torch.tensor(x, dtype=torch.float32, device=DEV)


def _mixed_case(seed=11):
    """R = 6 requests, each a contiguous run of seg whose rows read scattered rows of V: all three renorm types, sI 1 and 1.5, a request without a text-dropped row,
    one without an image-dropped row, one with CFG off. The renorm_min of 0.375 is exact in bf16: like
    bagel_cfg_euler_step, the kernel clamps with the fp32 value, where torch's clamp of a bf16 tensor gives bf16(min)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    R, C = 6, 64
    counts = [150, 97, 230, 61, 128, 200]
    M = sum(counts)
    seg = torch.cat([torch.full((n,), q, dtype=torch.int64) for q, n in enumerate(counts)])
    V = torch.randn(3 * M + 17, C, device=DEV, generator=g).to(torch.bfloat16)
    perm = torch.randperm(3 * M + 17, generator=torch.Generator().manual_seed(seed + 1))
    rm, rtx, rim = perm[:M].clone(), perm[M:2 * M].clone(), perm[2 * M:3 * M].clone()
    p = dict(sT=[4.0, 3.0, 4.0, 2.5, 4.0, 5.0], sI=[1.5, 1.0, 1.5, 1.5, 1.5, 1.5], rmin=[0.0, 0.0, 0.375, 0.0, 0.0, 0.0],
             rtype=[0, 1, 2, 0, 2, 1], on=[1, 1, 1, 1, 1, 0])
    rtx[seg == 3] = -1            # request 3: no text-dropped branch -> plain update
    rim[seg == 2] = -1            # request 2: sI 1.5 but no image-dropped row -> text CFG only
    rim[seg == 1] = -1
    x = torch.randn(M, C, device=DEV, generator=g)
    return dict(R=R, M=M, C=C, seg=seg, V=V, rm=rm, rtx=rtx, rim=rim, x=x, **p)


def _launch(c, x, ws=None, dt=0.037):
    ops = _ops()
    ws = ops.cfg_batch_workspace(c["M"], c["R"], DEV) if ws is None else ws
    ops.cfg_euler_step_batch(c["V"], _i32(c["seg"].tolist()), _i32(c["rm"].tolist()), _i32(c["rtx"].tolist()),
                             _i32(c["rim"].tolist()), x, ws, _f32(c["sT"]), _f32(c["sI"]), _f32(c["rmin"]),
                             _i32(c["rtype"]), _i32(c["on"]), _f32([dt]))


def _norm(t, **kw):
    """bf16 norm of a bf16 tensor from an exact (fp64) sum of squares: the kernel's fp32 sums differ from it by ~1e-6
    relative, so a norm flips by one bf16 ulp only next to a rounding boundary (a request's "global" norm covers
    thousands of elements, where a different fp32 order flips it far more often)."""
    return torch.norm(t.double(), **kw).to(torch.bfloat16)


def _host_step(c, dt=0.037):
    """bagel.py:873-907 + :746 per request, restated with torch bf16 tensor ops on the host like
    test_cfg_euler_matches_reference_arithmetic."""
    Vh = c["V"].cpu()
    x = c["x"].cpu().clone()
    names = ["global", "channel", "text_channel"]
    for q in range(c["R"]):
        r = torch.nonzero(c["seg"] == q).reshape(-1)
        v_ = Vh[c["rm"][r]]
        use = c["on"][q] and bool((c["rtx"][r] >= 0).all()) and c["sT"][q] > 1
        if not use:
            w = v_
        else:
            sT, rt = c["sT"][q], names[c["rtype"][q]]
            img = bool((c["rim"][r] >= 0).all()) and c["sI"][q] > 1
            sI = c["sI"][q]
            vT_ = Vh[c["rtx"][r]]
            vI_ = Vh[c["rim"][r]] if img else None
            u = vT_ + sT * (v_ - vT_)
            if rt == "text_channel":
                sc = (_norm(v_, dim=-1, keepdim=True) / (_norm(u, dim=-1, keepdim=True) + 1e-8)).clamp(
                    min=c["rmin"][q], max=1.0)
                ut = u * sc
                w = vI_ + sI * (ut - vI_) if img else ut
            else:
                w_ = vI_ + sI * (u - vI_) if img else u
                if rt == "global":
                    nv, nw = _norm(v_), _norm(w_)
                else:
                    nv, nw = _norm(v_, dim=-1, keepdim=True), _norm(w_, dim=-1, keepdim=True)
                w = w_ * (nv / (nw + 1e-8)).clamp(min=c["rmin"][q], max=1.0)
        x[r] = x[r] - w * torch.tensor(dt)
    return x


def test_cfg_batch_matches_per_request_host_arithmetic():
    c = _mixed_case()
    x = c["x"].clone()
    _launch(c, x)
    ref = _host_step(c)
    diff = (x.cpu() - ref).abs()
    # identical rounding points; only the fp32 sum-of-squares order differs, which can flip a bf16 norm by 1 ulp
    assert diff.max().item() <= 2e-3 and (diff > 0).float().mean().item() < 0.02
    # rows with CFG off or without a text-dropped branch take exactly x - bf16(v dt)
    plain = (c["seg"] == 3) | (c["seg"] == 5)
    v_plain = c["V"].cpu()[c["rm"][plain]].float()
    want = c["x"].cpu()[plain] - (v_plain * torch.tensor(0.037, dtype=torch.float32)).to(torch.bfloat16).float()
    assert torch.equal(x.cpu()[plain], want)


@pytest.mark.parametrize("rt", ["channel", "text_channel"])
@pytest.mark.parametrize("sI", [1.0, 1.5])
def test_cfg_batch_one_segment_is_bit_identical_to_cfg_euler_step(rt, sI):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(5)
    M, C = 1000, 64
    V = torch.randn(3 * (M + 20), C, device=DEV, generator=g).to(torch.bfloat16)    # three branch slabs of M + 20 rows
    x = torch.randn(M, C, device=DEV, generator=g)
    rows = torch.arange(10, 10 + M, device=DEV, dtype=torch.int32)                  # rows 10 .. M + 9 of each slab
    a = x.clone()
    ops.cfg_euler_step(V[:M + 20], V[M + 20:2 * M + 40], V[2 * M + 40:3 * M + 60] if sI > 1 else None, rows, a,
                       torch.zeros(2, device=DEV), 4.0, sI, 0.1, rt, 0.0, torch.tensor([0.037], device=DEV))
    b = x.clone()
    ops.cfg_euler_step_batch(V, torch.zeros(M, dtype=torch.int32, device=DEV), rows, rows + (M + 20),
                             rows + (2 * M + 40), b, ops.cfg_batch_workspace(M, 1, DEV), _f32([4.0]), _f32([sI]),
                             _f32([0.1]), _i32([ops.RENORM[rt]]), _i32([1]), _f32([0.037]))
    assert torch.equal(a, b)


def test_cfg_batch_determinism_and_graph_replay():
    ops = _ops()
    c = _mixed_case(seed=3)
    c["rtype"] = [0, 0, 0, 0, 1, 2]
    outs = []
    for _ in range(2):
        x = c["x"].clone()
        _launch(c, x)
        outs.append(x)
    assert torch.equal(outs[0], outs[1])
    # graph: device-resident parameters, captured once, replayed
    args = dict(seg=_i32(c["seg"].tolist()), rm=_i32(c["rm"].tolist()), rtx=_i32(c["rtx"].tolist()),
                rim=_i32(c["rim"].tolist()), sT=_f32(c["sT"]), sI=_f32(c["sI"]), rmin=_f32(c["rmin"]),
                rtype=_i32(c["rtype"]), on=_i32(c["on"]), dt=_f32([0.037]))
    ws = ops.cfg_batch_workspace(c["M"], c["R"], DEV)
    xg = c["x"].clone()

    def step():
        ops.cfg_euler_step_batch(c["V"], args["seg"], args["rm"], args["rtx"], args["rim"], xg, ws, args["sT"],
                                 args["sI"], args["rmin"], args["rtype"], args["on"], args["dt"])

    step()                 # warm
    xg.copy_(c["x"])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    xg.copy_(c["x"])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(xg, outs[0])


def test_cfg_batch_launches_do_not_grow_with_requests():
    from bagel_b200 import _cabi
    ops = _ops()
    counts = []
    for R in (1, 8, 64):
        M = 40 * R
        V = torch.randn(M, 64, device=DEV).to(torch.bfloat16)
        rows = torch.arange(M, dtype=torch.int32, device=DEV)
        seg = (rows // 40).contiguous()
        n0 = _cabi.launch_count()
        ops.cfg_euler_step_batch(V, seg, rows, rows, torch.full_like(rows, -1), torch.zeros(M, 64, device=DEV),
                                 ops.cfg_batch_workspace(M, R, DEV), torch.full((R,), 4.0, device=DEV),
                                 torch.ones(R, device=DEV), torch.zeros(R, device=DEV),
                                 torch.zeros(R, dtype=torch.int32, device=DEV), torch.ones(R, dtype=torch.int32, device=DEV),
                                 _f32([0.1]))
        counts.append(_cabi.launch_count() - n0)
    assert counts[0] == counts[1] == counts[2] == 3, counts


# ----------------------------------------------------------------------------------------------------------- sampler

@pytest.fixture(scope="module")
def tiny():
    return helpers.build_product_bagel(fixtures.TINY_LM, DEV)


def _t2i_batch(model, prompts, sizes, seeds, scales, renorm, intervals, steps=6):
    """T2I contexts for every request (main = [text], cfg_text empty, cfg_img = [text]) -> generate_image_batch."""
    from bagel_b200.qwen2_navit import NaiveCache
    R = len(prompts)
    L = model.config.llm_config.num_hidden_layers
    tok = helpers.IntTokenizer()
    gp, kv, rp = model.prepare_prompts([0] * R, [0] * R, prompts, tok, helpers.NEW_TOKEN_IDS)
    cache = model.forward_cache_update_text(NaiveCache(L), **gp)
    gp2, kv2, rp2 = model.prepare_prompts([0] * R, [0] * R, prompts, tok, helpers.NEW_TOKEN_IDS)
    cache_i = model.forward_cache_update_text(NaiveCache(L), **gp2)
    gi = model.prepare_vae_latent(kv, rp, sizes, helpers.NEW_TOKEN_IDS,
                                  generators=[torch.Generator().manual_seed(s) for s in seeds])
    ct = model.prepare_vae_latent_cfg([0] * R, [0] * R, sizes)
    ci = model.prepare_vae_latent_cfg(kv2, rp2, sizes)
    lat = model.generate_image_batch(
        past_key_values=cache, **gi, num_timesteps=steps, timestep_shift=3.0,
        cfg_text_scale=[s[0] for s in scales], cfg_img_scale=[s[1] for s in scales], cfg_interval=intervals,
        cfg_renorm_min=[0.0] * R, cfg_renorm_type=renorm,
        cfg_text_packed_position_ids=ct["cfg_packed_position_ids"],
        cfg_text_packed_query_indexes=ct["cfg_packed_query_indexes"], cfg_text_key_values_lens=ct["cfg_key_values_lens"],
        cfg_text_packed_key_value_indexes=ct["cfg_packed_key_value_indexes"], cfg_text_past_key_values=NaiveCache(L),
        cfg_img_packed_position_ids=ci["cfg_packed_position_ids"],
        cfg_img_packed_query_indexes=ci["cfg_packed_query_indexes"], cfg_img_key_values_lens=ci["cfg_key_values_lens"],
        cfg_img_packed_key_value_indexes=ci["cfg_packed_key_value_indexes"], cfg_img_past_key_values=cache_i)
    torch.cuda.synchronize()
    return [t.clone() for t in lat]


BASE = dict(prompts=["5 17 900 33 2", "8 8 100 4 77 650 12", "3 1 4 1 5", "9 2 6"],
            sizes=[(64, 64), (64, 96), (32, 64), (64, 32)], seeds=[1, 2, 3, 4],
            scales=[(4.0, 1.5), (4.0, 1.5), (3.0, 1.0), (4.0, 2.0)],
            renorm=["global", "global", "channel", "global"], intervals=[(0.4, 1.0)] * 4)


def _change(j, what):
    k = {key: list(v) for key, v in BASE.items()}
    if what == "seed":
        k["seeds"][j] = 99
    elif what == "prompt":
        k["prompts"][j] = " ".join(str((int(t) * 7 + 1) % 997) for t in k["prompts"][j].split())
    elif what == "scales":
        k["scales"][j] = (2.0, 1.25)
    elif what == "renorm":
        k["renorm"][j] = "text_channel"
    return k


@pytest.mark.parametrize("what", ["seed", "prompt", "scales", "renorm"])
def test_requests_are_independent(tiny, what):
    base = _t2i_batch(tiny, **BASE)
    j = 1
    other = _t2i_batch(tiny, **_change(j, what))
    assert not torch.equal(base[j], other[j]), "the change did not reach its own request"
    for q in range(4):
        if q != j:
            assert torch.equal(base[q], other[q]), (what, q)


@pytest.mark.parametrize("intervals,steps", [
    ([(0.4, 1.0), (0.0, 1.0), (0.4, 1.0), (0.6, 0.9)], 6),     # every step on the all-branch plan
    ([(0.6, 1.0), (0.6, 1.0), (0.6, 0.9), (0.7, 1.0)], 12),    # the last three steps (t <= 0.6) on the main plan
])
def test_graph_equals_eager(tiny, intervals, steps):
    from bagel_b200 import bagel as bmod
    keys = []
    orig = bmod.FlowRunner._launch

    def launch(self, key):
        keys.append(key)
        return orig(self, key)

    kw = dict(BASE, intervals=intervals, steps=steps)
    bmod.FlowRunner._launch = launch
    try:
        tiny.use_cuda_graph = True
        a = _t2i_batch(tiny, **kw)
        tiny.use_cuda_graph = False
        b = _t2i_batch(tiny, **kw)
    finally:
        tiny.use_cuda_graph = True
        bmod.FlowRunner._launch = orig
    _, _, cfg_on, full = bmod._flow_batch_schedule(steps, 3.0, intervals, [3, 3, 2, 3])
    assert keys == 2 * ["full" if f else "main" for f in full]
    if steps == 12:
        assert full.count(False) == 3      # main plan: eager, captured, replayed
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_one_graph_replay_per_step(tiny, monkeypatch):
    from bagel_b200 import _cabi
    replays = []
    orig = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), orig(self))[1])
    counts = {}
    from bagel_b200 import bagel as bmod
    orig_step = bmod.BatchFlowRunner.step

    def step(self, i):
        n0 = _cabi.launch_count()
        orig_step(self, i)
        counts.setdefault(len(self.st["sT"]), []).append(_cabi.launch_count() - n0)

    monkeypatch.setattr(bmod.BatchFlowRunner, "step", step)
    for R in (2, 4):
        kw = {k: v[:R] for k, v in BASE.items()}
        kw["intervals"] = [(0.0, 1.0)] * R
        n = len(replays)
        _t2i_batch(tiny, **kw, steps=10)
        assert len(replays) - n == 9 - 1        # step 0 eager, step 1 captured (+ one replay), then one replay each
        assert all(c == 0 for c in counts[R][2:]), counts[R]      # no launch outside the graph after warm-up


# --------------------------------------------------------------------------------------------------------- inferencer

@pytest.fixture(scope="module")
def gold():
    return load_file(os.path.join(os.path.dirname(__file__), "golden", "inferencer_tiny.safetensors"))


@pytest.fixture(scope="module")
def inferencer():
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV, max_latent_size=16, vae_downsample=2)
    vae = helpers.tiny_vae(DEV)
    vae.sample = False
    return InterleaveInferencer(model, vae, fixtures.ToyTokenizer(), ImageTransform(64, 32, 4), ImageTransform(112, 56, 14),
                                helpers.NEW_TOKEN_IDS)


def _cfg(kw):
    return {k: kw[k] for k in ("cfg_text_scale", "cfg_img_scale", "cfg_interval", "cfg_renorm_min", "cfg_renorm_type")}


def test_gen_image_batch_matches_reference_golden(inferencer, gold):
    steps = dict(num_timesteps=KW["num_timesteps"], timestep_shift=KW["timestep_shift"])
    imgs = inferencer.gen_image_batch([dict(text=TEXT, image_shapes=(32, 48), seed=21, **_cfg(KW)),
                                       dict(text=TEXT, image=fixtures.inferencer_image(), seed=22, **_cfg(KW))], **steps)
    assert imgs[0].size == (48, 32) and imgs[1].size == (56, 40)
    _check_image("batch t2i", imgs[0], gold["t2i.image"])
    _check_image("batch edit", imgs[1], gold["edit.image"])


def test_mixed_batch_matches_single_requests(inferencer):
    im = fixtures.inferencer_image()
    im2 = im.resize((40, 72))
    reqs = [
        dict(text=TEXT, image_shapes=(32, 48), seed=1),
        dict(text="8 8 100 4 77 650 12", image=im, seed=2, cfg_renorm_type="channel"),
        dict(text="3 1 4", image_shapes=(64, 32), seed=3, cfg_text_scale=1.0),
        dict(text=TEXT, image=im2, seed=4, cfg_img_scale=1.0, cfg_renorm_type="text_channel"),
        dict(text="9 2 6 5", image_shapes=(48, 48), seed=5, cfg_interval=(0.0, 0.7), cfg_renorm_type="text_channel"),
        dict(text="7 7 7", image=im, seed=6, cfg_interval=(0.0, 0.7), cfg_text_scale=2.0, cfg_img_scale=2.0),
        dict(text="1 2", image_shapes=(32, 32), seed=7, cfg_renorm_min=0.5),
    ]
    steps = dict(num_timesteps=6, timestep_shift=3.0)
    got = inferencer.gen_image_batch(reqs, **steps)
    for i, r in enumerate(reqs):
        r = dict(r)
        torch.manual_seed(r.pop("seed"))
        want = inferencer(image=r.pop("image", None), text=r.pop("text"), **r, **steps)["image"]
        assert got[i].size == want.size, (i, got[i].size, want.size)
        _check_image(f"request {i}", got[i], torch.from_numpy(np.asarray(want).copy()))


@pytest.fixture(scope="module")
def sampled(inferencer):
    """The same model with a VAE that samples its DiagonalGaussian (the VAE-encode noise of an edit is drawn)."""
    from bagel_b200.inferencer import InterleaveInferencer
    vae = helpers.tiny_vae(DEV)
    vae.sample = True
    return InterleaveInferencer(inferencer.model, vae, inferencer.tokenizer, inferencer.vae_transform,
                                inferencer.vit_transform, inferencer.new_token_ids)


def test_edit_encode_noise_is_the_single_request_draw(sampled):
    """_encode_image draws the noise torch.manual_seed(s) + forward_cache_update_vae's encode draws, and leaves the
    caller's CUDA RNG where it was."""
    from bagel_b200.transforms import pil_img2rgb
    m = sampled.model
    img = sampled.vae_transform.resize_transform(pil_img2rgb(fixtures.inferencer_image()))
    gi, _, _ = m.prepare_vae_images([0], [0], [img], sampled.vae_transform, helpers.NEW_TOKEN_IDS)
    torch.manual_seed(22)
    want = sampled.vae_model.encode(gi["padded_images"])[0]
    state = torch.cuda.get_rng_state()
    got = sampled._encode_image(sampled.vae_transform(img), 22)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert torch.equal(got, want)
    assert not torch.equal(sampled._encode_image(sampled.vae_transform(img), 23), want)


def test_sampled_vae_batch_matches_single_requests(sampled):
    steps = dict(num_timesteps=KW["num_timesteps"], timestep_shift=KW["timestep_shift"])
    reqs = [dict(text=TEXT, image=fixtures.inferencer_image(), seed=22, **_cfg(KW)),
            dict(text=TEXT, image_shapes=(32, 48), seed=21, **_cfg(KW)),
            dict(text="8 8 100 4", image=fixtures.inferencer_image().resize((40, 72)), seed=5, **_cfg(KW))]
    got = sampled.gen_image_batch(reqs, **steps)
    for i, r in enumerate(reqs):
        r = dict(r)
        torch.manual_seed(r.pop("seed"))
        want = sampled(image=r.pop("image", None), text=r.pop("text"), **r, **steps)["image"]
        assert got[i].size == want.size
        _check_image(f"sampled request {i}", got[i], torch.from_numpy(np.asarray(want).copy()))
