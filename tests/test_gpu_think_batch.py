"""-m gpu: batched interleaved requests. bagel_sample_rows_mixed_bf16 against bagel_sample_rows_bf16 /
bagel_argmax_rows_bf16 row by row, its determinism and graph replay; bagel_decode_advance_stop_limits against
bagel_decode_advance_stop and a host restatement; gather_requests; Bagel.generate_text_batch with per-request budgets,
sampling and temperatures; InterleaveInferencer.call_batch against sequential inferencer(...) calls and the reference's
inferencer golden, and its seeded sampling."""
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
NT = dict(helpers.NEW_TOKEN_IDS)


def _ops():
    from bagel_b200 import ops
    return ops


def _keys(vals):
    return torch.from_numpy(np.array(vals, dtype=np.uint64).view(np.int64)).to(DEV)


def _inv_t(temps):
    """0 for a greedy row, else 1.0f / T in fp32 (what the host hands the mixed kernel)."""
    return torch.from_numpy(np.array([0.0 if t is None else np.float32(1.0) / np.float32(t) for t in temps],
                                     dtype=np.float32)).to(DEV)


# ------------------------------------------------------------------------------------------------------- mixed sampler

@pytest.mark.parametrize("V,ld", [(1024, 1024), (1031, 1031), (152064, 152072)])
def test_mixed_sampler_equals_single_setting_kernels(V, ld):
    ops = _ops()
    temps = [None, 1.0, 0.3, None, 0.6, None, 2.5, 0.3, None, 1.0]      # None: greedy
    B = len(temps)
    g = torch.Generator().manual_seed(V)
    logits = (torch.randn(B, ld, generator=g) * 2).to(torch.bfloat16)
    logits[5] = float("nan")                       # an all-NaN greedy row and an all-NaN sampled row
    logits[9] = float("nan")
    logits[3, V // 2] = float("nan")               # a NaN among the values of a greedy row
    logits[1, 7] = float("-inf")
    logits = logits.to(DEV)[:, :V]
    keys = _keys([(0x1234 + 77 * i) | (i << 32) for i in range(B - 1)] + [0xDEADBEEFCAFEF00D])
    inv = _inv_t(temps)
    for step in (0, 7, 123456):
        step_dev = torch.tensor([step], dtype=torch.int32, device=DEV)
        tok = torch.full((B,), -7, dtype=torch.int64, device=DEV)
        tok32 = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        ops.sample_rows_mixed(logits, inv, keys, step_dev, tok, tok32)
        assert torch.equal(tok.to(torch.int32), tok32)
        greedy = torch.empty(B, dtype=torch.int64, device=DEV)
        ops.argmax_rows(logits, greedy)
        for b, t in enumerate(temps):
            if t is None:
                want = greedy[b]
            else:
                one = torch.empty(B, dtype=torch.int64, device=DEV)
                ops.sample_rows(logits, t, keys, step_dev, one)
                want = one[b]
            assert int(tok[b]) == int(want), (V, step, b, t)
        assert int(tok[5]) == 0 and int(tok[9]) == 0


def test_mixed_sampler_determinism_and_graph_replay():
    ops = _ops()
    B, V = 6, 4096
    logits = torch.randn(B, V, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).to(DEV)
    keys = _keys([11 | (i << 32) for i in range(B)])
    inv = _inv_t([0.9, None, 0.3, None, 1.7, 0.9])
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    tok = torch.empty(B, dtype=torch.int64, device=DEV)

    def eager(step):
        step_dev.fill_(step)
        ops.sample_rows_mixed(logits, inv, keys, step_dev, tok)
        return tok.clone()

    eager(0)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.sample_rows_mixed(logits, inv, keys, step_dev, tok)
    draws = {}
    for step in (3, 9, 3, 10):
        want = eager(step)
        assert torch.equal(want, eager(step)), "same keys and step, same tokens"
        step_dev.fill_(step)
        tok.fill_(-1)
        graph.replay()
        assert torch.equal(tok, want), "graph replay equals eager"
        draws[step] = want
    assert all(int(draws[s][1]) == int(draws[3][1]) for s in (9, 10)), "a greedy row ignores the step"
    assert not all(torch.equal(draws[3], draws[s]) for s in (9, 10)), "the step counter changes the sampled rows"


# ------------------------------------------------------------------------------------------------------- limits kernel

def _stop_state(B, seed, rows):
    g = torch.Generator().manual_seed(seed)
    m = dict(seq_len=torch.randint(0, 900, (B,), generator=g).to(torch.int32),
             pos=torch.randint(0, 5000, (B,), generator=g),
             tokens=torch.randint(0, 1000, (B,), generator=g),
             finished=(torch.rand(B, generator=g) < 0.2).to(torch.int32),
             history=torch.full((rows, B), -9, dtype=torch.int64))
    m["tokens32"] = m["tokens"].to(torch.int32)
    return m, g


@pytest.mark.parametrize("B", [1, 37, 1024])
def test_limits_kernel_with_equal_limits_is_decode_advance_stop(B):
    ops = _ops()
    rows, end, pad = 6, 77, -1
    m, g = _stop_state(B, B, rows)
    a = {k: v.to(DEV) for k, v in m.items()}
    b = {k: v.to(DEV) for k, v in m.items()}
    sa, sb = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    ua, ub = torch.full((1,), -5, dtype=torch.int32, device=DEV), torch.full((1,), -5, dtype=torch.int32, device=DEV)
    lim = torch.full((B,), rows, dtype=torch.int32, device=DEV)
    for step in range(rows + 2):
        nxt = torch.where(torch.rand(B, generator=g) < 0.15, torch.full((B,), end),
                          torch.randint(0, 1000, (B,), generator=g)).to(DEV)
        ops.decode_advance_stop(a["seq_len"], a["pos"], a["tokens"], a["tokens32"], nxt, a["history"], sa,
                                a["finished"], ua, end, pad)
        ops.decode_advance_stop_limits(b["seq_len"], b["pos"], b["tokens"], b["tokens32"], nxt, b["history"], sb,
                                       b["finished"], ub, end, lim, pad)
        for k in a:
            assert torch.equal(a[k], b[k]), (step, k)
        assert torch.equal(sa, sb) and torch.equal(ua, ub)


@pytest.mark.parametrize("B", [5, 300])
def test_limits_kernel_matches_host_restatement(B):
    ops = _ops()
    rows, end, pad = 9, 77, -1
    m, g = _stop_state(B, 100 + B, rows)
    limits = torch.randint(1, rows + 3, (B,), generator=g).to(torch.int32)     # some beyond the history
    d = {k: v.to(DEV) for k, v in m.items()}
    m = {k: v.clone() for k, v in m.items()}
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    unfinished = torch.full((1,), -5, dtype=torch.int32, device=DEV)
    for step in range(rows + 3):
        nxt = torch.where(torch.rand(B, generator=g) < 0.1, torch.full((B,), end),
                          torch.randint(0, 1000, (B,), generator=g))
        ops.decode_advance_stop_limits(d["seq_len"], d["pos"], d["tokens"], d["tokens32"], nxt.to(DEV), d["history"],
                                       step_dev, d["finished"], unfinished, end, limits.to(DEV), pad)
        for b in range(B):
            if m["finished"][b]:
                if step < rows:
                    m["history"][step, b] = pad
                continue
            if step < rows:
                m["history"][step, b] = m["tokens"][b]
            if int(nxt[b]) == end or step + 1 >= int(limits[b]):
                m["finished"][b] = 1
            else:
                m["seq_len"][b] += 1
                m["pos"][b] += 1
                m["tokens"][b] = nxt[b]
                m["tokens32"][b] = int(nxt[b])
        for k in m:
            assert torch.equal(d[k].cpu(), m[k]), (step, k)
        assert int(step_dev) == step + 1
        assert int(unfinished) == int((m["finished"] == 0).sum())


# ------------------------------------------------------------------------------------------------------ gather + decode

def test_gather_requests_copies_the_member_blocks():
    from bagel_b200.qwen2_navit import NaiveCache, gather_requests
    L, kv = 3, [5, 0, 7, 2, 4]
    c = NaiveCache(L)
    for li in range(L):
        c.key_cache[li] = torch.randn(sum(kv), 2, 64, device=DEV).to(torch.bfloat16)
        c.value_cache[li] = torch.randn(sum(kv), 2, 64, device=DEV).to(torch.bfloat16)
    start = np.cumsum([0] + kv)
    for members in ([3, 0], [2], [0, 1, 4], [4, 3, 2, 1, 0]):
        idx = torch.cat([torch.arange(start[q], start[q] + kv[q]) for q in members]).to(DEV)
        g = gather_requests(c, kv, members)
        for li in range(L):
            assert torch.equal(g.key_cache[li], c.key_cache[li][idx]) and torch.equal(g.value_cache[li], c.value_cache[li][idx])


@pytest.fixture(scope="module")
def tiny():
    return helpers.build_product_bagel(fixtures.TINY_LM, DEV)


def _text_context(model, prompts):
    from bagel_b200.qwen2_navit import NaiveCache
    B = len(prompts)
    gi, kv, rp = model.prepare_prompts([0] * B, [0] * B, prompts, helpers.IntTokenizer(), NT)
    cache = model.forward_cache_update_text(NaiveCache(model.config.llm_config.num_hidden_layers), **gi)
    return cache, model.prepare_start_tokens(kv, rp, NT)


PROMPTS = ["5 17 900 33 2", "8 8 100 4 77 650 12", "1 2 3", "999 0 999"]


def test_per_request_budgets_sampling_and_end_tokens(tiny):
    """Each row of a per-request decode is the row the scalar decode with its own setting gives, cut at its own budget
    or at the end token."""
    cache, gs = _text_context(tiny, PROMPTS)
    seeds = [5, 6, 7, 8]
    greedy = [t.tolist() for t in tiny.generate_text_batch(cache, max_length=24, **gs)]
    sampled = {T: [t.tolist() for t in tiny.generate_text_batch(cache, max_length=24, do_sample=True, temperature=T,
                                                                   seeds=seeds, **gs)] for T in (0.7, 1.3)}
    eos = next(t for t in greedy[0][3:] if t not in greedy[0][:3])
    settings = [(None, 5), (0.7, 24), (None, 24), (1.3, 11)]        # (temperature or greedy, budget)
    got = [t.tolist() for t in tiny.generate_text_batch(
        cache, max_length=[n for _, n in settings], do_sample=[t is not None for t, _ in settings],
        temperature=[t or 1.0 for t, _ in settings], end_token_id=eos, seeds=seeds, **gs)]
    for q, (T, n) in enumerate(settings):
        full = (greedy if T is None else sampled[T])[q][:n]
        want = full[:full.index(eos)] if eos in full else full
        assert got[q] == want, (q, got[q], want)
    # explicit keys: a request's draws follow its key, not its index (rows 0 and 2 share a prompt)
    cache, gs = _text_context(tiny, ["1 2 3", "5 6", "1 2 3"])
    kw = dict(max_length=[12] * 3, do_sample=True, temperature=0.7)
    row = [t.tolist() for t in tiny.generate_text_batch(cache, keys=[99, 5, 99], **kw, **gs)]
    assert row[0] == row[2]
    assert row[0] != [t.tolist() for t in tiny.generate_text_batch(cache, keys=[98, 5, 99], **kw, **gs)][0]


class _Recorder:
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


def _record(monkeypatch):
    from bagel_b200 import _cabi
    rec = _Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    return rec


def test_mixed_decode_step_is_one_graph_replay(tiny, monkeypatch):
    cache, gs = _text_context(tiny, PROMPTS)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
    rec = _record(monkeypatch)
    n = 12
    out = tiny.generate_text_batch(cache, max_length=[n, 5, n, 9], do_sample=[False, True, True, False],
                                   temperature=[1.0, 0.3, 0.8, 1.0], **gs)
    assert [len(t) for t in out] == [n, 5, n, 9]
    L = fixtures.TINY_LM.num_hidden_layers
    ctx, calls = rec.calls[:2 * L], rec.calls[2 * L:]
    assert ctx == ["bagel_copy_rows_bf16"] * (2 * L)
    half = len(calls) // 2
    assert calls[:half] == calls[half:]
    assert calls[half - 2:half] == ["bagel_sample_rows_mixed_bf16", "bagel_decode_advance_stop_limits"]
    assert len(replays) == n - 1


def test_mixed_loop_stops_soon_after_the_last_request(tiny, monkeypatch):
    cache, gs = _text_context(tiny, PROMPTS)
    tiny.use_cuda_graph = False
    try:
        rec = _record(monkeypatch)
        limits = [3, 9, 5, 4]
        never = fixtures.TINY_LM.vocab_size + 5
        out = tiny.generate_text_batch(cache, max_length=[40] + limits[1:], do_sample=[False, True, False, True],
                                       temperature=0.5, end_token_id=never, **gs)
        assert [len(t) for t in out] == [40] + limits[1:]
        rec.calls.clear()
        out = tiny.generate_text_batch(cache, max_length=limits, do_sample=[False, True, False, True],
                                       temperature=0.5, end_token_id=never, **gs)
        assert [len(t) for t in out] == limits
        steps = rec.calls.count("bagel_decode_advance_stop_limits")
        k = max(limits)
        assert k <= steps <= k + 2 * tiny.STOP_POLL - 1, (k, steps)
    finally:
        tiny.use_cuda_graph = True


# ---------------------------------------------------------------------------------------------------------- call_batch

@pytest.fixture(scope="module")
def inferencer():
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV, max_latent_size=16, vae_downsample=2)
    vae = helpers.tiny_vae(DEV)
    vae.sample = False
    return InterleaveInferencer(model, vae, fixtures.ToyTokenizer(), ImageTransform(64, 32, 4), ImageTransform(112, 56, 14),
                                helpers.NEW_TOKEN_IDS)


STEPS = dict(num_timesteps=KW["num_timesteps"], timestep_shift=KW["timestep_shift"])


def _single(inf, r):
    r = dict(r)
    torch.manual_seed(r.pop("seed"))
    return inf(image=r.pop("image", None), text=r.pop("text", None), **r, **STEPS)


def _tokens(text):
    inv = {v: k for k, v in fixtures.ToyTokenizer.SPECIAL.items()}
    return [inv[w] if w in inv else int(w) for w in text.split()]


def _margin(inf, r, prefix):
    """top-1 minus top-2 logit of the single-request decode of r after [bos] + prefix (teacher-forced), on the
    context interleave_inference builds for it."""
    from bagel_b200.inferencer import GEN_THINK_SYSTEM_PROMPT, VLM_THINK_SYSTEM_PROMPT
    from bagel_b200.transforms import pil_img2rgb
    und = r.get("understanding_output", False)
    torch.manual_seed(r["seed"])
    ctx = inf.init_gen_context()
    if r.get("think"):
        ctx = inf.update_context_text(VLM_THINK_SYSTEM_PROMPT if und else GEN_THINK_SYSTEM_PROMPT, ctx)
    if r.get("image") is not None:
        ctx = inf.update_context_image(inf.vae_transform.resize_transform(pil_img2rgb(r["image"])), ctx, vae=not und)
    if r.get("text") is not None:
        ctx = inf.update_context_text(r["text"], ctx)
    m = inf.model
    kv, rp = ctx["kv_lens"][0], ctx["ropes"][0]
    ids = torch.tensor([NT["bos_token_id"]] + list(prefix))
    n = ids.numel()
    out = m.language_model.forward_inference(
        packed_query_sequence=m.language_model.model.embed_tokens(ids), query_lens=torch.tensor([n], dtype=torch.int32),
        packed_query_position_ids=torch.arange(rp, rp + n), packed_query_indexes=torch.arange(kv, kv + n),
        past_key_values=ctx["past_key_values"], key_values_lens=torch.tensor([kv], dtype=torch.int32),
        packed_key_value_indexes=torch.arange(kv), update_past_key_values=False, is_causal=True, mode="und")
    top2 = m.language_model.lm_head(out.packed_query_sequence[-1:]).float().topk(2).values[0]
    return float(top2[0] - top2[1])


def _check_against_sequential(inf, reqs):
    got = inf.call_batch(reqs, **STEPS)
    assert len(got) == len(reqs)
    forked = 0
    for q, r in enumerate(reqs):
        want = _single(inf, r)
        assert (got[q]["text"] is None) == (want["text"] is None), q
        assert (got[q]["image"] is None) == (want["image"] is None), q
        same_text = got[q]["text"] == want["text"]
        if not same_text:
            a, b = _tokens(got[q]["text"]), _tokens(want["text"])
            s = next(k for k in range(max(len(a), len(b))) if k >= len(a) or k >= len(b) or a[k] != b[k])
            mg = _margin(inf, r, b[:s])
            # batched and sequential runs differ only by bf16 rounding (GEMM routes and decode-attention splits depend
            # on the batch); a different pick needs a top-2 margin within that noise
            assert mg <= 0.07, f"request {q} forked at text token {s} with margin {mg:.4f}"
            forked += 1
        if want["image"] is not None and same_text:
            assert got[q]["image"].size == want["image"].size, q
            _check_image(f"request {q}", got[q]["image"], torch.from_numpy(np.asarray(want["image"]).copy()))
    assert forked <= len(reqs) // 4, f"{forked} of {len(reqs)} requests forked"
    return got


def test_mixed_batch_matches_sequential_calls(inferencer):
    im = fixtures.inferencer_image()
    im2 = im.resize((40, 72))
    reqs = [
        dict(text=TEXT, image_shapes=(32, 48), seed=1, cfg_text_scale=4.0),                                    # T2I
        dict(text="8 8 100 4", think=True, max_think_token_n=5, image_shapes=(48, 32), seed=2,
             cfg_renorm_type="channel"),                                                                       # T2I + think
        dict(text="3 1 4", image=im, seed=3, cfg_img_scale=2.0, cfg_renorm_type="text_channel"),                # edit
        dict(text=TEXT, image=im2, think=True, max_think_token_n=7, seed=4, cfg_interval=(0.0, 0.7)),          # edit + think
        dict(text="9 2 6", image=im, understanding_output=True, max_think_token_n=6, seed=5),                  # understanding
        dict(text="7 7 7", image=im2, understanding_output=True, think=True, max_think_token_n=9, seed=6),     # und + think
        dict(text="12 400 7", understanding_output=True, max_think_token_n=4, seed=7),                         # text only
        dict(seed=8),                                                                                          # nothing
    ]
    got = _check_against_sequential(inferencer, reqs)
    assert got[7] == {"image": None, "text": None}
    # each text stops at its own budget at the latest: start token + at most max_think_token_n - 1 tokens
    for q, r in enumerate(reqs):
        if got[q]["text"] is not None:
            assert len(_tokens(got[q]["text"])) <= r["max_think_token_n"] - 1, q


def test_golden_think_and_understanding_inside_a_batch(inferencer):
    gold = load_file(os.path.join(os.path.dirname(__file__), "golden", "inferencer_tiny.safetensors"))
    cfg = {k: KW[k] for k in ("cfg_text_scale", "cfg_img_scale", "cfg_interval", "cfg_renorm_min", "cfg_renorm_type")}
    reqs = [
        dict(text="5 5 5", image_shapes=(32, 32), seed=3),
        dict(text=TEXT, think=True, max_think_token_n=5, do_sample=False, image_shapes=(32, 48), seed=24, **cfg),
        dict(image=fixtures.inferencer_image(), text=TEXT, understanding_output=True, max_think_token_n=6,
             do_sample=False, seed=23),
        dict(text=TEXT, image_shapes=(32, 48), seed=21, **cfg),
    ]
    got = inferencer.call_batch(reqs, **STEPS)
    _check_image("t2i in a think batch", got[3]["image"], gold["t2i.image"])
    forks = []
    for name, q in (("think", 1), ("und", 2)):
        mine = _tokens(got[q]["text"])
        ref = _tokens(bytes(gold[f"{name}.text"].tolist()).decode("utf-8"))
        print(name, "tokens", mine, "reference", ref)
        assert len(mine) == len(ref) and mine[:2] == ref[:2], (name, mine, ref)
        if mine != ref:
            forks.append(name)
        elif name == "think":
            _check_image("think in a batch", got[q]["image"], gold["think.image"])
    if forks:
        pytest.xfail(f"greedy continuation forked on a bf16 tie: {forks}")


SAMPLED = [
    dict(text="5 17 900 33 2", image=None, understanding_output=True, max_think_token_n=10, do_sample=True,
         text_temperature=0.8, seed=11),
    dict(text="8 8 100 4", think=True, max_think_token_n=8, do_sample=True, text_temperature=0.8,
         image_shapes=(32, 32), seed=12),
    dict(text="3 1 4 1 5", image="IMG", understanding_output=True, think=True, max_think_token_n=9, do_sample=True,
         text_temperature=1.2, seed=13),
    dict(text="9 2 6", think=True, max_think_token_n=6, do_sample=True, text_temperature=0.3,
         image_shapes=(32, 48), seed=14),
]


def _sampled(changes=None, order=None):
    reqs = [dict(r, image=fixtures.inferencer_image() if r["image"] == "IMG" else None) if "image" in r else dict(r)
            for r in SAMPLED]
    for q, ch in (changes or {}).items():
        reqs[q].update(ch)
    return [reqs[q] for q in (order or range(len(reqs)))]


def _same(a, b, q, exact_image=True):
    assert a["text"] == b["text"], (q, a["text"], b["text"])
    if a["image"] is None:
        assert b["image"] is None
    elif exact_image:
        assert np.array_equal(np.asarray(a["image"]), np.asarray(b["image"])), q
    else:
        _check_image(f"request {q}", a["image"], torch.from_numpy(np.asarray(b["image"]).copy()))


def test_sampled_requests_are_seeded_and_independent(inferencer):
    base = inferencer.call_batch(_sampled(), **STEPS)
    again = inferencer.call_batch(_sampled(), **STEPS)
    for q in range(len(SAMPLED)):
        _same(base[q], again[q], q)
    assert len({r["text"] for r in base}) == len(SAMPLED)
    # permuting the batch permutes the outputs
    order = [2, 0, 3, 1]
    perm = inferencer.call_batch(_sampled(order=order), **STEPS)
    for k, q in enumerate(order):
        _same(perm[k], base[q], q, exact_image=False)
    # another request's seed or prompt (same length: the same batch shapes) leaves a request unchanged
    for changes in ({1: dict(seed=99)}, {1: dict(text="7 7 100 5")}):
        other = inferencer.call_batch(_sampled(changes), **STEPS)
        # (the random tiny model's logits in this context are so peaked that its thought may not change with the seed;
        # its init noise does)
        assert other[1]["text"] != base[1]["text"] or not np.array_equal(np.asarray(other[1]["image"]),
                                                                         np.asarray(base[1]["image"])), \
            "the change did not reach its own request"
        for q in (0, 2, 3):
            _same(other[q], base[q], q)
