"""-m gpu: batched image understanding. The on-device sampler (bagel_sample_rows_bf16) against the NumPy Philox4x32-10 +
fp64 Gumbel restatement, its determinism, row independence and distribution; the per-request stop kernel
(bagel_decode_advance_stop) bit for bit; Bagel.chat_batch against sequential Bagel.chat and the reference's chat
output; per-request EOS; one graph replay per decode step."""
import random

import numpy as np
import pytest
import torch
from scipy import stats

import helpers
from oracle import fixtures
from sampling_oracle import gumbel_scores, philox4x32_10

pytestmark = pytest.mark.gpu
DEV = "cuda"
NT = dict(helpers.NEW_TOKEN_IDS)


def _ops():
    from bagel_b200 import ops
    return ops


def _keys(vals):
    return torch.from_numpy(np.array(vals, dtype=np.uint64).view(np.int64)).to(DEV)


# ------------------------------------------------------------------------------------------------------------- sampler

@pytest.mark.parametrize("V,ld", [(1024, 1024), (1031, 1031), (152064, 152072)])
@pytest.mark.parametrize("T", [1.0, 0.6, 2.5])
def test_sampler_matches_philox_gumbel_reference(V, ld, T):
    ops = _ops()
    B = 6
    g = torch.Generator().manual_seed(V + int(T * 10))
    logits = (torch.randn(B, ld, generator=g) * 2).to(torch.bfloat16).to(DEV)[:, :V]
    keys = [(0x1234 + 77 * i) | (i << 32) for i in range(B - 1)] + [0xDEADBEEFCAFEF00D]
    checked = 0
    for step in (0, 7, 123456):
        step_dev = torch.tensor([step], dtype=torch.int32, device=DEV)
        tok = torch.empty(B, dtype=torch.int64, device=DEV)
        tok32 = torch.empty(B, dtype=torch.int32, device=DEV)
        ops.sample_rows(logits, T, _keys(keys), step_dev, tok, tok32)
        got = tok.cpu().numpy()
        assert np.array_equal(got, tok32.cpu().numpy())
        lf = logits.float().cpu().numpy()
        for b in range(B):
            s = gumbel_scores(lf[b], T, keys[b], step)
            top2 = np.sort(s)[-2:]
            if top2[1] - top2[0] > 1e-5 * max(1.0, abs(top2[1])):
                assert got[b] == int(np.argmax(s)), (b, step)
                checked += 1
    assert checked >= 3 * B - 1


def test_sampler_largest_word_does_not_bypass_the_logits():
    """Key (seed 0x1234, request 0), step 28: the Philox word of logit j = 91538 is 0xffffff01. A uniform built from its
    top 24 bits, (2^24 - 1 + 0.5) * 2^-24, rounds to 1.0 in fp32 and gives that logit a score of +inf whatever its
    value. With the logit at -30 below all the others the draw must not land on it and must equal the reference pick."""
    ops = _ops()
    V, j, key, step = 152064, 91538, 0x1234, 28
    word = philox4x32_10(np.array([step, j >> 2, 0, 0], dtype=np.uint32), np.array([key, 0], dtype=np.uint32))[j & 3]
    assert int(word) >> 8 == 0xFFFFFF
    logits = torch.zeros(1, V, dtype=torch.bfloat16)
    logits[0, j] = -30.0
    step_dev = torch.tensor([step], dtype=torch.int32, device=DEV)
    for T in (1.0, 0.5):
        tok = torch.empty(1, dtype=torch.int64, device=DEV)
        ops.sample_rows(logits.to(DEV), T, _keys([key]), step_dev, tok)
        s = gumbel_scores(logits[0].float().numpy(), T, key, step)
        top2 = np.sort(s)[-2:]
        assert top2[1] - top2[0] > 1e-5 * max(1.0, abs(top2[1]))
        assert int(tok) != j and int(tok) == int(np.argmax(s)), (T, int(tok))


def test_sampler_determinism_and_graph_replay():
    ops = _ops()
    B, V = 5, 4096
    logits = torch.randn(B, V, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).to(DEV)
    keys = _keys([11 | (i << 32) for i in range(B)])
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    tok = torch.empty(B, dtype=torch.int64, device=DEV)

    def eager(step):
        step_dev.fill_(step)
        ops.sample_rows(logits, 0.9, keys, step_dev, tok)
        return tok.clone()

    eager(0)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.sample_rows(logits, 0.9, keys, step_dev, tok)
    draws = {}
    for step in (3, 9, 3, 10):
        want = eager(step)
        assert torch.equal(want, eager(step)), "same seed and step, same tokens"
        step_dev.fill_(step)
        tok.fill_(-1)
        graph.replay()
        assert torch.equal(tok, want), "graph replay equals eager"
        draws[step] = want
    assert not all(torch.equal(draws[3], draws[s]) for s in (9, 10)), "the step counter changes the draw"


def test_sampler_row_independence():
    ops = _ops()
    V = 2048
    g = torch.Generator().manual_seed(5)
    row = torch.randn(1, V, generator=g).to(torch.bfloat16).to(DEV)
    key = 987654321 | (3 << 32)
    step_dev = torch.tensor([17], dtype=torch.int32, device=DEV)
    alone = torch.empty(1, dtype=torch.int64, device=DEV)
    ops.sample_rows(row, 1.3, _keys([key]), step_dev, alone)
    for B, at in ((2, 1), (7, 4), (33, 0)):
        others = torch.randn(B, V, generator=g).to(torch.bfloat16).to(DEV)
        others[at] = row[0]
        keys = [random.Random(B).getrandbits(63) for _ in range(B)]
        keys[at] = key
        tok = torch.empty(B, dtype=torch.int64, device=DEV)
        ops.sample_rows(others, 1.3, _keys(keys), step_dev, tok)
        assert int(tok[at]) == int(alone[0]), (B, at)


@pytest.mark.parametrize("T", [0.7, 1.6])
def test_sampler_distribution_chi_square(T):
    """One 64-way row over 100 000 step counters: the draws follow softmax(l / T) (Pearson chi-square, 63 dof)."""
    ops = _ops()
    V, N = 64, 100_000
    lq = torch.empty(V).uniform_(-2.0, 2.0, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
    logits = lq.reshape(1, V).to(DEV)
    keys = _keys([4242 | (1 << 32)])
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = torch.empty(N, dtype=torch.int64, device=DEV)
    for s in range(N):
        ops.sample_rows(logits, T, keys, step_dev, out[s:s + 1])
        step_dev += 1
    counts = np.bincount(out.cpu().numpy(), minlength=V)
    p = torch.softmax(lq.double() / T, 0).numpy()
    expected = N * p
    assert expected.min() > 5
    chi2 = float(((counts - expected) ** 2 / expected).sum())
    pval = stats.chi2.sf(chi2, V - 1)
    assert pval > 1e-3, (chi2, pval)


# -------------------------------------------------------------------------------------------------------- stop kernel

@pytest.mark.parametrize("B", [1, 37, 1024])
def test_decode_advance_stop_bit_exact(B):
    ops = _ops()
    g = torch.Generator().manual_seed(B)
    max_length, end, pad = 6, 77, -1
    seq_len = torch.randint(0, 900, (B,), generator=g).to(torch.int32)
    pos = torch.randint(0, 5000, (B,), generator=g)
    tokens = torch.randint(0, 1000, (B,), generator=g)
    tokens32 = tokens.to(torch.int32)
    finished = (torch.rand(B, generator=g) < 0.2).to(torch.int32)
    history = torch.full((max_length, B), -9, dtype=torch.int64)
    m = dict(seq_len=seq_len, pos=pos, tokens=tokens, tokens32=tokens32, finished=finished, history=history)
    d = {k: v.to(DEV) for k, v in m.items()}
    m = {k: v.clone() for k, v in m.items()}
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    unfinished = torch.full((1,), -5, dtype=torch.int32, device=DEV)
    for step in range(max_length + 2):         # two steps past max_length: nothing is written out of range
        nxt = torch.where(torch.rand(B, generator=g) < 0.15, torch.full((B,), end), torch.randint(0, 1000, (B,), generator=g))
        ops.decode_advance_stop(d["seq_len"], d["pos"], d["tokens"], d["tokens32"], nxt.to(DEV), d["history"], step_dev,
                                d["finished"], unfinished, end, pad)
        for b in range(B):                     # Python model of the kernel
            if m["finished"][b]:
                if step < max_length:
                    m["history"][step, b] = pad
                continue
            if step < max_length:
                m["history"][step, b] = m["tokens"][b]
            if int(nxt[b]) == end or step + 1 >= max_length:
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
    assert int(unfinished) == 0


# ----------------------------------------------------------------------------------------------------------- chat_batch

def _img(seed, h, w):
    return torch.rand(3, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def _answer_tokens(text):
    inv = {v: k for k, v in fixtures.ToyTokenizer.SPECIAL.items()}
    return [inv[w] if w in inv else int(w) for w in text.split()]


def _seq_context(model, tok, imgs, prompt):
    """Bagel.chat's context for one request: (cache, kv len, rope position) before decoding."""
    from bagel_b200.qwen2_navit import NaiveCache
    cache, kv, rp = NaiveCache(model.config.llm_config.num_hidden_layers), [0], [0]
    for im in imgs:
        gi, kv, rp = model.prepare_vit_images(kv, rp, [im], lambda x: x, NT)
        cache = model.forward_cache_update_vit(cache, **gi)
    gi, kv, rp = model.prepare_prompts(kv, rp, [prompt], tok, NT)
    return model.forward_cache_update_text(cache, **gi), kv[0], rp[0]


def _margin(model, tok, req, prefix):
    """top-1 minus top-2 logit of sequential decoding after the inputs [bos] + prefix (teacher-forced)."""
    cache, kv, rp = _seq_context(model, tok, *req)
    ids = torch.tensor([NT["bos_token_id"]] + list(prefix))
    n = ids.numel()
    out = model.language_model.forward_inference(
        packed_query_sequence=model.language_model.model.embed_tokens(ids), query_lens=torch.tensor([n], dtype=torch.int32),
        packed_query_position_ids=torch.arange(rp, rp + n), packed_query_indexes=torch.arange(kv, kv + n),
        past_key_values=cache, key_values_lens=torch.tensor([kv], dtype=torch.int32),
        packed_key_value_indexes=torch.arange(kv), update_past_key_values=False, is_causal=True, mode="und")
    top2 = model.language_model.lm_head(out.packed_query_sequence[-1:]).float().topk(2).values[0]
    return float(top2[0] - top2[1])


def _check_against_sequential(model, reqs, max_length):
    tok = fixtures.ToyTokenizer()
    got = model.chat_batch(tok, NT, lambda x: x, reqs, max_length=max_length)
    assert len(got) == len(reqs)
    diverged = 0
    for i, req in enumerate(reqs):
        want = model.chat(tok, NT, lambda x: x, req[0], req[1], max_length=max_length)
        if got[i] == want:
            continue
        a, b = _answer_tokens(got[i]), _answer_tokens(want)
        s = next(k for k in range(max(len(a), len(b))) if k >= len(a) or k >= len(b) or a[k] != b[k])
        m = _margin(model, tok, req, b[:s])
        # the batched and the sequential run differ only by bf16 rounding (GEMM routes and decode-attention splits depend
        # on the batch); a different pick needs a top-2 margin within that noise
        assert m <= 0.07, f"request {i} diverged at answer token {s} with margin {m:.4f}"
        diverged += 1
    assert diverged <= len(reqs) // 4, f"{diverged} of {len(reqs)} requests diverged"
    return got


def test_chat_batch_matches_golden_and_sequential_chat(golden_dir):
    import os
    from safetensors.torch import load_file
    gold = load_file(os.path.join(golden_dir, "chat_tiny.safetensors"))
    want = bytes(gold["chat.text"].tolist()).decode("utf-8")
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, "cuda")
    reqs = [
        ([], "12 400 7"),
        ([_img(1, 28, 42)], "9 9 33"),
        (fixtures.vit_images(), "5 17 900 33 2 describe"),          # the reference's chat() golden request
        ([_img(2, 56, 28), _img(3, 14, 14)], "1 2 3 4 5 6 7 8"),
        ([_img(4, 42, 42)], "88"),
        ([], "300 301"),
    ]
    got = _check_against_sequential(model, reqs, max_length=8)
    assert got[2] == want, (got[2], want)


def test_chat_batch_80_requests_fused_qkv_decode():
    """80 requests: above 64 rows the decode step takes the fused QKV epilogue (head_dim 128)."""
    model = helpers.build_product_bagel_with_vit(fixtures.TINY128_LM, "cuda")
    rnd = random.Random(0)
    reqs = [([_img(rnd.randint(0, 10 ** 6), 14 * rnd.randint(1, 4), 14 * rnd.randint(1, 4))
              for _ in range(rnd.choice([0, 1, 1, 2]))],
             " ".join(str(rnd.randint(0, 999)) for _ in range(rnd.randint(1, 10)))) for _ in range(80)]
    _check_against_sequential(model, reqs, max_length=6)


def test_chat_batch_sampling_is_seeded():
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, "cuda")
    tok = fixtures.ToyTokenizer()
    reqs = [([], "1 2 3"), ([_img(7, 28, 28)], "4 5"), (fixtures.vit_images(), "6")]
    runs = []
    for _ in range(2):
        torch.manual_seed(123)
        runs.append(model.chat_batch(tok, NT, lambda x: x, reqs, max_length=10, do_sample=True, temperature=0.8))
    assert runs[0] == runs[1]
    a = model.chat_batch(tok, NT, lambda x: x, reqs, max_length=10, do_sample=True, temperature=0.8, seeds=[5, 6, 7])
    assert a == model.chat_batch(tok, NT, lambda x: x, reqs, max_length=10, do_sample=True, temperature=0.8,
                                 seeds=[5, 6, 7])


# ---------------------------------------------------------------------------------------------- stopping and launches

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


def _text_context(model, prompts):
    from bagel_b200.qwen2_navit import NaiveCache
    B = len(prompts)
    gi, kv, rp = model.prepare_prompts([0] * B, [0] * B, prompts, helpers.IntTokenizer(), NT)
    cache = model.forward_cache_update_text(NaiveCache(model.config.llm_config.num_hidden_layers), **gi)
    return cache, model.prepare_start_tokens(kv, rp, NT)


def _first_new(stream, lo=3):
    """(index, token) of the first token at index >= lo that does not occur earlier in the stream."""
    for k in range(lo, len(stream)):
        if stream[k] not in stream[:k]:
            return k, stream[k]
    raise AssertionError("no fresh token in the stream")


def test_per_request_eos():
    model = helpers.build_product_bagel(fixtures.TINY_LM, "cuda")
    prompts = ["5 17 900 33 2", "8 8 100 4 77 650 12", "1 2 3", "999 0 999"]
    cache, gs = _text_context(model, prompts)
    full = [t.tolist() for t in model.generate_text_batch(cache, max_length=24, **gs)]
    assert all(len(t) == 24 and t[0] == NT["bos_token_id"] for t in full)
    k, eos = _first_new(full[0])
    got = [t.tolist() for t in model.generate_text_batch(cache, max_length=24, end_token_id=eos, **gs)]
    for f, g in zip(full, got):
        assert g == (f[:f.index(eos)] if eos in f else f)
    assert got[0] == full[0][:k]
    assert max(len(g) for g in got) > len(got[0]), "the other requests continue after request 0 stops"


def test_loop_stops_soon_after_the_last_request(monkeypatch):
    model = helpers.build_product_bagel(fixtures.TINY_LM, "cuda")
    cache, gs = _text_context(model, ["8 8 100 4 77 650 12"] * 4)
    full = [t.tolist() for t in model.generate_text_batch(cache, max_length=40, **gs)]
    k, eos = _first_new(full[0])
    assert all(f == full[0] for f in full)
    model.use_cuda_graph = False
    rec = _record(monkeypatch)
    got = [t.tolist() for t in model.generate_text_batch(cache, max_length=40, end_token_id=eos, **gs)]
    assert got == [full[0][:k]] * 4
    steps = rec.calls.count("bagel_decode_advance_stop")
    assert k <= steps <= k + 2 * model.STOP_POLL - 1, (k, steps)


@pytest.mark.parametrize("do_sample", [False, True])
def test_one_graph_replay_per_decode_step(monkeypatch, do_sample):
    model = helpers.build_product_bagel(fixtures.TINY_LM, "cuda")
    cache, gs = _text_context(model, helpers.PROMPTS)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
    rec = _record(monkeypatch)
    n = 12
    out = model.generate_text_batch(cache, max_length=n, do_sample=do_sample, **gs)
    assert all(len(t) == n for t in out)
    L = fixtures.TINY_LM.num_hidden_layers
    ctx, calls = rec.calls[:2 * L], rec.calls[2 * L:]
    assert ctx == ["bagel_copy_rows_bf16"] * (2 * L)
    # step 0 eagerly, step 1 inside the capture, then no library call at all: every later step is one replay
    half = len(calls) // 2
    assert calls[:half] == calls[half:]
    pick = "bagel_sample_rows_bf16" if do_sample else "bagel_argmax_rows_bf16"
    assert calls[half - 2:half] == [pick, "bagel_decode_advance_stop"]
    # the capture replays once to run step 1, then steps 2 .. n-1 replay once each
    assert len(replays) == n - 1
