"""-m gpu: decode-step penalties. bagel_apply_penalties_bf16 driven over many steps with its incremental state against
the NumPy penalty oracle, bit for bit (B up to 128, V = 152064 with a padded ld and V = 1031, repetitive streams,
rows that finish partway, rows with penalties off, step 0, every combination of the three penalties);
Bagel.generate_text_batch on the tiny model eager (each step's logits before and after the kernel against the oracle,
greedy picks) and captured; penalties off change nothing; one graph replay per step; chat_batch and call_batch give a
request the same text in a batch as alone."""
import numpy as np
import pytest
import torch

import helpers
import penalty_oracle as po
from oracle import fixtures

pytestmark = pytest.mark.gpu
DEV = "cuda"
NT = dict(helpers.NEW_TOKEN_IDS)


def _ops():
    from bagel_b200 import ops
    return ops


def _f32(vals):
    return torch.tensor(vals, dtype=torch.float32, device=DEV)


# (repetition, frequency, presence): every combination of the three on / off, with different values
COMBOS = [(1.0, 0.0, 0.0), (1.05, 0.0, 0.0), (1.0, 0.7, 0.0), (1.0, 0.0, -1.5), (0.8, -0.3, 0.0), (1.3, 0.0, 0.4),
          (1.0, 2.0, 2.0), (1 / 1.05, -2.0, -0.25), (2.5, 0.1, 1.0)]


def _streams(B, S, V, rng):
    """Per row: the tokens fed at steps 0..S-1 (step 0's is the start token) and the step after which the row is
    finished (S: never). Even rows repeat a few tokens heavily; every third row finishes partway."""
    toks, fin = [], []
    for b in range(B):
        pool = rng.integers(0, V, 1 + b % 4) if b % 2 == 0 else np.arange(V)
        s = rng.choice(pool, S)
        s[0] = rng.integers(0, V)
        toks.append(s)
        fin.append(int(rng.integers(1, S - 1)) if b % 3 == 1 else S)
    return np.array(toks), fin


def _logits(B, V, ld, gen):
    x = torch.randn(B, ld, generator=gen) * 4
    x[:, ::97] = 0.0
    x[:, 5::211] = float("-inf")
    x[:, 11::307] = float("nan")
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("B,V,ld,S", [(128, 152064, 152072, 24), (37, 1031, 1031, 80), (5, 1031, 1040, 200)])
def test_kernel_matches_oracle_over_steps(B, V, ld, S):
    ops = _ops()
    rng = np.random.default_rng(B)
    gen = torch.Generator().manual_seed(V)
    stream, fin = _streams(B, S, V, rng)
    settings = [COMBOS[b % len(COMBOS)] for b in range(B)]
    rp, fp, pp = (_f32([s[i] for s in settings]) for i in range(3))
    seen = ops.penalty_state(B, S, DEV)
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    for step in range(S):
        # a finished row keeps the token it had when it finished, as decode_advance_stop leaves it
        fed = [stream[b, min(step, fin[b])] for b in range(B)]
        tokens = torch.tensor(fed, dtype=torch.int64, device=DEV)
        finished = torch.tensor([int(step > fin[b]) for b in range(B)], dtype=torch.int32, device=DEV)
        step_dev.fill_(step)
        before = _logits(B, V, ld, gen)
        full = before.to(DEV)
        ops.apply_penalties(full[:, :V], rp, fp, pp, tokens, finished, step_dev, seen)
        full = full.cpu()
        after = full[:, :V]
        assert torch.equal(po.bits(full[:, V:]), po.bits(before[:, V:])), "the padding of a row changed"
        for b in range(B):
            g = stream[b, 1:min(step, fin[b]) + 1]
            want = po.apply(before[b, :V], g, *settings[b])
            assert torch.equal(po.bits(after[b]), po.bits(want)), (step, b, settings[b])
            if step == 0 or po.is_off(*settings[b]):
                assert torch.equal(po.bits(after[b]), po.bits(before[b, :V])), (step, b)
    # the state holds each penalised row's distinct tokens and their counts
    st = seen.cpu().numpy()
    for b in range(B):
        if po.is_off(*settings[b]):
            assert st[b, 0] == 0
            continue
        ids, counts = np.unique(stream[b, 1:min(S - 1, fin[b]) + 1], return_counts=True)
        n = st[b, 0]
        assert n == ids.size
        got = dict(zip(st[b, 1:1 + n], st[b, 1 + S:1 + S + n]))
        assert got == dict(zip(ids, counts))


def test_kernel_replays_in_a_graph():
    ops = _ops()
    B, V, S = 6, 1031, 12
    rng = np.random.default_rng(3)
    stream, _ = _streams(B, S, V, rng)
    rp, fp, pp = (_f32([COMBOS[b + 1][i] for b in range(B)]) for i in range(3))
    before = _logits(B, V, V, torch.Generator().manual_seed(1)).to(DEV)
    logits = before.clone()
    tokens = torch.tensor(stream[:, 0], dtype=torch.int64, device=DEV)
    finished = torch.zeros(B, dtype=torch.int32, device=DEV)
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    seen = ops.penalty_state(B, S, DEV)
    ops.apply_penalties(logits, rp, fp, pp, tokens, finished, step_dev, seen)     # step 0, eager
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.apply_penalties(logits, rp, fp, pp, tokens, finished, step_dev, seen)
    for step in range(1, S):
        logits.copy_(before)
        tokens.copy_(torch.from_numpy(stream[:, step]))
        step_dev.fill_(step)
        graph.replay()
        got = logits.cpu()
        for b in range(B):
            want = po.apply(before[b].cpu(), stream[b, 1:step + 1], *(COMBOS[b + 1]))
            assert torch.equal(po.bits(got[b]), po.bits(want)), (step, b)


# ------------------------------------------------------------------------------------------------------- end to end

@pytest.fixture(scope="module")
def tiny():
    return helpers.build_product_bagel(fixtures.TINY_LM, DEV)


def _text_context(model, prompts):
    from bagel_b200.qwen2_navit import NaiveCache
    B = len(prompts)
    gi, kv, rp = model.prepare_prompts([0] * B, [0] * B, prompts, helpers.IntTokenizer(), NT)
    cache = model.forward_cache_update_text(NaiveCache(model.config.llm_config.num_hidden_layers), **gi)
    return cache, model.prepare_start_tokens(kv, rp, NT)


PROMPTS = ["5 17 900 33 2", "8 8 100 4 77 650 12", "1 2 3", "999 0 999", "4 4 4 4", "31 41 59 26 53"]
PEN = dict(repetition_penalty=[1.3, None, 1.05, 0.9, 2.0, 1.0], presence_penalty=[0.0, 1.5, None, -0.5, 0.3, 0.0],
           frequency_penalty=[0.5, 0.0, 0.2, None, -1.0, 0.0])
MIXED = dict(do_sample=[False, True, False, True, True, False], temperature=[1.0, 1.4, 1.0, 0.8, 1.2, 1.0],
             top_p=[None, 0.9, None, None, 0.8, None], max_length=[24, 24, 10, 24, 17, 24], end_token_id=7)


def _settings():
    """PEN per request as (repetition, frequency, presence), off values for None."""
    return [(1.0 if r is None else r, 0.0 if f is None else f, 0.0 if p is None else p)
            for r, f, p in zip(PEN["repetition_penalty"], PEN["frequency_penalty"], PEN["presence_penalty"])]


def _gen(model, cache, gs, **kw):
    kw = dict(dict(max_length=20, seeds=[5, 6, 7, 8, 9, 10]), **kw)
    return [t.tolist() for t in model.generate_text_batch(cache, **kw, **gs)]


def test_eager_steps_equal_the_oracle(tiny, monkeypatch):
    from bagel_b200 import ops
    cache, gs = _text_context(tiny, PROMPTS)
    records = []
    real = ops.apply_penalties

    def recording(logits, *args):
        before = logits.cpu()
        real(logits, *args)
        records.append((before, logits.cpu()))
    monkeypatch.setattr(ops, "apply_penalties", recording)
    tiny.use_cuda_graph = False
    try:
        eager = _gen(tiny, cache, gs, **MIXED, **PEN)
    finally:
        tiny.use_cuda_graph = True
    monkeypatch.setattr(ops, "apply_penalties", real)
    assert len(records) >= max(MIXED["max_length"]) - 1
    settings = _settings()
    checked = 0
    for step, (before, after) in enumerate(records):
        for b, out in enumerate(eager):
            # tokens fed at steps 1..step, frozen once the request finished (its output has len(out) - 1 of them)
            g = out[1:min(step, len(out) - 1) + 1]
            want = po.apply(before[b], g, *settings[b])
            assert torch.equal(po.bits(after[b]), po.bits(want)), (step, b)
            if not MIXED["do_sample"][b] and step + 1 < len(out):
                assert int(torch.argmax(after[b].float())) == out[step + 1], (step, b)
                checked += 1
            if step and g and not po.is_off(*settings[b]) and not torch.equal(after[b], before[b]):
                checked += 1
    assert checked > 30
    # the penalties change something, and the captured run gives the same tokens
    assert eager != _gen(tiny, cache, gs, **MIXED)
    assert _gen(tiny, cache, gs, **MIXED, **PEN) == eager


def test_penalties_off_change_nothing(tiny):
    cache, gs = _text_context(tiny, PROMPTS)
    B = len(PROMPTS)
    offs = (dict(repetition_penalty=None, presence_penalty=None, frequency_penalty=None),
            dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0),
            dict(repetition_penalty=[1.0] * B, presence_penalty=[None] * B, frequency_penalty=[0.0] * B))
    for run in (dict(), dict(do_sample=True, temperature=1.3), dict(do_sample=True, temperature=1.3, top_k=5,
                                                                     top_p=0.9), MIXED):
        plain = _gen(tiny, cache, gs, **run)
        for off in offs:
            assert _gen(tiny, cache, gs, **run, **off) == plain, (run, off)
    # requests with penalties off keep their tokens while the others set them
    plain = _gen(tiny, cache, gs, **MIXED)
    pen = _gen(tiny, cache, gs, **MIXED, **PEN)
    for b, setting in enumerate(_settings()):
        if po.is_off(*setting):
            assert pen[b] == plain[b], b
    assert pen != plain


def test_off_penalties_launch_what_no_penalties_launch(tiny, monkeypatch):
    from bagel_b200 import _cabi
    cache, gs = _text_context(tiny, PROMPTS[:3])
    tiny.generate_text_batch(cache, max_length=6, do_sample=True, temperature=0.9, **gs)    # sizes every workspace
    lib = _cabi.lib()
    seqs = []
    for kw in (dict(), dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=[0.0, None, 0.0])):
        rec = _Recorder(lib)
        monkeypatch.setattr(_cabi, "_lib", rec)
        tiny.generate_text_batch(cache, max_length=6, do_sample=True, temperature=0.9, **kw, **gs)
        seqs.append(rec.calls)
    assert seqs[0] == seqs[1]
    assert "bagel_apply_penalties_bf16" not in seqs[0]


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


@pytest.mark.parametrize("filtered", [False, True])
def test_penalised_decode_step_is_one_graph_replay(tiny, monkeypatch, filtered):
    from bagel_b200 import _cabi
    cache, gs = _text_context(tiny, PROMPTS)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
    rec = _Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    n = 12
    kw = dict(top_p=0.9) if filtered else {}
    out = tiny.generate_text_batch(cache, max_length=n, do_sample=True, temperature=0.8, repetition_penalty=1.05,
                                   presence_penalty=0.5, frequency_penalty=0.5, **kw, **gs)
    assert all(len(t) == n for t in out)
    L = fixtures.TINY_LM.num_hidden_layers
    ctx, calls = rec.calls[:2 * L], rec.calls[2 * L:]
    assert ctx == ["bagel_copy_rows_bf16"] * (2 * L)
    half = len(calls) // 2
    assert calls[:half] == calls[half:]
    pick = "bagel_sample_rows_filtered_bf16" if filtered else "bagel_sample_rows_mixed_bf16"
    assert calls[half - 4:half] == ["bagel_gemm_bf16", "bagel_apply_penalties_bf16", pick,
                                    "bagel_decode_advance_stop_limits"], calls[half - 4:half]
    assert len(replays) == n - 1


@pytest.mark.parametrize("sampled", [False, True])
def test_chat_batch_with_penalties_same_in_a_batch_as_alone(sampled):
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV)
    tok = fixtures.ToyTokenizer()
    reqs = [(fixtures.vit_images(), "6 1"), ([], "1 2 3"), ([], "4 5")]
    kw = dict(max_length=12, do_sample=sampled, temperature=1.4)
    batch = model.chat_batch(tok, NT, lambda x: x, reqs, seeds=[5, 6, 7], top_p=[0.7, None, 0.9],
                             repetition_penalty=[1.2, None, 1.05], frequency_penalty=[0.5, 0.0, 1.0],
                             presence_penalty=[0.3, 1.0, None], **kw)
    alone = model.chat_batch(tok, NT, lambda x: x, reqs[:1], seeds=[5], top_p=0.7, repetition_penalty=1.2,
                             frequency_penalty=0.5, presence_penalty=0.3, **kw)
    assert batch[0] == alone[0]
    if not sampled:         # chat_batch keys a sampled request's draws by its index, so only request 0 compares
        alone = model.chat_batch(tok, NT, lambda x: x, reqs[2:], top_p=0.9, repetition_penalty=1.05,
                                 frequency_penalty=1.0, **kw)
        assert batch[2] == alone[0]


@pytest.mark.parametrize("sampled", [False, True])
def test_call_batch_with_penalties_same_in_a_batch_as_alone(sampled):
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV, max_latent_size=16, vae_downsample=2)
    vae = helpers.tiny_vae(DEV)
    vae.sample = False
    inf = InterleaveInferencer(model, vae, fixtures.ToyTokenizer(), ImageTransform(64, 32, 4),
                               ImageTransform(112, 56, 14), helpers.NEW_TOKEN_IDS)
    steps = dict(num_timesteps=3, timestep_shift=3.0)
    und = dict(text="5 17 900 33 2", understanding_output=True, max_think_token_n=12, do_sample=sampled,
               text_temperature=1.4, top_p=0.8, repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.2,
               seed=11)
    others = [dict(text="3 1 4", understanding_output=True, max_think_token_n=6, do_sample=True, top_k=3,
                   presence_penalty=1.5, seed=12),
              dict(text="9 2 6", understanding_output=True, max_think_token_n=8, seed=13)]
    batch = inf.call_batch([others[0], und, others[1]], **steps)
    alone = inf.call_batch([und], **steps)
    assert batch[1]["text"] == alone[0]["text"]
    plain = inf.call_batch([others[1]], **steps)
    assert batch[2]["text"] == plain[0]["text"]
