"""-m gpu: truncated sampling. bagel_sample_rows_filtered_bf16 against the NumPy filter oracle (V = 152064, small and
odd V, strided rows, bf16 ties, -inf, all-NaN, a different setting on every row); with every filter off against
bagel_sample_rows_mixed_bf16 bit for bit; its distribution (chi-square against the truncated softmax); determinism,
graph replay and row independence; Bagel.generate_text_batch, chat_batch and InterleaveInferencer.call_batch with
filters on the tiny model."""
import numpy as np
import pytest
import torch
from scipy import stats

import helpers
import sampling_filter_oracle as sfo
from oracle import fixtures

pytestmark = pytest.mark.gpu
DEV = "cuda"
NT = dict(helpers.NEW_TOKEN_IDS)
EPS = 1e-5          # relative top-p mass band in which either neighbouring threshold is accepted


def _ops():
    from bagel_b200 import ops
    return ops


def _keys(vals):
    return torch.from_numpy(np.array(vals, dtype=np.uint64).view(np.int64)).to(DEV)


def _f32(vals):
    return torch.tensor(vals, dtype=torch.float32, device=DEV)


def _inv_t(temps):
    return _f32([0.0 if t is None else np.float32(1.0) / np.float32(t) for t in temps])


def _run(logits, temps, ks, ps, ms, keys, step):
    ops = _ops()
    B = logits.shape[0]
    tok = torch.full((B,), -7, dtype=torch.int64, device=DEV)
    tok32 = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    ops.sample_rows_filtered(logits, _inv_t(temps), torch.tensor(ks, dtype=torch.int32, device=DEV), _f32(ps), _f32(ms),
                             _keys(keys), torch.tensor([step], dtype=torch.int32, device=DEV), tok, tok32)
    assert torch.equal(tok.to(torch.int32), tok32)
    return tok.cpu().numpy()


# (temperature or None for greedy, top_k, top_p, min_p): a different mix on every row
SETTINGS = [
    (1.0, 50, 1.0, 0.0), (0.7, 0, 0.9, 0.0), (1.3, 0, 1.0, 0.05), (0.5, 20, 0.8, 0.02), (1.0, 1, 1.0, 0.0),
    (2.0, 0, 0.3, 0.0), (None, 5, 0.5, 0.1), (0.9, 1000, 0.95, 0.0), (1.0, 3, 1.0, 0.5), (0.3, 0, 0.999, 0.001),
    (1.6, 7, 0.6, 0.2), (1.0, 0, 1.0, 0.0),
]


def _rows(V, ld, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(SETTINGS)
    logits = (torch.randn(B, ld, generator=g) * 3).to(torch.bfloat16)
    logits[1] = (torch.randint(-12, 13, (ld,), generator=g) / 4.0).to(torch.bfloat16)     # heavy ties
    logits[3] = (torch.randint(-40, 9, (ld,), generator=g) / 8.0).to(torch.bfloat16)
    logits[10] = (torch.randint(-3, 4, (ld,), generator=g) * 0.5).to(torch.bfloat16)
    logits[2, ::3] = float("-inf")
    logits[7, : V // 2] = float("-inf")
    logits[5] = float("nan")                      # all-NaN sampled row
    return logits


@pytest.mark.parametrize("V,ld", [(152064, 152072), (1024, 1024), (1031, 1037)])
def test_filtered_sampler_matches_oracle(V, ld):
    logits = _rows(V, ld, V).to(DEV)[:, :V]
    rows = logits.float().cpu().numpy().astype(np.float64)
    B = len(SETTINGS)
    keys = [(0x5151 + 31 * i) | (i << 32) for i in range(B)]
    temps, ks, ps, ms = (list(c) for c in zip(*SETTINGS))
    checked = 0
    for step in (0, 4099):
        got = _run(logits, temps, ks, ps, ms, keys, step)
        greedy = torch.empty(B, dtype=torch.int64, device=DEV)
        _ops().argmax_rows(logits, greedy)
        for b, (T, k, p, m) in enumerate(SETTINGS):
            if T is None:
                assert got[b] == int(greedy[b]), b
                continue
            inv_t = float(np.float32(1.0) / np.float32(T))
            cands = sfo.floors(rows[b], inv_t, k, p, m, eps=EPS)
            want, decided = sfo.draw(rows[b], T, keys[b], step, cands[0])
            if got[b] != want:
                alt = [sfo.draw(rows[b], T, keys[b], step, f)[0] for f in cands[1:]]
                assert got[b] in alt, (V, step, b, got[b], want, cands)
            elif decided:
                checked += 1
            assert b == 5 or sfo.kept(rows[b], min(cands))[got[b]], (b, got[b])
        assert got[5] == 0, "all-NaN row"
    assert checked >= 2 * (B - 2) - 2, checked


@pytest.mark.parametrize("V,ld", [(152064, 152064), (1031, 1031)])
def test_filters_off_is_the_mixed_sampler(V, ld):
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    temps = [None, 1.0, 0.3, None, 0.6, 2.5, 0.8, None]
    B = len(temps)
    logits = (torch.randn(B, ld, generator=g) * 2).to(torch.bfloat16)
    logits[6] = float("nan")
    logits[1, 5] = float("-inf")
    logits = logits.to(DEV)[:, :V]
    keys = [(77 + i) | (i << 32) for i in range(B)]
    for step in (0, 12):
        mixed = torch.empty(B, dtype=torch.int64, device=DEV)
        ops.sample_rows_mixed(logits, _inv_t(temps), _keys(keys), torch.tensor([step], dtype=torch.int32, device=DEV),
                              mixed)
        want = mixed.cpu().numpy()
        # off, and settings that keep every finite logit (k >= V); greedy rows ignore filters that are set
        off = _run(logits, temps, [0, V, 0, 9, V + 5, 0, 0, 3], [1.0] * 3 + [0.2] + [1.0] * 3 + [0.5],
                   [0.0] * 3 + [0.3] + [0.0] * 4, keys, step)
        assert np.array_equal(off, want), (step, off, want)


@pytest.mark.parametrize("which", ["top_k", "top_p", "min_p"])
def test_filtered_distribution_chi_square(which):
    """4 launches of 1024 rows with the same logits and distinct keys: the draws follow the truncated, renormalised
    softmax (Pearson chi-square over the kept tokens; none outside them)."""
    V, B, T = 48, 1024, 0.9
    lq = torch.empty(V).uniform_(-2.0, 2.0, generator=torch.Generator().manual_seed(21)).to(torch.bfloat16)
    logits = lq.reshape(1, V).expand(B, V).contiguous().to(DEV)
    setting = dict(top_k=(10, 1.0, 0.0), top_p=(0, 0.7, 0.0), min_p=(0, 1.0, 0.25))[which]
    row = lq.double().numpy()
    inv_t = float(np.float32(1.0) / np.float32(T))
    (floor,) = sfo.floors(row, inv_t, *setting)
    p = sfo.truncated_softmax(row, T, floor)
    draws = np.concatenate([_run(logits, [T] * B, [setting[0]] * B, [setting[1]] * B, [setting[2]] * B,
                                 [(9000 + i) | (7 << 32) for i in range(B)], step) for step in range(4)])
    keep = p > 0
    assert 3 <= keep.sum() < V
    counts = np.bincount(draws, minlength=V)
    assert counts[~keep].sum() == 0, "a draw outside the kept set"
    expected = draws.size * p[keep]
    assert expected.min() > 5
    chi2 = float(((counts[keep] - expected) ** 2 / expected).sum())
    pval = stats.chi2.sf(chi2, int(keep.sum()) - 1)
    assert pval > 1e-3, (which, chi2, pval)


def test_filtered_determinism_replay_and_row_independence():
    ops = _ops()
    V = 4099
    logits = _rows(V, V, 11).to(DEV)
    B = len(SETTINGS)
    temps, ks, ps, ms = (list(c) for c in zip(*SETTINGS))
    keys = [(123 + i) | (i << 32) for i in range(B)]
    base = _run(logits, temps, ks, ps, ms, keys, 5)
    assert np.array_equal(base, _run(logits, temps, ks, ps, ms, keys, 5)), "two launches"
    # graph replay equals eager
    args = (_inv_t(temps), torch.tensor(ks, dtype=torch.int32, device=DEV), _f32(ps), _f32(ms), _keys(keys),
            torch.tensor([5], dtype=torch.int32, device=DEV))
    tok = torch.empty(B, dtype=torch.int64, device=DEV)
    ops.sample_rows_filtered(logits, *args, tok)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.sample_rows_filtered(logits, *args, tok)
    tok.fill_(-1)
    graph.replay()
    assert np.array_equal(tok.cpu().numpy(), base)
    # permuted rows: each row keeps its token
    perm = np.random.default_rng(2).permutation(B)
    got = _run(logits[torch.from_numpy(perm).to(DEV)], [temps[i] for i in perm], [ks[i] for i in perm],
               [ps[i] for i in perm], [ms[i] for i in perm], [keys[i] for i in perm], 5)
    assert np.array_equal(got, base[perm])
    # other rows' settings change, row 0 and row 3 do not
    other = [(t, 2, 0.5, 0.3) if i not in (0, 3) else (t, k, p, m) for i, (t, k, p, m) in enumerate(SETTINGS)]
    t2, k2, p2, m2 = (list(c) for c in zip(*other))
    t2 = [1.0 if (t is None and i not in (0, 3)) else t for i, t in enumerate(t2)]
    got = _run(logits, t2, k2, p2, m2, keys, 5)
    assert got[0] == base[0] and got[3] == base[3]


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


PROMPTS = ["5 17 900 33 2", "8 8 100 4 77 650 12", "1 2 3", "999 0 999"]
FILT = dict(top_k=[5, 0, 40, None], top_p=[None, 0.8, 0.9, 1.0], min_p=[0.0, 0.05, None, 0.2])


def _gen(model, cache, gs, **kw):
    kw = dict(dict(max_length=16, do_sample=True, temperature=1.5, seeds=[5, 6, 7, 8]), **kw)
    return [t.tolist() for t in model.generate_text_batch(cache, **kw, **gs)]


def test_generate_text_batch_with_filters(tiny):
    cache, gs = _text_context(tiny, PROMPTS)
    captured = _gen(tiny, cache, gs, **FILT)
    tiny.use_cuda_graph = False
    try:
        eager = _gen(tiny, cache, gs, **FILT)
    finally:
        tiny.use_cuda_graph = True
    assert captured == eager
    plain = _gen(tiny, cache, gs)
    assert _gen(tiny, cache, gs, top_k=0, top_p=1.0, min_p=0.0) == plain
    assert _gen(tiny, cache, gs, top_k=[None] * 4, top_p=[None] * 4, min_p=[None] * 4) == plain
    # top_k = 1 is greedy; a request's tokens do not depend on the other requests' filters
    greedy = [t.tolist() for t in tiny.generate_text_batch(cache, max_length=16, **gs)]
    assert _gen(tiny, cache, gs, top_k=1) == greedy
    other = _gen(tiny, cache, gs, top_k=[5, 1, 2, 1], top_p=[None, 0.3, 0.5, None], min_p=[0.0, 0.5, None, 0.9])
    assert other[0] == captured[0]
    assert other[1] == greedy[1] and other[3] == greedy[3]


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


def test_filtered_decode_step_is_one_graph_replay(tiny, monkeypatch):
    from bagel_b200 import _cabi
    cache, gs = _text_context(tiny, PROMPTS)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
    rec = _Recorder(_cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    n = 12
    out = tiny.generate_text_batch(cache, max_length=n, do_sample=True, temperature=0.8, top_p=0.9, **gs)
    assert all(len(t) == n for t in out)
    L = fixtures.TINY_LM.num_hidden_layers
    ctx, calls = rec.calls[:2 * L], rec.calls[2 * L:]
    assert ctx == ["bagel_copy_rows_bf16"] * (2 * L)
    half = len(calls) // 2
    assert calls[:half] == calls[half:]
    assert calls[half - 2:half] == ["bagel_sample_rows_filtered_bf16", "bagel_decode_advance_stop_limits"]
    assert len(replays) == n - 1


def test_chat_batch_with_top_p_same_in_a_batch_as_alone():
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV)
    tok = fixtures.ToyTokenizer()
    reqs = [(fixtures.vit_images(), "6 1"), ([], "1 2 3"), ([], "4 5")]
    kw = dict(max_length=10, do_sample=True, temperature=1.4)
    batch = model.chat_batch(tok, NT, lambda x: x, reqs, seeds=[5, 6, 7], top_p=[0.7, None, 0.9], **kw)
    alone = model.chat_batch(tok, NT, lambda x: x, reqs[:1], seeds=[5], top_p=0.7, **kw)
    assert batch[0] == alone[0]


def test_call_batch_with_top_p_same_in_a_batch_as_alone():
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, DEV, max_latent_size=16, vae_downsample=2)
    vae = helpers.tiny_vae(DEV)
    vae.sample = False
    inf = InterleaveInferencer(model, vae, fixtures.ToyTokenizer(), ImageTransform(64, 32, 4),
                               ImageTransform(112, 56, 14), helpers.NEW_TOKEN_IDS)
    steps = dict(num_timesteps=3, timestep_shift=3.0)
    und = dict(text="5 17 900 33 2", understanding_output=True, max_think_token_n=10, do_sample=True,
               text_temperature=1.4, top_p=0.8, seed=11)
    others = [dict(text="3 1 4", understanding_output=True, max_think_token_n=6, do_sample=True, top_k=3, seed=12),
              dict(text="9 2 6", understanding_output=True, max_think_token_n=8, seed=13)]
    batch = inf.call_batch([others[0], und, others[1]], **steps)
    alone = inf.call_batch([und], **steps)
    assert batch[1]["text"] == alone[0]["text"]
