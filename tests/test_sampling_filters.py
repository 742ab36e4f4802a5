"""Host side of truncated sampling (no GPU): the filter oracle's thresholds against brute-force definitions on rows with
heavy ties, its kept set against transformers' top-k / top-p / min-p warpers chained in generate's order, and the
argument checks of Bagel.generate_text_batch, Bagel.chat_batch and InterleaveInferencer.call_batch."""
import numpy as np
import pytest
import torch

import helpers
from sampling_filter_oracle import floors, kept, thresholds


def _bf16_row(rng, V, ties):
    """bf16-valued logits; with ties, from a coarse grid so that most values repeat."""
    x = rng.integers(-40, 41, V) / 4.0 if ties else rng.normal(0.0, 3.0, V)
    return torch.tensor(x, dtype=torch.float32).to(torch.bfloat16).double().numpy()


def _brute(row, inv_t, k, p, m):
    """Each filter applied in turn, by direct counts and sums per candidate value."""
    keep = np.isfinite(row)
    if k:
        keep &= np.array([(row[keep] > v).sum() < k for v in row])
    if p is not None and p < 1:
        lmax = row[np.isfinite(row)].max()
        e = np.where(keep, np.exp((row - lmax) * float(np.float32(inv_t))), 0.0)
        total = e.sum()
        # a value is kept when the mass strictly above it has not reached p yet
        keep &= np.array([e[row > v].sum() < p * total for v in row])
    if m:
        lmax = row[np.isfinite(row)].max()
        x = (row.astype(np.float32) - np.float32(lmax)) * np.float32(inv_t)
        keep &= x >= np.float32(np.log(np.float32(m)))
    return keep


@pytest.mark.parametrize("seed", range(8))
def test_oracle_thresholds_equal_brute_force(seed):
    rng = np.random.default_rng(seed)
    for trial in range(12):
        V = int(rng.integers(1, 300))
        row = _bf16_row(rng, V, ties=trial % 3 != 0)
        if trial % 4 == 1:
            row[rng.integers(0, V, V // 5)] = -np.inf
        inv_t = float(np.float32(1.0) / np.float32(rng.choice([0.3, 0.7, 1.0, 1.9])))
        k = int(rng.choice([0, 1, 2, 5, 17, V, V + 3]))
        p = float(rng.choice([1.0, 0.05, 0.5, 0.9, 0.99]))
        m = float(rng.choice([0.0, 0.01, 0.1, 0.5]))
        (floor,) = floors(row, inv_t, k, p, m)[:1]
        assert np.array_equal(kept(row, floor), _brute(row, inv_t, k, p, m)), (seed, trial, k, p, m)
        # the maximum is always kept
        fin = row[np.isfinite(row)]
        if fin.size:
            assert floor <= fin.max()


def test_oracle_edge_rows():
    nan = np.full(7, np.nan)
    assert thresholds(nan, 1.0, 3, 0.5, 0.1) == (-np.inf, {-np.inf}, {-np.inf})
    row = np.array([1.0, 1.0, 1.0, 0.5, -np.inf, np.nan])
    assert thresholds(row, 1.0, top_k=2)[0] == 1.0           # ties at the boundary are kept
    assert kept(row, floors(row, 1.0, top_k=2)[0]).sum() == 3
    assert thresholds(row, 1.0, top_k=9)[0] == -np.inf        # more than the finite logits: keep them all
    assert kept(row, floors(row, 1.0, top_k=9)[0]).sum() == 4


def _hf_kept(row, T, k, p, m):
    from transformers.generation.logits_process import MinPLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    scores = torch.tensor(row / T, dtype=torch.float32)[None]
    ids = torch.zeros((1, 1), dtype=torch.long)
    if k:
        scores = TopKLogitsWarper(top_k=k)(ids, scores)
    if p is not None and p < 1:
        scores = TopPLogitsWarper(top_p=p)(ids, scores)
    if m:
        scores = MinPLogitsWarper(min_p=m)(ids, scores)
    return torch.isfinite(scores[0]).numpy()


@pytest.mark.parametrize("seed", range(6))
def test_oracle_kept_set_equals_transformers_warpers(seed):
    rng = np.random.default_rng(100 + seed)
    checked = 0
    for trial in range(40):
        V = int(rng.integers(8, 2000))
        row = np.unique(_bf16_row(rng, V, ties=False))     # no ties at all
        rng.shuffle(row)
        T = float(rng.choice([0.3, 0.7, 1.0, 1.5]))
        inv_t = float(np.float32(1.0) / np.float32(T))
        k = int(rng.choice([0, 1, 7, 50, row.size]))
        p = float(rng.choice([1.0, 0.3, 0.8, 0.95]))
        m = float(rng.choice([0.0, 0.02, 0.2]))
        fl = floors(row, inv_t, k, p, m, eps=1e-4)
        if len(fl) > 1:
            continue        # a boundary within fp32 noise of the threshold: the two sides may differ
        assert np.array_equal(kept(row, fl[0]), _hf_kept(row, T, k, p, m)), (seed, trial, k, p, m)
        checked += 1
    assert checked >= 30


# ---------------------------------------------------------------------------------------------- argument checks

@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel(device="cpu", load=False)


KW = dict(past_key_values=None, packed_key_value_indexes=None, key_values_lens=[3, 4], packed_start_tokens=None,
          packed_query_position_ids=None)

BAD = [
    (dict(top_k=-1), "top_k"), (dict(top_k=2.5), "top_k"), (dict(top_k=True), "top_k"), (dict(top_k=[3, -2]), "top_k"),
    (dict(top_p=0.0), "top_p"), (dict(top_p=1.5), "top_p"), (dict(top_p=[0.5, float("nan")]), "top_p"),
    (dict(min_p=1.0), "min_p"), (dict(min_p=-0.1), "min_p"), (dict(min_p=[0.1, 2.0]), "min_p"),
    (dict(top_k=[5]), "top_k has 1 entries"), (dict(top_p=[0.5, 0.5, 0.5]), "top_p has 3 entries"),
    (dict(min_p=[0.1]), "min_p has 1 entries"),
]


@pytest.mark.parametrize("bad,match", BAD)
def test_generate_text_batch_refuses_bad_filters(model, bad, match):
    with pytest.raises(ValueError, match=match):
        model.generate_text_batch(**KW, max_length=5, do_sample=True, temperature=0.7, **bad)


def test_generate_text_batch_accepts_filters_that_are_off(model):
    # nothing to decode: the checks pass and no device work starts
    for kw in (dict(top_k=0, top_p=1.0, min_p=0.0), dict(top_k=[None, 3], top_p=[1.0, None], min_p=[0.0, 0.5]),
               dict(top_k=7, top_p=0.9, min_p=0.05)):
        out = model.generate_text_batch(**KW, max_length=[0, 0], do_sample=True, temperature=0.3, **kw)
        assert [t.numel() for t in out] == [0, 0]


@pytest.mark.parametrize("bad,match", BAD[:10])
def test_chat_batch_refuses_bad_filters(model, bad, match):
    reqs = [([], "1 2"), ([], "3")]
    with pytest.raises(ValueError, match=match):
        model.chat_batch(helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS, None, reqs, max_length=4, do_sample=True, **bad)
    with pytest.raises(ValueError, match="top_k has 3 entries"):
        model.chat_batch(helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS, None, reqs, max_length=4, do_sample=True,
                         top_k=[1, 2, 3])


def test_call_batch_refuses_bad_filters(model):
    from bagel_b200.inferencer import InterleaveInferencer
    inf = InterleaveInferencer(model, None, helpers.IntTokenizer(), None, None, helpers.NEW_TOKEN_IDS)
    for bad, match in BAD[:10]:
        bad = {k: v[-1] if isinstance(v, list) else v for k, v in bad.items()}
        with pytest.raises(ValueError, match=match):
            inf.call_batch([dict(text="1", understanding_output=True, do_sample=True), dict(text="2", **bad)])
    # the filter keys are known; off values (and requests with no input) run nothing
    assert inf.call_batch([dict(top_k=None, top_p=1.0, min_p=0.0), dict(top_k=3, top_p=0.9, min_p=0.1)]) == \
        [{"image": None, "text": None}] * 2
