"""Host side of the decode-step penalties (no GPU): the penalty oracle against transformers'
RepetitionPenaltyLogitsProcessor (prompt ignored), its presence / frequency arithmetic against a direct restatement of
the formula with one rounding per operation (on values where a fused multiply-add would round differently), and the
argument checks of Bagel.generate_text_batch, Bagel.chat_batch and InterleaveInferencer.call_batch."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import helpers
import penalty_oracle as po


def _row(rng, V):
    """bf16 logits with negative, zero, -0, -inf and NaN entries."""
    x = torch.tensor(rng.normal(0.0, 4.0, V), dtype=torch.float32)
    x[rng.integers(0, V, V // 10)] = 0.0
    x[rng.integers(0, V, V // 20)] = -0.0
    x[rng.integers(0, V, V // 20)] = float("-inf")
    x[rng.integers(0, V, V // 30)] = float("nan")
    return x.to(torch.bfloat16)


def _same(a, b):
    return torch.equal(po.bits(a), po.bits(b))


def _hf(row, prompt, generated, penalty):
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    ids = torch.tensor([list(prompt) + list(generated)], dtype=torch.long)
    proc = RepetitionPenaltyLogitsProcessor(penalty, prompt_ignore_length=len(prompt))
    return proc(ids, row.float()[None].clone())[0].to(torch.bfloat16)


@pytest.mark.parametrize("seed", range(6))
def test_repetition_oracle_equals_transformers(seed):
    rng = np.random.default_rng(seed)
    for trial in range(25):
        V = int(rng.integers(16, 3000))
        row = _row(rng, V)
        prompt = rng.integers(0, V, int(rng.integers(1, 40))).tolist()
        n = int(rng.integers(0, 200))
        # heavy repetition on some trials: a few tokens, many times
        pool = rng.integers(0, V, 5) if trial % 2 else np.arange(V)
        generated = rng.choice(pool, n).tolist()
        if trial % 5 == 0:          # tokens whose logit is NaN, -inf, zero
            generated += [int(i) for i in torch.nonzero(~torch.isfinite(row.float()) | (row == 0))[:6, 0]]
        penalty = float(rng.choice([1.05, 1.3, 2.0, 0.7, 1 / 1.05, 1.0, 17.0]))
        want = _hf(row, prompt, generated, penalty)
        got = po.apply(row, generated, rp=penalty)
        nan = torch.isnan(want.float())
        assert torch.equal(nan, torch.isnan(got.float())), (seed, trial)
        assert _same(got[~nan], want[~nan]), (seed, trial, penalty)
        # the prompt's tokens are not penalised unless generated too
        only_prompt = sorted(set(prompt) - set(generated))
        assert _same(got[only_prompt], row[only_prompt])


def test_oracle_edge_values():
    row = torch.tensor([2.0, -2.0, 0.0, -0.0, float("-inf"), float("nan"), float("inf"), 3.0], dtype=torch.bfloat16)
    got = po.apply(row, [0, 1, 2, 3, 4, 5, 6, 0], rp=2.0, fp=0.5, pp=0.25)
    # 2/2 - 0.5*2 - 0.25; -2*2 - 0.5 - 0.25; 0/2 - 0.75; -0/2 - 0.75; -inf; NaN (bits kept); inf; untouched
    want = torch.tensor([-0.25, -4.75, -0.75, -0.75, float("-inf"), float("nan"), float("inf"), 3.0],
                        dtype=torch.bfloat16)
    assert _same(got[[0, 1, 2, 3, 4, 6, 7]], want[[0, 1, 2, 3, 4, 6, 7]])
    assert _same(got[5:6], row[5:6])
    neg_nan = torch.tensor([-1, 0x7FC1, 0x3F80], dtype=torch.int16).view(torch.bfloat16)     # NaN payloads are kept
    assert _same(po.apply(neg_nan, [0, 1, 2], rp=1.3, fp=0.5, pp=0.5)[:2], neg_nan[:2])
    assert _same(po.apply(row, [], rp=1.3, fp=1.0, pp=1.0), row)                 # nothing generated: unchanged
    assert _same(po.apply(row, [0, 1, 7], rp=1.0, fp=0.0, pp=-0.0), row)        # every penalty off
    assert po.is_off(1.0, 0.0, 0.0) and not po.is_off(1.0, 0.0, 1e-30)


def _f32(x):
    """Round an exact rational to the nearest float32, ties to even."""
    c = np.float32(float(x))
    best = None
    for v in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(v)) - x)
        even = (int(np.array(v, np.float32).view(np.int32)) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, v)
    return best[1]


def _restated(l, c, rp, fp, pp):
    """The formula for one logit, one float32 rounding per operation, then bf16 round to nearest even."""
    l, rp, fp, pp = (np.float32(v) for v in (l, rp, fp, pp))
    r = _f32(Fraction(float(l)) * Fraction(float(rp))) if l < 0 else _f32(Fraction(float(l)) / Fraction(float(rp)))
    r = _f32(Fraction(float(r)) - _f32(Fraction(float(fp)) * c))
    r = _f32(Fraction(float(r)) - Fraction(float(pp)))
    return torch.tensor([float(r)], dtype=torch.float32).to(torch.bfloat16)


def _fused(l, c, rp, fp, pp):
    """The same with r - fp * c as one fused operation (a single rounding)."""
    l, rp, fp, pp = (np.float32(v) for v in (l, rp, fp, pp))
    r = _f32(Fraction(float(l)) * Fraction(float(rp))) if l < 0 else _f32(Fraction(float(l)) / Fraction(float(rp)))
    r = _f32(Fraction(float(r)) - Fraction(float(fp)) * c)
    r = _f32(Fraction(float(r)) - Fraction(float(pp)))
    return torch.tensor([float(r)], dtype=torch.float32).to(torch.bfloat16)


def test_presence_frequency_oracle_equals_restatement():
    rng = np.random.default_rng(7)
    for trial in range(300):
        V = 12
        row = _row(rng, V)
        generated = rng.integers(0, V, int(rng.integers(0, 30))).tolist()
        rp = float(rng.choice([1.0, 1.05, 0.8]))
        fp = float(np.float32(rng.uniform(-2, 2)))
        pp = float(rng.choice([0.0, np.float32(rng.uniform(-2, 2))]))
        got = po.apply(row, generated, rp, fp, pp)
        for t in range(V):
            c = generated.count(t)
            l = float(row[t])
            if c == 0 or np.isnan(l):
                assert _same(got[t:t + 1], row[t:t + 1])
            elif np.isfinite(l):
                assert _same(got[t:t + 1], _restated(l, c, rp, fp, pp)), (trial, t, l, c, rp, fp, pp)


def test_frequency_penalty_is_not_fused():
    """Values where r - fp * c rounded once (FMA) and twice end on different bf16 values: the oracle takes the
    twice-rounded one."""
    rng = np.random.default_rng(11)
    n = 1 << 21
    l = torch.tensor(rng.uniform(-8, 8, n), dtype=torch.float32).to(torch.bfloat16).float().numpy()
    fp = rng.uniform(-2, 2, n).astype(np.float32)
    c = rng.integers(1, 64, n)
    rp = np.float32(1.05)
    with np.errstate(over="ignore"):
        r = np.where(l < 0, l * rp, l / rp).astype(np.float32)
    unfused = (r - (fp * c.astype(np.float32)).astype(np.float32)).astype(np.float32)
    # a screen only: every candidate is checked exactly below
    fused = (r.astype(np.float64) - fp.astype(np.float64) * c).astype(np.float32)
    bf = lambda x: torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    cand = np.nonzero(bf(unfused) != bf(fused))[0]
    checked = 0
    for i in cand[:40]:
        want = _restated(l[i], int(c[i]), rp, fp[i], 0.0)
        if _same(want, _fused(l[i], int(c[i]), rp, fp[i], 0.0)):
            continue
        row = torch.tensor([l[i]], dtype=torch.float32).to(torch.bfloat16)
        got = po.apply(row, [0] * int(c[i]), float(rp), float(fp[i]), 0.0)
        assert _same(got, want), (l[i], c[i], fp[i])
        checked += 1
    assert checked >= 10, checked


# ---------------------------------------------------------------------------------------------- argument checks

@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel(device="cpu", load=False)


KW = dict(past_key_values=None, packed_key_value_indexes=None, key_values_lens=[3, 4], packed_start_tokens=None,
          packed_query_position_ids=None)

BAD = [
    (dict(repetition_penalty=0.0), "repetition_penalty"), (dict(repetition_penalty=-1.05), "repetition_penalty"),
    (dict(repetition_penalty=float("nan")), "repetition_penalty"),
    (dict(repetition_penalty=float("inf")), "repetition_penalty"),
    (dict(repetition_penalty=True), "repetition_penalty"),
    (dict(repetition_penalty=[1.05, 1e-60]), "repetition_penalty"),
    (dict(presence_penalty=2.5), "presence_penalty"), (dict(presence_penalty=[0.5, float("nan")]), "presence_penalty"),
    (dict(presence_penalty=False), "presence_penalty"), (dict(frequency_penalty=-2.01), "frequency_penalty"),
    (dict(frequency_penalty=[0.1, "0.2"]), "frequency_penalty"), (dict(frequency_penalty=True), "frequency_penalty"),
    (dict(repetition_penalty=[1.1]), "repetition_penalty has 1 entries"),
    (dict(presence_penalty=[0.5, 0.5, 0.5]), "presence_penalty has 3 entries"),
    (dict(frequency_penalty=[0.1]), "frequency_penalty has 1 entries"),
]


@pytest.mark.parametrize("bad,match", BAD)
def test_generate_text_batch_refuses_bad_penalties(model, bad, match):
    with pytest.raises(ValueError, match=match):
        model.generate_text_batch(**KW, max_length=5, **bad)


def test_penalty_plan():
    from bagel_b200.bagel import _penalties
    off = (dict(), dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0),
           dict(repetition_penalty=[None, 1.0], presence_penalty=[0.0, None], frequency_penalty=[-0.0, 0]),
           dict(repetition_penalty=1, presence_penalty=0, frequency_penalty=0))
    for kw in off:
        assert _penalties(2, kw.get("repetition_penalty"), kw.get("presence_penalty"),
                          kw.get("frequency_penalty")) is None, kw
    plan = _penalties(3, [1.05, None, 1.0], 0.5, [None, -2.0, 0.0])
    assert plan == ([float(np.float32(1.05)), 1.0, 1.0], [0.0, -2.0, 0.0], [0.5, 0.5, 0.5])
    assert _penalties(1, 2, None, None) == ([2.0], [0.0], [0.0])


def test_generate_text_batch_accepts_penalties_that_are_off(model):
    # nothing to decode: the checks pass and no device work starts
    for kw in (dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0),
               dict(repetition_penalty=[None, 1.05], presence_penalty=[0.0, -2.0], frequency_penalty=[2.0, None]),
               dict(repetition_penalty=0.5, presence_penalty=2, frequency_penalty=-2)):
        out = model.generate_text_batch(**KW, max_length=[0, 0], **kw)
        assert [t.numel() for t in out] == [0, 0]


@pytest.mark.parametrize("bad,match", BAD[:12])
def test_chat_batch_refuses_bad_penalties(model, bad, match):
    reqs = [([], "1 2"), ([], "3")]
    with pytest.raises(ValueError, match=match):
        model.chat_batch(helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS, None, reqs, max_length=4, **bad)
    with pytest.raises(ValueError, match="frequency_penalty has 3 entries"):
        model.chat_batch(helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS, None, reqs, max_length=4,
                         frequency_penalty=[0.1, 0.2, 0.3])


def test_call_batch_refuses_bad_penalties(model):
    from bagel_b200.inferencer import InterleaveInferencer
    inf = InterleaveInferencer(model, None, helpers.IntTokenizer(), None, None, helpers.NEW_TOKEN_IDS)
    for bad, match in BAD[:12]:
        bad = {k: v[-1] if isinstance(v, list) else v for k, v in bad.items()}
        with pytest.raises(ValueError, match=match):
            inf.call_batch([dict(text="1", understanding_output=True), dict(text="2", **bad)])
    # the penalty keys are known; off values (and requests with no input) run nothing
    assert inf.call_batch([dict(repetition_penalty=None, presence_penalty=0.0, frequency_penalty=0.0),
                           dict(repetition_penalty=1.05, presence_penalty=0.5, frequency_penalty=-0.5)]) == \
        [{"image": None, "text": None}] * 2
