"""Host logic of batched interleaved requests (no GPU): the text-round packer gives every present request exactly
prepare_prompts' layout for it alone and carries absent requests unchanged; InterleaveInferencer.call_batch's round
schedule follows interleave_inference per request; request validation and refusals; gather_requests' cases that copy
nothing."""
import random

import pytest
import torch

import helpers
from bagel_b200.inferencer import InterleaveInferencer, call_batch_schedule
from bagel_b200.qwen2_navit import NaiveCache, gather_requests

NT = helpers.NEW_TOKEN_IDS


@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel(device="cpu", load=False)


def _block(gi, q, ql):
    """Request q's part of a text round, its indexes relative to its own block."""
    cl = gi["key_values_lens"].to(torch.int64)
    b0 = int((cl + ql)[:q].sum())
    q0 = int(ql[:q].sum())
    qs = slice(q0, q0 + int(ql[q]))
    return dict(text_token_lens=gi["text_token_lens"][q:q + 1], key_values_lens=gi["key_values_lens"][q:q + 1],
                packed_text_ids=gi["packed_text_ids"][qs], packed_text_position_ids=gi["packed_text_position_ids"][qs],
                packed_text_indexes=gi["packed_text_indexes"][qs] - b0,
                packed_key_value_indexes=gi["packed_key_value_indexes"][int(cl[:q].sum()):int(cl[:q + 1].sum())] - b0)


@pytest.mark.parametrize("seed", range(6))
def test_prompts_round_matches_prepare_prompts_per_request(model, seed):
    rnd = random.Random(seed)
    R = rnd.randint(1, 7)
    prompts = [None if rnd.random() < 0.4 else " ".join(str(rnd.randint(0, 999)) for _ in range(rnd.randint(0, 9)))
               for _ in range(R)]
    kv0 = [rnd.randint(0, 30) for _ in range(R)]
    rp0 = [rnd.randint(0, 6) for _ in range(R)]
    tok = helpers.IntTokenizer()
    gi, kv, rp = model.prepare_prompts_round(kv0, rp0, prompts, tok, NT)
    ql = gi["text_token_lens"].to(torch.int64)
    assert int(ql.sum()) == gi["packed_text_ids"].numel()
    for q, p in enumerate(prompts):
        got = _block(gi, q, ql)
        if p is None:
            assert int(ql[q]) == 0 and kv[q] == kv0[q] and rp[q] == rp0[q]
            assert int(got["key_values_lens"]) == kv0[q]
            assert torch.equal(got["packed_key_value_indexes"], torch.arange(kv0[q]))
            continue
        want, kv1, rp1 = model.prepare_prompts([kv0[q]], [rp0[q]], [p], tok, NT)
        assert kv[q] == kv1[0] and rp[q] == rp1[0]
        for k, v in want.items():
            assert torch.equal(got[k], v), (q, k)
    # every row of the packed sequence is used exactly once
    used = torch.cat([gi["packed_text_indexes"], gi["packed_key_value_indexes"]])
    assert torch.equal(used.sort().values, torch.arange(int(ql.sum()) + sum(kv0)))


def test_prompts_round_with_every_text_is_prepare_prompts(model):
    tok = helpers.IntTokenizer()
    a = model.prepare_prompts_round([3, 0, 7], [1, 0, 2], ["1 2", "3", ""], tok, NT)
    b = model.prepare_prompts([3, 0, 7], [1, 0, 2], ["1 2", "3", ""], tok, NT)
    assert a[1:] == b[1:] and set(a[0]) == set(b[0]) and all(torch.equal(a[0][k], b[0][k]) for k in a[0])


IMG = object()      # the schedule reads only whether a request has an image


def test_schedule_of_a_mixed_set():
    reqs = [
        dict(text="a"),                                                  # 0 T2I
        dict(text="a", think=True),                                      # 1 T2I + think
        dict(text="a", image=IMG),                                       # 2 edit
        dict(text="a", image=IMG, think=True),                           # 3 edit + think
        dict(text="a", image=IMG, understanding_output=True),            # 4 understanding
        dict(text="a", image=IMG, understanding_output=True, think=True),   # 5 understanding + think
        dict(),                                                          # 6 nothing: no round at all
        dict(text="a", understanding_output=True),                       # 7 text-only understanding
        dict(image=IMG, think=True),                                     # 8 image-only generation with think
        dict(image=None, text=None, think=True),                         # 9 nothing either
    ]
    s = call_batch_schedule(reqs)
    assert s == {
        "system": [1, 3, 5, 8],
        "system_cfg_img": [1, 3, 8],
        "vae": [2, 3, 8],
        "vit": [2, 3, 4, 5, 8],
        "prompt": [0, 1, 2, 3, 4, 5, 7],
        "prompt_cfg_img": [0, 1, 2, 3],
        "decode": [1, 3, 4, 5, 7, 8],
        "thought": [1, 3, 8],
        "generate": [0, 1, 2, 3, 8],
    }
    # a pure function of each request: a request's rounds do not depend on the others
    for q, r in enumerate(reqs):
        alone = call_batch_schedule([r])
        assert {k: (v == [0]) for k, v in alone.items()} == {k: (q in v) for k, v in s.items()}, q
    assert not any(call_batch_schedule([]).values())


def _inferencer(model):
    return InterleaveInferencer(model, None, helpers.IntTokenizer(), None, None, NT)


def test_request_validation_and_refusals(model):
    inf = _inferencer(model)
    with pytest.raises(ValueError, match="unknown request keys"):
        inf.call_batch([dict(text="1"), dict(text="2", cfg_scale=3.0)])
    with pytest.raises(NotImplementedError, match="TaylorSeer"):
        inf.call_batch([dict(text="1", enable_taylorseer=True)])
    with pytest.raises(ValueError, match="Unsupported input type"):
        inf.call_batch([dict(text="1", image="not an image")])
    with pytest.raises(ValueError, match="text must be a string"):
        inf.call_batch([dict(text=5)])
    # no input at all: nothing to run, like __call__
    assert inf.call_batch([dict(), dict(think=True, seed=3)]) == [{"image": None, "text": None}] * 2
    assert inf.call_batch([]) == []
    # enable_taylorseer=False is the default setting, accepted
    assert inf.call_batch([dict(enable_taylorseer=False)]) == [{"image": None, "text": None}]


def test_generate_text_batch_per_request_argument_checks(model):
    kw = dict(past_key_values=None, packed_key_value_indexes=None, key_values_lens=[3, 4], packed_start_tokens=None,
              packed_query_position_ids=None)
    with pytest.raises(ValueError, match="max_length has 1 entries"):
        model.generate_text_batch(**kw, max_length=[5])
    with pytest.raises(ValueError, match="temperature"):
        model.generate_text_batch(**kw, max_length=5, do_sample=[False, True], temperature=[1.0, 0.0])
    with pytest.raises(ValueError, match="keys"):
        model.generate_text_batch(**kw, max_length=[5, 6], keys=[1])
    # no request has a budget: nothing to decode
    out = model.generate_text_batch(**kw, max_length=[0, -2], do_sample=True, temperature=0.3)
    assert [t.numel() for t in out] == [0, 0]
    mb = helpers.build_product_bagel(device="cpu", load=False, dtype_mode="B")
    with pytest.raises(NotImplementedError):
        mb.generate_text_batch(**kw, max_length=[5, 6])


def test_gather_requests_without_copies():
    L = 3
    c = NaiveCache(L)
    for li in range(L):
        c.key_cache[li] = torch.randn(9, 2, 4)
        c.value_cache[li] = torch.randn(9, 2, 4)
    # the members' blocks are the whole cache (request 1 has no rows): a new cache over the same tensors
    g = gather_requests(c, [4, 0, 5], [0, 2])
    assert g is not c and g.key_cache is not c.key_cache
    assert all(g.key_cache[li] is c.key_cache[li] and g.value_cache[li] is c.value_cache[li] for li in range(L))
    g.key_cache[0] = None                  # replacing an entry of the new cache leaves the source alone
    assert c.key_cache[0] is not None
    # no member rows
    e = gather_requests(c, [4, 0, 5], [1])
    assert e.num_layers == L and e.seq_lens == 0
    assert gather_requests(NaiveCache(L), [0, 0], [0, 1]).seq_lens == 0
