"""n samples per request in batched text decode, without a GPU: the shared-prefix decode plan's slab layout and write
slots (decode_prepare's arithmetic restated on the host), the replication fallback, the per-sample Philox keys, the
argument checks of generate_text_batch / chat_batch (raised before any prefill) and of the C entry."""
import numpy as np
import pytest
import torch

import helpers
from bagel_b200 import _cabi, build
from bagel_b200.bagel import _sample_keys
from bagel_b200.qwen2_navit import SHARED_MIN_CTX_PER_SAMPLE, SHARED_MIN_SAMPLES, ForwardPlan
from oracle import fixtures


@pytest.fixture(scope="module")
def lm128():
    return helpers.build_product_bagel(fixtures.TINY128_LM, device="cpu", load=False).language_model.model


@pytest.fixture(scope="module")
def lm64():
    return helpers.build_product_bagel(fixtures.TINY_LM, device="cpu", load=False).language_model.model


def _ragged(seed):
    g = np.random.default_rng(seed)
    R = int(g.integers(1, 9))
    ctx = g.integers(0, 40, R).tolist()
    ns = g.integers(1, 7, R).tolist()
    ctx[int(g.integers(R))] = 0
    ns[int(g.integers(R))] = 1
    i = int(g.integers(R))
    ns[i] = SHARED_MIN_SAMPLES + int(g.integers(0, 30))       # a request for which the shared layout pays
    ctx[i] = SHARED_MIN_CTX_PER_SAMPLE * ns[i] + int(g.integers(0, 100))
    return ctx, ns, int(g.integers(1, 20))


@pytest.mark.parametrize("seed", range(12))
def test_shared_plan_layout(lm128, seed):
    ctx, ns, T = _ragged(seed)
    p = ForwardPlan.decode_shared(lm128, ctx, ns, T)
    sh = p.shared
    assert sh is not None and p.ctx_src is None
    R, B = len(ctx), sum(ns)
    assert p.batch == p.n == B
    assert p.total_kv == sum(ctx) + sum(ns) * T
    assert sh.cu_rows.tolist() == np.cumsum([0] + ns).tolist() and sh.max_group_rows == max(ns)
    assert sh.prefix_len.tolist() == ctx
    pb, sb, base = sh.prefix_begin.tolist(), sh.suffix_begin.tolist(), p.cu_k.tolist()
    owner = np.zeros(p.total_kv, dtype=np.int64) - 1
    r = 0
    for i in range(R):
        # request i's region: its context, then one suffix of T rows per sample, contiguous
        lo = pb[i]
        assert lo == (0 if i == 0 else pb[i - 1] + ctx[i - 1] + ns[i - 1] * T)
        assert (owner[lo:lo + ctx[i]] == -1).all()
        owner[lo:lo + ctx[i]] = i
        for j in range(ns[i]):
            assert sb[r] == lo + ctx[i] + j * T
            assert (owner[sb[r]:sb[r] + T] == -1).all()
            owner[sb[r]:sb[r] + T] = 1000 + r
            # decode_prepare: kv_rows = base + seq_len, seqused = seq_len + 1, seq_len = ctx + tokens so far
            for step in range(T):
                seq_len = ctx[i] + step
                assert base[r] + seq_len == sb[r] + step
                assert seq_len + 1 - ctx[i] == step + 1        # the kernel's suffix length
            r += 1
    assert (owner >= 0).all(), "every slab row belongs to a context or a suffix"
    # the context rows are placed once, in cache order
    want_ctx = [pb[i] + t for i in range(R) for t in range(ctx[i])]
    assert p.ctx_rows.tolist() == want_ctx
    assert p.max_k == max(c for c in ctx) + T


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("why", ["head_dim64", "few_samples", "short_context"])
def test_fallback_plan_is_decode_over_repeated_rows(lm64, lm128, seed, why):
    ctx, ns, T = _ragged(seed)
    lm = lm64
    if why == "few_samples":     # no request with SHARED_MIN_SAMPLES samples: replication measured faster
        ns = [min(n, SHARED_MIN_SAMPLES - 1) for n in ns]
        lm = lm128
    if why == "short_context":   # every request with many samples has a short context per sample
        ctx = [min(c, SHARED_MIN_CTX_PER_SAMPLE * n - 1) for c, n in zip(ctx, ns)]
        lm = lm128
    p = ForwardPlan.decode_shared(lm, ctx, ns, T)
    rep = [c for c, n in zip(ctx, ns) for _ in range(n)]
    want = ForwardPlan.decode(lm, rep, T)
    assert p.shared is None
    for name in ("batch", "n", "n_ctx", "total_kv", "max_q", "max_k", "fuse_qkv"):
        assert getattr(p, name) == getattr(want, name), name
    for name in ("cu_q", "cu_k", "ctx_rows"):
        assert torch.equal(getattr(p, name), getattr(want, name)), name
    # each placed row copies its request's cache rows
    start = np.cumsum([0] + ctx)
    assert p.ctx_src.tolist() == [start[i] + t for i, n in enumerate(ns) for _ in range(n) for t in range(ctx[i])]


def test_sample_keys():
    R, seeds = 5, [7, 2 ** 33 + 5, 0, 123456789, 2 ** 32 - 1]
    ones = _sample_keys(seeds, [1] * R)
    assert ones == [(sd & 0xFFFFFFFF) | (i << 32) for i, sd in enumerate(seeds)]      # the keys without num_samples
    ns = [3, 1, 4, 1, 2]
    ks = _sample_keys(seeds, ns)
    assert len(set(ks)) == len(ks) == sum(ns)
    assert [ks[f] for f in np.cumsum([0] + ns)[:-1]] == ones                          # sample 0 keeps its key
    assert ks[1] == (7 | ((0 + 5 * 1) << 32)) and ks[-1] == ((2 ** 32 - 1) | ((4 + 5 * 1) << 32))
    assert len(set(_sample_keys([9] * R, ns))) == sum(ns)                              # one seed for all: distinct


# ---------------------------------------------------------------------------------------------- argument checks

@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel(device="cpu", load=False)


KW = dict(past_key_values=None, packed_key_value_indexes=None, key_values_lens=[3, 4], packed_start_tokens=None,
          packed_query_position_ids=None)

BAD = [
    (dict(num_samples=0), "num_samples must be"), (dict(num_samples=-1), "num_samples must be"),
    (dict(num_samples=True), "num_samples must be"), (dict(num_samples=2.0), "num_samples must be"),
    (dict(num_samples=[2, 0]), "num_samples must be"), (dict(num_samples=[2, False]), "num_samples must be"),
    (dict(num_samples=[2, 1.5]), "num_samples must be"), (dict(num_samples=[2]), "num_samples has 1 entries"),
    (dict(num_samples=[1, 2, 3]), "num_samples has 3 entries"),
]


@pytest.mark.parametrize("bad,match", BAD)
def test_generate_text_batch_refuses_bad_num_samples(model, bad, match):
    with pytest.raises(ValueError, match=match):
        model.generate_text_batch(**KW, max_length=5, **bad)


def test_generate_text_batch_checks_per_request_lists_and_keys(model):
    with pytest.raises(ValueError, match="temperature has 3 entries for 2 requests"):
        model.generate_text_batch(**KW, max_length=5, do_sample=True, temperature=[1.0, 1.0, 1.0], num_samples=[2, 1])
    with pytest.raises(ValueError, match="top_k has 3 entries"):
        model.generate_text_batch(**KW, max_length=5, do_sample=True, top_k=[1, 2, 3], num_samples=[2, 1])
    with pytest.raises(ValueError, match="2 keys for 3 samples"):
        model.generate_text_batch(**KW, max_length=5, keys=[1, 2], num_samples=[2, 1])
    with pytest.raises(ValueError, match="3 seeds for 2 requests"):
        model.generate_text_batch(**KW, max_length=5, seeds=[1, 2, 3], num_samples=2)


def test_generate_text_batch_nothing_to_decode(model):
    out = model.generate_text_batch(**KW, max_length=[0, 0], num_samples=[2, 3])
    assert [len(x) for x in out] == [2, 3] and all(t.numel() == 0 for x in out for t in x)
    out = model.generate_text_batch(**KW, max_length=0, num_samples=None)
    assert [t.numel() for t in out] == [0, 0]


@pytest.mark.parametrize("bad,match", BAD)
def test_chat_batch_refuses_bad_num_samples_before_prefill(model, bad, match, monkeypatch):
    def no_prefill(*a, **kw):
        raise AssertionError("prefill ran before the argument check")

    monkeypatch.setattr(model, "prepare_vit_image_round", no_prefill)
    monkeypatch.setattr(model, "prepare_prompts", no_prefill)
    reqs = [([], "1 2"), ([], "3")]
    with pytest.raises(ValueError, match=match):
        model.chat_batch(helpers.IntTokenizer(), helpers.NEW_TOKEN_IDS, None, reqs, max_length=4, **bad)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _cabi.lib()


def test_shared_attention_argument_validation_without_gpu(lib):
    f = lib.bagel_attn_decode_shared_bf16
    # (q, k, v, out, cu_rows, prefix_begin, prefix_len, suffix_begin, seqused_k, groups, rows, max_group_rows,
    #  Hq, Hk, head_dim, max_seqlen_k, scale, ld_q, ld_k, ld_v, ld_out, stream)
    args = [None] * 9 + [2, 5, 3, 28, 4, 128, 100, 0.088, 3584, 512, 512, 3584, None]

    def call(**kw):
        a = list(args)
        for i, val in kw.items():
            a[int(i[1:])] = val
        return f(*a)

    assert call(a14=64) == -1 and b"head_dim" in lib.bagel_last_error()
    assert call(a12=12, a13=4) == -1 and b"GQA group 3" in lib.bagel_last_error()
    assert call(a12=28, a13=0) == -1
    assert call(a12=30, a13=4) == -1
    assert call(a11=0) == -1 and b"max_group_rows" in lib.bagel_last_error()
    assert call(a11=6) == -1                                     # more rows in a group than rows
    assert call(a9=-1) == -1
    assert call(a9=70000, a10=70000, a11=1) == -1 and b"groups x passes" in lib.bagel_last_error()
    assert call(a17=3583) == -2
    assert call(a1=8) == -2                                      # k not 16-byte aligned
    assert call(a17=3576) == -5 and b"shorter than a row" in lib.bagel_last_error()
    assert call(a20=256) == -5
