"""-m gpu: n samples per request in batched text decode. The shared-prefix decode attention (attn_decode_shared.cu)
against fp64 attention over the same bf16 inputs for every GQA group, ragged groups and prefixes, strided q/out and
large-logit outliers, at every key split; its independence of group order and of the other rows of a pass; decode with
num_samples against decode over the context replicated per row (teacher-forced logits and picks); the head_dim 64
replication fallback; the unchanged step when every n_i = 1; per-sample stopping and settings; chat_batch."""
import json

import numpy as np
import pytest
import torch

import gemm_oracle as go
import helpers
from oracle import fixtures
from sampling_oracle import gumbel_scores

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
NT = dict(helpers.NEW_TOKEN_IDS)
ATOL, RTOL = 1e-2, 2e-2   # the tolerances of test_gpu_attn_routes.py's decode route test
GROUPS = {1: (4, 4), 2: (8, 4), 4: (16, 4), 7: (28, 4), 8: (8, 1)}   # G -> (Hq, Hk)
S = 4                     # rows per CTA pass of the shared kernel


def _ops():
    from bagel_b200 import ops
    return ops


def _cu(lens):
    return torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=DEV)


def _i32(x):
    return torch.tensor(list(x), dtype=torch.int32, device=DEV)


def _case(ns, ctx, used, Hq, Hk, seed, q_pad=0, outliers=False, spare=3):
    """Slab with each group's prefix once and one suffix region per row (contents of spare rows are finite noise)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    B = sum(ns)
    pb, sb = [], []
    at = 0
    r = 0
    for n, c in zip(ns, ctx):
        pb.append(at)
        at += c + spare
        for _ in range(n):
            sb.append(at)
            at += used[r] + spare
            r += 1
    k = torch.randn(at, Hk, 128, device=DEV, generator=g).to(BF)
    v = torch.randn(at, Hk, 128, device=DEV, generator=g).to(BF)
    qbuf = torch.randn(B, Hq * 128 + q_pad, device=DEV, generator=g).to(BF)
    q = qbuf[:, :Hq * 128].view(B, Hq, 128) if q_pad else qbuf.view(B, Hq, 128)
    if outliers:
        G = Hq // Hk
        r = 0
        for i, (n, c) in enumerate(zip(ns, ctx)):
            for _ in range(n):
                # one key far above the rest in the prefix (shared) and one in this row's suffix
                if c:
                    k[pb[i] + c // 2, 0] = (q[r, 0].float() * 3).to(BF)
                k[sb[r] + used[r] - 1, 0] = (q[r, G - 1].float() * 4).to(BF)
                r += 1
    seqused = []
    r = 0
    for n, c in zip(ns, ctx):
        for _ in range(n):
            seqused.append(c + used[r])
            r += 1
    return dict(q=q, k=k, v=v, ns=ns, ctx=ctx, used=used, pb=pb, sb=sb, seqused=seqused)


def _run(c, out=None):
    return _ops().attn_decode_shared(c["q"], c["k"], c["v"], _cu(c["ns"]), _i32(c["pb"]), _i32(c["ctx"]),
                                     _i32(c["sb"]), _i32(c["seqused"]), max(c["ns"]),
                                     max(c["seqused"]), out=out)


def _ref(c):
    q, k, v = c["q"], c["k"], c["v"]
    Hq, Hk = q.shape[1], k.shape[1]
    out = torch.zeros(q.shape, dtype=torch.float64, device=DEV)
    r = 0
    for i, (n, ctx) in enumerate(zip(c["ns"], c["ctx"])):
        for _ in range(n):
            rows = list(range(c["pb"][i], c["pb"][i] + ctx)) + list(range(c["sb"][r], c["sb"][r] + c["used"][r]))
            idx = torch.tensor(rows, device=DEV, dtype=torch.long)
            kk = k[idx].double().transpose(0, 1).repeat_interleave(Hq // Hk, dim=0)
            vv = v[idx].double().transpose(0, 1).repeat_interleave(Hq // Hk, dim=0)
            s = q[r].double()[:, None, :] @ kk.transpose(1, 2) * 128 ** -0.5
            out[r] = (torch.softmax(s, -1) @ vv)[:, 0]
            r += 1
    return out


def _split(groups_passes, Hk, max_k, sms):
    """The shared kernel's key-split rule (attn_decode's, over (pass, kv head) pairs)."""
    pairs, split = groups_passes * Hk, 1
    while split < 8 and pairs * split * 2 <= 2 * sms:
        split *= 2
    while split > 1 and (max_k + split - 1) // split < 64:
        split //= 2
    return split


def _cases():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(0)
    out = []
    for G, (Hq, Hk) in GROUPS.items():
        # every group size and prefix length of interest in one ragged batch
        ns = [1, 2, 3, S, S + 1, 2 * S + 3, 32]
        ctx = [0, 1, 15, 16, 17, 1300, 4100]
        used = [int(u) for u in rng.integers(1, 140, sum(ns))]
        used[0], used[1] = 1, 128
        out.append((f"G{G}-ragged", dict(ns=ns, ctx=ctx, used=used, Hq=Hq, Hk=Hk, q_pad=0)))
        # fewer (pass, kv head) pairs: the key split grows to 2, 4 and 8
        for ns1, ctx1 in (([3], [4100]), ([S + 1, 2], [1300, 17]), ([2] * 5, [700] * 5), ([2] * 20, [300] * 20)):
            used1 = [int(u) for u in rng.integers(1, 100, sum(ns1))]
            out.append((f"G{G}-{ns1}-{ctx1[0]}", dict(ns=ns1, ctx=ctx1, used=used1, Hq=Hq, Hk=Hk, q_pad=256)))
    for name, kw in out:
        passes = max(-(-n // S) for n in kw["ns"])
        kw["split"] = _split(len(kw["ns"]) * passes, kw["Hk"], max(c + u for c, u in zip(
            np.repeat(kw["ctx"], kw["ns"]), kw["used"])), sms)
    return out


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_shared_kernel_against_fp64(cases):
    splits = set()
    for name, kw in cases:
        for outl in (False, True):
            c = _case(kw["ns"], kw["ctx"], kw["used"], kw["Hq"], kw["Hk"], seed=len(name) + outl, q_pad=kw["q_pad"],
                      outliers=outl)
            B, Hq = sum(kw["ns"]), kw["Hq"]
            obuf = torch.full((B, Hq * 128 + 64), float("nan"), device=DEV, dtype=BF)
            out = _run(c, out=obuf[:, :Hq * 128].view(B, Hq, 128))
            assert torch.isnan(obuf[:, Hq * 128:]).all(), f"{name}: out's gap columns were written"
            assert torch.isfinite(out).all(), name
            torch.testing.assert_close(out.double(), _ref(c), atol=ATOL, rtol=RTOL, msg=lambda m: f"{name}: {m}")
            assert torch.equal(out, _run(c)), f"{name}: repeated call differs"
        splits.add(kw["split"])
    assert splits == {1, 2, 4, 8}, splits


def test_shared_kernel_group_permutation_and_row_independence():
    Hq, Hk = GROUPS[7]
    ns, ctx = [3, 1, 6, 2], [900, 0, 257, 33]
    used = [5, 17, 1, 40, 3, 3, 3, 64, 9, 2, 2, 77]
    c = _case(ns, ctx, used, Hq, Hk, seed=5)
    out = _run(c)
    perm = [2, 0, 3, 1]
    first = np.cumsum([0] + ns)
    rows = [r for i in perm for r in range(first[i], first[i + 1])]
    cp = dict(c, q=c["q"][rows].contiguous(), ns=[ns[i] for i in perm], ctx=[ctx[i] for i in perm],
              pb=[c["pb"][i] for i in perm], sb=[c["sb"][r] for r in rows], used=[used[r] for r in rows],
              seqused=[c["seqused"][r] for r in rows])
    assert torch.equal(_run(cp), out[rows]), "permuting the groups must permute the output bit for bit"
    # equal rows of one group give equal bits, wherever they sit in the pass
    c2 = dict(c)
    q2 = c["q"].clone()
    q2[first[2]:first[3]] = q2[first[2]]
    sb2 = list(c["sb"])
    sb2[first[2]:first[3]] = [c["sb"][first[2]]] * ns[2]
    u2 = list(c["seqused"])
    u2[first[2]:first[3]] = [c["seqused"][first[2]]] * ns[2]
    c2.update(q=q2, sb=sb2, seqused=u2)
    o2 = _run(c2)
    for r in range(first[2], first[3]):
        assert torch.equal(o2[r], o2[first[2]]), r
    # a row's output does not depend on the other rows of its group (row first[2] kept its inputs, the others changed)
    assert torch.equal(o2[first[2]], out[first[2]])


def _observe(fn, path):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        events = json.load(f).get("traceEvents", [])
    ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    return len(ks), [tuple(e.get("args", {}).get("grid") or ()) for e in ks if "attn_decode_shared_kernel" in e["name"]]


def test_shared_kernel_splits_observed(tmp_path):
    if not go.IN_CHILD:
        # a fresh process: a torch.profiler session that follows earlier ones in the same process may record only part
        # of the kernel events (see gemm_oracle.run_in_child)
        out = go.run_in_child(__file__, "test_shared_kernel_splits_observed")
        print(out[out.find("shared route proof"):].splitlines()[0])
        return
    inputs = [(kw, _case(kw["ns"], kw["ctx"], kw["used"], kw["Hq"], kw["Hk"], seed=1)) for _, kw in _cases()]
    for _, c in inputs:       # first launches (module load, smem attribute) outside the profiled window
        _run(c)
    n, grids = _observe(lambda: [_run(c) for _, c in inputs], tmp_path / "shared.json")
    if n == 0:
        pytest.skip("torch.profiler recorded no CUDA kernel events on this machine")
    assert len(grids) == len(inputs)
    for (kw, _), grid in zip(inputs, grids):
        if grid:
            passes = max(-(-m // S) for m in kw["ns"])
            assert grid == (kw["split"], kw["Hk"], len(kw["ns"]) * passes), (kw["ns"], grid)
    splits = {g[0] for g in grids if g}
    assert splits == {1, 2, 4, 8}, splits
    print(f"shared route proof: {len(grids)} launches, splits observed {sorted(splits)}")


# ------------------------------------------------------------------------------------------------------------ decode

def _text_context(model, prompts):
    from bagel_b200.qwen2_navit import NaiveCache
    B = len(prompts)
    gi, kv, rp = model.prepare_prompts([0] * B, [0] * B, prompts, helpers.IntTokenizer(), NT)
    cache = model.forward_cache_update_text(NaiveCache(model.config.llm_config.num_hidden_layers), **gi)
    return cache, model.prepare_start_tokens(kv, rp, NT)


def _replicated(cache, gs, ns):
    """The context of request i repeated n_i times, as independent requests."""
    from bagel_b200.qwen2_navit import gather_requests
    kv = torch.as_tensor(gs["key_values_lens"]).cpu()
    members = [i for i, n in enumerate(ns) for _ in range(n)]
    rc = gather_requests(cache, kv, members)
    m = torch.tensor(members)
    kvr = kv[m]
    return rc, dict(key_values_lens=kvr, packed_key_value_indexes=torch.arange(int(kvr.sum())),
                    packed_start_tokens=torch.as_tensor(gs["packed_start_tokens"]).cpu()[m],
                    packed_query_position_ids=torch.as_tensor(gs["packed_query_position_ids"]).cpu()[m])


def _flat(nested):
    return [t for ts in nested for t in ts]


# request 2 has 5 samples and a context of >= 64 tokens per sample: the batch takes the shared layout
PROMPTS3 = ["5 17 900 33 2", "8 8 100 4 77 650 12", " ".join(str(7 * i % 997) for i in range(330))]
NS = [3, 1, 5]


def _teacher_forced_logits(model, cache, gs, fed, ns=None):
    """Each step's logits [T, rows, V] of the decode state, fed the token sequences `fed` [T, rows] (row r's token at
    step s, the start token at step 0)."""
    ops = _ops()
    d = model._decode_state(cache, gs["key_values_lens"], gs["packed_start_tokens"], gs["packed_query_position_ids"],
                            fed.shape[0], ns)
    out = []
    for s in range(fed.shape[0]):
        assert torch.equal(d["tokens"], fed[s].to(DEV))
        d["body"]()
        out.append(d["logits"].float().clone())
        ops.decode_advance(d["seq_len"], d["pos"], d["tokens"], d["history"], d["step_dev"])
        if s + 1 < fed.shape[0]:
            d["tokens"].copy_(fed[s + 1].to(DEV))
            d["tokens32"].copy_(fed[s + 1].to(DEV, torch.int32))
    return torch.stack(out)


@pytest.fixture(scope="module", params=["tiny128", "7b-2layer"])
def decode_model(request):
    if request.param == "tiny128":
        return helpers.build_product_bagel(fixtures.TINY128_LM, "cuda")
    from bagel_b200 import synthetic
    return synthetic.build_random_bagel(num_layers=2)


@pytest.mark.parametrize("do_sample", [False, True])
def test_decode_matches_replicated_context(decode_model, do_sample):
    model = decode_model
    T = 12
    cache, gs = _text_context(model, PROMPTS3)
    rc, rgs = _replicated(cache, gs, NS)
    keys = [(0x5EED + 31 * r) | (r << 32) for r in range(sum(NS))]
    temp = 0.9
    want = model.generate_text_batch(rc, max_length=T, do_sample=do_sample, temperature=temp, keys=keys, **rgs)
    got = model.generate_text_batch(cache, max_length=T, do_sample=do_sample, temperature=temp, keys=keys,
                                     num_samples=NS, **gs)
    assert [len(x) for x in got] == NS
    got = _flat(got)
    assert all(len(t) == T for t in want) and all(len(t) == T for t in got)
    fed = torch.stack([t.cpu() for t in want], 1)                           # [T, rows], the start token first
    ls = _teacher_forced_logits(model, cache, gs, fed, NS)
    lr = _teacher_forced_logits(model, rc, rgs, fed)
    # the two layouts differ only in the order of the attention sums: logits agree to bf16 rounding noise
    err = (ls - lr).abs().max().item()
    scale = lr.abs().max().item()
    print(f"teacher-forced logits: max |shared - replicated| = {err:.4g} (|logit| max {scale:.3g})")
    assert err <= 0.02 * scale + 0.02, (err, scale)
    # the picks agree wherever the top-1 / top-2 margin of the (Gumbel) score exceeds that noise
    for r in range(sum(NS)):
        a, b = got[r].tolist(), want[r].tolist()
        if a == b:
            continue
        s = next(k for k in range(T) if a[k] != b[k])
        row = lr[s - 1, r].cpu().numpy()
        sc = gumbel_scores(row, temp, keys[r], s - 1) if do_sample else row
        top2 = np.sort(sc)[-2:]
        assert top2[1] - top2[0] <= 2 * (err / (temp if do_sample else 1.0)) + 1e-6, (r, s, top2)


def test_fallback_head64_is_replication_bit_for_bit():
    model = helpers.build_product_bagel(fixtures.TINY_LM, "cuda")
    cache, gs = _text_context(model, PROMPTS3)
    rc, rgs = _replicated(cache, gs, NS)
    keys = [(77 + r) | (r << 32) for r in range(sum(NS))]
    for do_sample in (False, True):
        want = model.generate_text_batch(rc, max_length=10, do_sample=do_sample, keys=keys, **rgs)
        got = _flat(model.generate_text_batch(cache, max_length=10, do_sample=do_sample, keys=keys, num_samples=NS,
                                              **gs))
        assert all(torch.equal(a, b) for a, b in zip(got, want))


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


def _record(monkeypatch, lib=None):
    from bagel_b200 import _cabi
    rec = _Recorder(lib or _cabi.lib())
    monkeypatch.setattr(_cabi, "_lib", rec)
    return rec


@pytest.mark.parametrize("do_sample", [False, True])
def test_all_ones_is_the_step_without_num_samples(monkeypatch, do_sample):
    model = helpers.build_product_bagel(fixtures.TINY128_LM, "cuda")
    model.use_cuda_graph = False      # every step's launches go through the library
    cache, gs = _text_context(model, PROMPTS3)
    from bagel_b200 import _cabi
    lib = _cabi.lib()
    runs = []
    for kw in (dict(), dict(num_samples=None), dict(num_samples=1), dict(num_samples=[1, 1, 1])):
        rec = _record(monkeypatch, lib)
        out = model.generate_text_batch(cache, max_length=8, do_sample=do_sample, seeds=[3, 4, 5], **gs, **kw)
        if kw.get("num_samples") is not None:
            assert all(len(x) == 1 for x in out)
            out = _flat(out)
        runs.append((rec.calls, [t.cpu() for t in out]))
    assert "bagel_attn_decode_shared_bf16" not in runs[0][0]
    for calls, toks in runs[1:]:
        assert calls == runs[0][0]
        assert all(torch.equal(a, b) for a, b in zip(toks, runs[0][1]))


def test_shared_step_launches_and_one_replay_per_step(monkeypatch):
    model = helpers.build_product_bagel(fixtures.TINY128_LM, "cuda")
    cache, gs = _text_context(model, PROMPTS3)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
    rec = _record(monkeypatch)
    n = 10
    out = model.generate_text_batch(cache, max_length=n, do_sample=True, num_samples=NS, **gs)
    assert [len(x) for x in out] == NS and all(len(t) == n for t in _flat(out))
    L = fixtures.TINY128_LM.num_hidden_layers
    assert rec.calls.count("bagel_attn_decode_shared_bf16") == 2 * L     # eager step 0 and the captured step 1
    assert "bagel_attn_varlen_fwd" not in rec.calls
    assert rec.calls[:2 * L] == ["bagel_copy_rows_bf16"] * (2 * L)       # the context placed once per layer, K and V
    assert len(replays) == n - 1


def test_per_sample_stop_and_settings():
    """Per-request settings reach every sample, and each sample stops, freezes and penalises on its own: the result
    equals the same decode over the replicated context with the settings listed per row (head_dim 64: that decode
    runs the same kernels on the same layout, so bit for bit)."""
    model = helpers.build_product_bagel(fixtures.TINY_LM, "cuda")
    cache, gs = _text_context(model, PROMPTS3)
    rc, rgs = _replicated(cache, gs, NS)
    keys = [(1234 + 7 * r) | (r << 32) for r in range(sum(NS))]
    per = dict(max_length=[12, 5, 16], do_sample=[True, False, True], temperature=[0.7, 1.0, 1.3], top_k=[20, None, 0],
               top_p=[None, None, 0.9], repetition_penalty=[1.3, None, 1.1], frequency_penalty=[None, 0.5, 0.2])
    row = {k: [v for v, n in zip(x, NS) for _ in range(n)] for k, x in per.items()}
    full = model.generate_text_batch(rc, keys=keys, **row, **rgs)
    stream = full[0].tolist()
    eos = next(t for t in stream[2:] if t not in stream[:2])
    want = model.generate_text_batch(rc, keys=keys, end_token_id=eos, **row, **rgs)
    got = model.generate_text_batch(cache, keys=keys, end_token_id=eos, num_samples=NS, **per, **gs)
    got = _flat(got)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    lens = [len(t) for t in got]
    assert lens[0] < 12 and max(lens) > lens[0], lens               # sample 0 froze while others went on
    assert all(n <= 12 for n in lens[:3]) and lens[3] <= 5 and all(n <= 16 for n in lens[4:]), lens


def test_shared_decode_per_sample_stop():
    """The same on the shared kernel (head_dim 128): sample 0 of request 0 stops at a token only it emits, the
    others go on and match their own decode without the stop."""
    model = helpers.build_product_bagel(fixtures.TINY128_LM, "cuda")
    cache, gs = _text_context(model, PROMPTS3)
    keys = [(99 + r) | (r << 32) for r in range(sum(NS))]
    full = _flat(model.generate_text_batch(cache, max_length=16, do_sample=True, keys=keys, num_samples=NS, **gs))
    s0 = full[0].tolist()
    k, eos = next((k, t) for k, t in enumerate(s0) if k >= 2 and t not in s0[:k])
    got = _flat(model.generate_text_batch(cache, max_length=16, do_sample=True, keys=keys, end_token_id=eos,
                                          num_samples=NS, **gs))
    assert got[0].tolist() == s0[:k]
    for f, g in zip(full, got):
        f = f.tolist()
        assert g.tolist() == (f[:f.index(eos)] if eos in f else f)
    assert max(len(g) for g in got) > k, "the other samples continue after sample 0 stops"


# --------------------------------------------------------------------------------------------------------- chat_batch

def _img(seed, h, w):
    return torch.rand(3, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def test_chat_batch_num_samples():
    model = helpers.build_product_bagel_with_vit(fixtures.TINY128_LM, "cuda")
    tok = fixtures.ToyTokenizer()
    long_prompt = " ".join(str(3 * i % 991) for i in range(400))      # >= 64 context tokens for each of 6 samples
    reqs = [(fixtures.vit_images(), "5 17 900 33 2 describe"), ([_img(4, 42, 42)], "88"), ([], long_prompt)]
    ident = lambda x: x  # noqa: E731
    chats = [model.chat(tok, NT, ident, req[0], req[1], max_length=8) for req in reqs]
    # greedy: n identical answers, each chat's answer (replicated layout, then the shared one)
    for ns in ([3, 1, 2], [3, 1, 6]):
        got = model.chat_batch(tok, NT, ident, reqs, max_length=8, num_samples=ns)
        assert [len(x) for x in got] == ns
        for want, answers in zip(chats, got):
            assert answers == [want] * len(answers)
    # None: today's List[str]
    assert model.chat_batch(tok, NT, ident, reqs, max_length=8) == chats
    # sampled: n strings per request; sample 0 uses the key the request has without num_samples
    kw = dict(max_length=10, do_sample=True, temperature=1.0, seeds=[5, 6, 7])
    one = model.chat_batch(tok, NT, ident, reqs, **kw)
    many = model.chat_batch(tok, NT, ident, reqs, num_samples=[5, 5, 6], **kw)
    assert [len(x) for x in many] == [5, 5, 6] and all(isinstance(s, str) for x in many for s in x)
    same = sum(m[0] == o for m, o in zip(many, one))
    assert same >= len(reqs) - 1, (many, one)       # up to a near-tie pick, sample 0 is the n = 1 answer
    assert any(len(set(x)) > 1 for x in many), "samples of a request are drawn independently"
