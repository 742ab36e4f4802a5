"""Host logic of batched image generation (no GPU): the packed LM-call layout of Bagel.generate_image_batch gives every
request exactly the samples its own single-request plan has (prepare_vae_latent -> prepare_vae_latent_cfg ->
_cfg_branches on that request alone), shifted to its block; the per-step plan choice and CFG table follow each
request's own interval; prepare_vae_image_round matches prepare_vae_images per request; per-request seeds draw the
init noise a single seeded request draws."""
import random

import pytest
import torch

import helpers
from bagel_b200.bagel import _branch_counts, _cfg_branches, _flow_batch_layout, _flow_batch_schedule

NT = helpers.NEW_TOKEN_IDS


@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel_with_vit(device="cpu", load=False)


class _Ctx:
    """Stands in for a NaiveCache that holds rows (the layout only asks whether a cache has any)."""
    key_cache = {0: torch.zeros(1)}


SCALES = [(4.0, 1.5), (4.0, 1.0), (1.0, 1.5), (1.0, 1.0), (2.5, 2.0)]     # 3, 2, 1, 1 and 3 branches
INTERVALS = [(0.4, 1.0), (0.0, 1.0), (0.6, 0.9), (0.0, 0.3)]


def _requests(rnd, R):
    reqs = []
    for _ in range(R):
        edit = rnd.random() < 0.5
        img_ctx = rnd.randint(3, 40) if edit else 0          # VAE + ViT rows of an edit's image
        txt = rnd.randint(2, 9)
        size = (16 * rnd.randint(1, 5), 16 * rnd.randint(1, 5))
        sT, sI = rnd.choice(SCALES)
        reqs.append(dict(main=(img_ctx + txt, 2 * edit + 1), text=(img_ctx, 2 * edit), img=(txt, 1), size=size,
                         sT=sT, sI=sI, iv=rnd.choice(INTERVALS)))
    return reqs


def _packed(model, reqs):
    sizes = [r["size"] for r in reqs]
    gi = model.prepare_vae_latent([r["main"][0] for r in reqs], [r["main"][1] for r in reqs], sizes, NT)
    ct = model.prepare_vae_latent_cfg([r["text"][0] for r in reqs], [r["text"][1] for r in reqs], sizes)
    ci = model.prepare_vae_latent_cfg([r["img"][0] for r in reqs], [r["img"][1] for r in reqs], sizes)
    text_cache = _Ctx() if any(r["text"][0] for r in reqs) else None
    br = _cfg_branches(
        (gi["packed_position_ids"], gi["packed_indexes"], _Ctx(), gi["key_values_lens"], gi["packed_key_value_indexes"]),
        (ct["cfg_packed_position_ids"], ct["cfg_packed_query_indexes"], text_cache, ct["cfg_key_values_lens"],
         ct["cfg_packed_key_value_indexes"]),
        (ci["cfg_packed_position_ids"], ci["cfg_packed_query_indexes"], _Ctx(), ci["cfg_key_values_lens"],
         ci["cfg_packed_key_value_indexes"]), 2.0, 2.0)
    return gi, br


def _single(model, r):
    gi = model.prepare_vae_latent([r["main"][0]], [r["main"][1]], [r["size"]], NT)
    ct = model.prepare_vae_latent_cfg([r["text"][0]], [r["text"][1]], [r["size"]])
    ci = model.prepare_vae_latent_cfg([r["img"][0]], [r["img"][1]], [r["size"]])
    br = _cfg_branches(
        (gi["packed_position_ids"], gi["packed_indexes"], None, gi["key_values_lens"], gi["packed_key_value_indexes"]),
        (ct["cfg_packed_position_ids"], ct["cfg_packed_query_indexes"], None, ct["cfg_key_values_lens"],
         ct["cfg_packed_key_value_indexes"]),
        (ci["cfg_packed_position_ids"], ci["cfg_packed_query_indexes"], None, ci["cfg_key_values_lens"],
         ci["cfg_packed_key_value_indexes"]), r["sT"], r["sI"])
    return gi, br


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("which", ["full", "main"])
def test_batch_layout_matches_single_request_plans(model, seed, which):
    rnd = random.Random(seed)
    reqs = _requests(rnd, rnd.randint(1, 7))
    R = len(reqs)
    gi, br = _packed(model, reqs)
    nbs = _branch_counts([r["sT"] for r in reqs], [r["sI"] for r in reqs])
    members = [list(range(R)), [q for q in range(R) if nbs[q] >= 2], [q for q in range(R) if nbs[q] >= 3]]
    if which == "main":
        members = members[:1]
    lay = _flow_batch_layout(gi["packed_seqlens"], gi["packed_vae_token_indexes"], gi["packed_text_indexes"], br, members)

    ql, kl = lay["query_lens"], lay["key_values_lens"]
    cq = torch.cumsum(ql, 0) - ql
    ck = torch.cumsum(kl, 0) - kl
    seen = {}
    for k, (b, q, row_off, q_off) in enumerate(lay["samples"]):
        seen.setdefault(b, []).append(q)
        assert int(cq[k]) == q_off
        gi1, br1 = _single(model, reqs[q])
        assert b < len(br1), "a request sits in a block its own plan does not have"
        want = br1[b]
        qs, ks = slice(int(cq[k]), int(cq[k] + ql[k])), slice(int(ck[k]), int(ck[k] + kl[k]))
        assert int(ql[k]) == int(gi1["packed_seqlens"][0])
        assert int(kl[k]) == int(want["key_values_lens"][0])
        assert torch.equal(lay["position_ids"][qs], want["packed_position_ids"])
        assert torch.equal(lay["packed_query_indexes"][qs] - row_off, want["packed_query_indexes"])
        assert torch.equal(lay["packed_key_value_indexes"][ks] - row_off, want["packed_key_value_indexes"])
        # expert routing rows and the latent rows the CFG kernel reads
        pv, pt = lay["packed_vae_token_indexes"], lay["packed_text_indexes"]
        assert torch.equal(pv[(pv >= qs.start) & (pv < qs.stop)] - q_off, gi1["packed_vae_token_indexes"])
        assert torch.equal(pt[(pt >= qs.start) & (pt < qs.stop)] - q_off, gi1["packed_text_indexes"])
        mine = lay["seg"] == q
        assert torch.equal(lay["rows"][b][mine] - q_off, gi1["packed_vae_token_indexes"])
        if b:
            src, dst = lay["copy"]
            sel = (dst >= qs.start) & (dst < qs.stop)
            assert torch.equal(dst[sel], torch.arange(qs.start, qs.stop))
            q0 = int(gi["packed_seqlens"][:q].to(torch.int64).sum())
            assert torch.equal(src[sel], torch.arange(q0, q0 + int(ql[k])))
    assert lay["rows"].shape[0] == len(members)
    for b, mem in enumerate(members):
        assert sorted(seen.get(b, [])) == mem
    for b in range(len(members)):                  # requests outside a block have no row in it
        for q in range(R):
            if q not in members[b]:
                assert torch.all(lay["rows"][b][lay["seg"] == q] == -1)
    # context placement: each block's member rows of its branch cache, to that sample's kv indexes
    kvl_all = {b: torch.as_tensor(br[b]["key_values_lens"]).to(torch.int64) for b in range(3)}
    for b, src, dst in lay["ctx"]:
        want_src, want_dst = [], []
        c0 = torch.cumsum(kvl_all[b], 0) - kvl_all[b]
        for k, (bb, q, row_off, _) in enumerate(lay["samples"]):
            if bb == b:
                want_src.append(torch.arange(int(c0[q]), int(c0[q] + kvl_all[b][q])))
                want_dst.append(lay["packed_key_value_indexes"][int(ck[k]):int(ck[k] + kl[k])])
        assert torch.equal(src, torch.cat(want_src)) and torch.equal(dst, torch.cat(want_dst))
    # every merged K/V row is used exactly once
    used = torch.cat([lay["packed_query_indexes"], lay["packed_key_value_indexes"]])
    assert torch.equal(used.sort().values, torch.arange(int((ql + kl).sum())))


@pytest.mark.parametrize("seed", range(4))
def test_schedule_follows_each_request(seed):
    rnd = random.Random(100 + seed)
    R = rnd.randint(1, 6)
    ivs = [rnd.choice(INTERVALS) for _ in range(R)]
    sc = [rnd.choice(SCALES) for _ in range(R)]
    nbs = _branch_counts([s[0] for s in sc], [s[1] for s in sc])
    steps, shift = rnd.choice([4, 12, 50]), rnd.choice([1.0, 3.0])
    ts, dts, cfg_on, full = _flow_batch_schedule(steps, shift, ivs, nbs)
    # make_flow_runner's schedule, per request alone
    t1 = torch.linspace(1, 0, steps)
    t1 = shift * t1 / (1 + (shift - 1) * t1)
    assert torch.equal(dts, t1[:-1] - t1[1:]) and torch.equal(ts, t1[:-1])
    for q, iv in enumerate(ivs):
        own = [bool(t > iv[0] and t <= iv[1]) for t in t1[:-1]]
        assert [row[q] for row in cfg_on] == own
    for i in range(steps - 1):
        assert full[i] == any(cfg_on[i][q] and nbs[q] > 1 for q in range(R))


def test_branch_counts_follow_cfg_branches():
    assert _branch_counts([4.0, 4.0, 1.0, 1.0, 1.5], [1.5, 1.0, 1.5, 1.0, 1.01]) == [3, 2, 1, 1, 3]


@pytest.mark.parametrize("seed", range(4))
def test_vae_round_packer_matches_per_request_packing(model, seed):
    rnd = random.Random(seed)
    R = rnd.randint(2, 6)
    has = [rnd.random() < 0.6 for _ in range(R)]
    has[rnd.randrange(R)] = True
    imgs = [torch.rand(3, 16 * rnd.randint(1, 4), 16 * rnd.randint(1, 4), generator=torch.Generator().manual_seed(q))
            if h else None for q, h in enumerate(has)]
    kv0 = [rnd.randint(0, 20) for _ in range(R)]
    rp0 = [rnd.randint(0, 5) for _ in range(R)]
    tf = lambda im: im
    gi, kv, rp = model.prepare_vae_image_round(kv0, rp0, imgs, tf, NT)
    gi2, kv2, rp2, tensors = model.prepare_vae_image_round(kv0, rp0, imgs, tf, NT, return_tensors=True)
    assert kv2 == kv and rp2 == rp and set(gi2) == set(gi)
    assert [t.data_ptr() for t in tensors] == [im.data_ptr() for im in imgs if im is not None]
    ql = gi["packed_seqlens"].to(torch.int64)
    cl = gi["key_values_lens"].to(torch.int64)
    k = 0
    voff = 0
    for q in range(R):
        b0 = int((cl + ql)[:q].sum())
        q0 = int(ql[:q].sum())
        qs = slice(q0, q0 + int(ql[q]))
        assert int(cl[q]) == kv0[q]
        assert torch.equal(gi["packed_key_value_indexes"][int(cl[:q].sum()):int(cl[:q + 1].sum())] - b0,
                           torch.arange(kv0[q]))
        if imgs[q] is None:
            assert int(ql[q]) == 0 and kv[q] == kv0[q] and rp[q] == rp0[q]
            continue
        want, kv1, rp1 = model.prepare_vae_images([kv0[q]], [rp0[q]], [imgs[q]], tf, NT)
        assert kv[q] == kv1[0] and rp[q] == rp1[0]
        assert torch.equal(gi["packed_seqlens"][q:q + 1], want["packed_seqlens"])
        assert torch.equal(gi["packed_position_ids"][qs], want["packed_position_ids"])
        assert torch.equal(gi["packed_indexes"][qs] - b0, want["packed_indexes"])
        assert gi["patchified_vae_latent_shapes"][k] == want["patchified_vae_latent_shapes"][0]
        h, w = want["patchified_vae_latent_shapes"][0]
        vs = slice(voff, voff + h * w)
        assert torch.equal(gi["packed_vae_token_indexes"][vs] - q0, want["packed_vae_token_indexes"])
        assert torch.equal(gi["packed_vae_position_ids"][vs], want["packed_vae_position_ids"])
        assert torch.equal(gi["packed_text_indexes"][2 * k:2 * k + 2] - q0, want["packed_text_indexes"])
        assert torch.equal(gi["packed_text_ids"][2 * k:2 * k + 2], want["packed_text_ids"])
        H, W = imgs[q].shape[1:]
        assert torch.equal(gi["padded_images"][k, :, :H, :W], want["padded_images"][0])
        assert torch.equal(gi["packed_timesteps"], want["packed_timesteps"])
        k += 1
        voff += h * w
    assert k == gi["padded_images"].shape[0] and voff == gi["packed_vae_token_indexes"].numel()


def test_request_seed_draws_the_single_request_init_noise(model):
    sizes = [(32, 48), (64, 16), (16, 16)]
    seeds = [21, 22, 12345]
    gi = model.prepare_vae_latent([3, 9, 0], [1, 3, 0], sizes, NT,
                                  generators=[torch.Generator().manual_seed(s) for s in seeds])
    ntok = (gi["packed_seqlens"].to(torch.int64) - 2).tolist()
    got = gi["packed_init_noises"].split(ntok)
    for q, (s, hw) in enumerate(zip(seeds, sizes)):
        torch.manual_seed(s)
        want = model.prepare_vae_latent([0], [0], [hw], NT)["packed_init_noises"]
        assert torch.equal(got[q], want)
    with pytest.raises(ValueError):
        model.prepare_vae_latent([0], [0], [(16, 16)], NT, generators=[])


def test_refusals():
    m = helpers.build_product_bagel(device="cpu", load=False)
    with pytest.raises(NotImplementedError):
        m.generate_image_batch(None, None, None, None, None, [18], None, None, None, None, None, [4.0], [1.0],
                               [(0.4, 1.0)], [0.0], ["global"], enable_taylorseer=True)
    mb = helpers.build_product_bagel(device="cpu", load=False, dtype_mode="B")
    with pytest.raises(NotImplementedError):
        mb.generate_image_batch(None, None, None, None, None, [18], None, None, None, None, None, [4.0], [1.0],
                                [(0.4, 1.0)], [0.0], ["global"])
