"""Host logic of batched understanding (no GPU): the image-round packer of Bagel.chat_batch gives every request exactly
the layout Bagel.chat's per-request packer sequence gives it, and the sampler's Philox4x32-10 restatement reproduces
the published known-answer vectors."""
import random

import numpy as np
import pytest
import torch

import helpers
from sampling_oracle import gumbel_scores, philox4x32_10, uniforms

NT = helpers.NEW_TOKEN_IDS


@pytest.fixture(scope="module")
def model():
    return helpers.build_product_bagel_with_vit(device="cpu", load=False)


def _rows_of(gi, i):
    """Request i's part of a batched packer output, with its indexes made relative to its own block / query span."""
    ql = gi["packed_seqlens"].to(torch.int64) if "packed_seqlens" in gi else gi["text_token_lens"].to(torch.int64)
    cl = gi["key_values_lens"].to(torch.int64)
    b0 = int((cl + ql)[:i].sum())
    q0 = int(ql[:i].sum())
    qs = slice(q0, q0 + int(ql[i]))
    out = {"key_values_lens": gi["key_values_lens"][i:i + 1],
           "packed_key_value_indexes": gi["packed_key_value_indexes"][int(cl[:i].sum()):int(cl[:i + 1].sum())] - b0}
    if "packed_seqlens" in gi:
        out.update(packed_seqlens=gi["packed_seqlens"][i:i + 1], packed_position_ids=gi["packed_position_ids"][qs],
                   packed_indexes=gi["packed_indexes"][qs] - b0)
        if int(ql[i]):
            k = int((ql[:i] > 0).sum())           # image number of request i within this round
            vl = gi["vit_token_seqlens"].to(torch.int64)
            v0 = int(vl[:k].sum())
            vs = slice(v0, v0 + int(vl[k]))
            out.update(vit_token_seqlens=gi["vit_token_seqlens"][k:k + 1], packed_vit_tokens=gi["packed_vit_tokens"][vs],
                       packed_vit_position_ids=gi["packed_vit_position_ids"][vs],
                       packed_vit_token_indexes=gi["packed_vit_token_indexes"][vs] - q0,
                       packed_text_indexes=gi["packed_text_indexes"][2 * k:2 * k + 2] - q0,
                       packed_text_ids=gi["packed_text_ids"][2 * k:2 * k + 2])
    else:
        out.update(text_token_lens=gi["text_token_lens"][i:i + 1], packed_text_ids=gi["packed_text_ids"][qs],
                   packed_text_position_ids=gi["packed_text_position_ids"][qs],
                   packed_text_indexes=gi["packed_text_indexes"][qs] - b0)
    return out


def _image(rnd):
    return torch.rand(3, 14 * rnd.randint(1, 5), 14 * rnd.randint(1, 5), generator=torch.Generator().manual_seed(rnd.randint(0, 999)))


@pytest.mark.parametrize("seed", range(4))
def test_round_packer_matches_per_request_chat_packing(model, seed):
    rnd = random.Random(seed)
    counts = [0, 1, 2, 3] + [rnd.randint(0, 3) for _ in range(rnd.randint(0, 3))]
    rnd.shuffle(counts)
    reqs = [([_image(rnd) for _ in range(c)], " ".join(str(rnd.randint(0, 999)) for _ in range(rnd.randint(0, 9))))
            for c in counts]
    tok, tf = helpers.IntTokenizer(), (lambda im: im)
    R = len(reqs)
    # batched: the packer sequence of chat_batch
    kv, rp, rounds = [0] * R, [0] * R, []
    for r in range(max(counts)):
        gi, kv, rp = model.prepare_vit_image_round(kv, rp, [im[r] if r < len(im) else None for im, _ in reqs], tf, NT)
        rounds.append(gi)
    gp, kv, rp = model.prepare_prompts(kv, rp, [p for _, p in reqs], tok, NT)
    gs = model.prepare_start_tokens(kv, rp, NT)
    for i, (imgs, prompt) in enumerate(reqs):
        # chat's sequence for request i alone
        kv1, rp1 = [0], [0]
        for r, im in enumerate(imgs):
            want, kv1, rp1 = model.prepare_vit_images(kv1, rp1, [im], tf, NT)
            got = _rows_of(rounds[r], i)
            assert set(got) == set(want)
            for k in want:
                assert torch.equal(got[k], want[k]) and got[k].dtype == want[k].dtype, (i, r, k)
        for r in range(len(imgs), len(rounds)):       # rounds without an image: no query rows, cache carried as is
            got = _rows_of(rounds[r], i)
            assert int(got["packed_seqlens"]) == 0 and got["packed_indexes"].numel() == 0
            assert int(got["key_values_lens"]) == kv1[0]
            assert torch.equal(got["packed_key_value_indexes"], torch.arange(kv1[0]))
        want, kv1, rp1 = model.prepare_prompts(kv1, rp1, [prompt], tok, NT)
        got = _rows_of(gp, i)
        for k in want:
            assert torch.equal(got[k], want[k]) and got[k].dtype == want[k].dtype, (i, "prompt", k)
        assert kv[i] == kv1[0] and rp[i] == rp1[0]
        want = model.prepare_start_tokens(kv1, rp1, NT)
        assert int(gs["key_values_lens"][i]) == int(want["key_values_lens"][0])
        assert int(gs["packed_query_position_ids"][i]) == int(want["packed_query_position_ids"][0])


# Random123 kat_vectors, philox4x32_10: (counter, key, expected output)
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
     (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert tuple(int(x) for x in got) == want
    batch = philox4x32_10(np.array([ctr, ctr], dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert all(tuple(int(x) for x in row) == want for row in batch)


def test_uniforms_and_scores_are_in_range():
    u = uniforms((7 << 32) | 12345, 3, 4099)
    assert u.min() > 0.0 and u.max() < 1.0
    assert np.all(u * 2 ** 23 - 0.5 == np.floor(u * 2 ** 23))       # (23-bit integer + 0.5) * 2^-23
    # the same value in fp32, as the kernel computes it: exact, and below 1 even for the largest word
    top = np.array([0xFFFFFFFF >> 9, 0xFFFFFF01 >> 9], dtype=np.uint32)
    u32 = (top.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    assert np.all(u32.astype(np.float64) == (top.astype(np.float64) + 0.5) * 2.0 ** -23) and np.all(u32 < 1.0)
    s = gumbel_scores(np.zeros(4099), 1.0, (7 << 32) | 12345, 3)
    assert np.isfinite(s).all() and np.argmax(s) == np.argmax(-np.log(-np.log(u)))
