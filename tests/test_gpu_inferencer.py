"""-m gpu: InterleaveInferencer end to end (SURVEY.md §8 a1) against outputs of the UNMODIFIED reference inferencer
(reference inferencer.py:23-313) run on CPU by tests/golden/make_golden.py::golden_inferencer on the same tiny
LM + SigLIP tower + VAE, the same tokenizer, transforms, prompts, input image and RNG seeds:
  text -> image, image + text -> image (edit), image + text -> text (understanding), think -> text -> image.
What this pins is the ORCHESTRATION: which contexts are built, in which order, where they are deep-copied for the two
CFG branches, what is fed back, and the image pre/post-processing; the kernels underneath have their own parity tests.
Images are compared in 8-bit levels (bf16 pipelines on different hardware cannot be bit-identical)."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

import helpers
from oracle import fixtures

pytestmark = pytest.mark.gpu
TEXT = "5 17 900 33 2"
KW = dict(num_timesteps=4, timestep_shift=3.0, cfg_text_scale=4.0, cfg_img_scale=1.5, cfg_interval=[0.4, 1.0],
          cfg_renorm_min=0.0, cfg_renorm_type="global")


@pytest.fixture(scope="module")
def gold():
    return load_file(os.path.join(os.path.dirname(__file__), "golden", "inferencer_tiny.safetensors"))


@pytest.fixture(scope="module")
def inferencer():
    from bagel_b200.inferencer import InterleaveInferencer
    from bagel_b200.transforms import ImageTransform
    model = helpers.build_product_bagel_with_vit(fixtures.TINY_LM, "cuda", max_latent_size=16, vae_downsample=2)
    vae = helpers.tiny_vae("cuda")
    vae.sample = False                      # DiagonalGaussian(sample=False), as in the fixture run
    return InterleaveInferencer(model, vae, fixtures.ToyTokenizer(), ImageTransform(64, 32, 4), ImageTransform(112, 56, 14),
                                helpers.NEW_TOKEN_IDS)


def _text(t):
    return bytes(t.tolist()).decode("utf-8")


def _check_image(name, img, ref):
    got = np.asarray(img).astype(np.int32)
    ref = ref.numpy().astype(np.int32)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    d = np.abs(got - ref)
    print(f"{name}: |d| mean {d.mean():.2f} levels, p99 {np.percentile(d, 99):.0f}, max {d.max()}")
    # random-init VAE decoder output is noise-like (std ~67 levels): a wrong context / branch / seed gives |d| ~ 75
    # bound for bf16 GPU-vs-CPU differences after resampling
    assert d.mean() <= 2.5 and np.percentile(d, 99) <= 12, f"{name}: mean {d.mean():.2f}, p99 {np.percentile(d, 99)}"


def _tokens(s):
    return [int(w) for w in s.split()]


def test_input_image_fixture_is_reproducible(gold):
    assert np.array_equal(np.asarray(fixtures.inferencer_image()), gold["input.image"].numpy())


def test_text_to_image(inferencer, gold):
    torch.manual_seed(21)
    r = inferencer(text=TEXT, image_shapes=(32, 48), **KW)
    assert r["text"] is None and r["image"].size == (48, 32)
    _check_image("t2i", r["image"], gold["t2i.image"])


def test_image_edit(inferencer, gold):
    """VAE + ViT image context, text; CFG-text context = image only, CFG-image context = text only (inferencer.py:241-252)."""
    torch.manual_seed(22)
    r = inferencer(image=fixtures.inferencer_image(), text=TEXT, **KW)
    assert r["image"].size == (56, 40)      # output takes the (resized) input image's shape
    _check_image("edit", r["image"], gold["edit.image"])


def test_image_understanding_text(inferencer, gold):
    torch.manual_seed(23)
    r = inferencer(image=fixtures.inferencer_image(), text=TEXT, understanding_output=True, max_think_token_n=6, do_sample=False)
    assert r["image"] is None
    got, ref = _tokens(r["text"]), _tokens(_text(gold["und.text"]))
    print("understanding tokens", got, "reference", ref)
    assert len(got) == len(ref)
    # greedy ids of a random-init tiny model sit on bf16-margin ties now and then (see test_generate_text_greedy): the
    # first tokens must agree, a later tie may fork the continuation
    assert got[:2] == ref[:2], (got, ref)
    if got != ref:
        pytest.xfail(f"greedy continuation forked on a bf16 tie: {got} vs {ref}")


def test_think_then_image(inferencer, gold):
    torch.manual_seed(24)
    r = inferencer(text=TEXT, think=True, max_think_token_n=5, do_sample=False, image_shapes=(32, 48), **KW)
    got, ref = _tokens(r["text"]), _tokens(_text(gold["think.text"]))
    print("think tokens", got, "reference", ref)
    assert got[:2] == ref[:2], (got, ref)
    if got != ref:
        pytest.xfail(f"greedy continuation forked on a bf16 tie: {got} vs {ref}")
    _check_image("think", r["image"], gold["think.image"])     # the thought is fed back as context for the image
