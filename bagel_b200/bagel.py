"""BAGEL unified model — host side of the H100-native build.

Same public surface as the reference's modeling/bagel/bagel.py (Bagel :57): the `prepare_*` packers
(:232-264, :552-641, :909-927) return dicts with the same keys / dtypes (key names are API — callers splat
them as kwargs), `forward_cache_update_text` (:267-297) prefill, the rectified-flow sampler `generate_image`
(:644-754) with `_forward_flow` (:757-907), and `generate_text` (:930-1000).

What is different underneath (GPU-first, not a port):
  * packers are vectorised index arithmetic (no per-token Python loops);
  * `generate_image` plans the whole run once (index maps, RoPE tables, all timestep embeddings, merged KV
    buffers with the read-only context already in place), batches the CFG branches into ONE packed LM call per
    step (they share weights; the reference runs them one after another), keeps x_t resident in HBM and issues
    a sync-free launch sequence per step, optionally replayed as a CUDA graph;
  * every tensor op on the per-step path is a kernel from bagel_b200.ops.
"""
from __future__ import annotations

import math
import numbers
import warnings
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import ops
from .config import BagelConfig
from .modeling_utils import MLPconnector, PositionEmbedding, TimestepEmbedder
from .qwen2_navit import ForwardPlan, NaiveCache, Qwen2ForCausalLM, _ranges

BF16 = torch.bfloat16


# --------------------------------------------------------------------------------------------------
# index helpers (host, int64)
# --------------------------------------------------------------------------------------------------
def get_flattened_position_ids_extrapolate(img_h, img_w, patch_size, max_num_patches_per_side):
    """row * max_side + col for every patch (reference data/data_utils.py:53-58)."""
    nh, nw = img_h // patch_size, img_w // patch_size
    return (torch.arange(nh)[:, None] * max_num_patches_per_side + torch.arange(nw)[None, :]).reshape(-1)


def get_flattened_position_ids_interpolate(img_h, img_w, patch_size, max_num_patches_per_side):
    """Bucketised fractional coordinates (reference data/data_utils.py:61-69)."""
    nh, nw = img_h // patch_size, img_w // patch_size
    edges = torch.arange(1 / max_num_patches_per_side, 1.0, 1 / max_num_patches_per_side)
    bh = torch.bucketize(torch.arange(0, 1 - 1e-6, 1 / nh), edges, right=True)
    bw = torch.bucketize(torch.arange(0, 1 - 1e-6, 1 / nw), edges, right=True)
    return (bh[:, None] * max_num_patches_per_side + bw[None, :]).reshape(-1)


def patchify(image: torch.Tensor, patch_size: int) -> torch.Tensor:
    """[C, H, W] -> [(H/p)*(W/p), p*p*C], each patch flattened (row-in-patch, col-in-patch, channel) — the
    order convert_conv2d_to_linear's W.permute(0,2,3,1) expects (reference data/data_utils.py:43-50)."""
    c, h, w = image.shape
    p = patch_size
    assert h % p == 0 and w % p == 0
    return image.reshape(c, h // p, p, w // p, p).permute(1, 3, 2, 4, 0).reshape(-1, p * p * c)


def _cfg_branches(main, text, img, cfg_text_scale: float, cfg_img_scale: float) -> List[Dict[str, Any]]:
    """The LM calls of one CFG velocity evaluation: the conditional branch, the text-CFG branch when
    cfg_text_scale > 1 and, only inside it, the image-CFG branch (the reference consumes the image branch only
    inside the text-CFG block, :873). Each argument is (packed_position_ids, packed_query_indexes, past_key_values,
    key_values_lens, packed_key_value_indexes)."""
    names = ("packed_position_ids", "packed_query_indexes", "past_key_values", "key_values_lens",
             "packed_key_value_indexes")
    branches = [main]
    if cfg_text_scale > 1.0:
        branches.append(text)
        if cfg_img_scale > 1.0:
            branches.append(img)
    return [dict(zip(names, b)) for b in branches]


def _branch_counts(cfg_text_scale: Sequence[float], cfg_img_scale: Sequence[float]) -> List[int]:
    """Per request, the number of LM branches _cfg_branches gives it alone (1 main, 2 + text, 3 + image)."""
    return [len(_cfg_branches((), (), (), sT, sI)) for sT, sI in zip(cfg_text_scale, cfg_img_scale)]


def _flow_batch_layout(packed_seqlens, packed_vae_token_indexes, packed_text_indexes, branches: Sequence[Dict[str, Any]],
                       members: Sequence[Sequence[int]]) -> Dict[str, Any]:
    """Host layout of one packed LM call of a batch of independent image requests (Bagel.generate_image_batch).

    branches[b] holds the packed inputs of branch b (0 main, 1 text-dropped, 2 image-dropped) over ALL requests, in
    the keys of _cfg_branches; members[b] lists the requests that take part in block b (blocks with no member are
    skipped). Block b holds, request after request, the sample [context rows, query rows] that branch b gives the
    request alone, shifted to the block's place: its position ids and kv len are the branch's, its query and kv indexes
    are the branch's minus the request's start in the branch packing plus its start in the merged one. The query rows of
    all blocks are packed in the same order (block, then request).

    Returns the ForwardPlan inputs (query_lens, position_ids, packed_query_indexes, key_values_lens,
    packed_key_value_indexes, packed_vae_token_indexes, packed_text_indexes), `ctx`: per block (branch, cache rows,
    merged rows) of the context K/V to place, `copy`: (main query rows, block query rows) of every query row outside
    block 0 (the latent-in rows of a request are the same in every branch), `rows`: [n_blocks, M] query row of each
    latent row in each block (-1: request not in the block), and `samples`: (block, request, merged start, query start)."""
    i64 = lambda t: torch.as_tensor(t).to("cpu", torch.int64).reshape(-1)
    ql = i64(packed_seqlens)
    R = int(ql.numel())
    cq = torch.cumsum(ql, 0) - ql                       # query start of each request in the main packing
    vae = i64(packed_vae_token_indexes)
    txt = i64(packed_text_indexes)
    ntok = ql - 2
    seg = torch.repeat_interleave(torch.arange(R), ntok)
    out: Dict[str, Any] = {k: [] for k in ("query_lens", "position_ids", "packed_query_indexes", "key_values_lens",
                                           "packed_key_value_indexes", "packed_vae_token_indexes",
                                           "packed_text_indexes", "ctx", "samples")}
    rows = []
    copy_src, copy_dst = [], []
    row_off = 0        # merged K/V row of the next sample
    q_off = 0          # query row of the next sample
    for b, mem in enumerate(members):
        mem = sorted(int(q) for q in mem)
        if not mem:
            rows.append(torch.full((int(ntok.sum()),), -1, dtype=torch.int64))
            continue
        br = branches[b]
        cache = br["past_key_values"]
        has_ctx = cache is not None and cache.key_cache[0] is not None
        kl = i64(br["key_values_lens"]) if has_ctx else torch.zeros(R, dtype=torch.int64)
        base = torch.cumsum(kl + ql, 0) - (kl + ql)     # request start in the branch's own packing
        ckv = torch.cumsum(kl, 0) - kl                  # its first cache row
        pos, pq = i64(br["packed_position_ids"]), i64(br["packed_query_indexes"])
        pkv = i64(br["packed_key_value_indexes"]) if has_ctx else torch.zeros(0, dtype=torch.int64)
        blk_q = torch.full((R,), -1, dtype=torch.int64)  # query start of each request within this block's rows
        src_rows, dst_rows = [], []
        for q in mem:
            qs = slice(int(cq[q]), int(cq[q] + ql[q]))
            ks = slice(int(ckv[q]), int(ckv[q] + kl[q]))
            shift = row_off - int(base[q])
            out["query_lens"].append(ql[q:q + 1])
            out["position_ids"].append(pos[qs])
            out["packed_query_indexes"].append(pq[qs] + shift)
            out["key_values_lens"].append(kl[q:q + 1])
            out["packed_key_value_indexes"].append(pkv[ks] + shift)
            src_rows.append(torch.arange(ks.start, ks.stop))
            dst_rows.append(pkv[ks] + shift)
            sel_v = (vae >= qs.start) & (vae < qs.stop)
            sel_t = (txt >= qs.start) & (txt < qs.stop)
            out["packed_vae_token_indexes"].append(vae[sel_v] - qs.start + q_off)
            out["packed_text_indexes"].append(txt[sel_t] - qs.start + q_off)
            out["samples"].append((b, q, row_off, q_off))
            blk_q[q] = q_off
            if b:
                copy_src.append(torch.arange(qs.start, qs.stop))
                copy_dst.append(torch.arange(q_off, q_off + int(ql[q])))
            row_off += int(kl[q] + ql[q])
            q_off += int(ql[q])
        if has_ctx:
            out["ctx"].append((b, torch.cat(src_rows), torch.cat(dst_rows)))
        r = torch.full((int(ntok.sum()),), -1, dtype=torch.int64)
        inb = blk_q[seg] >= 0
        r[inb] = vae[inb] - cq[seg[inb]] + blk_q[seg[inb]]
        rows.append(r)
    for k in ("query_lens", "position_ids", "packed_query_indexes", "key_values_lens", "packed_key_value_indexes",
              "packed_vae_token_indexes", "packed_text_indexes"):
        out[k] = torch.cat(out[k])
    cat0 = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64)
    out["copy"] = (cat0(copy_src), cat0(copy_dst))
    out["rows"] = torch.stack(rows)
    out["seg"] = seg
    out["n"] = q_off
    return out


def _flow_batch_schedule(num_timesteps: int, timestep_shift: float, cfg_interval: Sequence[Sequence[float]],
                         nbs: Sequence[int]):
    """The shared schedule of a batch and its per-step CFG switches: (ts, dts, cfg_on [steps][R], full [steps]).
    cfg_on[i][q] is make_flow_runner's test for request q alone; step i runs the all-branch plan when a request that has a
    text-dropped branch has CFG on."""
    ts = torch.linspace(1, 0, num_timesteps)
    ts = timestep_shift * ts / (1 + (timestep_shift - 1) * ts)
    dts = ts[:-1] - ts[1:]
    ts = ts[:-1]
    cfg_on = [[bool(t > iv[0] and t <= iv[1]) for iv in cfg_interval] for t in ts]
    full = [any(on and nb > 1 for on, nb in zip(row, nbs)) for row in cfg_on]
    return ts, dts, cfg_on, full


def _sampling_filters(B: int, do_sample, top_k, top_p, min_p,
                      who: str = "generate_text_batch") -> Optional[Tuple[List[int], List[float], List[float]]]:
    """generate_text_batch's top_k / top_p / min_p (each None, one value, or one per request), checked: per-request
    lists (0, 1.0, 0.0 where off) for ops.sample_rows_filtered, or None when no sampled request sets a filter."""
    def expand(name, x):
        if x is None or isinstance(x, numbers.Real):
            return [x] * B
        x = list(x)
        if len(x) != B:
            raise ValueError(f"{who}: {name} has {len(x)} entries for {B} requests")
        return x

    def top_k_ok(k):
        return isinstance(k, numbers.Integral) and not isinstance(k, bool) and k >= 0

    def real(v):
        return isinstance(v, numbers.Real) and not isinstance(v, bool)

    ks = [0 if k is None else k for k in expand("top_k", top_k)]
    ps = [1.0 if p is None else p for p in expand("top_p", top_p)]
    ms = [0.0 if m is None else m for m in expand("min_p", min_p)]
    if not all(top_k_ok(k) for k in ks):
        raise ValueError(f"{who}: top_k must be None or an int >= 0, got {top_k!r}")
    if not all(real(p) and 0.0 < p <= 1.0 for p in ps):
        raise ValueError(f"{who}: top_p must be None or in (0, 1], got {top_p!r}")
    if not all(real(m) and 0.0 <= m < 1.0 for m in ms):
        raise ValueError(f"{who}: min_p must be None or in [0, 1), got {min_p!r}")
    sampled = [do_sample] * B if isinstance(do_sample, numbers.Real) else list(do_sample)
    if len(sampled) != B:
        return None         # generate_text_batch reports the wrong length of do_sample
    if not any(s and (k > 0 or p < 1.0 or m > 0.0) for s, k, p, m in zip(sampled, ks, ps, ms)):
        return None
    return [int(k) for k in ks], [float(p) for p in ps], [float(m) for m in ms]


def _penalties(B: int, repetition_penalty, presence_penalty, frequency_penalty,
               who: str = "generate_text_batch") -> Optional[Tuple[List[float], List[float], List[float]]]:
    """generate_text_batch's repetition_penalty (finite, > 0; None or 1: off), presence_penalty and frequency_penalty
    (finite, in [-2, 2]; None or 0: off), each None, one value, or one per request, checked: per-request lists
    (repetition, frequency, presence) for ops.apply_penalties, or None when every request has all three off."""
    def expand(name, x):
        if x is None or isinstance(x, numbers.Real):
            return [x] * B
        x = list(x)
        if len(x) != B:
            raise ValueError(f"{who}: {name} has {len(x)} entries for {B} requests")
        return x

    def real(v):
        return isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(v)

    def positive_f32(r):         # the device divides by the fp32 value: it must be neither 0 nor inf
        with np.errstate(over="ignore"):
            return real(r) and r > 0.0 and 0.0 < np.float32(r) < np.inf

    rs = [1.0 if r is None else r for r in expand("repetition_penalty", repetition_penalty)]
    ps = [0.0 if p is None else p for p in expand("presence_penalty", presence_penalty)]
    fs = [0.0 if f is None else f for f in expand("frequency_penalty", frequency_penalty)]
    if not all(positive_f32(r) for r in rs):
        raise ValueError(f"{who}: repetition_penalty must be None or finite and > 0, got {repetition_penalty!r}")
    for name, xs, x in (("presence_penalty", ps, presence_penalty), ("frequency_penalty", fs, frequency_penalty)):
        if not all(real(v) and -2.0 <= v <= 2.0 for v in xs):
            raise ValueError(f"{who}: {name} must be None or in [-2, 2], got {x!r}")
    # the device compares the fp32 values with the off values, so a value that rounds to one is off too
    rs, fs, ps = ([float(np.float32(v)) for v in xs] for xs in (rs, fs, ps))
    if all(r == 1.0 and f == 0.0 and p == 0.0 for r, f, p in zip(rs, fs, ps)):
        return None
    return rs, fs, ps


def _num_samples(R: int, num_samples, who: str = "generate_text_batch") -> Optional[List[int]]:
    """num_samples (None, one int >= 1, or one per request), checked: one count per request, or None."""
    if num_samples is None:
        return None
    ns = [num_samples] * R if isinstance(num_samples, numbers.Number) else list(num_samples)
    if len(ns) != R:
        raise ValueError(f"{who}: num_samples has {len(ns)} entries for {R} requests")
    if not all(isinstance(n, numbers.Integral) and not isinstance(n, bool) and n >= 1 for n in ns):
        raise ValueError(f"{who}: num_samples must be an int >= 1 or one per request, got {num_samples!r}")
    return [int(n) for n in ns]


def _sample_keys(seeds: Sequence[int], ns: Sequence[int]) -> List[int]:
    """Philox key of sample j of request i among R: (seeds[i] & 0xFFFFFFFF) | ((i + R * j) << 32), request-major. With
    every n_i = 1 this is request i's key (seed, i); no two samples share a key."""
    R = len(ns)
    return [(int(sd) & 0xFFFFFFFF) | ((i + R * j) << 32) for i, (sd, n) in enumerate(zip(seeds, ns)) for j in range(n)]


def _per_sample(x, ns: List[int]):
    """A per-request setting as generate_text_batch takes it (None, one value, or one per request) for the decode rows
    of num_samples ns: one value stays, a per-request list repeats each entry n_i times."""
    if x is None or isinstance(x, numbers.Number):
        return x
    x = list(x)
    if len(x) != len(ns):
        return x            # the row-level check reports the wrong length
    return [v for v, n in zip(x, ns) for _ in range(n)]


def _capture_graph(launch: Callable[[], None], what: str) -> Optional[torch.cuda.CUDAGraph]:
    """Capture launch() as a CUDA graph and replay it once (capture does not execute the work). Capture is an
    optimisation and the eager launch sequence is the same work: on failure, warn, synchronise and return None."""
    try:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launch()
        graph.replay()
        return graph
    except Exception as e:
        warnings.warn(f"bagel_b200: CUDA graph capture of {what} failed, continuing eagerly: {e}")
        torch.cuda.synchronize()
        return None


class _Affine:
    """weight/bias holder for vae2llm / llm2vae."""

    def __init__(self):
        self.weight = self.bias = None

    def load(self, sd, prefix, device):
        self.weight = sd[prefix + "weight"].to(device, BF16).contiguous()
        self.bias = sd[prefix + "bias"].to(device, BF16).contiguous()

    def __call__(self, x):
        return ops.gemm(x.to(BF16).contiguous(), self.weight, bias=self.bias)


class Bagel:
    def __init__(self, language_model: Qwen2ForCausalLM, vit_model, config: BagelConfig):
        self.language_model = language_model
        self.config = config
        self.device = language_model.device
        # "A": bf16 weights + autocast (app.py:111); "B": fp32 master weights + autocast (eval drivers) — see qwen2_navit.py
        self.dtype_mode = language_model.model.dtype_mode
        # opt-in block-scaled FP8 MLP of the generation expert (inference only; bagel_b200/fp8.py)
        self.fp8_gen_mlp = language_model.model.fp8_gen_mlp
        sdt = language_model.model.stream_dtype
        llm = config.llm_config
        self.hidden_size = llm.hidden_size
        self.use_moe = "Mo" in llm.layer_module
        self.num_heads = llm.num_attention_heads
        if config.visual_gen:
            self.latent_patch_size = config.latent_patch_size
            self.timestep_shift = config.timestep_shift
            self.latent_downsample = config.vae_config.downsample * config.latent_patch_size
            self.max_latent_size = config.max_latent_size
            self.latent_channel = config.vae_config.z_channels
            self.patch_latent_dim = self.latent_patch_size ** 2 * self.latent_channel
            self.time_embedder = TimestepEmbedder(self.hidden_size)
            self.vae2llm = _Affine()
            self.llm2vae = _Affine()
            self.latent_pos_embed = PositionEmbedding(self.max_latent_size, self.hidden_size, self.device, sdt)
        if config.visual_und:
            self.vit_model = vit_model
            self.vit_patch_size = config.vit_config.patch_size
            self.vit_max_num_patch_per_side = config.vit_max_num_patch_per_side
            self.vit_hidden_size = config.vit_config.hidden_size
            self.connector = MLPconnector(self.vit_hidden_size, self.hidden_size, config.connector_act)
            self.vit_pos_embed = PositionEmbedding(self.vit_max_num_patch_per_side, self.hidden_size, self.device, sdt)
        self.get_flattened_position_ids = (get_flattened_position_ids_interpolate if config.interpolate_pos
                                           else get_flattened_position_ids_extrapolate)
        self.use_cuda_graph = True
        self._graph_cache: Dict[Any, Any] = {}

    def eval(self):
        return self

    # ------------------------------------------------------------------------------------------
    # weights (reference key schema, SURVEY.md §8b)
    # ------------------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = False):
        """Reference key schema. strict=True: every expected tensor must be present and nothing may be left over
        (KeyError lists both); strict=False: unexpected keys are ignored, but the heads this configuration needs
        (vae2llm / llm2vae / time_embedder for visual_gen, connector for visual_und) must still be there — a model with
        `None` weights would only fail later inside a kernel call."""
        lm_sd = {k[len("language_model."):]: v for k, v in sd.items() if k.startswith("language_model.")}
        unexpected = ["language_model." + k for k in self.language_model.load_state_dict(lm_sd, strict=False)]
        used = set()
        missing: List[str] = []

        def need(keys):
            miss = [k for k in keys if k not in sd]
            missing.extend(miss)
            used.update(keys)
            return not miss

        if self.config.visual_gen:
            if need(["time_embedder.mlp.0.weight", "time_embedder.mlp.0.bias", "time_embedder.mlp.2.weight",
                     "time_embedder.mlp.2.bias"]):
                self.time_embedder.load(sd, "time_embedder.", self.device)
            if need(["vae2llm.weight", "vae2llm.bias"]):
                self.vae2llm.load(sd, "vae2llm.", self.device)
            if need(["llm2vae.weight", "llm2vae.bias"]):
                self.llm2vae.load(sd, "llm2vae.", self.device)
            self.latent_pos_embed.load(sd.get("latent_pos_embed.pos_embed"))   # frozen sincos table: optional
            used.add("latent_pos_embed.pos_embed")
        if self.config.visual_und:
            if need(["connector.fc1.weight", "connector.fc1.bias", "connector.fc2.weight", "connector.fc2.bias"]):
                self.connector.load(sd, "connector.", self.device)
            self.vit_pos_embed.load(sd.get("vit_pos_embed.pos_embed"))
            used.add("vit_pos_embed.pos_embed")
            vit_sd = {k[len("vit_model."):]: v for k, v in sd.items() if k.startswith("vit_model.")}
            used.update("vit_model." + k for k in vit_sd)
            if self.vit_model is not None and hasattr(self.vit_model, "load_state_dict"):
                if vit_sd:
                    self.vit_model.load_state_dict(vit_sd)
                else:
                    missing.append("vit_model.*")
        unexpected += [k for k in sd if not k.startswith("language_model.") and k not in used]
        if missing:
            raise KeyError(f"bagel_b200.Bagel.load_state_dict: missing weights {missing[:12]}"
                           + (f" (+{len(missing) - 12} more)" if len(missing) > 12 else ""))
        if strict and unexpected:
            raise KeyError(f"bagel_b200.Bagel.load_state_dict: unexpected keys {unexpected[:12]}")
        return self

    # ------------------------------------------------------------------------------------------
    # packers
    # ------------------------------------------------------------------------------------------
    def prepare_prompts(self, curr_kvlens, curr_rope, prompts, tokenizer, new_token_ids):
        return self.prepare_prompts_round(curr_kvlens, curr_rope, list(prompts), tokenizer, new_token_ids)

    def prepare_prompts_round(self, curr_kvlens, curr_rope, prompts, tokenizer, new_token_ids):
        """One text round of a batch of independent requests, with prepare_vit_image_round's contract: prompts[i] is
        request i's text or None. A request with a text gets the layout prepare_prompts gives that text alone
        ([bos] + tokens + [eos]); a request without one contributes zero query tokens, its cached rows are carried
        unchanged and its kv len and rope position stay."""
        bos, eos = new_token_ids["bos_token_id"], new_token_ids["eos_token_id"]
        ids = [[] if p is None else [bos] + list(tokenizer.encode(p)) + [eos] for p in prompts]
        tl = torch.tensor([len(x) for x in ids], dtype=torch.int64)
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        rope = torch.tensor(list(curr_rope), dtype=torch.int64)
        sample_start = torch.cumsum(cl + tl, 0) - (cl + tl)
        generation_input = {
            "text_token_lens": tl.to(torch.int),
            "packed_text_ids": torch.tensor([t for x in ids for t in x], dtype=torch.long),
            "packed_text_position_ids": _ranges(rope, tl),
            "packed_text_indexes": _ranges(sample_start + cl, tl),
            "packed_key_value_indexes": _ranges(sample_start, cl),
            "key_values_lens": cl.to(torch.int),
        }
        return generation_input, (cl + tl).tolist(), (rope + tl).tolist()

    def prepare_vae_latent(self, curr_kvlens, curr_rope, image_sizes, new_token_ids,
                           generators: Optional[Sequence[torch.Generator]] = None):
        """generators: optional CPU generator per sample for its init noise (independent requests each with their own
        seed); by default every sample draws from the global CPU generator, in sample order, like the reference."""
        ds = self.latent_downsample
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        rope = torch.tensor(list(curr_rope), dtype=torch.int64)
        ntok = torch.tensor([(H // ds) * (W // ds) for H, W in image_sizes], dtype=torch.int64)
        ql = ntok + 2
        q_start = torch.cumsum(ql, 0) - ql
        b_start = torch.cumsum(cl + ql, 0) - (cl + ql)
        B = len(image_sizes)
        dim = self.latent_channel * self.latent_patch_size ** 2
        # init noise: drawn per sample, in sample order, from the global CPU generator exactly like the reference
        gens = [None] * B if generators is None else list(generators)
        if len(gens) != B:
            raise ValueError(f"prepare_vae_latent: {len(gens)} generators for {B} samples")
        noises = [torch.randn(int(n), dim, generator=g) for n, g in zip(ntok, gens)]
        pos = [self.get_flattened_position_ids(H, W, ds, max_num_patches_per_side=self.max_latent_size)
               for H, W in image_sizes]
        generation_input = {
            "packed_text_ids": torch.tensor([new_token_ids["start_of_image"], new_token_ids["end_of_image"]] * B,
                                            dtype=torch.long),
            "packed_text_indexes": torch.stack([q_start, q_start + ntok + 1], dim=1).reshape(-1),
            "packed_init_noises": torch.cat(noises, dim=0),
            "packed_vae_position_ids": torch.cat(pos, dim=0),
            "packed_vae_token_indexes": _ranges(q_start + 1, ntok),
            "packed_seqlens": ql.to(torch.int),
            "packed_position_ids": torch.repeat_interleave(rope, ql),
            "key_values_lens": cl.to(torch.int),
            "packed_indexes": _ranges(b_start + cl, ql),
            "packed_key_value_indexes": _ranges(b_start, cl),
        }
        return generation_input

    def prepare_vae_latent_cfg(self, curr_kvlens, curr_rope, image_sizes):
        ds = self.latent_downsample
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        rope = torch.tensor(list(curr_rope), dtype=torch.int64)
        ql = torch.tensor([(H // ds) * (W // ds) + 2 for H, W in image_sizes], dtype=torch.int64)
        b_start = torch.cumsum(cl + ql, 0) - (cl + ql)
        return {
            "cfg_packed_position_ids": torch.repeat_interleave(rope, ql),
            "cfg_key_values_lens": cl.to(torch.int),
            "cfg_packed_query_indexes": _ranges(b_start + cl, ql),
            "cfg_packed_key_value_indexes": _ranges(b_start, cl),
        }

    def prepare_start_tokens(self, curr_kvlens, curr_rope, new_token_ids):
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        # NB: like the reference (:909-927) these indexes do NOT leave a slot for the query token; generate_text
        # shifts sample i by i at the first step (:955-958).
        b_start = torch.cumsum(cl, 0) - cl
        B = len(curr_kvlens)
        return {
            "packed_start_tokens": torch.tensor([new_token_ids["bos_token_id"]] * B, dtype=torch.long),
            "packed_query_position_ids": torch.tensor(list(curr_rope), dtype=torch.long),
            "key_values_lens": cl.to(torch.int),
            "packed_key_value_indexes": _ranges(b_start, cl),
        }

    # ------------------------------------------------------------------------------------------
    # prefill
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_cache_update_text(self, past_key_values: NaiveCache, packed_text_ids, packed_text_position_ids,
                                  text_token_lens, packed_text_indexes, packed_key_value_indexes, key_values_lens):
        emb = self.language_model.model.embed_tokens(packed_text_ids)
        out = self.language_model.forward_inference(
            packed_query_sequence=emb, query_lens=text_token_lens,
            packed_query_position_ids=packed_text_position_ids, packed_query_indexes=packed_text_indexes,
            past_key_values=past_key_values, packed_key_value_indexes=packed_key_value_indexes,
            key_values_lens=key_values_lens, update_past_key_values=True, is_causal=True, mode="und")
        return out.past_key_values

    # ------------------------------------------------------------------------------------------
    # image understanding context: SigLIP tokens (reference bagel.py:299-415)
    # ------------------------------------------------------------------------------------------
    def prepare_vit_images(self, curr_kvlens, curr_rope, images, transforms, new_token_ids):
        return self.prepare_vit_image_round(curr_kvlens, curr_rope, list(images), transforms, new_token_ids)

    def prepare_vit_image_round(self, curr_kvlens, curr_rope, images, transforms, new_token_ids):
        """One image round of a batch of independent requests: images[i] is request i's next image, or None when it
        has no image in this round (prepare_vit_images is the round in which every request has one). A request with an
        image gets the same position ids, kv lens and row layout (relative to its block) as prepare_vit_images on that
        image alone. A request without one contributes zero query tokens: its block holds only its cached rows, carried
        unchanged, and its kv len and rope position stay."""
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        rope = torch.tensor(list(curr_rope), dtype=torch.int64)
        has = torch.tensor([im is not None for im in images], dtype=torch.bool)
        tokens, pos = [], []
        for image in (im for im in images if im is not None):
            if hasattr(transforms, "patches") and hasattr(image, "size") and not torch.is_tensor(image):
                # device-side image path (transforms.DeviceImageTransform): resize + normalise + patchify on the GPU,
                # bit-identical to the host path below
                w_, h_ = transforms.resize_transform.target_size(*image.size)
                tokens.append(transforms.patches(image, self.vit_patch_size))
            else:
                t = transforms(image)
                h_, w_ = t.size(1), t.size(2)
                tokens.append(patchify(t, self.vit_patch_size))
            pos.append(self.get_flattened_position_ids(h_, w_, self.vit_patch_size,
                                                       max_num_patches_per_side=self.vit_max_num_patch_per_side))
        ntok = torch.zeros(len(images), dtype=torch.int64)
        ntok[has] = torch.tensor([x.shape[0] for x in tokens], dtype=torch.int64)
        ql = torch.where(has, ntok + 2, torch.zeros_like(ntok))
        q_start = torch.cumsum(ql, 0) - ql
        b_start = torch.cumsum(cl + ql, 0) - (cl + ql)
        generation_input = {
            "packed_text_ids": torch.tensor([new_token_ids["start_of_image"], new_token_ids["end_of_image"]] * len(tokens),
                                            dtype=torch.long),
            "packed_text_indexes": torch.stack([q_start[has], q_start[has] + ntok[has] + 1], dim=1).reshape(-1),
            "vit_token_seqlens": ntok[has].to(torch.int),
            "packed_vit_tokens": torch.cat(tokens, dim=0),
            "packed_vit_position_ids": torch.cat(pos, dim=0),
            "packed_vit_token_indexes": _ranges(q_start[has] + 1, ntok[has]),
            "packed_position_ids": torch.repeat_interleave(rope, ql),
            "packed_seqlens": ql.to(torch.int),
            "packed_indexes": _ranges(b_start + cl, ql),
            "packed_key_value_indexes": _ranges(b_start, cl),
            "key_values_lens": cl.to(torch.int),
        }
        # an image block shares ONE rope position; the counter then advances by 1 (reference :340-343)
        return generation_input, (cl + ql).tolist(), (rope + has.to(torch.int64)).tolist()

    def _vit_features(self, packed_vit_tokens, packed_vit_position_ids, vit_token_seqlens) -> torch.Tensor:
        """SigLIP tower (per-image varlen) + connector: [sum tokens, LM hidden] bf16."""
        vl = torch.as_tensor(vit_token_seqlens).to("cpu", torch.int64)
        cu = torch.cat([torch.zeros(1, dtype=torch.int64), vl.cumsum(0)]).to(torch.int32)
        feats = self.vit_model(packed_pixel_values=packed_vit_tokens,
                               packed_flattened_position_ids=packed_vit_position_ids, cu_seqlens=cu,
                               max_seqlen=int(vl.max()))
        return self.connector(feats)

    def _prefill_vit_features(self, past_key_values: NaiveCache, feats, packed_text_ids, packed_text_indexes,
                              packed_vit_token_indexes, packed_vit_position_ids, packed_position_ids, packed_seqlens,
                              packed_indexes, packed_key_value_indexes, key_values_lens) -> NaiveCache:
        """LM prefill of image blocks whose SigLIP + connector features are `feats` (reference :390-410)."""
        dev = self.device
        lm = self.language_model.model
        n = int(torch.as_tensor(packed_seqlens).sum())
        seq = torch.zeros((n, self.hidden_size), dtype=BF16, device=dev)
        emb = lm.embed_tokens(torch.as_tensor(packed_text_ids))
        ops.copy_rows(emb, seq, dst_rows=torch.as_tensor(packed_text_indexes).to(dev, torch.int32))
        # + vit_pos_embed[pos], scattered to the image rows of the packed sequence (reference :390-395)
        ops.latent_embed_add(feats, None, self.vit_pos_embed.pos_embed,
                             torch.as_tensor(packed_vit_position_ids).to(dev, torch.int64).contiguous(), seq,
                             torch.as_tensor(packed_vit_token_indexes).to(dev, torch.int32))
        out = self.language_model.forward_inference(
            packed_query_sequence=seq, query_lens=packed_seqlens, packed_query_position_ids=packed_position_ids,
            packed_query_indexes=packed_indexes, past_key_values=past_key_values,
            packed_key_value_indexes=packed_key_value_indexes, key_values_lens=key_values_lens,
            update_past_key_values=True, is_causal=False, mode="und")
        return out.past_key_values

    @torch.no_grad()
    def forward_cache_update_vit(self, past_key_values: NaiveCache, packed_text_ids, packed_text_indexes,
                                 packed_vit_tokens, packed_vit_token_indexes, packed_vit_position_ids,
                                 vit_token_seqlens, packed_position_ids, packed_seqlens, packed_indexes,
                                 packed_key_value_indexes, key_values_lens):
        if self.dtype_mode == "B":
            raise NotImplementedError("dtype_mode='B' covers the LM, the text / VAE prefills and the sampler; the SigLIP tower "
                                      "runs its bf16-stream path only (mode A)")
        feats = self._vit_features(packed_vit_tokens, packed_vit_position_ids, vit_token_seqlens)
        return self._prefill_vit_features(past_key_values, feats, packed_text_ids, packed_text_indexes,
                                          packed_vit_token_indexes, packed_vit_position_ids, packed_position_ids,
                                          packed_seqlens, packed_indexes, packed_key_value_indexes, key_values_lens)

    # ------------------------------------------------------------------------------------------
    # image editing context: clean VAE latents at t=0 (reference bagel.py:417-550)
    # ------------------------------------------------------------------------------------------
    def prepare_vae_images(self, curr_kvlens, curr_rope, images, transforms, new_token_ids, timestep=0):
        return self.prepare_vae_image_round(curr_kvlens, curr_rope, list(images), transforms, new_token_ids, timestep)

    def prepare_vae_image_round(self, curr_kvlens, curr_rope, images, transforms, new_token_ids, timestep=0,
                                return_tensors: bool = False):
        """One VAE image round of a batch of independent requests, with prepare_vit_image_round's contract: images[i] is
        request i's image or None. A request with an image gets the layout prepare_vae_images gives that image alone; a
        request without one contributes zero query tokens, keeps its kv len and its rope position. padded_images and
        patchified_vae_latent_shapes list the present images only, in request order. return_tensors=True also returns
        the transformed images themselves ([C, H, W] each, present images only), for a caller that encodes them one by
        one."""
        ds = self.latent_downsample
        cl = torch.tensor(list(curr_kvlens), dtype=torch.int64)
        rope = torch.tensor(list(curr_rope), dtype=torch.int64)
        has = torch.tensor([im is not None for im in images], dtype=torch.bool)
        tensors = [transforms(im) for im in images if im is not None]
        shapes = [(t.shape[1] // ds, t.shape[2] // ds) for t in tensors]
        ntok = torch.zeros(len(images), dtype=torch.int64)
        ntok[has] = torch.tensor([h * w for h, w in shapes], dtype=torch.int64)
        ql = torch.where(has, ntok + 2, torch.zeros_like(ntok))
        q_start = torch.cumsum(ql, 0) - ql
        b_start = torch.cumsum(cl + ql, 0) - (cl + ql)
        B = len(tensors)
        C = tensors[0].shape[0]
        Hm, Wm = max(t.shape[1] for t in tensors), max(t.shape[2] for t in tensors)
        padded = torch.zeros((B, C, Hm, Wm), device=tensors[0].device)   # stays on the GPU with DeviceImageTransform
        for i, t in enumerate(tensors):
            padded[i, :, : t.shape[1], : t.shape[2]] = t
        generation_input = {
            "padded_images": padded,
            "patchified_vae_latent_shapes": shapes,
            "packed_vae_position_ids": torch.cat([self.get_flattened_position_ids(
                t.size(1), t.size(2), ds, max_num_patches_per_side=self.max_latent_size) for t in tensors], dim=0),
            "packed_timesteps": torch.tensor([timestep]),
            "packed_vae_token_indexes": _ranges(q_start[has] + 1, ntok[has]),
            "packed_text_ids": torch.tensor([new_token_ids["start_of_image"], new_token_ids["end_of_image"]] * B,
                                            dtype=torch.long),
            "packed_text_indexes": torch.stack([q_start[has], q_start[has] + ntok[has] + 1], dim=1).reshape(-1),
            "packed_position_ids": torch.repeat_interleave(rope, ql),
            "packed_seqlens": ql.to(torch.int),
            "packed_indexes": _ranges(b_start + cl, ql),
            "packed_key_value_indexes": _ranges(b_start, cl),
            "key_values_lens": cl.to(torch.int),
        }
        out = generation_input, (cl + ql).tolist(), (rope + has.to(torch.int64)).tolist()
        return (*out, tensors) if return_tensors else out

    @torch.no_grad()
    def forward_cache_update_vae(self, vae_model, past_key_values: NaiveCache, padded_images,
                                 patchified_vae_latent_shapes, packed_vae_position_ids, packed_timesteps,
                                 packed_vae_token_indexes, packed_text_ids, packed_text_indexes, packed_position_ids,
                                 packed_seqlens, packed_indexes, key_values_lens, packed_key_value_indexes):
        latents = vae_model.encode(padded_images)                      # [B, z, Hm/8, Wm/8]
        return self._prefill_vae_latents(past_key_values, self._patchify_latents(latents, patchified_vae_latent_shapes),
                                         packed_vae_position_ids, packed_timesteps, packed_vae_token_indexes,
                                         packed_text_ids, packed_text_indexes, packed_position_ids, packed_seqlens,
                                         packed_indexes, key_values_lens, packed_key_value_indexes)

    def _patchify_latents(self, latents, patchified_vae_latent_shapes) -> torch.Tensor:
        """VAE latents [z, >= h*p, >= w*p] each -> packed 2x2-patch rows [sum h*w, p*p*z] bf16, (p, q, c) order
        (reference :517-518)."""
        p, zc = self.latent_patch_size, self.latent_channel
        rows = []
        for lat, (h, w) in zip(latents, patchified_vae_latent_shapes):
            lat = lat[:, : h * p, : w * p].reshape(zc, h, p, w, p)
            rows.append(lat.permute(1, 3, 2, 4, 0).reshape(h * w, p * p * zc))
        return torch.cat(rows, dim=0).to(self.device, BF16).contiguous()

    def _prefill_vae_latents(self, past_key_values: NaiveCache, packed_latent, packed_vae_position_ids,
                             packed_timesteps, packed_vae_token_indexes, packed_text_ids, packed_text_indexes,
                             packed_position_ids, packed_seqlens, packed_indexes, key_values_lens,
                             packed_key_value_indexes) -> NaiveCache:
        """LM prefill of clean-latent image blocks whose patchified VAE latents are `packed_latent` (reference :500-550)."""
        dev = self.device
        lm = self.language_model.model
        modeB = self.dtype_mode == "B"
        n = int(torch.as_tensor(packed_seqlens).sum())
        seq = torch.zeros((n, self.hidden_size), dtype=lm.stream_dtype, device=dev)
        emb = lm.embed_tokens(torch.as_tensor(packed_text_ids))
        (ops.copy_rows_f32 if modeB else ops.copy_rows)(emb, seq, dst_rows=torch.as_tensor(packed_text_indexes).to(dev, torch.int32))
        proj = ops.gemm(packed_latent, self.vae2llm.weight, bias=self.vae2llm.bias)
        t_emb = self.time_embedder(torch.as_tensor(packed_timesteps).to(dev, torch.float32).reshape(-1)[:1])
        (ops.latent_embed_add_f32 if modeB else ops.latent_embed_add)(
            proj, t_emb[0], self.latent_pos_embed.pos_embed,
            torch.as_tensor(packed_vae_position_ids).to(dev, torch.int64).contiguous(), seq,
            torch.as_tensor(packed_vae_token_indexes).to(dev, torch.int32))
        extra = {}
        if self.use_moe:
            extra = dict(mode="gen", packed_vae_token_indexes=packed_vae_token_indexes,
                         packed_text_indexes=packed_text_indexes)
        out = self.language_model.forward_inference(
            packed_query_sequence=seq, query_lens=packed_seqlens, packed_query_position_ids=packed_position_ids,
            packed_query_indexes=packed_indexes, past_key_values=past_key_values, key_values_lens=key_values_lens,
            packed_key_value_indexes=packed_key_value_indexes, update_past_key_values=True, is_causal=False, **extra)
        return out.past_key_values

    # ------------------------------------------------------------------------------------------
    # rectified-flow sampler
    # ------------------------------------------------------------------------------------------
    def _build_flow_plan(self, branches: List[Dict[str, Any]], packed_seqlens, packed_vae_token_indexes,
                         packed_text_indexes):
        """One ForwardPlan covering all CFG branches as extra samples of the packed batch, plus merged KV
        buffers with every branch's (read-only) context rows placed once."""
        lm = self.language_model.model
        n = int(torch.as_tensor(packed_seqlens).sum())
        ql, pos, qidx, kvl, kvidx, vae, txt = [], [], [], [], [], [], []
        row_off = 0
        ctx_pairs = []
        for b, br in enumerate(branches):
            kl = torch.as_tensor(br["key_values_lens"]).to("cpu", torch.int64)
            has_ctx = br["past_key_values"] is not None and br["past_key_values"].key_cache[0] is not None
            if not has_ctx:
                kl = torch.zeros_like(kl)
            total_b = n + int(kl.sum())
            ql.append(torch.as_tensor(packed_seqlens).to("cpu", torch.int64))
            pos.append(torch.as_tensor(br["packed_position_ids"]).to("cpu", torch.int64))
            qidx.append(torch.as_tensor(br["packed_query_indexes"]).to("cpu", torch.int64) + row_off)
            kvl.append(kl)
            ki = torch.as_tensor(br["packed_key_value_indexes"]).to("cpu", torch.int64) if has_ctx else torch.zeros(0, dtype=torch.int64)
            kvidx.append(ki + row_off)
            if has_ctx:
                ctx_pairs.append((br["past_key_values"], (ki + row_off).to(self.device, torch.int32)))
            vae.append(torch.as_tensor(packed_vae_token_indexes).to("cpu", torch.int64) + b * n)
            txt.append(torch.as_tensor(packed_text_indexes).to("cpu", torch.int64) + b * n)
            row_off += total_b
        plan = ForwardPlan(lm, query_lens=torch.cat(ql), position_ids=torch.cat(pos),
                           packed_query_indexes=torch.cat(qidx), key_values_lens=torch.cat(kvl),
                           packed_key_value_indexes=torch.cat(kvidx), is_causal=False,
                           mode="gen" if self.use_moe else "und",
                           packed_vae_token_indexes=torch.cat(vae), packed_text_indexes=torch.cat(txt))
        kbuf, vbuf = lm.alloc_kv(plan)
        for cache, rows in ctx_pairs:
            lm.place_context(cache, rows, kbuf, vbuf)
        return plan, kbuf, vbuf

    def _velocity(self, st: Dict[str, Any], key: str, t_row: torch.Tensor, x_src: torch.Tensor, head: bool = True) -> int:
        """Latent-in (bagel.py:796-806) -> packed LM call over all CFG branches -> llm2vae (:832). Fills
        st['v_all'][b*n:(b+1)*n] with branch b's outputs for every packed row; returns the branch count.
        head=False stops after the last decoder layer (TaylorSeer caches / replaces that tensor)."""
        lm = self.language_model.model
        plan, kbuf, vbuf, nb = st[key]
        n = st["n"]
        modeB = self.dtype_mode == "B"
        embed_add = ops.latent_embed_add_f32 if modeB else ops.latent_embed_add
        copy_rows = ops.copy_rows_f32 if modeB else ops.copy_rows
        seq = lm._buf("xa", plan.n, self.hidden_size, lm.stream_dtype)
        ops.cast_f32_to_bf16(x_src, out=st["x_bf16"])
        ops.gemm(st["x_bf16"], self.vae2llm.weight, bias=self.vae2llm.bias, out=st["proj"])
        for b in range(nb):
            embed_add(st["proj"], t_row, self.latent_pos_embed.pos_embed, st["vae_pos"], seq[b * n:(b + 1) * n], st["vae_rows"])
            copy_rows(st["text_emb"], seq[b * n:(b + 1) * n], dst_rows=st["text_rows"])
        lm.run_layers(seq, plan, kbuf, vbuf, final_norm=False)
        if head:
            self._velocity_head(st, key)
        return nb

    def _velocity_head(self, st: Dict[str, Any], key: str):
        """Final norm + llm2vae (bagel.py:832) over the hidden state in the LM's "xa" workspace."""
        lm = self.language_model.model
        plan, _, _, nb = st[key]
        out = lm.final_norm(plan, for_linear=True)
        ops.gemm(out, self.llm2vae.weight, bias=self.llm2vae.bias, out=st["v_all"][: nb * st["n"]])

    def _cfg_update(self, st: Dict[str, Any], nb: int, scales: Tuple[float, float], renorm_min: float,
                    renorm_type: str, x_dst: torch.Tensor, dt: float, dt_dev: Optional[torch.Tensor] = None):
        """CFG combine + renorm (bagel.py:873-905) fused with the Euler update x -= v*dt (:746)."""
        n, v = st["n"], st["v_all"]
        sT, sI = scales
        v_text = v[n:2 * n] if (nb >= 2 and sT > 1.0) else None
        v_img = v[2 * n:3 * n] if (nb >= 3 and sI > 1.0 and v_text is not None) else None
        ops.cfg_euler_step(v[:n], v_text, v_img, st["vae_rows"], x_dst, st["norms"],
                           sT if v_text is not None else 1.0, sI if v_img is not None else 1.0, renorm_min,
                           renorm_type, dt, dt_dev)

    def _flow_state(self, x_t, packed_seqlens, packed_vae_token_indexes, packed_text_indexes,
                    packed_vae_position_ids, packed_text_ids, nb: int) -> Dict[str, Any]:
        dev = self.device
        lm = self.language_model.model
        n = int(torch.as_tensor(packed_seqlens).sum())
        vae_idx = torch.as_tensor(packed_vae_token_indexes).to("cpu", torch.int64)
        txt_idx = torch.as_tensor(packed_text_indexes).to("cpu", torch.int64)
        M = int(vae_idx.numel())
        st: Dict[str, Any] = {"n": n, "M": M, "vae_idx": vae_idx, "txt_idx": txt_idx}
        st["x"] = x_t.to(dev, torch.float32, non_blocking=True).contiguous().clone()
        st["x_bf16"] = torch.empty((M, self.patch_latent_dim), dtype=BF16, device=dev)
        st["proj"] = torch.empty((M, self.hidden_size), dtype=BF16, device=dev)
        st["v_all"] = torch.empty((nb * n, self.patch_latent_dim), dtype=BF16, device=dev)
        st["norms"] = torch.zeros(2, dtype=torch.float32, device=dev)
        st["vae_rows"] = vae_idx.to(dev, torch.int32)
        st["text_rows"] = txt_idx.to(dev, torch.int32)
        st["vae_pos"] = torch.as_tensor(packed_vae_position_ids).to(dev, torch.int64).contiguous()
        st["text_emb"] = lm.embed_tokens(torch.as_tensor(packed_text_ids))
        return st

    @torch.no_grad()
    def make_flow_runner(self, packed_text_ids, packed_text_indexes, packed_init_noises, packed_vae_position_ids,
                         packed_vae_token_indexes, packed_seqlens, packed_position_ids, packed_indexes,
                         past_key_values: NaiveCache, key_values_lens, packed_key_value_indexes,
                         num_timesteps: int = 24, timestep_shift: float = 1.0, cfg_renorm_min: float = 0.0,
                         cfg_renorm_type: str = "global", cfg_interval: Optional[Sequence[float]] = (0, 1),
                         cfg_text_scale: float = 1.0, cfg_text_packed_query_indexes=None,
                         cfg_text_packed_position_ids=None, cfg_text_past_key_values: Optional[NaiveCache] = None,
                         cfg_text_key_values_lens=None, cfg_text_packed_key_value_indexes=None,
                         cfg_img_scale: float = 1.0, cfg_img_packed_query_indexes=None,
                         cfg_img_packed_position_ids=None, cfg_img_past_key_values: Optional[NaiveCache] = None,
                         cfg_img_key_values_lens=None, cfg_img_packed_key_value_indexes=None,
                         cfg_type: str = "parallel", enable_taylorseer: bool = False) -> "FlowRunner":
        """Plan a whole denoising run (same arguments as generate_image); FlowRunner.step(i) then executes
        velocity evaluation + CFG + Euler update number i as a sync-free kernel sequence."""
        if cfg_renorm_type not in ops.RENORM:
            raise NotImplementedError(f"{cfg_renorm_type} is not supported")
        if enable_taylorseer and self.dtype_mode == "B":
            raise NotImplementedError("enable_taylorseer=True is implemented for dtype_mode='A' only (bf16 factor planes)")
        dev = self.device

        # ---- schedule (host; identical arithmetic to the reference :693-696) ----
        ts = torch.linspace(1, 0, num_timesteps)
        ts = timestep_shift * ts / (1 + (timestep_shift - 1) * ts)
        dts = ts[:-1] - ts[1:]
        ts = ts[:-1]
        cfg_on = [bool(t > cfg_interval[0] and t <= cfg_interval[1]) for t in ts]

        branches = _cfg_branches(
            (packed_position_ids, packed_indexes, past_key_values, key_values_lens, packed_key_value_indexes),
            (cfg_text_packed_position_ids, cfg_text_packed_query_indexes, cfg_text_past_key_values,
             cfg_text_key_values_lens, cfg_text_packed_key_value_indexes),
            (cfg_img_packed_position_ids, cfg_img_packed_query_indexes, cfg_img_past_key_values,
             cfg_img_key_values_lens, cfg_img_packed_key_value_indexes), cfg_text_scale, cfg_img_scale)
        nbmax = len(branches)
        # every LM workspace at its final size BEFORE the first launch / graph capture: the 'full' (all-branch) steps
        # need nbmax*n rows, the 'main' steps n — growing a buffer in between would free memory a captured graph replays into
        n_rows = int(torch.as_tensor(packed_seqlens).sum())
        self.language_model.model.reserve(nbmax * n_rows, nbmax * int(torch.as_tensor(packed_text_indexes).numel()))
        st = self._flow_state(packed_init_noises, packed_seqlens, packed_vae_token_indexes, packed_text_indexes,
                              packed_vae_position_ids, packed_text_ids, nbmax)
        st["t_emb"] = self.time_embedder(ts.to(dev))  # every timestep of the run at once: [num_timesteps-1, H]
        if any(cfg_on) and nbmax > 1:
            st["full"] = (*self._build_flow_plan(branches, packed_seqlens, st["vae_idx"], st["txt_idx"]), nbmax)
        if (not all(cfg_on)) or nbmax == 1:
            st["main"] = (*self._build_flow_plan(branches[:1], packed_seqlens, st["vae_idx"], st["txt_idx"]), 1)
        return FlowRunner(self, st, dts.tolist(), cfg_on, (cfg_text_scale, cfg_img_scale), cfg_renorm_min,
                          cfg_renorm_type, nbmax, torch.as_tensor(packed_seqlens).to("cpu", torch.int64),
                          enable_taylorseer=enable_taylorseer)

    @torch.no_grad()
    def generate_image(self, *args, **kwargs):
        """Rectified-flow Euler sampler (reference bagel.py:644-754), same signature as the reference; returns the
        tuple of per-sample latents [h*w, 64] fp32 (on the model's device)."""
        runner = self.make_flow_runner(*args, **kwargs)
        for i in range(runner.num_steps):
            runner.step(i)
        return runner.latents()

    # ------------------------------------------------------------------------------------------
    # batched image generation of independent requests
    # ------------------------------------------------------------------------------------------
    def _build_flow_batch_plan(self, lay: Dict[str, Any], branches: Sequence[Dict[str, Any]]):
        """ForwardPlan + merged K/V buffers of a _flow_batch_layout, each block's context rows placed from its branch
        cache (only the member requests' rows), and the device copy map of the latent-in rows outside block 0."""
        lm = self.language_model.model
        dev = self.device
        plan = ForwardPlan(lm, query_lens=lay["query_lens"], position_ids=lay["position_ids"],
                           packed_query_indexes=lay["packed_query_indexes"], key_values_lens=lay["key_values_lens"],
                           packed_key_value_indexes=lay["packed_key_value_indexes"], is_causal=False,
                           mode="gen" if self.use_moe else "und", packed_vae_token_indexes=lay["packed_vae_token_indexes"],
                           packed_text_indexes=lay["packed_text_indexes"])
        kbuf, vbuf = lm.alloc_kv(plan)
        for b, src, dst in lay["ctx"]:
            if src.numel():
                lm.place_context(branches[b]["past_key_values"], dst.to(dev, torch.int32), kbuf, vbuf,
                                 src_rows=src.to(dev, torch.int32))
        src, dst = lay["copy"]
        copies = (src.to(dev, torch.int32), dst.to(dev, torch.int32)) if src.numel() else None
        return plan, kbuf, vbuf, copies

    def _velocity_batch(self, st: Dict[str, Any], key: str, t_row: torch.Tensor, x_src: torch.Tensor):
        """_velocity + _velocity_head for a batch plan: the latent-in rows are computed once for the main block and
        copied to the requests' rows in the other blocks (the same values _velocity computes for each branch)."""
        lm = self.language_model.model
        plan, kbuf, vbuf, copies = st[key]
        n = st["n"]
        seq = lm._buf("xa", plan.n, self.hidden_size, lm.stream_dtype)
        ops.cast_f32_to_bf16(x_src, out=st["x_bf16"])
        ops.gemm(st["x_bf16"], self.vae2llm.weight, bias=self.vae2llm.bias, out=st["proj"])
        ops.latent_embed_add(st["proj"], t_row, self.latent_pos_embed.pos_embed, st["vae_pos"], seq[:n], st["vae_rows"])
        ops.copy_rows(st["text_emb"], seq[:n], dst_rows=st["text_rows"])
        if copies is not None:
            ops.copy_rows(seq, seq, src_rows=copies[0], dst_rows=copies[1])
        lm.run_layers(seq, plan, kbuf, vbuf, final_norm=False)
        out = lm.final_norm(plan, for_linear=True)
        ops.gemm(out, self.llm2vae.weight, bias=self.llm2vae.bias, out=st["v_all"][: plan.n])

    @torch.no_grad()
    def generate_image_batch(self, packed_text_ids, packed_text_indexes, packed_init_noises, packed_vae_position_ids,
                             packed_vae_token_indexes, packed_seqlens, packed_position_ids, packed_indexes,
                             past_key_values: NaiveCache, key_values_lens, packed_key_value_indexes,
                             cfg_text_scale: Sequence[float], cfg_img_scale: Sequence[float],
                             cfg_interval: Sequence[Sequence[float]], cfg_renorm_min: Sequence[float],
                             cfg_renorm_type: Sequence[str], num_timesteps: int = 24, timestep_shift: float = 1.0,
                             cfg_text_packed_query_indexes=None, cfg_text_packed_position_ids=None,
                             cfg_text_past_key_values: Optional[NaiveCache] = None, cfg_text_key_values_lens=None,
                             cfg_text_packed_key_value_indexes=None, cfg_img_packed_query_indexes=None,
                             cfg_img_packed_position_ids=None, cfg_img_past_key_values: Optional[NaiveCache] = None,
                             cfg_img_key_values_lens=None, cfg_img_packed_key_value_indexes=None,
                             enable_taylorseer: bool = False) -> List[torch.Tensor]:
        """generate_image for R independent requests in one packed denoising run. The packed inputs are those of
        generate_image over all R samples; cfg_text_scale, cfg_img_scale, cfg_interval, cfg_renorm_min and
        cfg_renorm_type are per-request lists, num_timesteps and timestep_shift are shared. Returns one [h*w, 64] fp32
        latent per request.

        Each request gets the branches _cfg_branches gives it alone: the LM call of a step holds a main block with every
        request, a text-dropped block with the requests that have cfg_text_scale > 1 and an image-dropped block with
        those that also have cfg_img_scale > 1, each sample attending to its own request's context for that branch. A
        step runs that all-branch plan when any request with a text-dropped branch has CFG on at its timestep, else the
        main block alone; bagel_cfg_euler_step_batch then applies each request's own CFG, renorm (a "global" norm covers
        the request's own rows) and Euler update, with the per-step CFG switch of every request read from a device
        table, so where FlowRunner captures the step, one graph per plan serves every step."""
        if enable_taylorseer:
            raise NotImplementedError("generate_image_batch: TaylorSeer is not implemented for batched requests; use "
                                      "generate_image(..., enable_taylorseer=True) per request")
        if self.dtype_mode == "B":
            raise NotImplementedError("generate_image_batch: the batched sampler is implemented for dtype_mode='A'")
        dev = self.device
        ql = torch.as_tensor(packed_seqlens).to("cpu", torch.int64)
        R = int(ql.numel())
        per_req = dict(cfg_text_scale=cfg_text_scale, cfg_img_scale=cfg_img_scale, cfg_interval=cfg_interval,
                       cfg_renorm_min=cfg_renorm_min, cfg_renorm_type=cfg_renorm_type)
        for k, val in per_req.items():
            if len(val) != R:
                raise ValueError(f"generate_image_batch: {k} has {len(val)} entries for {R} requests")
        for rt in cfg_renorm_type:
            if rt not in ops.RENORM:
                raise NotImplementedError(f"{rt} is not supported")
        nbs = _branch_counts(cfg_text_scale, cfg_img_scale)
        ts, dts, cfg_on, full = _flow_batch_schedule(num_timesteps, timestep_shift, cfg_interval, nbs)
        branches = _cfg_branches(
            (packed_position_ids, packed_indexes, past_key_values, key_values_lens, packed_key_value_indexes),
            (cfg_text_packed_position_ids, cfg_text_packed_query_indexes, cfg_text_past_key_values,
             cfg_text_key_values_lens, cfg_text_packed_key_value_indexes),
            (cfg_img_packed_position_ids, cfg_img_packed_query_indexes, cfg_img_past_key_values,
             cfg_img_key_values_lens, cfg_img_packed_key_value_indexes), 2.0, 2.0)
        members = [list(range(R)), [q for q in range(R) if nbs[q] >= 2], [q for q in range(R) if nbs[q] >= 3]]
        lays = {}
        if any(full):
            lays["full"] = _flow_batch_layout(ql, packed_vae_token_indexes, packed_text_indexes, branches, members)
        if not all(full):
            lays["main"] = _flow_batch_layout(ql, packed_vae_token_indexes, packed_text_indexes, branches, members[:1])
        big = lays.get("full", lays.get("main"))
        # every LM workspace at its final size before the first launch / graph capture (DESIGN §2)
        self.language_model.model.reserve(big["n"], int(big["packed_text_indexes"].numel()))
        st = self._flow_state(packed_init_noises, ql, packed_vae_token_indexes, packed_text_indexes,
                              packed_vae_position_ids, packed_text_ids, 1)
        st["v_all"] = torch.empty((big["n"], self.patch_latent_dim), dtype=BF16, device=dev)
        st["t_emb"] = self.time_embedder(ts.to(dev))
        for key, lay in lays.items():
            st[key] = self._build_flow_batch_plan(lay, branches)
        rows = big["rows"]
        i32 = lambda t: torch.as_tensor(t).to(dev, torch.int32).contiguous()
        none = torch.full_like(rows[0], -1)
        st["seg"] = i32(big["seg"])
        st["row_main"] = i32(rows[0])
        st["row_text"] = i32(rows[1] if rows.shape[0] > 1 else none)
        st["row_img"] = i32(rows[2] if rows.shape[0] > 2 else none)
        st["sT"] = torch.tensor([float(x) for x in cfg_text_scale], dtype=torch.float32, device=dev)
        st["sI"] = torch.tensor([float(x) for x in cfg_img_scale], dtype=torch.float32, device=dev)
        st["renorm_min"] = torch.tensor([float(x) for x in cfg_renorm_min], dtype=torch.float32, device=dev)
        st["renorm_type"] = i32([ops.RENORM[x] for x in cfg_renorm_type])
        st["cfg_ws"] = ops.cfg_batch_workspace(st["M"], R, dev)
        cfg_tab = i32([[int(x) for x in row] for row in cfg_on]).reshape(len(cfg_on), R)
        runner = BatchFlowRunner(self, st, dts.tolist(), full, cfg_tab, ql, big["n"])
        for i in range(runner.num_steps):
            runner.step(i)
        return list(runner.latents())

    # ------------------------------------------------------------------------------------------
    # text decode
    # ------------------------------------------------------------------------------------------
    def _decode_state(self, past_key_values: Optional[NaiveCache], key_values_lens, packed_start_tokens,
                      packed_query_position_ids, max_length: int,
                      num_samples: Optional[Sequence[int]] = None) -> Dict[str, Any]:
        """Device state of a decode of `max_length` steps and its step body (embedding gather -> `run_layers` on a
        decode `ForwardPlan` -> final norm -> lm_head into `logits`). Every buffer the body touches is fixed, so the
        body is graph-replayable. num_samples (one int >= 1 per request): request i continues as that many decode rows,
        request-major, over one copy of its context (ForwardPlan.decode_shared); the per-row state starts from the
        request's start token, position and context length."""
        dev = self.device
        lm = self.language_model.model
        cfg = lm.config
        L, w = cfg.num_hidden_layers, cfg.num_key_value_heads * cfg.head_dim
        kv = torch.as_tensor(key_values_lens).to("cpu", torch.int64)
        if num_samples is None:
            plan = ForwardPlan.decode(lm, kv, max_length)
        else:
            plan = ForwardPlan.decode_shared(lm, kv, num_samples, max_length)
            rows = torch.repeat_interleave(torch.arange(kv.numel()), torch.as_tensor(list(num_samples)))
            kv = kv[rows]
            packed_start_tokens = torch.as_tensor(packed_start_tokens).cpu()[rows]
            packed_query_position_ids = torch.as_tensor(packed_query_position_ids).cpu()[rows]
        B = int(kv.numel())
        # zero-filled, not torch.empty: attention multiplies the masked probabilities (exactly 0) with whatever sits in the
        # spare rows of a slab — 0 x NaN/Inf garbage would poison the output (the attention kernel fetches whole 128-key
        # blocks by TMA; only the single-query d=128 kernel clamps its loads to the rows in use)
        kbuf = torch.zeros((L, plan.total_kv, w), dtype=BF16, device=dev)
        vbuf = torch.zeros((L, plan.total_kv, w), dtype=BF16, device=dev)
        if past_key_values is not None and past_key_values.key_cache[0] is not None and plan.n_ctx:
            lm.place_context(past_key_values, plan.ctx_rows, kbuf, vbuf, src_rows=plan.ctx_src)
        st: Dict[str, Any] = {"B": B}
        st["seq_len"] = seq_len = kv.to(dev, torch.int32)
        st["pos"] = pos = torch.as_tensor(packed_query_position_ids).to(dev, torch.int64).clone()
        st["tokens"] = torch.as_tensor(packed_start_tokens).to(dev, torch.int64).clone()
        st["tokens32"] = tokens32 = st["tokens"].to(torch.int32)
        st["history"] = torch.zeros((max_length, B), dtype=torch.int64, device=dev)
        st["step_dev"] = torch.zeros(1, dtype=torch.int32, device=dev)
        x = lm._buf("xa", B, cfg.hidden_size)      # run_layers' input workspace: the gather needs no extra copy
        st["logits"] = logits = torch.empty((B, cfg.vocab_size), dtype=BF16, device=dev)
        head = self.language_model.lm_head

        def body():
            """One decode step; every input/output is a fixed device buffer (graph-replayable)."""
            ops.copy_rows(lm.embed_tokens.weight, x, src_rows=tokens32, M=B)
            ops.rope_table_into(pos, lm.inv_freq, plan.cos, plan.sin, True)
            ops.decode_prepare(plan.cu_k, seq_len, plan.q_rows, plan.seqused_k)
            out = lm.run_layers(x, plan, kbuf, vbuf)     # decoder layers + final norm
            ops.gemm(out, head.weight, bias=head.bias, out=logits)

        st["body"] = body
        return st

    @torch.no_grad()
    def generate_text(self, past_key_values: NaiveCache, packed_key_value_indexes, key_values_lens,
                      packed_start_tokens, packed_query_position_ids, max_length: int, do_sample: bool = False,
                      temperature: float = 1.0, end_token_id: Optional[int] = None):
        """Greedy / sampled decode, one token per sample per step (reference bagel.py:930-1000). Returns [steps, B]
        token ids on the model's device. As in the reference, generation stops when SAMPLE 0 emits `end_token_id`
        (:996) and the stopping token is not returned.

        GPU-first execution (the reference re-allocates and re-scatters the whole KV cache per layer per token and
        rebuilds index tensors with host loops): the KV cache is copied ONCE into per-sample slabs with room for
        `max_length` new tokens; sequence lengths, RoPE positions, write slots and the token history live on the
        device. A step is embedding gather -> `run_layers` on a decode `ForwardPlan` (the QKV projection appends K/V
        in place, attention reads `seqused_k`) -> final norm -> lm_head -> argmax, captured once as a CUDA graph and
        replayed per token. The only host<->device traffic per step is the 8-byte EOS check the reference also
        performs."""
        if self.dtype_mode == "B":
            raise NotImplementedError("generate_text: the device-resident decode loop is implemented for dtype_mode='A'")
        dev = self.device
        B = int(torch.as_tensor(key_values_lens).numel())
        if max_length <= 0:
            return torch.zeros((0, B), dtype=torch.int64, device=dev)
        d = self._decode_state(past_key_values, key_values_lens, packed_start_tokens, packed_query_position_ids,
                               max_length)
        seq_len, pos, tokens, tokens32, history, step_dev = (d[k] for k in ("seq_len", "pos", "tokens", "tokens32",
                                                                            "history", "step_dev"))
        logits, body = d["logits"], d["body"]

        def greedy_step():
            body()
            ops.decode_advance(seq_len, pos, tokens, history, step_dev)   # history[step] = current tokens; lens += 1
            ops.argmax_rows(logits, tokens, tokens32)

        graph = None
        steps = 0
        for step in range(max_length):
            if graph is not None:
                graph.replay()
            elif do_sample:
                body()
                ops.decode_advance(seq_len, pos, tokens, history, step_dev)
                probs = torch.softmax(logits.float() / temperature, dim=-1)
                nxt = torch.multinomial(probs, num_samples=1).squeeze(1)
                tokens.copy_(nxt)
                tokens32.copy_(nxt.to(torch.int32))
            elif step == 1 and self.use_cuda_graph:
                # step 0 ran eagerly and sized every LM workspace the step uses, so the capture allocates none
                graph = _capture_graph(greedy_step, "the decode step")
                if graph is None:
                    greedy_step()
            else:
                greedy_step()
            steps += 1
            if end_token_id is not None and int(tokens[0]) == end_token_id:
                break
        return history[:steps].clone()

    # unfinished-request count: read every STOP_POLL steps, one read behind, so the host never waits on the step it
    # just queued; at most 2 * STOP_POLL - 1 steps run after the last request has finished
    STOP_POLL = 4
    HISTORY_PAD = -1      # history entry of a finished request (no token id is negative)

    @torch.no_grad()
    def generate_text_batch(self, past_key_values: NaiveCache, packed_key_value_indexes, key_values_lens,
                            packed_start_tokens, packed_query_position_ids, max_length: Union[int, Sequence[int]],
                            do_sample: Union[bool, Sequence[bool]] = False,
                            temperature: Union[float, Sequence[float]] = 1.0, end_token_id: Optional[int] = None,
                            seeds: Optional[Sequence[int]] = None,
                            keys: Optional[Sequence[int]] = None, top_k=None, top_p=None,
                            min_p=None, repetition_penalty=None, presence_penalty=None,
                            frequency_penalty=None, num_samples=None) -> Union[List[torch.Tensor], List[List[torch.Tensor]]]:
        """Decode a batch of independent requests (same inputs as generate_text). Returns one LongTensor per request on
        the model's device: its tokens from the start token up to, not including, its own `end_token_id`, at most
        `max_length` of them. A finished request's token, sequence length and position freeze while the others go on.

        Greedy picks the first maximum (argmax_rows); do_sample=True draws from softmax(logits / temperature) on the
        device (Gumbel-max over Philox4x32-10, ops.sample_rows). Request i's draws are keyed by (seed, i): `seeds=None`
        takes one 32-bit base seed from torch.default_generator (so torch.manual_seed fixes it) for every request,
        otherwise request i uses seeds[i]. `keys` (one 64-bit Philox key per request) replaces that key, for a caller
        whose draws must not depend on a request's index. Either way a step is one CUDA-graph replay (after an eager
        first step), and the host only reads the device's count of unfinished requests, lagged, to stop early.

        max_length, do_sample and temperature may each be one value per request instead of one for all. The step then
        picks every row with ops.sample_rows_mixed (greedy rows take argmax_rows' pick, sampled rows sample_rows' pick
        at their own temperature) and stops each request at its own limit with ops.decode_advance_stop_limits.

        top_k (int, None or 0: off), top_p (in (0, 1], None or 1: off) and min_p (in [0, 1), None or 0: off), each one
        value or one per request, truncate a sampled request's distribution as Hugging Face generate's warpers do, in
        that order (greedy requests ignore them): the draw keeps the logits at or above the largest of the three
        thresholds, computed on the device inside the step (ops.sample_rows_filtered; include/bagel_b200.h has the
        exact definitions, ties at the top-k and top-p boundaries are kept). When no sampled request sets one, the step
        runs exactly the launches it runs without them.

        repetition_penalty (finite, > 0; None or 1: off), presence_penalty and frequency_penalty (finite, in [-2, 2];
        None or 0: off), each one value or one per request, penalise the tokens the request has generated in this call,
        greedy and sampled requests alike, before temperature and the filters (Hugging Face's order: processors, then
        warpers). With c_t the number of times token t was emitted so far (the start token and the prompt do not count),
        each logit with c_t > 0 becomes bf16(((l < 0 ? l * rp : l / rp) - fp * c_t) - pp) in fp32, one rounding per
        operation (ops.apply_penalties; include/bagel_b200.h). The repetition penalty is Hugging Face's
        RepetitionPenaltyLogitsProcessor with prompt_ignore_length = the prompt's length, up to the final bf16 rounding;
        presence and frequency are the OpenAI / vLLM penalties. The state costs 8 bytes per request per step of
        max_length. When every request has all three off, the step runs exactly the launches it runs without them.

        num_samples (an int >= 1, or one per request) asks for n_i samples of request i: the call then returns one list
        of n_i token tensors per request. Sample j of request i is a decode row of its own with the request's settings
        and its own stop, penalty state and Philox key (seed_i & 0xFFFFFFFF) | ((i + R * j) << 32), R requests, so
        sample 0 keeps the key the request has without num_samples; `keys` then holds one key per sample, sum(n_i)
        of them, request-major. When ForwardPlan.decode_shared's rule picks the shared layout, the context is placed in
        the KV slab once per request and the decode attention reads it once per 4 samples (ops.attn_decode_shared);
        otherwise each sample gets a copy of it. With every n_i = 1 the step is exactly the step without num_samples."""
        if self.dtype_mode == "B":
            raise NotImplementedError("generate_text_batch: the device-resident decode loop is implemented for dtype_mode='A'")
        dev = self.device
        B = int(torch.as_tensor(key_values_lens).numel())
        ns = _num_samples(B, num_samples)
        if ns is not None:
            # request-level checks, then every per-request setting becomes a per-row one
            _sampling_filters(B, do_sample, top_k, top_p, min_p)
            _penalties(B, repetition_penalty, presence_penalty, frequency_penalty)
            for name, x in (("max_length", max_length), ("do_sample", do_sample), ("temperature", temperature)):
                if not isinstance(x, numbers.Number) and len(list(x)) != B:
                    raise ValueError(f"generate_text_batch: {name} has {len(list(x))} entries for {B} requests")
            if keys is None:
                if seeds is None:
                    base = int(torch.randint(0, 2 ** 32, (1,), dtype=torch.int64))
                    seeds = [base] * B
                elif len(seeds) != B:
                    raise ValueError(f"generate_text_batch: {len(seeds)} seeds for {B} requests")
                keys = _sample_keys(seeds, ns)
            elif len(keys) != sum(ns):
                raise ValueError(f"generate_text_batch: {len(keys)} keys for {sum(ns)} samples")
            max_length, do_sample, temperature, top_k, top_p, min_p, repetition_penalty, presence_penalty, \
                frequency_penalty = (_per_sample(x, ns) for x in (
                    max_length, do_sample, temperature, top_k, top_p, min_p, repetition_penalty, presence_penalty,
                    frequency_penalty))
            B = sum(ns)
        plan_samples = ns if ns is not None and max(ns) > 1 else None    # all ones: the step without num_samples
        filters = _sampling_filters(B, do_sample, top_k, top_p, min_p)
        penalties = _penalties(B, repetition_penalty, presence_penalty, frequency_penalty)
        per_request = filters is not None or penalties is not None or not all(
            isinstance(x, numbers.Real) for x in (max_length, do_sample, temperature))
        if per_request:
            max_length, do_sample, temperature = (
                [x] * B if isinstance(x, numbers.Real) else list(x) for x in (max_length, do_sample, temperature))
            for name, x in (("max_length", max_length), ("do_sample", do_sample), ("temperature", temperature)):
                if len(x) != B:
                    raise ValueError(f"generate_text_batch: {name} has {len(x)} entries for {B} requests")
            if any(s and not (0.0 < float(t) < float("inf")) for s, t in zip(do_sample, temperature)):
                raise ValueError("generate_text_batch: do_sample=True needs a finite temperature > 0")
            limits = [max(int(n), 0) for n in max_length]
            steps_max = max(limits, default=0)
        else:
            if do_sample and not (0.0 < float(temperature) < float("inf")):
                raise ValueError("generate_text_batch: do_sample=True needs a finite temperature > 0")
            steps_max = max_length
        if steps_max <= 0:
            return self._by_request([torch.zeros(0, dtype=torch.int64, device=dev) for _ in range(B)], ns)
        if keys is None:
            if seeds is None:
                base = int(torch.randint(0, 2 ** 32, (1,), dtype=torch.int64))
                seeds = [base] * B
            elif len(seeds) != B:
                raise ValueError(f"generate_text_batch: {len(seeds)} seeds for {B} requests")
            keys = _sample_keys(seeds, [1] * B)
        elif len(keys) != B:
            raise ValueError(f"generate_text_batch: {len(keys)} keys for {B} requests")
        d = self._decode_state(past_key_values, key_values_lens, packed_start_tokens, packed_query_position_ids,
                               steps_max, plan_samples)
        body, logits, history, step_dev = d["body"], d["logits"], d["history"], d["step_dev"]
        keys = torch.from_numpy(np.array([int(k) & 0xFFFFFFFFFFFFFFFF for k in keys], dtype=np.uint64).view(np.int64)).to(dev)
        nxt = torch.empty(B, dtype=torch.int64, device=dev)
        finished = torch.zeros(B, dtype=torch.int32, device=dev)
        unfinished = torch.full((1,), B, dtype=torch.int32, device=dev)

        if per_request:
            # 1.0f / T in fp32, as bagel_sample_rows_bf16 derives its inverse temperature; 0 marks a greedy row. A request
            # with no budget runs one step (the kernel's smallest) and is cut to nothing below.
            inv_t = torch.from_numpy(np.array([np.float32(1.0) / np.float32(t) if s else np.float32(0.0)
                                               for s, t in zip(do_sample, temperature)], dtype=np.float32)).to(dev)
            lim_dev = torch.tensor([max(n, 1) for n in limits], dtype=torch.int32, device=dev)
            if filters is not None:
                k_dev = torch.tensor(filters[0], dtype=torch.int32, device=dev)
                p_dev, m_dev = (torch.tensor(f, dtype=torch.float32, device=dev) for f in filters[1:])
            if penalties is not None:
                rep_dev, freq_dev, pres_dev = (torch.tensor(x, dtype=torch.float32, device=dev) for x in penalties)
                seen = ops.penalty_state(B, steps_max, dev)

            def step_fn():
                body()
                if penalties is not None:
                    ops.apply_penalties(logits, rep_dev, freq_dev, pres_dev, d["tokens"], finished, step_dev, seen)
                if filters is None:
                    ops.sample_rows_mixed(logits, inv_t, keys, step_dev, nxt)
                else:
                    ops.sample_rows_filtered(logits, inv_t, k_dev, p_dev, m_dev, keys, step_dev, nxt)
                ops.decode_advance_stop_limits(d["seq_len"], d["pos"], d["tokens"], d["tokens32"], nxt, history,
                                               step_dev, finished, unfinished, end_token_id, lim_dev, self.HISTORY_PAD)
        else:
            def step_fn():
                body()
                if do_sample:
                    ops.sample_rows(logits, temperature, keys, step_dev, nxt)
                else:
                    ops.argmax_rows(logits, nxt)
                ops.decode_advance_stop(d["seq_len"], d["pos"], d["tokens"], d["tokens32"], nxt, history, step_dev,
                                        finished, unfinished, end_token_id, self.HISTORY_PAD)

        count_host = torch.zeros(2, dtype=torch.int32, pin_memory=True)
        pending = None        # (event, slot) of the last count copy not yet read
        graph = None
        steps = 0
        for step in range(steps_max):
            if graph is not None:
                graph.replay()
            elif step == 1 and self.use_cuda_graph:
                # step 0 ran eagerly and sized every LM workspace the step uses, so the capture allocates none
                graph = _capture_graph(step_fn, "the batched decode step")
                if graph is None:
                    step_fn()
            else:
                step_fn()
            steps += 1
            if end_token_id is not None and steps % self.STOP_POLL == 0:
                slot = (steps // self.STOP_POLL) % 2
                count_host[slot:slot + 1].copy_(unfinished, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                if pending is not None:
                    pending[0].synchronize()
                    if int(count_host[pending[1]]) == 0:
                        break
                pending = (ev, slot)
        hist = history[:steps]
        lens = (hist != self.HISTORY_PAD).sum(0).tolist()
        if per_request:
            lens = [min(n, lim) for n, lim in zip(lens, limits)]
        return self._by_request([hist[:n, i].clone() for i, n in enumerate(lens)], ns)

    @staticmethod
    def _by_request(outs: List[Any], ns: Optional[List[int]]):
        """Per-row results as generate_text_batch returns them: as they are, or one list of n_i per request."""
        if ns is None:
            return outs
        first = np.cumsum([0] + ns)
        return [outs[a:b] for a, b in zip(first[:-1], first[1:])]

    @torch.no_grad()
    def chat_batch(self, tokenizer, new_token_ids, image_transform, requests: Sequence[Tuple[Sequence[Any], str]],
                   max_length: int, do_sample: bool = False, temperature: float = 1.0,
                   seeds: Optional[Sequence[int]] = None, top_k=None, top_p=None, min_p=None,
                   repetition_penalty=None, presence_penalty=None, frequency_penalty=None,
                   num_samples=None) -> Union[List[str], List[List[str]]]:
        """`chat` for a batch of independent requests, each `(images, prompt)` with any number of images (zero
        included); returns one answer per request, cut at its own <|im_end|> as `chat` does.

        The context is built as `chat` builds it for each request on its own: image r of a request attends to its
        images before r, never to later ones or to other requests. One SigLIP call covers every image of every
        request; then one LM prefill per image round r holds the r-th image of every request that has one (the others
        take part with no query tokens and their cached rows carried unchanged); then one prefill of all prompts and
        one `generate_text_batch` (top_k, top_p, min_p, repetition_penalty, presence_penalty and frequency_penalty as
        there, one value or one per request; the penalties count the answer's tokens only, not the images or the
        prompt).

        num_samples (an int >= 1, or one per request) returns n_i answers per request, as generate_text_batch's
        num_samples: each request's context is built once, whatever its n_i."""
        if self.dtype_mode == "B":
            raise NotImplementedError("chat_batch: the SigLIP prefill and the decode loop are implemented for dtype_mode='A'")
        # refuse bad settings before any prefill
        _sampling_filters(len(requests), do_sample, top_k, top_p, min_p, "chat_batch")
        _penalties(len(requests), repetition_penalty, presence_penalty, frequency_penalty, "chat_batch")
        ns = _num_samples(len(requests), num_samples, "chat_batch")
        images = [list(imgs) for imgs, _ in requests]
        R = len(requests)
        newlens, new_rope = [0] * R, [0] * R
        rounds = []
        for r in range(max((len(x) for x in images), default=0)):
            gi, newlens, new_rope = self.prepare_vit_image_round(
                newlens, new_rope, [x[r] if r < len(x) else None for x in images], image_transform, new_token_ids)
            rounds.append(gi)
        past_key_values = NaiveCache(self.config.llm_config.num_hidden_layers)
        if rounds:
            feats = self._vit_features(torch.cat([gi["packed_vit_tokens"] for gi in rounds], dim=0),
                                       torch.cat([gi["packed_vit_position_ids"] for gi in rounds], dim=0),
                                       torch.cat([gi["vit_token_seqlens"] for gi in rounds], dim=0))
            off = 0
            for gi in rounds:
                gi = dict(gi)
                n = gi.pop("packed_vit_tokens").shape[0]
                gi.pop("vit_token_seqlens")
                past_key_values = self._prefill_vit_features(past_key_values, feats[off:off + n], **gi)
                off += n
        generation_input, newlens, new_rope = self.prepare_prompts(
            curr_kvlens=newlens, curr_rope=new_rope, prompts=[p for _, p in requests], tokenizer=tokenizer,
            new_token_ids=new_token_ids)
        past_key_values = self.forward_cache_update_text(past_key_values, **generation_input)
        generation_input = self.prepare_start_tokens(newlens, new_rope, new_token_ids)
        answers = self.generate_text_batch(
            past_key_values=past_key_values, max_length=max_length, do_sample=do_sample, temperature=temperature,
            end_token_id=new_token_ids["eos_token_id"], seeds=seeds, top_k=top_k, top_p=top_p, min_p=min_p,
            repetition_penalty=repetition_penalty, presence_penalty=presence_penalty,
            frequency_penalty=frequency_penalty, num_samples=ns, **generation_input)

        def text(t):
            return tokenizer.decode(t).split("<|im_end|>")[0].split("<|im_start|>")[1]
        if ns is None:
            return [text(t) for t in answers]
        return [[text(t) for t in ts] for ts in answers]

    # ------------------------------------------------------------------------------------------
    # training-mode forward (losses only, no backward): reference Bagel.forward, bagel.py:101-229
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, sequence_length: int, packed_text_ids, packed_text_indexes, sample_lens: List[int],
                packed_position_ids, nested_attention_masks=None, split_lens: List[int] = None,
                attn_modes: List[str] = None, ce_loss_indexes=None, packed_label_ids=None, packed_vit_tokens=None,
                packed_vit_token_indexes=None, packed_vit_position_ids=None, vit_token_seqlens=None, padded_latent=None,
                patchified_vae_latent_shapes=None, packed_latent_position_ids=None, packed_vae_token_indexes=None,
                packed_timesteps=None, mse_loss_indexes=None, noise: Optional[torch.Tensor] = None):
        """The reference's training forward on a packed batch -> dict(mse=..., ce=...) (forward only: this build has no
        autograd; useful for evaluation losses / distillation targets with the inference kernels).

        Attention structure (data/data_utils.py:13-40, 72-103): every sample is a list of splits that are 'causal' (text),
        'full' (an image everyone after it may look at) or 'noise' (a noised image only it itself sees); a split attends to
        all earlier non-noise splits of its sample plus itself. That is exactly a chain of prefill calls on a growing KV
        cache — so instead of a block-sparse mask over the whole packed sequence, each split runs through the varlen
        attention kernel against [cache || itself] (causal flag for text) and is appended to the cache unless it is
        noise. Experts as in training: text + ViT tokens -> und weights, VAE tokens -> gen weights, with the training
        modules' all-bf16 q/k-norm + RoPE flow (`train_numerics`). `split_lens` / `attn_modes` (the reference's
        flex-attention inputs) are required; `nested_attention_masks` carries no extra information and is ignored.
        `noise` overrides the torch.randn_like draw of :184."""
        if split_lens is None or attn_modes is None:
            raise NotImplementedError("Bagel.forward needs split_lens and attn_modes (dense nested_attention_masks alone "
                                      "cannot be mapped onto the varlen attention kernel)")
        if self.dtype_mode != "A":
            raise NotImplementedError("Bagel.forward is implemented for dtype_mode='A'")
        if self.fp8_gen_mlp:
            raise NotImplementedError("Bagel.forward (training numerics) is not implemented with fp8_gen_mlp=True, which "
                                      "is an inference mode: load the model with fp8_gen_mlp=False")
        dev = self.device
        lm = self.language_model.model
        L = int(sequence_length)
        H = self.hidden_size
        i32 = lambda t: torch.as_tensor(t).to(dev, torch.int32).contiguous()
        seq = torch.zeros((L, H), dtype=BF16, device=dev)
        text_idx = torch.as_tensor(packed_text_indexes).to("cpu", torch.int64)
        ops.copy_rows(lm.embed_tokens(torch.as_tensor(packed_text_ids)), seq, dst_rows=i32(text_idx))
        kind = torch.zeros(L, dtype=torch.int8)          # 0 text (und), 1 ViT (und), 2 VAE (gen)
        if self.config.visual_und and packed_vit_tokens is not None:
            vl = torch.as_tensor(vit_token_seqlens).to("cpu", torch.int64)
            cu = torch.cat([torch.zeros(1, dtype=torch.int64), vl.cumsum(0)]).to(torch.int32)
            feats = self.connector(self.vit_model(packed_pixel_values=packed_vit_tokens,
                                                  packed_flattened_position_ids=packed_vit_position_ids, cu_seqlens=cu,
                                                  max_seqlen=int(vl.max())))
            ops.latent_embed_add(feats, None, self.vit_pos_embed.pos_embed,
                                 torch.as_tensor(packed_vit_position_ids).to(dev, torch.int64).contiguous(), seq,
                                 i32(packed_vit_token_indexes))
            kind[torch.as_tensor(packed_vit_token_indexes).to("cpu", torch.int64)] = 1
        mse = None
        if self.config.visual_gen and padded_latent is not None:
            p, zc = self.latent_patch_size, self.latent_channel
            rows = []
            for lat, (h, w) in zip(torch.as_tensor(padded_latent), patchified_vae_latent_shapes):
                lat = lat[:, : h * p, : w * p].reshape(zc, h, p, w, p)
                rows.append(lat.permute(1, 3, 2, 4, 0).reshape(h * w, p * p * zc))
            clean = torch.cat(rows, dim=0).to(dev, torch.float32)
            if noise is None:
                noise = torch.randn_like(clean)
            noise = noise.to(dev, torch.float32)
            t = torch.sigmoid(torch.as_tensor(packed_timesteps).to(dev, torch.float32))
            t = self.timestep_shift * t / (1 + (self.timestep_shift - 1) * t)
            x_t = ((1 - t[:, None]) * clean + t[:, None] * noise).contiguous()      # flow-matching interpolation (:185-187)
            proj = ops.gemm(ops.cast_f32_to_bf16(x_t), self.vae2llm.weight, bias=self.vae2llm.bias)
            t_emb = self.time_embedder(t)                                            # per token [M, H]
            vae_idx = torch.as_tensor(packed_vae_token_indexes).to("cpu", torch.int64)
            vae_rows = i32(vae_idx)
            vae_pos = torch.as_tensor(packed_latent_position_ids).to(dev, torch.int64).contiguous()
            off = 0
            for (h, w) in patchified_vae_latent_shapes:     # all tokens of an image share its timestep embedding row
                n = h * w
                ops.latent_embed_add(proj[off:off + n], t_emb[off], self.latent_pos_embed.pos_embed, vae_pos[off:off + n], seq,
                                     vae_rows[off:off + n])
                off += n
            kind[vae_idx] = 2
        # ---- the LM: one chained prefill per split ----
        hidden = torch.empty((L, H), dtype=BF16, device=dev)
        pos_all = torch.as_tensor(packed_position_ids).to("cpu", torch.int64)
        nl = lm.config.num_hidden_layers
        s_iter = iter(zip(split_lens, attn_modes))
        start = 0
        for slen in sample_lens:
            cache, kv_len, done = NaiveCache(nl), 0, 0
            while done < slen:
                n, amode = next(s_iter)
                if amode not in ("causal", "full", "noise"):
                    raise ValueError(f"unknown attn mode {amode!r}")
                r0 = start + done
                k = kind[r0:r0 + n]
                vae_rel = torch.nonzero(k == 2).reshape(-1)
                extra = {}
                if self.use_moe and vae_rel.numel():
                    extra = dict(mode="gen", packed_vae_token_indexes=vae_rel, packed_text_indexes=torch.nonzero(k != 2).reshape(-1))
                out = lm.forward_inference(
                    packed_query_sequence=seq[r0:r0 + n], query_lens=torch.tensor([n], dtype=torch.int32),
                    packed_query_position_ids=pos_all[r0:r0 + n], packed_query_indexes=torch.arange(kv_len, kv_len + n),
                    past_key_values=cache, key_values_lens=torch.tensor([kv_len], dtype=torch.int32),
                    packed_key_value_indexes=torch.arange(kv_len), update_past_key_values=(amode != "noise"),
                    is_causal=(amode == "causal"), train_numerics=True, **extra)
                hidden[r0:r0 + n] = out.packed_query_sequence
                if amode != "noise":
                    kv_len += n
                done += n
            if done != slen:
                raise ValueError("split_lens do not add up to sample_lens")
            start += slen
        self._last_hidden_state = hidden
        # ---- heads / losses (:214-227) ----
        if self.config.visual_gen and padded_latent is not None:
            mrows = torch.nonzero(torch.as_tensor(mse_loss_indexes).to("cpu")).reshape(-1)
            hm = torch.empty((mrows.numel(), H), dtype=BF16, device=dev)
            ops.copy_rows(hidden, hm, src_rows=i32(mrows))
            preds = ops.gemm(hm, self.llm2vae.weight, bias=self.llm2vae.bias)
            target = noise - clean                           # v_t = dx_t/dt = x_1 - x_0
            mse = (preds - target[t > 0]) ** 2
        ce = None
        if ce_loss_indexes is not None:
            crow = torch.nonzero(torch.as_tensor(ce_loss_indexes).to("cpu")).reshape(-1)
            hc = torch.empty((crow.numel(), H), dtype=BF16, device=dev)
            ops.copy_rows(hidden, hc, src_rows=i32(crow))
            logits = self.language_model.lm_head(hc)
            ce = torch.nn.functional.cross_entropy(logits.float(), torch.as_tensor(packed_label_ids).to(dev), reduction="none")
        return dict(mse=mse, ce=ce)

    __call__ = forward

    # ------------------------------------------------------------------------------------------
    # evaluation entry point: images + prompt -> text (reference bagel.py:1004-1075)
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def chat(self, tokenizer, new_token_ids, image_transform, images, prompt, max_length: int,
             do_sample: bool = False, temperature: float = 1.0):
        """Same call order as the reference: one SigLIP prefill per image (prepare_vit_images ->
        forward_cache_update_vit), then the prompt (prepare_prompts -> forward_cache_update_text), then greedy / sampled
        decode from <|im_start|> until <|im_end|>; returns the decoded answer between the two markers."""
        past_key_values = NaiveCache(self.config.llm_config.num_hidden_layers)
        newlens, new_rope = [0], [0]
        for image in images:
            generation_input, newlens, new_rope = self.prepare_vit_images(
                curr_kvlens=newlens, curr_rope=new_rope, images=[image], transforms=image_transform,
                new_token_ids=new_token_ids)
            past_key_values = self.forward_cache_update_vit(past_key_values, **generation_input)
        generation_input, newlens, new_rope = self.prepare_prompts(
            curr_kvlens=newlens, curr_rope=new_rope, prompts=[prompt], tokenizer=tokenizer, new_token_ids=new_token_ids)
        past_key_values = self.forward_cache_update_text(past_key_values, **generation_input)
        generation_input = self.prepare_start_tokens(newlens, new_rope, new_token_ids)
        unpacked_latent = self.generate_text(
            past_key_values=past_key_values, max_length=max_length, do_sample=do_sample, temperature=temperature,
            end_token_id=new_token_ids["eos_token_id"], **generation_input)
        output = tokenizer.decode(unpacked_latent[:, 0])
        return output.split("<|im_end|>")[0].split("<|im_start|>")[1]

    @torch.no_grad()
    def _forward_flow(self, x_t, timestep, packed_vae_token_indexes, packed_vae_position_ids, packed_text_ids,
                      packed_text_indexes, packed_indexes, packed_position_ids, packed_seqlens, key_values_lens,
                      past_key_values, packed_key_value_indexes, cfg_renorm_min=0.0, cfg_renorm_type="global",
                      cfg_text_scale=1.0, cfg_text_packed_position_ids=None, cfg_text_packed_query_indexes=None,
                      cfg_text_key_values_lens=None, cfg_text_past_key_values=None,
                      cfg_text_packed_key_value_indexes=None, cfg_img_scale=1.0, cfg_img_packed_position_ids=None,
                      cfg_img_packed_query_indexes=None, cfg_img_key_values_lens=None, cfg_img_past_key_values=None,
                      cfg_img_packed_key_value_indexes=None, cfg_type="parallel", model_pred_cache_dic=None,
                      model_pred_current=None, model_pred_text_cache_dic=None, model_pred_text_current=None,
                      model_pred_img_cache_dic=None, model_pred_img_current=None):
        """One velocity evaluation v_t [M, C] bf16 (reference :757-907). Implemented as a single Euler step of
        the fused path on x = 0 with dt = -1, which returns exactly the CFG-combined velocity."""
        if any(a is not None for a in (model_pred_cache_dic, model_pred_current, model_pred_text_cache_dic,
                                       model_pred_text_current, model_pred_img_cache_dic, model_pred_img_current)):
            # the reference threads its TaylorSeer caches through _forward_flow (:770-775); here the step cache belongs to
            # the planned run (FlowRunner) — a single stateless evaluation cannot honour it, so refuse instead of
            # silently computing a full step
            raise NotImplementedError("TaylorSeer caches are not accepted by _forward_flow; use "
                                      "generate_image(..., enable_taylorseer=True)")
        dev = self.device
        t = torch.as_tensor(timestep).to("cpu", torch.float32).reshape(-1)
        assert t.unique().numel() == 1
        branches = _cfg_branches(
            (packed_position_ids, packed_indexes, past_key_values, key_values_lens, packed_key_value_indexes),
            (cfg_text_packed_position_ids, cfg_text_packed_query_indexes, cfg_text_past_key_values,
             cfg_text_key_values_lens, cfg_text_packed_key_value_indexes),
            (cfg_img_packed_position_ids, cfg_img_packed_query_indexes, cfg_img_past_key_values,
             cfg_img_key_values_lens, cfg_img_packed_key_value_indexes), cfg_text_scale, cfg_img_scale)
        nb = len(branches)
        st = self._flow_state(x_t, packed_seqlens, packed_vae_token_indexes, packed_text_indexes,
                              packed_vae_position_ids, packed_text_ids, nb)
        st["t_emb"] = self.time_embedder(t[:1].to(dev))
        st["full"] = (*self._build_flow_plan(branches, packed_seqlens, st["vae_idx"], st["txt_idx"]), nb)
        self._velocity(st, "full", st["t_emb"][0], st["x"])
        v_out = torch.zeros_like(st["x"])  # x' = 0 - bf16(v * -1) = v
        self._cfg_update(st, nb, (cfg_text_scale, cfg_img_scale), cfg_renorm_min, cfg_renorm_type, v_out, -1.0)
        return v_out.to(BF16)


class FlowRunner:
    """A planned denoising run: x_t resident in HBM, one sync-free launch sequence per step. The per-step inputs
    that change (timestep embedding row, dt) live in fixed device buffers, so the launch sequence of a step is
    captured ONCE per branch set as a CUDA graph and replayed for the remaining steps."""

    def __init__(self, model: Bagel, st, dts, cfg_on, scales, renorm_min, renorm_type, nbmax, seqlens,
                 enable_taylorseer: bool = False, rows_max: Optional[int] = None):
        self.model, self.st, self.dts, self.cfg_on = model, st, dts, cfg_on
        self.scales, self.renorm_min, self.renorm_type, self.nbmax = scales, renorm_min, renorm_type, nbmax
        self.seqlens = seqlens
        self.num_steps = len(dts)
        dev = model.device
        self.dts_dev = torch.tensor(dts, dtype=torch.float32, device=dev)
        self.dt_cur = torch.zeros(1, dtype=torch.float32, device=dev)
        self.t_cur = torch.zeros_like(st["t_emb"][0])
        # CUDA graphs pay off only when a step is launch-bound. Capturing ~430 launches (twice, one graph per branch
        # set) costs ~0.7 s during which the GPU idles; at BAGEL-7B / 1024^2 / batch 8 a step is 0.8 s of GPU work
        # behind ~20 ms of asynchronous launches, so eager replay loses nothing there (measured: 39.4 s vs 40.1 s
        # per generate_image). Estimate the step from its linear-layer FLOPs at ~1 PFLOP/s.
        lcfg = model.language_model.model.config
        Hd, Id = lcfg.hidden_size, lcfg.intermediate_size
        qkv_o = (lcfg.num_attention_heads * 2 + lcfg.num_key_value_heads * 2) * lcfg.head_dim
        rows = nbmax * st["n"] if rows_max is None else rows_max      # packed rows of the largest LM call of a step
        flops_step = 2.0 * rows * lcfg.num_hidden_layers * Hd * (qkv_o + 3 * Id)
        self.use_cuda_graph = bool(getattr(model, "use_cuda_graph", True)) and flops_step / 1.0e15 < 0.05
        self._graphs: Dict[str, Any] = {}
        self._graph_gen: Dict[str, int] = {}
        self._eager_done: Dict[str, int] = {}
        # TaylorSeer (reference bagel.py:680-684): one schedule per branch; factor planes of the last decoder
        # layer's output for every packed row of every branch, [7 orders, nbmax*n, H] bf16
        self.taylor = None
        if enable_taylorseer:
            from .taylorseer import TaylorSeerSchedule
            self.taylor = [TaylorSeerSchedule(len(dts) + 1) for _ in range(nbmax)]
            self.factors = torch.empty((TaylorSeerSchedule.MAX_ORDER + 1, nbmax * st["n"], model.hidden_size),
                                       dtype=BF16, device=dev)

    def _body(self, key: str):
        if self.taylor is not None:     # layers only; the cache update / extrapolation and the head follow eagerly
            self.model._velocity(self.st, key, self.t_cur, self.st["x"], head=False)
            return
        m, st = self.model, self.st
        on = key == "full"
        nb = m._velocity(st, key, self.t_cur, st["x"])
        m._cfg_update(st, nb, self.scales if on else (1.0, 1.0), self.renorm_min, self.renorm_type, st["x"], 0.0,
                      self.dt_cur)

    @torch.no_grad()
    def step(self, i: int):
        key = "full" if (self.cfg_on[i] and self.nbmax > 1) else "main"
        self.t_cur.copy_(self.st["t_emb"][i])
        self.dt_cur.copy_(self.dts_dev[i:i + 1])
        if self.taylor is not None:
            return self._step_taylorseer(key)
        self._launch(key)

    def _step_taylorseer(self, key: str):
        """One evaluation with the step cache. Branches are extra samples of one packed LM call, so the layers run
        whenever ANY active branch needs a fully computed step (with the reference's schedules the active branches
        always agree); branches on an extrapolated step get their rows of the last-layer output replaced."""
        m, st = self.model, self.st
        lm = m.language_model.model
        nb = st[key][3]
        n, H = st["n"], m.hidden_size
        scheds = self.taylor[:nb]
        types = [s.begin_step() for s in scheds]
        if any(t == "full" for t in types):
            self._launch(key)                                # embeddings + all decoder layers -> "xa"
        xa = lm._buf("xa", nb * n, H)
        for b, s in enumerate(scheds):
            rows = slice(b * n, (b + 1) * n)
            if s.type == "full":
                n_deriv, dist = s.full_update_args()
                ops.taylor_update(xa[rows], self.factors[:, rows], n_deriv, dist)
            else:
                n_f, x = s.taylor_args()
                ops.taylor_eval(self.factors[:, rows], n_f, x, xa[rows])
            s.end_step()
        m._velocity_head(st, key)
        on = key == "full"
        m._cfg_update(st, nb, self.scales if on else (1.0, 1.0), self.renorm_min, self.renorm_type, st["x"], 0.0,
                      self.dt_cur)

    def _launch(self, key: str):
        lm = self.model.language_model.model
        g = self._graphs.get(key)
        if g is not None:
            if self._graph_gen.get(key) == lm._ws_gen:
                g.replay()
                return
            # some LM workspace was re-allocated since the capture (another, larger forward ran between two steps):
            # the graph holds pointers into freed buffers -> drop it and capture again on the current ones
            del self._graphs[key]
        if self.use_cuda_graph and self._eager_done.get(key, 0) >= 1:
            # everything is warm (workspaces allocated, kernel attributes set): capture this step
            graph = _capture_graph(lambda: self._body(key), "the denoising step")
            if graph is not None:
                self._graphs[key] = graph
                self._graph_gen[key] = lm._ws_gen
                return
            self.use_cuda_graph = False
        self._body(key)
        self._eager_done[key] = self._eager_done.get(key, 0) + 1

    def latents(self):
        return self.st["x"].split((self.seqlens - 2).tolist())


class BatchFlowRunner(FlowRunner):
    """FlowRunner of Bagel.generate_image_batch: the same launch / capture / workspace-generation logic, with the
    batch's velocity evaluation and bagel_cfg_euler_step_batch as the step body. Besides t_cur and dt_cur, the step
    copies its row of the device CFG table [steps, R] into cfg_cur, so one captured graph per plan serves every step."""

    def __init__(self, model: Bagel, st, dts, full, cfg_tab: torch.Tensor, seqlens, rows_max: int):
        super().__init__(model, st, dts, full, None, None, None, 2 if "full" in st else 1, seqlens, rows_max=rows_max)
        self.cfg_tab = cfg_tab
        self.cfg_cur = torch.zeros_like(cfg_tab[0])

    @torch.no_grad()
    def step(self, i: int):
        self.cfg_cur.copy_(self.cfg_tab[i])
        super().step(i)

    def _body(self, key: str):
        m, st = self.model, self.st
        m._velocity_batch(st, key, self.t_cur, st["x"])
        ops.cfg_euler_step_batch(st["v_all"], st["seg"], st["row_main"], st["row_text"], st["row_img"], st["x"],
                                 st["cfg_ws"], st["sT"], st["sI"], st["renorm_min"], st["renorm_type"], self.cfg_cur,
                                 self.dt_cur)
