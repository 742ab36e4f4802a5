"""Packed (NaViT) Qwen2 / Mixture-of-Transformers language model — host side.

Mirrors the inference API of the reference's modeling/bagel/qwen2_navit.py (NaiveCache :207-221,
Qwen2Model.forward_inference :1018-1092, Qwen2ForCausalLM.forward_inference :1157-1188, and the MoT layer /
attention they call :499-600, :757-831) with the same argument names and meaning, but executes every layer as a
fixed sequence of hand-written sm_90a kernels (bagel_b200.ops). There is no nn.Module / autograd here: weights
are plain device tensors in fused layouts (QKV concatenated, gate/up interleaved for the SwiGLU epilogue).

Numerics: `dtype_mode="A"` (default) follows the reference with bf16 weights under autocast (app.py:111 +
inferencer.py:233): bf16 residual stream, fp32 accumulation inside every kernel, the reference's bf16 rounding points
kept. `dtype_mode="B"` follows the reference with fp32 master weights under autocast (the eval drivers,
eval/gen/gen_images_mp.py:159-175 + :73; SURVEY.md §8a dtype table): fp32 residual stream, fp32 RMSNorm weights and
outputs, unrounded fp32 RoPE tables, fp32 q/k-norm arithmetic — every nn.Linear still runs bf16 x bf16 -> bf16 (GEMM
weights are the fp32 checkpoint values cast to bf16 once at load, which is what autocast does on every call).

MoT routing (reference: ~20 index gathers/scatters per layer, qwen2_navit.py:526-548, 593-594, 781-787,
808-819): every row runs through the gen-expert GEMM; the few text rows (2 per image while denoising) are
gathered once per GEMM, run through the und-expert weights, and scattered over their rows by the GEMM epilogue.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from . import fp8 as _fp8
from . import ops
from .config import Qwen2Config

BF16 = torch.bfloat16


def _ranges(starts: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """concat_i arange(starts[i], starts[i] + lens[i])"""
    lens = lens.to(torch.int64)
    total = int(lens.sum())
    if total == 0:
        return torch.zeros(0, dtype=torch.int64)
    excl = torch.cumsum(lens, 0) - lens
    return torch.repeat_interleave(starts.to(torch.int64) - excl, lens) + torch.arange(total, dtype=torch.int64)


class NaiveCache:
    """Per-layer packed KV tensors [sum_kv, Hk, D] (or None) — reference qwen2_navit.py:207-221.
    Deep-copyable (inferencer.py:230-253 relies on copy.deepcopy of whole contexts)."""

    def __init__(self, num_layers: int):
        self.key_cache: Dict[int, Optional[torch.Tensor]] = {k: None for k in range(num_layers)}
        self.value_cache: Dict[int, Optional[torch.Tensor]] = {k: None for k in range(num_layers)}

    @property
    def num_layers(self) -> int:
        return len(self.key_cache)

    @property
    def seq_lens(self) -> int:
        return 0 if self.key_cache[0] is None else self.key_cache[0].shape[0]


def gather_requests(cache: NaiveCache, key_values_lens, members) -> NaiveCache:
    """A new packed cache holding only the blocks of requests `members` (in that order) of `cache`, whose request q
    owns key_values_lens[q] rows in request order: one copy_rows per layer and K / V. When the members' blocks are
    already the whole cache, the new cache shares its tensors (cache tensors are replaced, never written in place)."""
    kv = torch.as_tensor(key_values_lens).to("cpu", torch.int64)
    start = torch.cumsum(kv, 0) - kv
    m = torch.as_tensor(list(members), dtype=torch.int64)
    src = _ranges(start[m], kv[m])
    out = NaiveCache(cache.num_layers)
    n = cache.seq_lens
    if src.numel() == 0:
        return out
    if src.numel() == n and torch.equal(src, torch.arange(n)):
        out.key_cache, out.value_cache = dict(cache.key_cache), dict(cache.value_cache)
        return out
    rows = src.to(cache.key_cache[0].device, torch.int32)
    for li in range(cache.num_layers):
        for srcs, dsts in ((cache.key_cache, out.key_cache), (cache.value_cache, out.value_cache)):
            t = srcs[li]
            dst = torch.empty((rows.numel(), *t.shape[1:]), dtype=t.dtype, device=t.device)
            ops.copy_rows(t.reshape(n, -1), dst.reshape(rows.numel(), -1), src_rows=rows)
            dsts[li] = dst
    return out


@dataclass
class BaseNavitOutputWithPast:
    packed_query_sequence: torch.Tensor = None
    past_key_values: Optional[NaiveCache] = None


class _Embedding:
    """model.embed_tokens: callable like nn.Embedding, gather done by bagel_copy_rows_bf16 (table bf16, or fp32 in
    dtype mode B — the rows are then copied as raw bytes)."""

    def __init__(self, weight: torch.Tensor):
        self.weight = weight

    def __call__(self, ids: torch.Tensor) -> torch.Tensor:
        ids32 = ids.to(device=self.weight.device, dtype=torch.int32)
        out = torch.empty((ids32.numel(), self.weight.shape[1]), dtype=self.weight.dtype, device=self.weight.device)
        (ops.copy_rows_f32 if self.weight.dtype == torch.float32 else ops.copy_rows)(self.weight, out, src_rows=ids32)
        return out


class _Linear:
    """lm_head etc.: callable like nn.Linear (bf16 in/out), runs bagel_gemm_bf16."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor] = None):
        self.weight, self.bias = weight, bias

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        shp = x.shape
        y = ops.gemm(x.reshape(-1, shp[-1]).to(BF16).contiguous(), self.weight, bias=self.bias)
        return y.reshape(*shp[:-1], self.weight.shape[0])


class _ExpertWeights:
    """One expert's ("" = und, "_moe_gen" = gen) weights of one decoder layer, in kernel layouts."""
    __slots__ = ("wqkv", "bqkv", "wo", "wgu", "wd", "ln_in", "ln_post", "q_norm", "k_norm", "fp8")
    # fp8: the gen expert's MLP as bagel_b200.fp8.GenMlpFp8 when the model has fp8_gen_mlp=True (wgu / wd are then None)


class _Layer:
    def __init__(self):
        self.und = _ExpertWeights()
        self.gen: Optional[_ExpertWeights] = None


# decode_shared() lays a batch out with a shared context prefix when some request has at least SHARED_MIN_SAMPLES
# samples and at least SHARED_MIN_CTX_PER_SAMPLE context tokens per sample
SHARED_MIN_SAMPLES = 5
SHARED_MIN_CTX_PER_SAMPLE = 64


class ForwardPlan:
    """Everything about one packed LM call that does not depend on the hidden states: int32 index maps on the
    device, cu_seqlens, RoPE tables, which QKV path runs. Built once per call (or once per denoising run, or once
    per decode) so the layer loop is pure kernel launches with no host<->device synchronisation (the reference
    syncs >= 2x per layer, :585-586). The constructor plans a packed prefill / denoising call; `decode()` plans
    the one-token-per-sample step of text generation."""
    shared: Optional["SharedPrefix"] = None     # set by decode_shared(): attention over a shared context prefix
    ctx_src: Optional[torch.Tensor] = None      # cache row of each ctx_rows entry (None: the cache rows in order)

    def __init__(self, lm: "Qwen2Model", query_lens, position_ids, packed_query_indexes, key_values_lens,
                 packed_key_value_indexes, is_causal: bool, mode: str, packed_vae_token_indexes=None,
                 packed_text_indexes=None, train_numerics: bool = False):
        dev = lm.device
        cfg = lm.config
        # head_dim 128: q/k-norm + RoPE + KV placement fused into the QKV GEMM epilogue
        self.fuse_qkv = cfg.head_dim == 128
        self.seqused_k = None
        ql = torch.as_tensor(query_lens).to("cpu", torch.int64).reshape(-1)
        self.batch = int(ql.numel())
        self.n = int(ql.sum())
        if key_values_lens is None:
            kl = torch.zeros_like(ql)
        else:
            kl = torch.as_tensor(key_values_lens).to("cpu", torch.int64).reshape(-1)
        self.n_ctx = int(kl.sum())
        self.total_kv = self.n + self.n_ctx
        tot = kl + ql
        self.max_q = int(ql.max()) if self.batch else 0
        self.max_k = int(tot.max()) if self.batch else 0
        z = torch.zeros(1, dtype=torch.int64)
        self.cu_q = torch.cat([z, ql.cumsum(0)]).to(dev, torch.int32)
        self.cu_k = torch.cat([z, tot.cumsum(0)]).to(dev, torch.int32)
        self.is_causal = bool(is_causal)
        self.mode = mode
        # q/k-norm + RoPE arithmetic in fp32 only in PackedAttentionMoT's gen branch (qwen2_navit.py:542-548); the dense
        # PackedAttention every other layer class uses is the bf16 flow whatever the mode (:325-336)
        self.fp32_flow = int((mode == "gen") and lm.layer_kind == "mot") + (2 if lm.dtype_mode == "B" else 0)
        if train_numerics:
            # the training-mode modules (PackedAttentionMoT.forward_train, qwen2_navit.py:406-449) have no fp32 upcast
            # around q/k-norm and RoPE: gen tokens take the same all-bf16 flow as und tokens, only the weights differ
            if lm.dtype_mode != "A":
                raise NotImplementedError("training-forward numerics are implemented for dtype_mode='A'")
            self.fp32_flow = 0
        self.q_rows = torch.as_tensor(packed_query_indexes).to(dev, torch.int32).contiguous()
        if self.n_ctx:
            self.ctx_rows = torch.as_tensor(packed_key_value_indexes).to(dev, torch.int32).contiguous()
            assert self.ctx_rows.numel() == self.n_ctx, "one packed key/value index per context row"
        else:
            self.ctx_rows = None
        self.expert = None
        self.text_rows = None
        if mode == "gen" and lm.use_moe:
            ex = torch.zeros(self.n, dtype=torch.uint8)
            vi = torch.as_tensor(packed_vae_token_indexes).to("cpu", torch.int64)
            ex[vi] = 1
            self.expert = ex.to(dev)
            ti = torch.as_tensor(packed_text_indexes).to("cpu", torch.int64)
            self.text_rows = ti.to(dev, torch.int32).contiguous() if ti.numel() else None
        pos = torch.as_tensor(position_ids).to(dev, torch.int64).contiguous()
        assert pos.numel() == self.n, "one position id per packed query token"
        # cos/sin take the dtype of the hidden stream (bf16 in mode A, fp32 in mode B): modeling_qwen2.py:150
        self.cos, self.sin = ops.rope_table(pos, lm.inv_freq, round_bf16=(lm.dtype_mode == "A"))

    @classmethod
    def decode(cls, lm: "Qwen2Model", key_values_lens, max_length: int) -> "ForwardPlan":
        """One new token per sample against per-sample K/V slabs: sample i owns rows [cu_k[i], cu_k[i+1]), its
        key_values_lens[i] context rows (ctx_rows) followed by room for `max_length` new ones. The per-step state is
        device-resident so that a step is replayable as a CUDA graph: ops.decode_prepare fills q_rows (the slab row each
        new K/V is written to) and seqused_k (keys in use), ops.rope_table_into fills cos/sin."""
        dev, D = lm.device, lm.config.head_dim
        kv = torch.as_tensor(key_values_lens).to("cpu", torch.int64).reshape(-1)
        cap = kv + max_length
        begin = torch.cumsum(cap, 0) - cap
        p = cls.__new__(cls)
        p.batch = p.n = B = int(kv.numel())
        p.n_ctx, p.total_kv = int(kv.sum()), int(cap.sum())
        p.max_q = 1
        p.max_k = int(cap.max())   # host upper bound of any sample's key count (sizes the key split of decode attention)
        p.cu_q = torch.arange(B + 1, dtype=torch.int32, device=dev)
        p.cu_k = torch.cat([begin, torch.tensor([p.total_kv])]).to(dev, torch.int32)
        p.ctx_rows = _ranges(begin, kv).to(dev, torch.int32)
        p.q_rows = torch.zeros(B, dtype=torch.int32, device=dev)
        p.seqused_k = torch.zeros(B, dtype=torch.int32, device=dev)
        p.cos = torch.empty((B, D // 2), dtype=torch.float32, device=dev)
        p.sin = torch.empty((B, D // 2), dtype=torch.float32, device=dev)
        p.is_causal, p.mode, p.fp32_flow = True, "und", 0
        p.expert = p.text_rows = None
        p.fuse_qkv = D == 128 and B > 64   # B <= 64: weight-streaming skinny GEMM + norm/RoPE kernel
        return p

    @classmethod
    def decode_shared(cls, lm: "Qwen2Model", key_values_lens, num_samples, max_length: int) -> "ForwardPlan":
        """`decode()` for num_samples[i] decode rows per request i (request-major), every row of request i continuing
        its key_values_lens[i] context rows. Request i owns one slab region: its context rows, placed once (ctx_rows),
        then one suffix of `max_length` rows per sample, so the slab has sum(ctx) + sum(n) * max_length rows and
        attention runs ops.attn_decode_shared over `shared`. cu_k[r] = suffix_begin[r] - ctx_i is the base that
        ops.decode_prepare adds seq_len[r] (= ctx_i + tokens so far) to: q_rows[r] is the row's next suffix row and
        seqused_k[r] its key count, prefix included.
        Batches where no request has n >= SHARED_MIN_SAMPLES samples and ctx >= SHARED_MIN_CTX_PER_SAMPLE * n context
        rows, and shapes the shared kernel does not take (head_dim 64, other GQA groups), get `decode()` over each
        request's context repeated per row instead, with ctx_src the cache row each placed row copies. On an H100 the
        shared kernel measured slower than attn_decode on the replicated layout at up to 4 samples (one pass: a
        quarter of the CTAs to stream the same prefix) and at 32 samples of a 797-token context, and faster at 8
        samples of 797 and 8 or 32 samples of 3721 tokens (README)."""
        cfg = lm.config
        kv = torch.as_tensor(key_values_lens).to("cpu", torch.int64).reshape(-1)
        ns = torch.as_tensor(num_samples).to("cpu", torch.int64).reshape(-1)
        assert ns.numel() == kv.numel() and bool((ns >= 1).all()), "one num_samples >= 1 per request"
        row_kv = torch.repeat_interleave(kv, ns)
        pays = bool(((ns >= SHARED_MIN_SAMPLES) & (kv >= SHARED_MIN_CTX_PER_SAMPLE * ns)).any())
        if not pays or not ops.attn_decode_shared_supported(cfg.num_attention_heads, cfg.num_key_value_heads,
                                                            cfg.head_dim):
            p = cls.decode(lm, row_kv, max_length)
            p.ctx_src = _ranges(torch.repeat_interleave(torch.cumsum(kv, 0) - kv, ns), row_kv).to(lm.device, torch.int32)
            return p
        dev = lm.device
        R, B = int(kv.numel()), int(ns.sum())
        cap = kv + ns * max_length
        begin = torch.cumsum(cap, 0) - cap
        req = torch.repeat_interleave(torch.arange(R), ns)
        first_row = torch.cumsum(ns, 0) - ns
        suffix_begin = begin[req] + kv[req] + (torch.arange(B) - first_row[req]) * max_length
        p = cls.decode(lm, row_kv, max_length)    # per-row state buffers, cos/sin, QKV path: as for B independent rows
        p.n_ctx, p.total_kv = int(kv.sum()), int(cap.sum())
        p.cu_k = torch.cat([suffix_begin - row_kv, torch.tensor([p.total_kv])]).to(dev, torch.int32)
        p.ctx_rows = _ranges(begin, kv).to(dev, torch.int32)
        z = torch.zeros(1, dtype=torch.int64)
        p.shared = SharedPrefix(cu_rows=torch.cat([z, ns.cumsum(0)]).to(dev, torch.int32),
                                prefix_begin=begin.to(dev, torch.int32), prefix_len=kv.to(dev, torch.int32),
                                suffix_begin=suffix_begin.to(dev, torch.int32), max_group_rows=int(ns.max()))
        return p


@dataclass
class SharedPrefix:
    """Index arrays (int32, on the device) of ops.attn_decode_shared for a ForwardPlan.decode_shared plan."""
    cu_rows: torch.Tensor
    prefix_begin: torch.Tensor
    prefix_len: torch.Tensor
    suffix_begin: torch.Tensor
    max_group_rows: int


class Qwen2Model:
    """The decoder stack (reference Qwen2Model, qwen2_navit.py:943-1092)."""

    def __init__(self, config: Qwen2Config, device="cuda", dtype_mode: str = "A", fp8_gen_mlp: bool = False):
        self.config = config
        self.device = torch.device(device)
        if dtype_mode not in ("A", "B"):
            raise ValueError("dtype_mode must be 'A' (bf16 weights + autocast) or 'B' (fp32 master weights + autocast)")
        self.dtype_mode = dtype_mode
        self.stream_dtype = torch.float32 if dtype_mode == "B" else BF16     # residual stream / norm weights / embeddings
        # decoder layer class (reference Decoder_layer_dict, qwen2_navit.py:936-940)
        kinds = {"Qwen2DecoderLayer": "dense", "Qwen2MoEDecoderLayer": "moe", "Qwen2MoTDecoderLayer": "mot"}
        if config.layer_module not in kinds:
            raise ValueError(f"unknown layer_module {config.layer_module!r}; expected one of {sorted(kinds)}")
        self.layer_kind = kinds[config.layer_module]
        self.use_moe = "Mo" in config.layer_module      # same test as the reference (:948): MoE and MoT
        # opt-in block-scaled FP8 gate/up/down of the generation expert (bagel_b200/fp8.py); everything else stays mode A
        self.fp8_gen_mlp = bool(fp8_gen_mlp)
        if self.fp8_gen_mlp:
            if dtype_mode != "A":
                raise NotImplementedError("fp8_gen_mlp=True is implemented for dtype_mode='A' (bf16 residual stream)")
            if not self.use_moe:
                raise ValueError(f"fp8_gen_mlp=True needs a generation expert (mlp_moe_gen); {config.layer_module} has none")
            if config.hidden_size % 128 or config.intermediate_size % 128:
                raise ValueError("fp8_gen_mlp=True needs hidden_size and intermediate_size to be multiples of 128 "
                                 f"(got {config.hidden_size}, {config.intermediate_size})")
        self.enable_taylorseer = False
        self.layers: List[_Layer] = [_Layer() for _ in range(config.num_hidden_layers)]
        self.embed_tokens: Optional[_Embedding] = None
        self.norm = None
        self.norm_moe_gen = None
        d = config.head_dim
        # same expression as the reference's default rope init (fp32), computed on the host then moved
        self.inv_freq = (1.0 / (config.rope_theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))).to(self.device)
        self._ws: Dict[str, torch.Tensor] = {}
        self._ws_gen = 0   # bumped on every workspace (re)allocation: CUDA graphs captured over older buffers are stale

    # ----------------------------------------------------------------------------------------------
    def _buf(self, name: str, rows: int, cols: int, dtype=BF16) -> torch.Tensor:
        """Grow-only activation workspace (no allocation inside the layer loop once warmed up)."""
        t = self._ws.get(name)
        if t is None or t.shape[0] < rows or t.shape[1] != cols or t.dtype != dtype:
            t = torch.empty((rows, cols), dtype=dtype, device=self.device)
            self._ws[name] = t
            self._ws_gen += 1
        return t[:rows]

    def reserve(self, rows: int, text_rows: int = 0) -> None:
        """Size every run_layers()/final_norm() workspace for `rows` packed tokens (and `text_rows` und-expert rows) up
        front, so a later, larger call cannot replace a buffer that a captured CUDA graph still points into."""
        cfg = self.config
        H, D, I = cfg.hidden_size, cfg.head_dim, cfg.intermediate_size
        Hq, Hk = cfg.num_attention_heads, cfg.num_key_value_heads
        for name in ("xa", "xb"):
            self._buf(name, rows, H, self.stream_dtype)
        for name, cols in (("h", H), ("out", H), ("qkv", (Hq + 2 * Hk) * D), ("q", Hq * D), ("att", Hq * D), ("act", I)):
            self._buf(name, rows, cols)
        if text_rows:
            for name, cols in (("h_text", H), ("att_text", Hq * D), ("act_text", I)):
                self._buf(name, text_rows, cols)
        if self.fp8_gen_mlp:
            self._fp8_bufs(rows)

    def _scales_buf(self, name: str, groups: int, rows: int) -> torch.Tensor:
        """Grow-only fp32 [groups, >= rows] buffer of K-block-major activation scales (leading dimension = capacity)."""
        t = self._ws.get(name)
        if t is None or t.shape[1] < rows or t.shape[0] != groups:
            t = torch.empty((groups, rows), dtype=torch.float32, device=self.device)
            self._ws[name] = t
            self._ws_gen += 1
        return t

    def _fp8_bufs(self, rows: int):
        """e4m3 copies of the MLP block's two GEMM inputs (h, act) and their scales."""
        H, I = self.config.hidden_size, self.config.intermediate_size
        return (self._buf("h_fp8", rows, H, ops.FP8), self._scales_buf("h_fp8_s", H // 128, rows),
                self._buf("act_fp8", rows, I, ops.FP8), self._scales_buf("act_fp8_s", I // 128, rows))

    def alloc_kv(self, plan: ForwardPlan):
        """Merged K/V buffers [total_kv, Hk*D] for every layer (the reference re-allocates these per layer per
        call, qwen2_navit.py:563-569)."""
        cfg = self.config
        w = cfg.num_key_value_heads * cfg.head_dim
        L = cfg.num_hidden_layers
        k = torch.empty((L, plan.total_kv, w), dtype=BF16, device=self.device)
        v = torch.empty((L, plan.total_kv, w), dtype=BF16, device=self.device)
        return k, v

    def place_context(self, cache: NaiveCache, rows: torch.Tensor, kbuf, vbuf, src_rows: Optional[torch.Tensor] = None):
        """Copy every layer's cached K/V rows to `rows` (int32, on the device) of the merged buffers (reference
        :565-569). src_rows (int32, on the device, as many as `rows`): place only these cache rows, cache row
        src_rows[i] to rows[i] (the requests of a batch that take part in one CFG branch)."""
        cfg = self.config
        m, w = rows.numel(), cfg.num_key_value_heads * cfg.head_dim
        for li in range(cfg.num_hidden_layers):
            pk, pv = cache.key_cache[li], cache.value_cache[li]
            if src_rows is None:
                assert pk is not None and pk.shape[0] == m, "cache rows must match key_values_lens"
            else:
                assert pk is not None and src_rows.numel() == m, "one cache row per destination row"
            n = pk.shape[0]
            ops.copy_rows(pk.reshape(n, w), kbuf[li], src_rows=src_rows, dst_rows=rows, M=m)
            ops.copy_rows(pv.reshape(n, w), vbuf[li], src_rows=src_rows, dst_rows=rows, M=m)

    # ----------------------------------------------------------------------------------------------
    def run_layers(self, x: torch.Tensor, plan: ForwardPlan, kbuf: torch.Tensor, vbuf: torch.Tensor,
                   final_norm: bool = True) -> torch.Tensor:
        """All decoder layers + final norm on a packed bf16 sequence x [n, H]. kbuf/vbuf: [L, total_kv, Hk*D]
        with the context rows already in place; the new K/V rows are written by the qk-norm/RoPE kernel.
        Pure kernel launches (CUDA-graph capturable). final_norm=False returns the last layer's output (the
        TaylorSeer feature, qwen2_navit.py:824-826) and leaves the norm to `final_norm()`."""
        cfg = self.config
        n, H = plan.n, cfg.hidden_size
        Hq, Hk, D, I = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.intermediate_size
        eps = cfg.rms_norm_eps
        routed = plan.expert is not None
        nt = plan.text_rows.numel() if (routed and plan.text_rows is not None) else 0
        # MoT duplicates norms + attention + MLP per expert; MoE (Qwen2MoEDecoderLayer, :834-933) only the MLP
        a_routed = routed and self.layer_kind == "mot"
        a_expert = plan.expert if a_routed else None
        nta = nt if a_routed else 0

        modeB = self.dtype_mode == "B"
        rmsnorm = ops.rmsnorm_f32 if modeB else ops.rmsnorm           # fp32 stream + fp32 weights -> bf16 GEMM input
        EPI_R = ops.EPI_RESID_F32 if modeB else ops.EPI_RESID         # residual add in the stream's dtype
        xa = self._buf("xa", n, H, self.stream_dtype)
        xb = self._buf("xb", n, H, self.stream_dtype)
        h = self._buf("h", n, H)
        qkv = self._buf("qkv", n, (Hq + 2 * Hk) * D)
        q = self._buf("q", n, Hq * D)
        att = self._buf("att", n, Hq * D)
        act = self._buf("act", n, I)
        fp8 = routed and self.fp8_gen_mlp     # the gen rows' MLP in block-scaled FP8
        if fp8:
            hq, hs, aq, as_ = self._fp8_bufs(n)
        if nt:
            ht = self._buf("h_text", nt, H)
            at = self._buf("att_text", nt, Hq * D)
            actt = self._buf("act_text", nt, I)
        if x.data_ptr() != xa.data_ptr():
            xa.copy_(x)

        for li, layer in enumerate(self.layers):
            main = layer.gen if routed else layer.und       # MLP weights every row runs through
            und = layer.und
            amain = layer.gen if a_routed else layer.und     # norm / attention weights every row runs through
            # ---- attention block ----
            rmsnorm(xa, und.ln_in, amain.ln_in if a_routed else None, a_expert, eps, out=h)
            if plan.fuse_qkv:
                # QKV GEMM with q/k-norm + RoPE + KV placement in its epilogue (no [n, 4608] round trip)
                ops.gemm_qkv_norm_rope(h, amain.wqkv, amain.bqkv, und.q_norm, und.k_norm,
                                       amain.q_norm if a_routed else None, amain.k_norm if a_routed else None, a_expert,
                                       plan.cos, plan.sin, q, kbuf[li], vbuf[li], plan.q_rows, Hq, Hk, eps, plan.fp32_flow)
                if nta:
                    ops.copy_rows(h, ht, src_rows=plan.text_rows)
                    ops.gemm_qkv_norm_rope(ht, und.wqkv, und.bqkv, und.q_norm, und.k_norm, amain.q_norm, amain.k_norm,
                                           a_expert, plan.cos, plan.sin, q, kbuf[li], vbuf[li], plan.q_rows, Hq, Hk,
                                           eps, plan.fp32_flow, row_map=plan.text_rows)
            else:
                ops.gemm(h, amain.wqkv, bias=amain.bqkv, out=qkv)
                if nta:
                    ops.copy_rows(h, ht, src_rows=plan.text_rows)
                    ops.gemm(ht, und.wqkv, bias=und.bqkv, row_map=plan.text_rows, out=qkv)
                ops.qk_norm_rope(qkv, und.q_norm, und.k_norm, amain.q_norm if a_routed else None,
                                 amain.k_norm if a_routed else None, a_expert, plan.cos, plan.sin, q, kbuf[li], vbuf[li],
                                 plan.q_rows, Hq, Hk, D, eps, plan.fp32_flow)
            if plan.shared is not None:
                sh = plan.shared
                ops.attn_decode_shared(q.view(n, Hq, D), kbuf[li].view(-1, Hk, D), vbuf[li].view(-1, Hk, D), sh.cu_rows,
                                       sh.prefix_begin, sh.prefix_len, sh.suffix_begin, plan.seqused_k,
                                       sh.max_group_rows, plan.max_k, out=att.view(n, Hq, D))
            else:
                ops.attn_varlen(q.view(n, Hq, D), kbuf[li].view(-1, Hk, D), vbuf[li].view(-1, Hk, D), plan.cu_q,
                                plan.cu_k, plan.max_q, plan.max_k, plan.is_causal, out=att.view(n, Hq, D),
                                seqused_k=plan.seqused_k)
            ops.gemm(att, amain.wo, resid=xa, epilogue=EPI_R, out=xb)
            if nta:
                ops.copy_rows(att, at, src_rows=plan.text_rows)
                ops.gemm(at, und.wo, resid=xa, row_map=plan.text_rows, epilogue=EPI_R, out=xb)
            # ---- MLP block ----
            rmsnorm(xb, und.ln_post, amain.ln_post if a_routed else None, a_expert, eps, out=h)
            if fp8:
                ops.quantize_fp8(h, 1, q=hq, scales=hs)
                ops.gemm_fp8(hq, hs, main.fp8.wgu, main.fp8.wgu_s, epilogue=ops.EPI_SWIGLU, out=act)
                ops.quantize_fp8(act, 1, q=aq, scales=as_)
                ops.gemm_fp8(aq, as_, main.fp8.wd, main.fp8.wd_s, resid=xb, epilogue=ops.EPI_RESID, out=xa)
            else:
                ops.gemm(h, main.wgu, epilogue=ops.EPI_SWIGLU, out=act)
                ops.gemm(act, main.wd, resid=xb, epilogue=EPI_R, out=xa)
            if nt:
                ops.copy_rows(h, ht, src_rows=plan.text_rows)
                ops.gemm(ht, und.wgu, epilogue=ops.EPI_SWIGLU, out=actt)
                ops.gemm(actt, und.wd, resid=xb, row_map=plan.text_rows, epilogue=EPI_R, out=xa)

        if not final_norm:
            return xa
        return self.final_norm(plan)

    def final_norm(self, plan: ForwardPlan, for_linear: bool = False) -> torch.Tensor:
        """Final (routed) RMSNorm of the hidden state left in the "xa" workspace (qwen2_navit.py:1075-1084). Mode B: the
        norm output is fp32 (what forward_inference returns); for_linear=True gives its bf16 cast, i.e. the operand the
        next nn.Linear (llm2vae / lm_head) sees under autocast."""
        n, H = plan.n, self.config.hidden_size
        routed = plan.expert is not None
        xa = self._buf("xa", n, H, self.stream_dtype)
        w1 = self.norm_moe_gen if routed else None
        if self.dtype_mode == "B":
            out = self._buf("out", n, H) if for_linear else self._buf("out32", n, H, torch.float32)
            return ops.rmsnorm_f32(xa, self.norm, w1, plan.expert, self.config.rms_norm_eps, out=out)
        out = self._buf("out", n, H)
        ops.rmsnorm(xa, self.norm, w1, plan.expert, self.config.rms_norm_eps, out=out)
        return out

    # ----------------------------------------------------------------------------------------------
    def forward_inference(self, packed_query_sequence, query_lens, packed_query_position_ids, packed_query_indexes,
                          past_key_values: Optional[NaiveCache] = None, key_values_lens=None,
                          packed_key_value_indexes=None, update_past_key_values=True, is_causal=True, mode="und",
                          packed_vae_token_indexes=None, packed_text_indexes=None,
                          train_numerics: bool = False) -> BaseNavitOutputWithPast:
        if self.enable_taylorseer:
            raise NotImplementedError("the TaylorSeer step cache lives in the planned sampler: call "
                                      "Bagel.generate_image(enable_taylorseer=True) (bagel_b200/bagel.py FlowRunner)")
        if not self.use_moe:
            mode = "und"
        has_ctx = past_key_values is not None and past_key_values.key_cache[0] is not None
        plan = ForwardPlan(self, query_lens, packed_query_position_ids, packed_query_indexes,
                           key_values_lens if has_ctx else None, packed_key_value_indexes if has_ctx else None,
                           is_causal, mode, packed_vae_token_indexes, packed_text_indexes, train_numerics)
        x = packed_query_sequence.to(self.device, self.stream_dtype)
        kbuf, vbuf = self.alloc_kv(plan)
        if plan.n_ctx:
            self.place_context(past_key_values, plan.ctx_rows, kbuf, vbuf)
        out = self.run_layers(x, plan, kbuf, vbuf).clone()
        if update_past_key_values:
            cfg = self.config
            for li in range(cfg.num_hidden_layers):
                past_key_values.key_cache[li] = kbuf[li].view(-1, cfg.num_key_value_heads, cfg.head_dim)
                past_key_values.value_cache[li] = vbuf[li].view(-1, cfg.num_key_value_heads, cfg.head_dim)
        return BaseNavitOutputWithPast(packed_query_sequence=out, past_key_values=past_key_values)

    __call__ = forward_inference


class Qwen2ForCausalLM:
    """Reference Qwen2ForCausalLM (qwen2_navit.py:1095-1188): `.model`, `.lm_head`, forward_inference(...)."""

    def __init__(self, config: Qwen2Config, device="cuda", dtype_mode: str = "A", fp8_gen_mlp: bool = False):
        self.config = config
        self.model = Qwen2Model(config, device, dtype_mode, fp8_gen_mlp)
        self.lm_head: Optional[_Linear] = None
        self.vocab_size = config.vocab_size

    @property
    def device(self):
        return self.model.device

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def eval(self):
        return self

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """`sd` uses the reference's parameter names (SURVEY.md §8b): model.layers.{i}.self_attn.q_proj.weight ...
        Builds the fused kernel layouts on the device."""
        cfg = self.config
        dev = self.model.device
        used = set()

        sdt = self.model.stream_dtype     # fp32 in dtype mode B: norm weights / embeddings keep the checkpoint precision

        def get(name, required=True, dtype=BF16):
            if name in sd:
                used.add(name)
                return sd[name].to(dev, dtype)
            if required:
                raise KeyError(f"missing weight {name}")
            return None

        def load_mlp(e: _ExpertWeights, m: str, gen: bool):
            if gen and self.model.fp8_gen_mlp:
                # quantised from the bf16 matrices, which are dropped afterwards: only the e4m3 copies stay on the device
                e.fp8 = _fp8.GenMlpFp8.from_reference(get(m + "gate_proj.weight"), get(m + "up_proj.weight"),
                                                      get(m + "down_proj.weight"))
                e.wgu = e.wd = None
            else:
                e.wgu = ops.interleave_gate_up(get(m + "gate_proj.weight"), get(m + "up_proj.weight"))
                e.wd = get(m + "down_proj.weight").contiguous()
                e.fp8 = None

        self.model.embed_tokens = _Embedding(get("model.embed_tokens.weight", dtype=sdt).contiguous())
        for li, layer in enumerate(self.model.layers):
            p = f"model.layers.{li}."
            for sfx, tgt in (("", "und"), ("_moe_gen", "gen")):
                if sfx and not self.model.use_moe:
                    continue
                e = _ExpertWeights()
                if sfx and self.model.layer_kind == "moe":
                    # Qwen2MoEDecoderLayer: only the MLP is duplicated (mlp_moe_gen); attention / norms are shared
                    load_mlp(e, p + f"mlp{sfx}.", bool(sfx))
                    u = layer.und
                    e.wqkv, e.bqkv, e.wo, e.ln_in, e.ln_post, e.q_norm, e.k_norm = (u.wqkv, u.bqkv, u.wo, u.ln_in,
                                                                                     u.ln_post, u.q_norm, u.k_norm)
                    setattr(layer, tgt, e)
                    continue
                a = p + "self_attn."
                e.wqkv = torch.cat([get(a + f"q_proj{sfx}.weight"), get(a + f"k_proj{sfx}.weight"),
                                    get(a + f"v_proj{sfx}.weight")], dim=0).contiguous()
                e.bqkv = torch.cat([get(a + f"q_proj{sfx}.bias"), get(a + f"k_proj{sfx}.bias"),
                                    get(a + f"v_proj{sfx}.bias")], dim=0).contiguous()
                e.wo = get(a + f"o_proj{sfx}.weight").contiguous()
                if cfg.qk_norm:
                    e.q_norm = get(a + f"q_norm{sfx}.weight", dtype=sdt).contiguous()
                    e.k_norm = get(a + f"k_norm{sfx}.weight", dtype=sdt).contiguous()
                else:
                    # nn.Identity in the reference (:247-252, :398-404); no shipped BAGEL config uses it and the fused
                    # QKV epilogue has no norm-free variant, so say so at load time instead of mis-computing later
                    raise NotImplementedError("bagel_b200: qk_norm=False is not implemented (every shipped BAGEL loader "
                                              "forces qk_norm=True, app.py:41)")
                load_mlp(e, p + f"mlp{sfx}.", bool(sfx))
                e.ln_in = get(p + f"input_layernorm{sfx}.weight", dtype=sdt).contiguous()
                e.ln_post = get(p + f"post_attention_layernorm{sfx}.weight", dtype=sdt).contiguous()
                setattr(layer, tgt, e)
        self.model.norm = get("model.norm.weight", dtype=sdt).contiguous()
        if self.model.use_moe:
            self.model.norm_moe_gen = get("model.norm_moe_gen.weight", dtype=sdt).contiguous()
        lw = get("lm_head.weight", required=False)
        if lw is None and cfg.tie_word_embeddings:
            lw = self.model.embed_tokens.weight.to(BF16)
        self.lm_head = _Linear(lw.contiguous()) if lw is not None else None
        unexpected = [k for k in sd if k not in used]
        if strict and unexpected:
            raise KeyError(f"unexpected keys: {unexpected[:8]}")
        return unexpected

    def forward_inference(self, *args, **kwargs) -> BaseNavitOutputWithPast:
        return self.model.forward_inference(*args, **kwargs)

    __call__ = forward_inference
