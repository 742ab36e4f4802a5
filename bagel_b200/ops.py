"""torch.Tensor-facing wrappers over the C ABI (include/bagel_b200.h). PyTorch is used only for device
memory and streams; every call below lands in a hand-written sm_90a kernel or raises."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _cabi

EPI_BIAS, EPI_RESID, EPI_SWIGLU, EPI_GELU, EPI_SILU, EPI_F32 = 0, 1, 2, 3, 4, 5
EPI_RESID_F32 = 7   # fp32 residual stream (dtype mode B): out32 = resid32 + bf16(acc + bias)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# Optional live timing of one kernel family inside a run (bench.py roofline): CUDA events on the launching stream.
_timer = {"tag": None, "events": []}


def kernel_timer_start(tag: str) -> None:
    _timer["tag"], _timer["events"] = tag, []


def kernel_timer_stop():
    """Returns the per-launch durations (ms) recorded since kernel_timer_start (synchronises)."""
    ev = _timer["events"]
    _timer["tag"], _timer["events"] = None, []
    if not ev:
        return []
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def _opt(t: Optional[torch.Tensor], dtype, name: str) -> None:
    if t is not None:
        _req(t, dtype, name)


def _req(t: torch.Tensor, dtype, name: str) -> None:
    if not torch.is_tensor(t):
        raise _cabi.BagelB200Error(f"{name}: expected a tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise _cabi.BagelB200Error(f"{name}: expected a CUDA tensor (bagel_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _cabi.BagelB200Error(f"{name}: expected {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1:
        raise _cabi.BagelB200Error(f"{name}: innermost dimension must be contiguous")


def interleave_gate_up(gate_w: torch.Tensor, up_w: torch.Tensor, block: int = 128) -> torch.Tensor:
    """[I,K],[I,K] -> [2I,K] with rows arranged (gate block of 128 | up block of 128) per 256 rows, the
    layout BAGEL_EPI_SWIGLU expects so one 256-wide tile holds matching gate/up columns."""
    I, K = gate_w.shape
    assert up_w.shape == (I, K) and I % block == 0
    g = gate_w.reshape(I // block, block, K)
    u = up_w.reshape(I // block, block, K)
    return torch.stack((g, u), dim=1).reshape(2 * I, K).contiguous()


def gemm(a: torch.Tensor, w: torch.Tensor, *, bias: Optional[torch.Tensor] = None,
         resid: Optional[torch.Tensor] = None, row_map: Optional[torch.Tensor] = None,
         epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(a @ w.T); a [M,K] bf16, w [N,K] bf16 (nn.Linear layout)."""
    _req(a, torch.bfloat16, "a")
    _req(w, torch.bfloat16, "w")
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    out_dtype = torch.float32 if epilogue in (EPI_F32, EPI_RESID_F32) else torch.bfloat16
    if out is None:
        assert row_map is None, "row_map scatter needs an explicit `out`"
        out = torch.empty((M, n_out), dtype=out_dtype, device=a.device)
    _req(out, out_dtype, "out")
    assert out.shape[1] == n_out
    if bias is not None:
        _req(bias, torch.bfloat16, "bias")
        assert bias.numel() == N
    ldr = 0
    if resid is not None:
        _req(resid, torch.float32 if epilogue == EPI_RESID_F32 else torch.bfloat16, "resid")
        ldr = resid.stride(0)
    if row_map is not None:
        _req(row_map, torch.int32, "row_map")
        assert row_map.numel() == M
    timed = _timer["tag"] == "swiglu" and epilogue == EPI_SWIGLU and M >= 1024
    if timed:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = _cabi.lib().bagel_gemm_bf16(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0),
                                     M, N, K, _ptr(bias), _ptr(resid), ldr, _ptr(row_map), epilogue, _stream())
    _cabi.check(rc, "bagel_gemm_bf16")
    if timed:
        e1.record()
        _timer["events"].append((e0, e1))
    return out


FP8 = torch.float8_e4m3fn


def quantize_fp8(x: torch.Tensor, block_rows: int = 1, *, q: Optional[torch.Tensor] = None,
                 scales: Optional[torch.Tensor] = None):
    """Block-scaled e4m3 quantisation of a bf16 [M, K] tensor (K % 128 == 0): returns (q [M, K] float8_e4m3fn,
    fp32 power-of-two scales). block_rows=1: one scale per 1 x 128 group, K-block major [K/128, M] (activations);
    block_rows=128: one per 128 x 128 block, [ceil(M/128), K/128] (weights). See bagel_quantize_fp8_bf16."""
    _req(x, torch.bfloat16, "x")
    M, K = x.shape
    if q is None:
        q = torch.empty((M, K), dtype=FP8, device=x.device)
    _req(q, FP8, "q")
    assert q.shape == (M, K)
    shape = (K // 128, M) if block_rows == 1 else ((M + 127) // 128, K // 128)
    if scales is None:
        scales = torch.empty(shape, dtype=torch.float32, device=x.device)
    _req(scales, torch.float32, "scales")
    assert scales.dim() == 2 and scales.shape[0] == shape[0] and scales.shape[1] >= shape[1]
    rc = _cabi.lib().bagel_quantize_fp8_bf16(_ptr(x), x.stride(0), _ptr(q), q.stride(0), _ptr(scales), scales.stride(0),
                                             M, K, int(block_rows), _stream())
    _cabi.check(rc, "bagel_quantize_fp8_bf16")
    return q, scales


def gemm_fp8(a: torch.Tensor, a_scales: torch.Tensor, w: torch.Tensor, w_scales: torch.Tensor, *,
             resid: Optional[torch.Tensor] = None, epilogue: int = EPI_RESID,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(dequant(a) @ dequant(w).T) with block-scaled e4m3 operands: a [M, K] with a_scales [K/128, >= M]
    (quantize_fp8 block_rows=1), w [N, K] with w_scales [N/64, K/128] (see bagel_b200.fp8 for the weight layouts).
    EPI_SWIGLU (w gate|up interleaved per 64 rows, out [M, N/2]) or EPI_RESID (out [M, N] = resid + y)."""
    _req(a, FP8, "a")
    _req(w, FP8, "w")
    _req(a_scales, torch.float32, "a_scales")
    _req(w_scales, torch.float32, "w_scales")
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and w_scales.is_contiguous() and w_scales.shape == (N // 64, K // 128)
    assert a_scales.shape[0] == K // 128 and a_scales.shape[1] >= M
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=a.device)
    _req(out, torch.bfloat16, "out")
    assert out.shape[1] == n_out
    ldr = 0
    if resid is not None:
        _req(resid, torch.bfloat16, "resid")
        ldr = resid.stride(0)
    rc = _cabi.lib().bagel_gemm_fp8(_ptr(a), a.stride(0), _ptr(a_scales), a_scales.stride(0), _ptr(w), w.stride(0),
                                    _ptr(w_scales), _ptr(out), out.stride(0), M, N, K, _ptr(resid), ldr, epilogue,
                                    _stream())
    _cabi.check(rc, "bagel_gemm_fp8")
    return out


def gemm_qkv_norm_rope(a, w, bias, q_w0, k_w0, q_w1, k_w1, expert, cos, sin, q_out, k_out, v_out, kv_rows, Hq, Hk,
                       eps: float, fp32_flow: bool, row_map=None):
    """Fused QKV projection + per-head q/k RMSNorm + RoPE + bf16 cast + K/V placement (head_dim 128)."""
    _req(a, torch.bfloat16, "a"); _req(w, torch.bfloat16, "w"); _req(bias, torch.bfloat16, "bias")
    M, K = a.shape
    assert w.shape == ((Hq + 2 * Hk) * 128, K)
    _qkv_tail_checks(M if row_map is None else None, q_w0, k_w0, q_w1, k_w1, expert, cos, sin, q_out, k_out, v_out, kv_rows,
                     Hq, Hk, 128, int(fp32_flow))
    _opt(row_map, torch.int32, "row_map")
    rc = _cabi.lib().bagel_gemm_qkv_norm_rope(
        _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(bias), M, K, _ptr(row_map), _ptr(q_w0), _ptr(k_w0),
        _ptr(q_w1), _ptr(k_w1), _ptr(expert), _ptr(cos), _ptr(sin), _ptr(q_out), q_out.stride(0), _ptr(k_out),
        _ptr(v_out), k_out.stride(0), _ptr(kv_rows), Hq, Hk, float(eps), int(fp32_flow), _stream())
    _cabi.check(rc, "bagel_gemm_qkv_norm_rope")


def _qkv_tail_checks(n_rows, q_w0, k_w0, q_w1, k_w1, expert, cos, sin, q_out, k_out, v_out, kv_rows, Hq, Hk, D, flow=0):
    """Shared argument checks of the two q/k-norm + RoPE + KV-placement entry points (raw pointers cross the C ABI)."""
    wdt = torch.float32 if flow >= 2 else torch.bfloat16      # flows 2, 3 (fp32 master weights) read fp32 norm weights
    for t, nm in ((q_w0, "q_w0"), (k_w0, "k_w0")):
        _req(t, wdt, nm)
        assert t.numel() == D, f"{nm}: expected {D} elements"
    _opt(q_w1, wdt, "q_w1"); _opt(k_w1, wdt, "k_w1")
    _opt(expert, torch.uint8, "expert")
    _req(cos, torch.float32, "cos"); _req(sin, torch.float32, "sin")
    assert cos.shape == sin.shape and cos.shape[-1] == D // 2 and cos.is_contiguous() and sin.is_contiguous()
    _req(q_out, torch.bfloat16, "q_out"); _req(k_out, torch.bfloat16, "k_out"); _req(v_out, torch.bfloat16, "v_out")
    assert q_out.shape[-1] >= Hq * D and k_out.shape[-1] >= Hk * D and v_out.shape[-1] >= Hk * D
    assert k_out.stride(0) == v_out.stride(0), "K and V buffers must share their row stride"
    _opt(kv_rows, torch.int32, "kv_rows")
    if n_rows is not None:
        assert cos.shape[0] >= n_rows and q_out.shape[0] >= n_rows
        if kv_rows is not None:
            assert kv_rows.numel() >= n_rows
        if expert is not None:
            assert expert.numel() >= n_rows


def attn_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q: torch.Tensor,
                cu_seqlens_k: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, causal: bool = False,
                softmax_scale: Optional[float] = None, out: Optional[torch.Tensor] = None,
                seqused_k: Optional[torch.Tensor] = None) -> torch.Tensor:
    """flash_attn_varlen_func contract (qwen2_navit.py:579-588): q [Sq,Hq,D], k/v [Sk,Hk,D] bf16."""
    _req(q, torch.bfloat16, "q"); _req(k, torch.bfloat16, "k"); _req(v, torch.bfloat16, "v")
    _req(cu_seqlens_q, torch.int32, "cu_seqlens_q"); _req(cu_seqlens_k, torch.int32, "cu_seqlens_k")
    Sq, Hq, D = q.shape
    Sk, Hk, _ = k.shape
    assert q.stride(1) == D and k.stride(1) == D and v.stride(1) == D, "heads must be contiguous"
    if out is None:
        out = torch.empty((Sq, Hq, D), dtype=torch.bfloat16, device=q.device)
    if softmax_scale is None:
        softmax_scale = D ** -0.5
    B = cu_seqlens_q.numel() - 1
    rc = _cabi.lib().bagel_attn_varlen_fwd(_ptr(q), _ptr(k), _ptr(v), _ptr(out), _ptr(cu_seqlens_q), _ptr(cu_seqlens_k),
                                           Sq, Sk, B, Hq, Hk, D, int(max_seqlen_q), int(max_seqlen_k), int(bool(causal)),
                                           float(softmax_scale), q.stride(0), k.stride(0), v.stride(0), out.stride(0),
                                           _ptr(seqused_k), _stream())
    _cabi.check(rc, "bagel_attn_varlen_fwd")
    return out


def rmsnorm(x: torch.Tensor, w0: torch.Tensor, w1: Optional[torch.Tensor] = None,
            expert: Optional[torch.Tensor] = None, eps: float = 1e-6, out: Optional[torch.Tensor] = None):
    _req(x, torch.bfloat16, "x"); _req(w0, torch.bfloat16, "w0")
    N, H = x.shape
    if out is None:
        out = torch.empty_like(x)
    if expert is not None:
        _req(expert, torch.uint8, "expert")
    rc = _cabi.lib().bagel_rmsnorm_bf16(_ptr(x), x.stride(0), _ptr(w0), _ptr(w1), _ptr(expert), _ptr(out), out.stride(0),
                                        N, H, float(eps), _stream())
    _cabi.check(rc, "bagel_rmsnorm_bf16")
    return out


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-6, out: Optional[torch.Tensor] = None):
    _req(x, torch.bfloat16, "x"); _req(w, torch.bfloat16, "w"); _req(b, torch.bfloat16, "b")
    N, H = x.shape
    if out is None:
        out = torch.empty_like(x)
    rc = _cabi.lib().bagel_layernorm_bf16(_ptr(x), x.stride(0), _ptr(w), _ptr(b), _ptr(out), out.stride(0), N, H,
                                          float(eps), _stream())
    _cabi.check(rc, "bagel_layernorm_bf16")
    return out


def rope_table(pos: torch.Tensor, inv_freq: torch.Tensor, round_bf16: bool = True):
    _req(pos, torch.int64, "pos"); _req(inv_freq, torch.float32, "inv_freq")
    N, half = pos.numel(), inv_freq.numel()
    cos = torch.empty((N, half), dtype=torch.float32, device=pos.device)
    sin = torch.empty_like(cos)
    rc = _cabi.lib().bagel_rope_table(_ptr(pos), _ptr(inv_freq), _ptr(cos), _ptr(sin), N, half, int(round_bf16), _stream())
    _cabi.check(rc, "bagel_rope_table")
    return cos, sin


def rope_table_into(pos: torch.Tensor, inv_freq: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, round_bf16: bool = True):
    """rope_table writing into caller-owned buffers (graph-replayable decode step)."""
    _req(pos, torch.int64, "pos"); _req(inv_freq, torch.float32, "inv_freq")
    _req(cos, torch.float32, "cos"); _req(sin, torch.float32, "sin")
    assert cos.is_contiguous() and sin.is_contiguous() and cos.numel() >= pos.numel() * inv_freq.numel() <= sin.numel()
    rc = _cabi.lib().bagel_rope_table(_ptr(pos), _ptr(inv_freq), _ptr(cos), _ptr(sin), pos.numel(), inv_freq.numel(),
                                      int(round_bf16), _stream())
    _cabi.check(rc, "bagel_rope_table")


def qk_norm_rope(qkv, q_w0, k_w0, q_w1, k_w1, expert, cos, sin, q_out, k_out, v_out, kv_rows, Hq, Hk, D,
                 eps: float, fp32_flow: bool):
    _req(qkv, torch.bfloat16, "qkv")
    N = qkv.shape[0]
    assert qkv.shape[1] >= (Hq + 2 * Hk) * D
    _qkv_tail_checks(N, q_w0, k_w0, q_w1, k_w1, expert, cos, sin, q_out, k_out, v_out, kv_rows, Hq, Hk, D, int(fp32_flow))
    rc = _cabi.lib().bagel_qk_norm_rope(_ptr(qkv), qkv.stride(0), _ptr(q_w0), _ptr(k_w0), _ptr(q_w1), _ptr(k_w1),
                                        _ptr(expert), _ptr(cos), _ptr(sin), _ptr(q_out), q_out.stride(0), _ptr(k_out),
                                        _ptr(v_out), k_out.stride(0), _ptr(kv_rows), N, Hq, Hk, D, float(eps),
                                        int(fp32_flow), _stream())
    _cabi.check(rc, "bagel_qk_norm_rope")


def copy_rows(src, dst, src_rows=None, dst_rows=None, M: Optional[int] = None):
    _req(src, torch.bfloat16, "src"); _req(dst, torch.bfloat16, "dst")
    if M is None:
        M = src_rows.numel() if src_rows is not None else (dst_rows.numel() if dst_rows is not None else src.shape[0])
    H = src.shape[-1]
    _opt(src_rows, torch.int32, "src_rows"); _opt(dst_rows, torch.int32, "dst_rows")
    if dst.shape[-1] < H:
        raise _cabi.BagelB200Error(f"copy_rows: dst rows are {dst.shape[-1]} wide, src rows {H}")
    if src_rows is not None and src_rows.numel() < M or dst_rows is not None and dst_rows.numel() < M:
        raise _cabi.BagelB200Error("copy_rows: index tensor shorter than M")
    if src_rows is None and src.shape[0] < M or dst_rows is None and dst.shape[0] < M:
        raise _cabi.BagelB200Error("copy_rows: M exceeds the rows of an un-indexed operand")
    rc = _cabi.lib().bagel_copy_rows_bf16(_ptr(src), src.stride(0), _ptr(src_rows), _ptr(dst), dst.stride(0),
                                          _ptr(dst_rows), M, H, _stream())
    _cabi.check(rc, "bagel_copy_rows_bf16")
    return dst


def latent_embed_add(proj, t_emb, pos_table, pos_ids, seq, dst_rows):
    """seq[dst_rows[i]] = bf16(bf16(proj[i] + t_emb) + pos_table[pos_ids[i]]); t_emb / dst_rows may be None."""
    M, H = proj.shape
    _req(proj, torch.bfloat16, "proj"); _opt(t_emb, torch.bfloat16, "t_emb"); _req(pos_table, torch.bfloat16, "pos_table")
    _req(pos_ids, torch.int64, "pos_ids"); _req(seq, torch.bfloat16, "seq"); _opt(dst_rows, torch.int32, "dst_rows")
    assert pos_table.shape[-1] == H and seq.shape[-1] >= H and pos_ids.numel() >= M
    assert t_emb is None or t_emb.numel() >= H
    assert (dst_rows.numel() >= M) if dst_rows is not None else (seq.shape[0] >= M)
    rc = _cabi.lib().bagel_latent_embed_add(_ptr(proj), proj.stride(0), _ptr(t_emb), _ptr(pos_table), pos_table.stride(0),
                                            _ptr(pos_ids), _ptr(seq), seq.stride(0), _ptr(dst_rows), M, H, _stream())
    _cabi.check(rc, "bagel_latent_embed_add")


RENORM = {"global": 0, "channel": 1, "text_channel": 2}


def cfg_euler_step(v, v_text, v_img, rows, x, norms_ws, cfg_text_scale, cfg_img_scale, renorm_min, renorm_type, dt,
                   dt_dev: Optional[torch.Tensor] = None):
    _req(x, torch.float32, "x")
    M, Cc = x.shape
    assert x.is_contiguous()
    _req(v, torch.bfloat16, "v"); _opt(v_text, torch.bfloat16, "v_text"); _opt(v_img, torch.bfloat16, "v_img")
    _req(rows, torch.int32, "rows"); _req(norms_ws, torch.float32, "norms_ws"); _opt(dt_dev, torch.float32, "dt_dev")
    assert rows.numel() >= M and norms_ws.numel() >= 2 and v.shape[-1] >= Cc
    for t in (v_text, v_img):
        assert t is None or t.stride(0) == v.stride(0), "CFG branches must share the row stride of v"
    rc = _cabi.lib().bagel_cfg_euler_step(_ptr(v), _ptr(v_text), _ptr(v_img), v.stride(0), _ptr(rows), _ptr(x),
                                          _ptr(norms_ws), M, Cc, float(cfg_text_scale), float(cfg_img_scale),
                                          float(renorm_min), RENORM[renorm_type], float(dt), _ptr(dt_dev), _stream())
    _cabi.check(rc, "bagel_cfg_euler_step")


def cfg_batch_workspace(M: int, R: int, device) -> torch.Tensor:
    """fp32 workspace of cfg_euler_step_batch for M latent rows of R requests."""
    return torch.zeros(2 * M + 2 * R, dtype=torch.float32, device=device)


def cfg_euler_step_batch(v, seg, row_main, row_text, row_img, x, workspace, cfg_text_scale, cfg_img_scale, renorm_min,
                         renorm_type, cfg_on, dt_dev):
    """Per-request CFG + renorm + Euler step (see include/bagel_b200.h): latent row r of request seg[r] reads rows
    row_main[r] / row_text[r] / row_img[r] (-1: no such branch) of v; a request's rows are contiguous in seg.
    Per-request parameters are device arrays of length R: scales / renorm_min fp32, renorm_type (ops.RENORM values) and
    cfg_on int32; dt_dev fp32[1]; workspace from cfg_batch_workspace."""
    _req(x, torch.float32, "x")
    M, Cc = x.shape
    assert x.is_contiguous()
    _req(v, torch.bfloat16, "v")
    for t, nm in ((seg, "seg"), (row_main, "row_main"), (row_text, "row_text"), (row_img, "row_img")):
        _req(t, torch.int32, nm)
        assert t.numel() >= M, f"{nm}: one entry per latent row"
    R = cfg_on.numel()
    for t, dt, nm in ((cfg_text_scale, torch.float32, "cfg_text_scale"), (cfg_img_scale, torch.float32, "cfg_img_scale"),
                      (renorm_min, torch.float32, "renorm_min"), (renorm_type, torch.int32, "renorm_type"),
                      (cfg_on, torch.int32, "cfg_on")):
        _req(t, dt, nm)
        assert t.numel() == R, f"{nm}: one entry per request"
    _req(dt_dev, torch.float32, "dt_dev"); _req(workspace, torch.float32, "workspace")
    assert workspace.numel() >= 2 * M + 2 * R and v.shape[-1] >= Cc
    rc = _cabi.lib().bagel_cfg_euler_step_batch(_ptr(v), v.stride(0), _ptr(seg), _ptr(row_main), _ptr(row_text),
                                                _ptr(row_img), _ptr(x), M, Cc, R, _ptr(cfg_text_scale),
                                                _ptr(cfg_img_scale), _ptr(renorm_min), _ptr(renorm_type), _ptr(cfg_on),
                                                _ptr(dt_dev), _ptr(workspace), _stream())
    _cabi.check(rc, "bagel_cfg_euler_step_batch")


def cast_f32_to_bf16(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, torch.float32, "x")
    assert x.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    rc = _cabi.lib().bagel_cast_f32_to_bf16(_ptr(x), _ptr(out), x.numel(), _stream())
    _cabi.check(rc, "bagel_cast_f32_to_bf16")
    return out


# ---------------------------------------------------------------------------------------------------------
# VAE ops (NHWC bf16)
# ---------------------------------------------------------------------------------------------------------
def conv2d_nhwc(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, stride: int = 1, pad: int = 0,
                out_hw=None, resid: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B,H,W,Cin], w [Cout,k,k,Cin] bf16 -> [B,Ho,Wo,Cout] = bf16(resid + bf16(conv(x) + bias))."""
    _req(x, torch.bfloat16, "x"); _req(w, torch.bfloat16, "w")
    assert x.is_contiguous() and w.is_contiguous()
    B, Hi, Wi, Cin = x.shape
    Cout, k, k2, Cin2 = w.shape
    assert k == k2 and Cin2 == Cin
    if out_hw is None:
        Ho = (Hi + 2 * pad - k) // stride + 1
        Wo = (Wi + 2 * pad - k) // stride + 1
    else:
        Ho, Wo = out_hw
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), dtype=torch.bfloat16, device=x.device)
    if resid is not None:
        _req(resid, torch.bfloat16, "resid")
        assert resid.shape == out.shape and resid.is_contiguous()
    rc = _cabi.lib().bagel_conv2d_nhwc_bf16(_ptr(x), B, Hi, Wi, Cin, _ptr(w), Cout, k, stride, pad, _ptr(bias), _ptr(resid),
                                            _ptr(out), Ho, Wo, _stream())
    _cabi.check(rc, "bagel_conv2d_nhwc_bf16")
    return out


_gn_ws = {}


def groupnorm_nhwc(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-6, swish: bool = True,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, torch.bfloat16, "x")
    assert x.is_contiguous()
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    key = (x.device, B)
    ws = _gn_ws.get(key)
    if ws is None:
        ws = torch.empty(int(_cabi.lib().bagel_groupnorm_workspace_bytes(B, 32)), dtype=torch.uint8, device=x.device)
        _gn_ws[key] = ws
    if out is None:
        out = torch.empty_like(x)
    rc = _cabi.lib().bagel_groupnorm_nhwc_bf16(_ptr(x), _ptr(w), _ptr(b), _ptr(out), _ptr(ws), B, HW, C, 32, float(eps),
                                               int(swish), _stream())
    _cabi.check(rc, "bagel_groupnorm_nhwc_bf16")
    return out


def upsample2x_nhwc(x: torch.Tensor) -> torch.Tensor:
    _req(x, torch.bfloat16, "x")
    assert x.is_contiguous()
    B, H, W, C = x.shape
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.bfloat16, device=x.device)
    rc = _cabi.lib().bagel_upsample2x_nhwc_bf16(_ptr(x), _ptr(y), B, H, W, C, _stream())
    _cabi.check(rc, "bagel_upsample2x_nhwc_bf16")
    return y


def softmax_rows(S: torch.Tensor, scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(S, torch.float32, "S")
    rows, L = S.shape
    if out is None:
        out = torch.empty((rows, L), dtype=torch.bfloat16, device=S.device)
    rc = _cabi.lib().bagel_softmax_rows_f32(_ptr(S), S.stride(0), _ptr(out), out.stride(0), rows, L, float(scale), _stream())
    _cabi.check(rc, "bagel_softmax_rows_f32")
    return out


def transpose(x: torch.Tensor) -> torch.Tensor:
    _req(x, torch.bfloat16, "x")
    R, Cc = x.shape
    y = torch.empty((Cc, R), dtype=torch.bfloat16, device=x.device)
    rc = _cabi.lib().bagel_transpose_bf16(_ptr(x), x.stride(0), _ptr(y), y.stride(0), R, Cc, _stream())
    _cabi.check(rc, "bagel_transpose_bf16")
    return y


# ---------------------------------------------------------------------------------------------------------
# text decode bookkeeping (device-resident)
# ---------------------------------------------------------------------------------------------------------
def decode_prepare(k_begin, seq_len, kv_rows, seqused):
    for t, nm in ((k_begin, "k_begin"), (seq_len, "seq_len"), (kv_rows, "kv_rows"), (seqused, "seqused")):
        _req(t, torch.int32, nm)
    assert k_begin.numel() >= seq_len.numel() + 1 and kv_rows.numel() >= seq_len.numel() <= seqused.numel()
    rc = _cabi.lib().bagel_decode_prepare(_ptr(k_begin), _ptr(seq_len), _ptr(kv_rows), _ptr(seqused), seq_len.numel(), _stream())
    _cabi.check(rc, "bagel_decode_prepare")


def argmax_rows(logits: torch.Tensor, tokens: torch.Tensor, tokens32: Optional[torch.Tensor] = None):
    _req(logits, torch.bfloat16, "logits"); _req(tokens, torch.int64, "tokens")
    B, V = logits.shape
    rc = _cabi.lib().bagel_argmax_rows_bf16(_ptr(logits), logits.stride(0), B, V, _ptr(tokens), _ptr(tokens32), _stream())
    _cabi.check(rc, "bagel_argmax_rows_bf16")


def decode_advance(seq_len, pos, tokens, history, step_dev):
    _req(seq_len, torch.int32, "seq_len"); _req(pos, torch.int64, "pos"); _req(tokens, torch.int64, "tokens")
    _req(history, torch.int64, "history"); _req(step_dev, torch.int32, "step_dev")
    assert pos.numel() == seq_len.numel() == tokens.numel() and history.is_contiguous() and history.shape[-1] == seq_len.numel()
    rc = _cabi.lib().bagel_decode_advance(_ptr(seq_len), _ptr(pos), _ptr(tokens), _ptr(history), _ptr(step_dev),
                                          seq_len.numel(), _stream())
    _cabi.check(rc, "bagel_decode_advance")


def sample_rows(logits: torch.Tensor, temperature: float, keys: torch.Tensor, step_dev: torch.Tensor,
                tokens: torch.Tensor, tokens32: Optional[torch.Tensor] = None):
    """tokens[b] = a draw from softmax(logits[b] / temperature) (Gumbel-max over Philox4x32-10 uniforms keyed by
    keys[b] = seed | request_id << 32, counter = (step_dev[0], j / 4)); see include/bagel_b200.h."""
    _req(logits, torch.bfloat16, "logits"); _req(keys, torch.int64, "keys"); _req(step_dev, torch.int32, "step_dev")
    _req(tokens, torch.int64, "tokens")
    _opt(tokens32, torch.int32, "tokens32")
    B, V = logits.shape
    assert keys.numel() == tokens.numel() == B and (tokens32 is None or tokens32.numel() == B)
    rc = _cabi.lib().bagel_sample_rows_bf16(_ptr(logits), logits.stride(0), B, V, float(temperature), _ptr(keys),
                                            _ptr(step_dev), _ptr(tokens), _ptr(tokens32), _stream())
    _cabi.check(rc, "bagel_sample_rows_bf16")


def decode_advance_stop(seq_len, pos, tokens, tokens32, next_tokens, history, step_dev, finished, unfinished,
                        end_token_id: Optional[int], pad: int):
    """Per-request stopping of a batched decode step (history [max_length, B]); see include/bagel_b200.h."""
    for t, dt, nm in ((seq_len, torch.int32, "seq_len"), (pos, torch.int64, "pos"), (tokens, torch.int64, "tokens"),
                      (tokens32, torch.int32, "tokens32"), (next_tokens, torch.int64, "next_tokens"),
                      (history, torch.int64, "history"), (step_dev, torch.int32, "step_dev"),
                      (finished, torch.int32, "finished"), (unfinished, torch.int32, "unfinished")):
        _req(t, dt, nm)
    B = seq_len.numel()
    assert pos.numel() == tokens.numel() == tokens32.numel() == next_tokens.numel() == finished.numel() == B
    assert history.dim() == 2 and history.is_contiguous() and history.shape[1] == B
    rc = _cabi.lib().bagel_decode_advance_stop(_ptr(seq_len), _ptr(pos), _ptr(tokens), _ptr(tokens32), _ptr(next_tokens),
                                               _ptr(history), _ptr(step_dev), _ptr(finished), _ptr(unfinished),
                                               -1 if end_token_id is None else int(end_token_id), history.shape[0],
                                               int(pad), B, _stream())
    _cabi.check(rc, "bagel_decode_advance_stop")


def taylor_update(feature: torch.Tensor, factors: torch.Tensor, n_deriv: int, dist: int, rows: Optional[int] = None):
    """TaylorSeer derivative_approximation (cache_utils/taylorseer.py:12-32) on factor planes [orders, cap_rows, H]
    (in place): plane 0 <- feature, plane i+1 <- bf16(bf16(plane_i_new - plane_i_old) / dist) for i < n_deriv."""
    _req(feature, torch.bfloat16, "feature"); _req(factors, torch.bfloat16, "factors")
    assert factors.dim() == 3 and factors.stride(2) == 1 and factors.stride(1) == factors.shape[2] and feature.stride(1) == 1
    M = feature.shape[0] if rows is None else int(rows)
    H = feature.shape[1]
    assert factors.shape[2] == H and factors.shape[1] >= M and factors.shape[0] >= n_deriv + 1
    rc = _cabi.lib().bagel_taylor_update_bf16(_ptr(feature), feature.stride(0), _ptr(factors), factors.stride(0),
                                              int(n_deriv), int(dist), M, H, _stream())
    _cabi.check(rc, "bagel_taylor_update_bf16")


def taylor_eval(factors: torch.Tensor, n_factors: int, x: int, out: torch.Tensor, rows: Optional[int] = None):
    """TaylorSeer taylor_formula (cache_utils/taylorseer.py:34-47): out = sum_i bf16(bf16(f_i / i!) * x^i)."""
    _req(factors, torch.bfloat16, "factors"); _req(out, torch.bfloat16, "out")
    assert factors.dim() == 3 and factors.stride(2) == 1 and factors.stride(1) == factors.shape[2] and out.stride(1) == 1
    M = out.shape[0] if rows is None else int(rows)
    H = out.shape[1]
    assert factors.shape[2] == H and factors.shape[1] >= M and 1 <= n_factors <= factors.shape[0]
    rc = _cabi.lib().bagel_taylor_eval_bf16(_ptr(factors), factors.stride(0), int(n_factors), int(x), _ptr(out),
                                            out.stride(0), M, H, _stream())
    _cabi.check(rc, "bagel_taylor_eval_bf16")
    return out


def siglip_rope2d(x: torch.Tensor, heads: int, head_stride: int, head_dim: int, pos_ids: torch.Tensor, cos_h, sin_h, cos_w,
                  sin_w) -> None:
    """In-place 2-D RoPE on `heads` consecutive heads of every row of x [n, >= heads*head_stride] (SigLIP rope=True)."""
    _req(x, torch.bfloat16, "x"); _req(pos_ids, torch.int64, "pos_ids")
    for t, nm in ((cos_h, "cos_h"), (sin_h, "sin_h"), (cos_w, "cos_w"), (sin_w, "sin_w")):
        _req(t, torch.float32, nm)
        assert t.is_contiguous() and t.shape[-1] == head_dim // 2
    n = x.shape[0]
    assert x.shape[1] >= heads * head_stride and pos_ids.numel() >= n
    rc = _cabi.lib().bagel_siglip_rope2d_bf16(_ptr(x), x.stride(0), n, heads, head_stride, head_dim, _ptr(pos_ids), _ptr(cos_h),
                                              _ptr(sin_h), _ptr(cos_w), _ptr(sin_w), _stream())
    _cabi.check(rc, "bagel_siglip_rope2d_bf16")


def rmsnorm_f32(x: torch.Tensor, w0: torch.Tensor, w1: Optional[torch.Tensor] = None, expert: Optional[torch.Tensor] = None,
                eps: float = 1e-6, out: Optional[torch.Tensor] = None, out_dtype=torch.bfloat16) -> torch.Tensor:
    """dtype mode B: fp32 hidden stream, fp32 norm weights; bf16 out (the next Linear's input) or fp32 out."""
    _req(x, torch.float32, "x"); _req(w0, torch.float32, "w0"); _opt(w1, torch.float32, "w1"); _opt(expert, torch.uint8, "expert")
    N, H = x.shape
    if out is None:
        out = torch.empty((N, H), dtype=out_dtype, device=x.device)
    assert out.dtype in (torch.bfloat16, torch.float32) and out.shape[0] >= N and out.shape[1] == H and out.stride(1) == 1
    rc = _cabi.lib().bagel_rmsnorm_f32(_ptr(x), x.stride(0), _ptr(w0), _ptr(w1), _ptr(expert), _ptr(out), out.stride(0),
                                       int(out.dtype == torch.float32), N, H, float(eps), _stream())
    _cabi.check(rc, "bagel_rmsnorm_f32")
    return out


def latent_embed_add_f32(proj, t_emb, pos_table, pos_ids, seq, dst_rows):
    """dtype mode B: seq32[dst_rows[i]] = fp32(bf16(proj[i] + t_emb) + pos_table32[pos_ids[i]])."""
    M, H = proj.shape
    _req(proj, torch.bfloat16, "proj"); _opt(t_emb, torch.bfloat16, "t_emb"); _req(pos_table, torch.float32, "pos_table")
    _req(pos_ids, torch.int64, "pos_ids"); _req(seq, torch.float32, "seq"); _opt(dst_rows, torch.int32, "dst_rows")
    assert pos_table.shape[-1] == H and seq.shape[-1] >= H and pos_ids.numel() >= M
    assert (dst_rows.numel() >= M) if dst_rows is not None else (seq.shape[0] >= M)
    rc = _cabi.lib().bagel_latent_embed_add_f32(_ptr(proj), proj.stride(0), _ptr(t_emb), _ptr(pos_table), pos_table.stride(0),
                                                _ptr(pos_ids), _ptr(seq), seq.stride(0), _ptr(dst_rows), M, H, _stream())
    _cabi.check(rc, "bagel_latent_embed_add_f32")


def copy_rows_f32(src: torch.Tensor, dst: torch.Tensor, src_rows=None, dst_rows=None, M: Optional[int] = None):
    """Row gather/scatter of fp32 rows through the bf16 copy kernel (a pure byte copy: each fp32 row is 2H bf16 lanes)."""
    _req(src, torch.float32, "src"); _req(dst, torch.float32, "dst")
    return copy_rows(src.view(torch.bfloat16), dst.view(torch.bfloat16), src_rows, dst_rows, M)


# ---------------------------------------------------------------------------------------------------------------------
# device-side image preprocessing (uint8 HWC images)
# ---------------------------------------------------------------------------------------------------------------------
def image_resize_bicubic_u8(src: torch.Tensor, Ho: int, Wo: int, taps_h, taps_v) -> torch.Tensor:
    """Pillow-exact 8-bit bicubic resize of a uint8 [Hi, Wi, 3] CUDA image. taps_* = (kk int32 [out, ksize], bounds int32
    [out, 2], ksize) from bagel_b200.transforms.pil_bicubic_coeffs, or None for an axis whose size does not change."""
    _req(src, torch.uint8, "src")
    assert src.dim() == 3 and src.shape[2] == 3 and src.is_contiguous()
    Hi, Wi = int(src.shape[0]), int(src.shape[1])
    assert (taps_h is not None) == (Wo != Wi) and (taps_v is not None) == (Ho != Hi)
    dst = torch.empty((Ho, Wo, 3), dtype=torch.uint8, device=src.device)
    tmp = torch.empty((Hi, Wo, 3), dtype=torch.uint8, device=src.device) if (taps_h is not None and taps_v is not None) else None
    kh, bh, ksh = taps_h if taps_h is not None else (None, None, 0)
    kv, bv, ksv = taps_v if taps_v is not None else (None, None, 0)
    for t, n_out in ((kh, Wo), (kv, Ho)):
        if t is not None:
            _req(t, torch.int32, "taps"); assert t.is_contiguous() and t.shape[0] == n_out
    rc = _cabi.lib().bagel_image_resize_bicubic_u8(_ptr(src), Hi, Wi, _ptr(dst), Ho, Wo, _ptr(tmp), _ptr(kh), _ptr(bh), int(ksh),
                                                   _ptr(kv), _ptr(bv), int(ksv), _stream())
    _cabi.check(rc, "bagel_image_resize_bicubic_u8")
    return dst


def image_normalize_u8(src: torch.Tensor, mean, std, patch: int = 0) -> torch.Tensor:
    """uint8 [H, W, 3] -> fp32 ((u8/255) - mean) / std: planar [3, H, W] (patch = 0) or patch rows [(H/p)(W/p), p*p*3]."""
    _req(src, torch.uint8, "src")
    assert src.dim() == 3 and src.shape[2] == 3 and src.is_contiguous()
    H, W = int(src.shape[0]), int(src.shape[1])
    if patch:
        out = torch.empty(((H // patch) * (W // patch), patch * patch * 3), dtype=torch.float32, device=src.device)
        ld = out.stride(0)
    else:
        out = torch.empty((3, H, W), dtype=torch.float32, device=src.device)
        ld = 0
    rc = _cabi.lib().bagel_image_normalize_u8(_ptr(src), H, W, float(mean[0]), float(mean[1]), float(mean[2]), float(std[0]),
                                              float(std[1]), float(std[2]), _ptr(out), ld, int(patch), _stream())
    _cabi.check(rc, "bagel_image_normalize_u8")
    return out
