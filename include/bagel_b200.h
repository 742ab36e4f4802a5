/* bagel_b200 — C ABI of the H100-native (sm_90a) kernels behind BAGEL's inference forward path.
 *
 * The reference (ByteDance-Seed/Bagel) is pure Python; the only native seam it has is
 * `flash_attn_varlen_func` (modeling/bagel/qwen2_navit.py:361,579; modeling/bagel/siglip_navit.py:232).
 * Every other GPU op is reached through torch (nn.Linear -> cuBLASLt, ATen elementwise, cuDNN conv).
 * This header is the boundary a maintainer would bind with ctypes (see INTEGRATION.md): plain pointers
 * and sizes, no torch types. Conventions for every entry point:
 *
 *   - all pointers are DEVICE pointers unless a parameter is documented as host;
 *   - the caller owns every buffer (inputs, outputs, workspaces); the library never allocates device memory;
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); no internal synchronisation, so calls
 *     are CUDA-graph capturable;
 *   - return value 0 on success, a negative BAGEL_ERR_* otherwise; `bagel_last_error()` gives the message
 *     (thread-local);
 *   - bf16 tensors are row-major with an explicit leading dimension in ELEMENTS.
 */
#ifndef BAGEL_B200_H_
#define BAGEL_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BAGEL_OK 0
#define BAGEL_ERR_SHAPE (-1)
#define BAGEL_ERR_ALIGN (-2)
#define BAGEL_ERR_ARCH (-3)
#define BAGEL_ERR_CUDA (-4)
#define BAGEL_ERR_ARG (-5)

const char* bagel_last_error(void);
/* ABI version of this header; bump on any signature change. */
int bagel_abi_version(void);
/* Number of kernels launched by this library in this process (monotonic; used by bench.py's gpu_launches). */
long long bagel_launch_count(void);

/* GEMM epilogues (bagel_gemm_bf16 `epilogue`). */
#define BAGEL_EPI_BIAS 0   /* C = bf16(acc + bias)                                   nn.Linear               */
#define BAGEL_EPI_RESID 1  /* C = bf16(resid + bf16(acc + bias))                     Linear + residual add   */
#define BAGEL_EPI_SWIGLU 2 /* C[:,j] = bf16(bf16(silu(bf16 g_j)) * bf16 u_j)         Qwen2MLP gate/up/act    */
#define BAGEL_EPI_GELU 3   /* C = bf16(gelu_tanh(bf16(acc + bias)))                  SiglipMLP / connector   */
#define BAGEL_EPI_SILU 4   /* C = bf16(silu(bf16(acc + bias)))                       TimestepEmbedder.mlp[0:2] */
#define BAGEL_EPI_F32 5    /* C (fp32 [M, ldc]) = acc + bias                         attention logits, VAE mid block */
#define BAGEL_EPI_RESID_F32 7 /* C (fp32) = resid (fp32 [*, ldr]) + bf16(acc + bias)    fp32 residual stream: dtype mode B
                              * (fp32 master weights under autocast, eval/gen/gen_images_mp.py:159-175, :73)            */

/* C[M,N] = epilogue(A[M,K] @ W[N,K]^T), bf16 in / fp32 accumulate (wgmma) / bf16 out.
 * Replaces nn.Linear at modeling/bagel/qwen2_navit.py:515-517,529-536 (q/k/v_proj{,_moe_gen}),
 * :589-594 (o_proj{,_moe_gen}), modeling/qwen2/modeling_qwen2.py:200-201 (gate/up/down_proj),
 * modeling/bagel/bagel.py:803,832 (vae2llm, llm2vae), modeling/bagel/modeling_utils.py:84-110,120-124.
 *   W        nn.Linear weight layout [N, K]. For BAGEL_EPI_SWIGLU, W is [2*I, K] with gate/up rows
 *            interleaved in blocks of 128 (rows 256t..256t+127 = gate rows 128t.., next 128 = up rows) and
 *            C is [M, I].
 *   bias     [N] bf16 or NULL.   resid  [*, ldr] bf16 (BAGEL_EPI_RESID only).
 *   row_map  optional int32[M]: A-row r is written to C row row_map[r] (and reads resid row row_map[r]);
 *            used to scatter the und-expert rows of a MoT layer back into the packed sequence.
 * K, N, lda, ldw, ldc, ldr must be multiples of 8; pointers 16-byte aligned.
 * M <= 64 (token-by-token decode, und-expert rows) takes a weight-streaming path: swapped operands, split-K over a
 * thread-block cluster, launched with programmatic stream serialization — its W tiles may be prefetched while the
 * kernel in front of it on `stream` is still running (A, bias, resid and C are only touched after that kernel has
 * completed). W must therefore not be written by the immediately preceding kernel; BAGEL_PDL=0 in the environment
 * turns the early launch off, BAGEL_GEMM_SKINNY=0 the whole path. */
int bagel_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M,
                    int N, int K, const void* bias, const void* resid, long long ldr, const int* row_map,
                    int epilogue, void* stream);

/* Block-scaled FP8 (float8_e4m3fn) quantiser, the opt-in FP8 path of the generation expert's MLP.
 * X bf16 [M, K] -> Q e4m3 [M, K] (one byte per value, leading dimension ldq in bytes) + fp32 scales. A group is
 * 1 x 128 values along K (block_rows = 1, activations) or 128 x 128 (block_rows = 128, weights). Each group's scale s is
 * the smallest power of two with amax <= 448 s, at least 2^-126, and 1 for an all-zero group; Q = e4m3(X / s), round to
 * nearest even. s is a power of two, so X / s is exact and Q * s is exactly a bf16 value.
 * Scale layouts:
 *   block_rows = 1    K-block major: scales[kb * lds + m] for row m and columns [128 kb, 128 kb + 128); lds >= M.
 *   block_rows = 128  scales[(m / 128) * lds + kb]; lds >= K / 128.
 * K % 128 == 0, ldx % 8 == 0, ldq % 16 == 0, X and Q 16-byte aligned; ldx, ldq >= K (BAGEL_ERR_ARG otherwise). */
int bagel_quantize_fp8_bf16(const void* X, long long ldx, void* Q, long long ldq, float* scales, long long lds, int M,
                            int K, int block_rows, void* stream);

/* C = epilogue(dequant(A) @ dequant(W)^T) with block-scaled e4m3 operands (see bagel_quantize_fp8_bf16):
 *   y[m, n] = sum_kb a_scales[kb * ld_as + m] * w_scales[(n / 64) * (K / 128) + kb] * (sum_{k in kb} A[m, k] W[n, k]),
 * each 128-wide K block's tensor-core sum scaled and added into a separate fp32 accumulator, then the bf16 epilogue:
 *   BAGEL_EPI_SWIGLU  W [2*I, K] with gate/up rows interleaved in blocks of 64 (rows 128t..128t+63 = gate rows 64t..,
 *                     next 64 = up rows 64t..); C [M, I] = bf16(bf16(silu(bf16 g)) * bf16 u).
 *   BAGEL_EPI_RESID   C [M, N] = bf16(resid + bf16(y)), resid [*, ldr] bf16.
 * A [M, K] e4m3 (lda bytes), a_scales as the block_rows = 1 quantiser writes them (ld_as >= M); W [N, K] e4m3 (ldw
 * bytes); w_scales fp32 [N / 64, K / 128] row-major: one scale per 64-row half of a 128-row tile and K block (a weight
 * quantised in 128 x 128 blocks repeats each block's scale for its two halves).
 * K % 128 == 0 and N % 128 == 0 (BAGEL_ERR_SHAPE); lda, ldw % 16 == 0, ldc, ldr % 8 == 0, A, W, C, resid 16-byte
 * aligned (BAGEL_ERR_ALIGN); lda, ldw >= K, ldc >= the output width (I or N), ldr >= N, and any other epilogue are
 * BAGEL_ERR_ARG. No bias, no row_map. */
int bagel_gemm_fp8(const void* A, long long lda, const float* a_scales, long long ld_as, const void* W, long long ldw,
                   const float* w_scales, void* C, long long ldc, int M, int N, int K, const void* resid, long long ldr,
                   int epilogue, void* stream);

/* QKV projection with the whole pre-attention tail fused into the GEMM epilogue (head_dim 128 only):
 *   [q|k|v] = A W^T + bias; per-head RMSNorm of q and k with expert-routed weights; RoPE; bf16 cast; q -> q_out,
 *   k / v -> merged KV buffers at row kv_rows[r]. One launch for bagel_gemm_bf16 + bagel_qk_norm_rope, without the
 *   [M, (Hq+2Hk)*128] round trip through HBM (north_star: "RMSNorm+RoPE fused into the QKV projection epilogue";
 *   reference modeling/bagel/qwen2_navit.py:515-557, 559-574). Arguments as in those two entry points; all per-row
 *   tables (expert, cos_t, sin_t, kv_rows) are indexed by the OUTPUT row (row_map[r] when row_map is given). */
int bagel_gemm_qkv_norm_rope(const void* A, long long lda, const void* W, long long ldw, const void* bias, int M, int K,
                             const int* row_map, const void* q_w0, const void* k_w0, const void* q_w1, const void* k_w1,
                             const uint8_t* expert, const float* cos_t, const float* sin_t, void* q_out, long long ld_q,
                             void* k_out, void* v_out, long long ld_kv, const int* kv_rows, int Hq, int Hk, float eps,
                             int fp32_flow, void* stream);

/* Packed variable-length attention forward; same contract as flash_attn_varlen_func as the reference calls it
 * (modeling/bagel/qwen2_navit.py:361-370, 579-588; modeling/bagel/siglip_navit.py:232-241):
 *   q [total_q, Hq, D], k/v [total_k, Hk, D], out [total_q, Hq, D] bf16 (row strides ld_* in elements);
 *   cu_seqlens_q / cu_seqlens_k int32 [batch+1] DEVICE arrays; Hq % Hk == 0 (GQA); D in {64, 128};
 *   causal != 0: bottom-right aligned mask (query i sees keys <= i + Lk - Lq), as flash-attn >= 2.1;
 *   softmax in fp32, scale = softmax_scale (reference default D^-0.5). max_seqlen_q sizes the grid (host int,
 *   exactly what the reference passes); max_seqlen_k (host int, <= 0 if unknown) only tunes the key split of the
 *   single-query path: when max_seqlen_q == 1 (text decode, D = 128) a split-KV kernel streams the cache instead.
 *   seqused_k (optional int32[batch], device): number of keys in use per sample when the K/V rows of sample b start at
 *   cu_seqlens_k[b] but the buffer has spare capacity (append-in-place decode; same meaning as flash-attn's seqused_k).
 *   The spare rows must hold FINITE values (e.g. a zero-initialised slab): whole 128-key blocks are fetched by TMA and the
 *   masked probabilities (exactly 0) are multiplied with them. */
int bagel_attn_varlen_fwd(const void* q, const void* k, const void* v, void* out, const int* cu_seqlens_q,
                          const int* cu_seqlens_k, int total_q, int total_k, int batch, int num_heads_q,
                          int num_heads_k, int head_dim, int max_seqlen_q, int max_seqlen_k, int causal,
                          float softmax_scale, long long ld_q, long long ld_k, long long ld_v, long long ld_out,
                          const int* seqused_k, void* stream);

/* y = bf16(w_e * bf16(x * rsqrt(mean(x^2) + eps))), e = expert[row] ? w1 : w0 (expert / w1 may be NULL).
 * Qwen2RMSNorm (modeling/qwen2/modeling_qwen2.py:54-59) with the MoT row routing of
 * modeling/bagel/qwen2_navit.py:781-787, 808-815, 1075-1082. x, y bf16 [N, H]. */
int bagel_rmsnorm_bf16(const void* x, long long ldx, const void* w0, const void* w1, const uint8_t* expert, void* y,
                       long long ldy, int N, int H, float eps, void* stream);

/* y = bf16((x - mean) * rsqrt(var + eps) * w + b): nn.LayerNorm of the SigLIP tower
 * (modeling/bagel/siglip_navit.py:269-271, 283, 294, 346, 370). x, y bf16 [N, H]; w, b bf16 [H]. */
int bagel_layernorm_bf16(const void* x, long long ldx, const void* w, const void* b, void* y, long long ldy, int N,
                         int H, float eps, void* stream);

/* cos/sin[N, half] = cos/sin(float(pos[r]) * inv_freq[c]), optionally rounded to bf16 values
 * (Qwen2RotaryEmbedding.forward, modeling/qwen2/modeling_qwen2.py:130-150; halves are duplicated there). */
int bagel_rope_table(const long long* pos, const float* inv_freq, float* cos_t, float* sin_t, int N, int half,
                     int round_bf16, void* stream);

/* Per-head RMSNorm(q,k) + RoPE + bf16 cast + placement of K/V rows into the merged KV buffer
 * (PackedAttentionMoT.forward_inference, modeling/bagel/qwen2_navit.py:518-519, 542-557, 559-574).
 *   qkv [N, (Hq+2Hk)*D] bf16; q_out [N, Hq*D]; k_out / v_out [rows, Hk*D] written at row kv_rows[r] (NULL: r);
 *   *_w0 und-expert norm weights [D], *_w1 gen-expert (NULL when not MoT), expert[N] routing flags (may be NULL);
 *   fp32_flow: rounding-point flow of the reference (SURVEY.md 8a dtype table):
 *     0 = bf16 weights, und / dense attention (bf16 at every op, bf16-rounded cos/sin);
 *     1 = bf16 weights, MoT gen branch (fp32 norm + RoPE, single bf16 cast);
 *     2 = fp32 master weights, und / dense (bf16(x*r) * w_fp32, fp32 RoPE with fp32 cos/sin);
 *     3 = fp32 master weights, MoT gen branch (everything fp32).
 *   flows 2 and 3 read q_w* / k_w* as FP32 [D] (bagel_gemm_qkv_norm_rope takes the same values). */
int bagel_qk_norm_rope(const void* qkv, long long ld_qkv, const void* q_w0, const void* k_w0, const void* q_w1,
                       const void* k_w1, const uint8_t* expert, const float* cos_t, const float* sin_t, void* q_out,
                       long long ld_q, void* k_out, void* v_out, long long ld_kv, const int* kv_rows, int N, int Hq,
                       int Hk, int D, float eps, int fp32_flow, void* stream);

/* dst[dst_rows[i]] = src[src_rows[i]] for i < M (either map may be NULL = identity); bf16 rows of H elements.
 * Token-embedding lookup (modeling/bagel/bagel.py:277, 796), modality gathers (qwen2_navit.py:526-548) and
 * cached-KV placement (qwen2_navit.py:565-569). */
int bagel_copy_rows_bf16(const void* src, long long lds, const int* src_rows, void* dst, long long ldd,
                         const int* dst_rows, int M, int H, void* stream);

/* seq[dst_rows[i]] = bf16(bf16(proj[i] + t_emb) + pos_table[pos_ids[i]])  (modeling/bagel/bagel.py:801-806);
 * t_emb NULL: seq = bf16(proj + pos_table[pos_ids]) (SigLIP patch embed + position embedding, siglip_navit.py:190-193;
 * connector output + vit_pos_embed, bagel.py:390-392). */
int bagel_latent_embed_add(const void* proj, long long ldp, const void* t_emb, const void* pos_table, long long ldt,
                           const long long* pos_ids, void* seq, long long lds, const int* dst_rows, int M, int H,
                           void* stream);

/* CFG combine + renorm + Euler update, x fp32 [M, C] in place (modeling/bagel/bagel.py:873-907, :746).
 *   v / v_text / v_img: bf16 llm2vae outputs of the main / text-dropped / image-dropped branches (row pitch ldv),
 *   latent token i lives at row rows[i] (NULL: i). v_text NULL or cfg_text_scale <= 1: plain x -= bf16(v*dt).
 *   renorm_type 0 "global" (needs norms_ws fp32[2]), 1 "channel", 2 "text_channel".
 *   dt_dev: optional device pointer to the step size; when non-NULL it overrides `dt` (the same captured CUDA graph
 *   can then be replayed for every step of a run). */
int bagel_cfg_euler_step(const void* v, const void* v_text, const void* v_img, long long ldv, const int* rows,
                         float* x, float* norms_ws, int M, int C, float cfg_text_scale, float cfg_img_scale,
                         float renorm_min, int renorm_type, float dt, const float* dt_dev, void* stream);

/* bagel_cfg_euler_step for a batch of independent requests (Bagel.generate_image_batch), x fp32 [M, C] in place.
 *   Latent row r belongs to request seg[r] in [0, R); the rows of one request are contiguous (one run of seg). Row r
 *   reads rows row_main[r], row_text[r], row_img[r] of the bf16 llm2vae output v (row pitch ldv); row_text / row_img
 *   are -1 when the request has no such branch.
 *   Per request q (device arrays of length R): cfg_text_scale[q], cfg_img_scale[q], renorm_min[q], renorm_type[q]
 *   (0 "global", 1 "channel", 2 "text_channel"; mixed in one launch) and cfg_on[q] for this step. Row r takes text CFG
 *   when cfg_on[q] != 0, row_text[r] >= 0 and cfg_text_scale[q] > 1, and image CFG inside it when also row_img[r] >= 0
 *   and cfg_img_scale[q] > 1; otherwise x -= bf16(v * dt). Every rounding point is that of bagel_cfg_euler_step with
 *   the request's parameters. "global" norms are summed over the request's own rows only, per row and then in a fixed
 *   order (no atomics): two launches give the same bits. The work per step is O(M + R).
 *   dt_dev: device pointer to the step size (required). workspace: 4-byte words [2 * M + 2 * R] of device memory
 *   (contents need no initialisation).
 *   No host reads, no allocations: capturable once for every step of a run. C <= 128. */
int bagel_cfg_euler_step_batch(const void* v, long long ldv, const int* seg, const int* row_main, const int* row_text,
                               const int* row_img, float* x, int M, int C, int R, const float* cfg_text_scale,
                               const float* cfg_img_scale, const float* renorm_min, const int* renorm_type,
                               const int* cfg_on, const float* dt_dev, float* workspace, void* stream);

/* y[i] = bf16(x[i]) — the autocast cast in front of vae2llm (modeling/bagel/bagel.py:803). */
int bagel_cast_f32_to_bf16(const float* x, void* y, long long n, void* stream);

/* 2-D convolution on NHWC bf16 activations as an im2col-free implicit GEMM on wgmma (FLUX VAE convs:
 * modeling/autoencoder.py:76-80 ResnetBlock, :102-108 Downsample (stride 2, pad right/bottom), :114-119 Upsample conv,
 * :43-48 AttnBlock 1x1, :139,170,221,248 conv_in/conv_out — cuDNN NCHW convolutions in the reference).
 *   x [B, Hi, Wi, Cin], w [Cout, ksize, ksize, Cin] (reference layout [Cout, Cin, kh, kw] permuted once at load),
 *   out [B, Ho, Wo, Cout] = bf16(resid + bf16(conv + bias)) (resid / bias may be NULL).
 *   ksize in {1, 3}; stride in {1, 2}; `pad` = zero padding on the left/top (right/bottom padding is implied by
 *   Ho, Wo: anything outside the input reads as zero). Cin %% 64 == 0, Cout %% 8 == 0 (pad channels / filters). */
int bagel_conv2d_nhwc_bf16(const void* x, int B, int Hi, int Wi, int Cin, const void* w, int Cout, int ksize, int stride,
                           int pad, const void* bias, const void* resid, void* out, int Ho, int Wo, void* stream);

/* GroupNorm(32 groups, affine) over NHWC bf16 [B, HW, C] + optional swish, fp32 statistics, deterministic two-stage
 * reduction (modeling/autoencoder.py:43, 75-89, 169, 190-191, 247, 269-270 with swish :34-35).
 * x, y bf16; w, b FP32 [C] (the reference keeps the VAE's parameters in fp32 and autocast runs group_norm in fp32);
 * workspace: bagel_groupnorm_workspace_bytes(B, 32) bytes of device memory. C in {128, 256, 512}. */
long long bagel_groupnorm_workspace_bytes(int B, int groups);
int bagel_groupnorm_nhwc_bf16(const void* x, const void* w, const void* b, void* y, void* workspace, int B,
                              long long HW, int C, int groups, float eps, int swish, void* stream);

/* y[b, 2h+i, 2w+j, :] = x[b, h, w, :] — nn.functional.interpolate(scale_factor=2, mode="nearest")
 * (modeling/autoencoder.py:117), NHWC bf16. */
int bagel_upsample2x_nhwc_bf16(const void* x, void* y, int B, int H, int W, int C, void* stream);

/* P[r, :] = bf16(softmax(S[r, :] * scale)), S fp32 — softmax of the single-head d=512 attention of the VAE mid
 * block (modeling/autoencoder.py:50-62, F.scaled_dot_product_attention). */
int bagel_softmax_rows_f32(const float* S, long long lds, void* P, long long ldp, int rows, int L, float scale,
                           void* stream);

/* y[c, r] = x[r, c], bf16 (V^T for the P*V GEMM of the VAE mid attention). */
int bagel_transpose_bf16(const void* x, long long ldx, void* y, long long ldy, int R, int C, void* stream);

/* Text decode helpers (modeling/bagel/bagel.py:930-1000, one token per sample per step, all state on the device so a
 * whole decode step is one replayable CUDA graph):
 *   bagel_decode_prepare: kv_rows[b] = k_begin[b] + seq_len[b] (slot of the new token), seqused[b] = seq_len[b] + 1;
 *   bagel_argmax_rows_bf16: tokens[b] = argmax_v logits[b, v] (first maximum, like torch.argmax), int64 out, and the
 *     same ids as int32 (row indices for the next embedding gather);
 *   bagel_decode_advance: seq_len[b] += 1; pos[b] += 1; history[step_dev[0], b] = tokens[b]; step_dev[0] += 1. */
int bagel_decode_prepare(const int* k_begin, const int* seq_len, int* kv_rows, int* seqused, int B, void* stream);
int bagel_argmax_rows_bf16(const void* logits, long long ld, int B, int V, long long* tokens, int* tokens32, void* stream);
int bagel_decode_advance(int* seq_len, long long* pos, const long long* tokens, long long* history, int* step_dev, int B,
                         void* stream);

/* Batched decode of independent requests (Bagel.generate_text_batch); state in device memory, graph-replayable:
 *   bagel_sample_rows_bf16: tokens[b] = a draw from softmax(logits[b, :] / temperature), by Gumbel-max:
 *     argmax_j (logit_j / T - log(-log u_j)), ties to the lowest index. u_j comes from Philox4x32-10 with key
 *     (low, high 32 bits of keys[b]) = (seed, request id) and counter (step_dev[0], j / 4, 0, 0), word j % 4; the 23 top
 *     bits x of that word give u = (x + 0.5) * 2^-23, exact in fp32 and strictly inside (0, 1). A row's draw depends
 *     only on its logits, key and the step.
 *     temperature finite and > 0 (greedy decoding is bagel_argmax_rows_bf16); tokens32 may be NULL.
 *   bagel_decode_advance_stop: per request b, with step = step_dev[0] and history [max_length, B]:
 *     finished[b] != 0: history[step, b] = pad; nothing else changes (its token, seq_len and pos stay frozen);
 *     otherwise history[step, b] = tokens[b], then if next[b] == end_token_id or step + 1 == max_length, finished[b] = 1;
 *     else seq_len[b] += 1, pos[b] += 1, tokens[b] = tokens32[b] = next[b].
 *     Then unfinished[0] = number of requests not finished, step_dev[0] += 1. Rows of history at step >= max_length are
 *     not written. B <= 1024; end_token_id < 0 never matches. */
int bagel_sample_rows_bf16(const void* logits, long long ld, int B, int V, float temperature, const long long* keys,
                           const int* step_dev, long long* tokens, int* tokens32, void* stream);
int bagel_decode_advance_stop(int* seq_len, long long* pos, long long* tokens, int* tokens32, const long long* next,
                              long long* history, int* step_dev, int* finished, int* unfinished, long long end_token_id,
                              int max_length, long long pad, int B, void* stream);

/* TaylorSeer step cache (reference modeling/cache_utils/taylorseer.py, enabled by generate_image(enable_taylorseer=True),
 * modeling/bagel/bagel.py:678-684; decoder-layer hooks modeling/bagel/qwen2_navit.py:773-777, 824-829).
 * factors: bf16 planes [order][rows][H], plane_stride elements apart, of the last decoder layer's output.
 * update  = derivative_approximation (:12-32) on a fully computed step:
 *           new[0] = feature; new[i+1] = bf16(bf16(new[i] - old[i]) / dist) for i < n_deriv  (in place).
 * eval    = taylor_formula (:34-47) on a skipped step: out = sum_{i<n_factors} bf16(bf16(f_i / i!) * x^i), bf16 adds,
 *           x = steps since the last fully computed one. Bit-exact w.r.t. torch's bf16 elementwise semantics. */
int bagel_taylor_update_bf16(const void* feature, long long ldf, void* factors, long long plane_stride, int n_deriv,
                             int dist, int rows, int H, void* stream);
int bagel_taylor_eval_bf16(const void* factors, long long plane_stride, int n_factors, int x, void* out, long long ldo,
                           int rows, int H, void* stream);

/* SigLIP 2-D RoPE, in place on `heads` consecutive heads (head_stride elements apart, e.g. the q and k heads of a fused
 * QKV buffer) of every token row (modeling/bagel/siglip_navit.py:102-142 RotaryEmbedding2D, :224-230): the first half of
 * a head is rotated with the row table, the second half with the column table of the token's patch position:
 *   out = bf16( fp32(x) * cos[pos] + rotate_half(fp32(x)) * sin[pos] ),   tables fp32 [max_h*max_w, head_dim/2]. */
int bagel_siglip_rope2d_bf16(void* x, long long ld, int n_tokens, int heads, int head_stride, int head_dim,
                             const long long* pos_ids, const float* cos_h, const float* sin_h, const float* cos_w,
                             const float* sin_w, void* stream);

/* dtype mode B (fp32 master weights + autocast): RMSNorm of an FP32 hidden stream with FP32 weights,
 * y = w_e * (x * rsqrt(mean(x^2) + eps)) with both products rounded to fp32 (modeling/qwen2/modeling_qwen2.py:54-59);
 * out_f32 = 1 stores that fp32 value (the final norm handed back to the caller), 0 stores bf16(y) — the autocast cast
 * in front of the next nn.Linear. Routing by expert[row] as bagel_rmsnorm_bf16. */
int bagel_rmsnorm_f32(const float* x, long long ldx, const float* w0, const float* w1, const uint8_t* expert, void* y,
                      long long ldy, int out_f32, int N, int H, float eps, void* stream);

/* bagel_latent_embed_add for an fp32 hidden stream: seq32[dst_rows[i]] = fp32(bf16(proj[i] + t_emb) + pos_table32[pos_ids[i]])
 * (modeling/bagel/bagel.py:801-806 with fp32 parameters: the frozen sincos table and the packed sequence are fp32). */
int bagel_latent_embed_add_f32(const void* proj, long long ldp, const void* t_emb, const float* pos_table, long long ldt,
                               const long long* pos_ids, float* seq, long long lds, const int* dst_rows, int M, int H,
                               void* stream);

/* Device-side image preprocessing (the reference does this on the host: data/transforms.py:15-115 -> PIL, then
 * data/data_utils.py:43-50 patchify). BIT-EXACT w.r.t. Pillow's 8-bit bicubic resampler (antialiased, a = -0.5) and torch's
 * ToTensor + Normalize arithmetic.
 *   bagel_image_resize_bicubic_u8: src uint8 [Hi, Wi, 3] -> dst uint8 [Ho, Wo, 3]; horizontal pass then vertical pass,
 *     out = clip8((2^21 + sum_k in[xmin+k] * kk[k]) >> 22); kk_* int32 [out_size, ksize_*] fixed-point taps (2^22) and
 *     bounds_* int32 [out_size, 2] = (xmin, n) per output index, both computed by the host exactly as Pillow's
 *     precompute_coeffs / normalize_coeffs_8bpc (bagel_b200.transforms.pil_bicubic_coeffs); tmp uint8 [Hi, Wo, 3].
 *   bagel_image_normalize_u8: value = ((u8 / 255) - mean[c]) / std[c] in fp32 (three roundings, as torch);
 *     patch == 0: out fp32 planar [3, H, W];  patch > 0: out fp32 [(H/patch)*(W/patch), ld] patch rows in (row-in-patch,
 *     col-in-patch, channel) order — the `packed_vit_tokens` layout. */
int bagel_image_resize_bicubic_u8(const uint8_t* src, int Hi, int Wi, uint8_t* dst, int Ho, int Wo, uint8_t* tmp,
                                  const int* kk_h, const int* bounds_h, int ksize_h, const int* kk_v, const int* bounds_v,
                                  int ksize_v, void* stream);
int bagel_image_normalize_u8(const uint8_t* src, int H, int W, float mean0, float mean1, float mean2, float std0, float std1,
                             float std2, float* out, long long ld, int patch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BAGEL_B200_H_ */
