// Packed variable-length flash attention forward for sm_90a (wgmma + TMA + mbarrier).
//
// Drop-in for the reference's only native seam, flash_attn_varlen_func (FA2, mma.sync) as called at
// modeling/bagel/qwen2_navit.py:361-370, 579-588 and modeling/bagel/siglip_navit.py:232-241:
//   out[Sq,Hq,D] = softmax(q k^T * scale [+ bottom-right causal mask]) v   per packed sample, GQA by Hq % Hk == 0,
//   bf16 in / fp32 softmax + accumulation / bf16 out.
//
// One CTA per 128-row query tile of one (sample, head), swept over that sample's keys in blocks of 128:
//   warp 8           TMA producer (one elected lane): the Q tile, then K_j / V_j through a smem ring
//   warpgroups 0, 1  64 query rows each: S = Q K_j^T (wgmma, both K-major, fp32 in registers) -> online softmax in
//                    registers -> P (bf16) stays in registers as the A operand of O += P V_j (wgmma, V MN-major)
// The two MMA warpgroups run out of phase on their own: one is in its softmax while the other's wgmmas occupy the tensor
// cores.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "host_util.h"
#include "attn_decode.h"

namespace bagel {

constexpr int kAttnThreads = 2 * 128 + 32;   // two MMA warpgroups + the producer warp (<= 224 registers per thread)
constexpr int kAttnMmaWarps = 8;
constexpr int kBlockM = 128;  // query rows per CTA (64 per MMA warpgroup)
constexpr int kBlockN = 128;  // keys per block

struct AttnParams {
  __nv_bfloat16* out;
  long long ld_out;  // elements between consecutive rows of out (= Hq*D for packed layout)
  const int* cu_q;   // [B+1]
  const int* cu_k;   // [B+1]
  const int* seqused_k;  // optional [B]: keys in use per sample (<= cu_k[b+1]-cu_k[b]); KV buffers with spare capacity
  int Hq, Hk;
  int causal;
  float scale_log2;  // softmax_scale * log2(e)
  int poly;          // every 4th score pair of unmasked key blocks takes the FMA-pipe exp2 (BAGEL_ATTN_POLY)
};

template <int D>
struct AttnCfg {
  static constexpr int kTileBytes = kBlockM * D * 2;  // the Q tile / one K block / one V block
  static constexpr int kStages = (D == 128) ? 4 : 6;
  static constexpr int kSmemBytes = kTileBytes + kStages * kTileBytes + 1024 + 256;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 2^x on the FMA pipe for a PAIR of scores (no MUFU): round-to-nearest split x = n + f through the 1.5 * 2^23 magic add,
// degree-3 minimax polynomial of 2^f on [-0.5, 0.5] (max relative error 1.0e-4, 40x below the bf16 rounding of P), and n added
// to the exponent field with one integer add. Valid for x <= ~100; x below -126 (masked-out -inf included) clamps to
// 2^-126, NOT to 0 — so it is only used in unmasked key blocks. The MUFU unit (16 exp2 / clk / SM) is the softmax's
// bottleneck; every 4th score pair goes through this path instead.
__device__ __forceinline__ float2 ex2_poly2(float2 x) {
  const float2 magic = make_float2(12582912.0f, 12582912.0f);
  const float2 c1 = make_float2(0.69328292f, 0.69328292f), c2 = make_float2(0.24221068f, 0.24221068f),
               c3 = make_float2(0.05500873f, 0.05500873f);
  x.x = fmaxf(x.x, -126.0f);
  x.y = fmaxf(x.y, -126.0f);
  const float2 t = make_float2(x.x + magic.x, x.y + magic.y);     // integer part in the low mantissa bits
  const float2 n = make_float2(t.x - magic.x, t.y - magic.y);     // exact
  const float2 f = make_float2(x.x - n.x, x.y - n.y);             // in [-0.5, 0.5]
  float2 q = make_float2(fmaf(f.x, c3.x, c2.x), fmaf(f.y, c3.y, c2.y));
  q = make_float2(fmaf(q.x, f.x, c1.x), fmaf(q.y, f.y, c1.y));
  q = make_float2(fmaf(q.x, f.x, 1.0f), fmaf(q.y, f.y, 1.0f));
  float2 r;
  r.x = __int_as_float(__float_as_int(q.x) + (__float_as_int(t.x) << 23));
  r.y = __int_as_float(__float_as_int(q.y) + (__float_as_int(t.y) << 23));
  return r;
}

// grid (query tiles, Hq, batch)
template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_varlen_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  using Cfg = AttnCfg<D>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kTileBytes = Cfg::kTileBytes;
  constexpr int kAtoms = D / 64;               // 64-column (128 B) swizzle atoms per row
  constexpr int kAtomBytes = kBlockM * 128;    // one [128 rows x 64 cols] box

  // causal: the LAST query tiles sweep the most keys — start them first
  const int qt = p.causal ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q_beg = p.cu_q[b];
  const int Lq = p.cu_q[b + 1] - q_beg;
  const int q0 = qt * kBlockM;
  if (q0 >= Lq) return;   // uniform over the CTA
  const int hk = h / (p.Hq / p.Hk);
  const int k_beg = p.cu_k[b];
  const int Lk = p.seqused_k ? p.seqused_k[b] : (p.cu_k[b + 1] - k_beg);
  const int shift = Lk - Lq;   // bottom-right aligned causal: key kv visible to query qi iff kv <= qi + shift
  int kv_end = Lk;
  if (p.causal) kv_end = max(0, min(Lk, min(Lq, q0 + kBlockM) - 1 + shift + 1));
  const int nblk = (kv_end + kBlockN - 1) / kBlockN;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + kTileBytes;    // ring: K_0, V_0, K_1, V_1, ...
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_kv + kStages * kTileBytes);
  uint64_t* q_full = bars;                 // [1]
  uint64_t* kv_full = bars + 1;            // [kStages]
  uint64_t* kv_empty = kv_full + kStages;  // [kStages]  one arrive per MMA warp

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], kAttnMmaWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 2) {
    // =========================== TMA producer ===========================
    if (elect_one_lane() && nblk > 0) {
      mbar_expect_tx(q_full, kTileBytes);
      for (int a = 0; a < kAtoms; ++a)
        tma_load_2d(smem_q + a * kAtomBytes, &tmQ, q_full, h * D + a * 64, q_beg + q0, kEvictFirst);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nblk; ++j) {
        for (int kv = 0; kv < 2; ++kv) {  // K_j then V_j
          mbar_wait(&kv_empty[stage], phase ^ 1);
          mbar_expect_tx(&kv_full[stage], kTileBytes);
          const CUtensorMap* tm = kv == 0 ? &tmK : &tmV;
          for (int a = 0; a < kAtoms; ++a)
            tma_load_2d(smem_kv + stage * kTileBytes + a * kAtomBytes, tm, &kv_full[stage], hk * D + a * 64,
                        k_beg + j * kBlockN, kEvictLast);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // =========================== S = QK^T, online softmax, O += PV ===========================
    const int half = wg;                                       // query rows [64 half, 64 half + 64) of the tile
    const int cq = 2 * (lane & 3);                             // fragment column offset
    const int row0 = half * 64 + (warp & 3) * 16 + (lane >> 2); // fragment rows row0 and row0 + 8
    const int qi[2] = {q0 + row0, q0 + row0 + 8};              // query index within the sample
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    if (nblk > 0) {
      mbar_wait(q_full, 0);
      const uint32_t q_addr = smem_u32(smem_q) + half * 64 * 128;
      const int tile_q_lo = q0 + half * 64;
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nblk; ++j) {
        // ---- S = Q K_j^T: K-major operands, D = kAtoms atoms of 64 columns, 4 k16 steps (+32 B) per atom ----
        float s[kBlockN / 2];
        mbar_wait(&kv_full[stage], phase);
        {
          const uint32_t k_addr = smem_u32(smem_kv + stage * kTileBytes);
          wgmma_fence();
#pragma unroll
          for (int a = 0; a < kAtoms; ++a)
#pragma unroll
            for (int k = 0; k < 4; ++k)
              wgmma_ss<kBlockN>(s, gmma_desc_kmajor_sw128(q_addr + a * kAtomBytes) + 2 * k,
                                gmma_desc_kmajor_sw128(k_addr + a * kAtomBytes) + 2 * k, (a | k) != 0);
          wgmma_commit();
          wgmma_wait<0>();
          gmma_fence_operand(s);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[stage]);
        if (++stage == kStages) { stage = 0; phase ^= 1; }

        // ---- online softmax over this thread's two rows (a row's 128 scores are spread over a lane quad) ----
        const int kv0 = j * kBlockN;
        const bool need_mask = (kv0 + kBlockN > Lk) || (p.causal && (kv0 + kBlockN - 1 > tile_q_lo + shift));
        if (need_mask) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int lim = p.causal ? min(Lk - 1, qi[r] + shift) : (Lk - 1);   // last visible key of this row
#pragma unroll
            for (int c = 0; c < kBlockN / 8; ++c)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (kv0 + 8 * c + cq + e > lim) s[4 * c + 2 * r + e] = -INFINITY;
          }
        }
        float neg_ms[2], alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float mx = -INFINITY;
#pragma unroll
          for (int c = 0; c < kBlockN / 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * r], s[4 * c + 2 * r + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m[r], mx);
          const float m_use = (m_new == -INFINITY) ? 0.f : m_new;   // a row with no visible key yet: p = 0
          alpha[r] = ex2((m[r] - m_use) * p.scale_log2);            // m = -inf -> 0
          m[r] = m_new;
          neg_ms[r] = -m_use * p.scale_log2;
        }
        // P = 2^(s scale - m scale) as bf16 A fragments of the P*V wgmma: keys 16kk .. 16kk + 15 are column blocks
        // 2kk (a0: row0, a1: row0 + 8) and 2kk + 1 (a2, a3)
        const bool poly = p.poly && !need_mask;
        float rs[2] = {0.f, 0.f};
        uint32_t pa[kBlockN / 16][4];
#pragma unroll
        for (int c = 0; c < kBlockN / 8; ++c) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const float2 x = make_float2(fmaf(s[4 * c + 2 * r], p.scale_log2, neg_ms[r]),
                                         fmaf(s[4 * c + 2 * r + 1], p.scale_log2, neg_ms[r]));
            const float2 e = (poly && (c & 3) == 3) ? ex2_poly2(x) : make_float2(ex2(x.x), ex2(x.y));
            rs[r] += e.x + e.y;
            pa[c >> 1][(c & 1) * 2 + r] = pack_bf16x2(e.x, e.y);
          }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          l[r] = l[r] * alpha[r] + rs[r];
#pragma unroll
          for (int c = 0; c < D / 8; ++c) {
            o[4 * c + 2 * r] *= alpha[r];
            o[4 * c + 2 * r + 1] *= alpha[r];
          }
        }

        // ---- O += P V_j: B = V block, MN-major (64-column halves kAtomBytes apart), 16 keys = 2048 B per k16 step ----
        mbar_wait(&kv_full[stage], phase);
        {
          const uint32_t v_addr = smem_u32(smem_kv + stage * kTileBytes);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kBlockN / 16; ++kk)
            wgmma_rs<D, 1>(o, pa[kk], gmma_desc_mnmajor_sw128(v_addr + kk * 2048, kAtomBytes), 1u);
          wgmma_commit();
          wgmma_wait<0>();
          gmma_fence_operand(o);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[stage]);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }

    // ---- epilogue: O / l -> bf16 -> global; rows that never saw a visible key produce 0, as flash-attn does ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float lr = l[r];
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      const float inv_l = (lr > 0.f && m[r] != -INFINITY) ? (1.f / lr) : 0.f;
      if (qi[r] >= Lq) continue;
      __nv_bfloat16* orow = p.out + (long long)(q_beg + qi[r]) * p.ld_out + h * D;
#pragma unroll
      for (int c = 0; c < D / 8; ++c)
        *reinterpret_cast<uint32_t*>(orow + 8 * c + cq) = pack_bf16x2(o[4 * c + 2 * r] * inv_l, o[4 * c + 2 * r + 1] * inv_l);
    }
  }
}

template <int D>
static int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p, int B,
                       int max_seqlen_q, cudaStream_t stream) {
  using Cfg = AttnCfg<D>;
  auto kern = attn_varlen_kernel<D>;
  static bool attr_done = false;
  if (!attr_done) {
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_done = true;
  }
  const int qtiles = (max_seqlen_q + kBlockM - 1) / kBlockM;
  if (p.Hq > 65535 || B > 65535) return set_error(BAGEL_ERR_SHAPE, "bagel_attn_varlen_fwd: too many heads / samples");
  kern<<<dim3(qtiles, p.Hq, B), kAttnThreads, Cfg::kSmemBytes, stream>>>(tmQ, tmK, tmV, p);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace bagel

using namespace bagel;

extern "C" int bagel_attn_varlen_fwd(const void* q, const void* k, const void* v, void* out, const int* cu_seqlens_q,
                                     const int* cu_seqlens_k, int total_q, int total_k, int batch, int num_heads_q,
                                     int num_heads_k, int head_dim, int max_seqlen_q, int max_seqlen_k, int causal,
                                     float softmax_scale, long long ld_q, long long ld_k, long long ld_v,
                                     long long ld_out, const int* seqused_k, void* stream) {
  if (head_dim != 64 && head_dim != 128)
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_varlen_fwd: head_dim must be 64 or 128 (got %d)", head_dim);
  if (num_heads_k <= 0 || num_heads_q % num_heads_k)
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_varlen_fwd: num_heads_q %% num_heads_k != 0");
  if (batch <= 0 || total_q < 0 || total_k < 0) return set_error(BAGEL_ERR_SHAPE, "bagel_attn_varlen_fwd: bad sizes");
  if ((ld_q % 8) || (ld_k % 8) || (ld_v % 8) || (ld_out % 8) || (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15))
    return set_error(BAGEL_ERR_ALIGN, "bagel_attn_varlen_fwd: row strides %% 8 and 16-byte aligned pointers required");
  if (int rc = require_sm90()) return rc;
  if (total_q == 0 || max_seqlen_q <= 0) return 0;
  // one query token per sample (text decode): HBM-bound split-KV kernel instead of the 128-row wgmma tiles.
  // A single query sees every key under both mask settings (bottom-right aligned causal), so `causal` is moot.
  if (attn_decode_supported(max_seqlen_q, head_dim, num_heads_q, num_heads_k))
    return attn_decode(q, k, v, out, cu_seqlens_q, cu_seqlens_k, seqused_k, batch, num_heads_q, num_heads_k,
                       max_seqlen_k, softmax_scale, ld_q, ld_k, ld_v, ld_out, static_cast<cudaStream_t>(stream));

  CUtensorMap tmQ, tmK, tmV;
  if (int rc = make_tmap_2d_bf16(&tmQ, q, (uint64_t)num_heads_q * head_dim, (uint64_t)total_q, (uint64_t)ld_q, 64, kBlockM)) return rc;
  const uint64_t rows_k = total_k > 0 ? (uint64_t)total_k : 1;
  if (int rc = make_tmap_2d_bf16(&tmK, k, (uint64_t)num_heads_k * head_dim, rows_k, (uint64_t)ld_k, 64, kBlockN)) return rc;
  if (int rc = make_tmap_2d_bf16(&tmV, v, (uint64_t)num_heads_k * head_dim, rows_k, (uint64_t)ld_v, 64, kBlockN)) return rc;

  AttnParams p{};
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ld_out = ld_out;
  p.cu_q = cu_seqlens_q;
  p.cu_k = cu_seqlens_k;
  p.seqused_k = seqused_k;
  p.Hq = num_heads_q;
  p.Hk = num_heads_k;
  p.causal = causal;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  // FMA-pipe exp2 for every 4th score pair: on for long non-causal sweeps (denoise, ViT at >= 2k keys), where MUFU limits the
  // softmax; off for short or causal ones, where it measured slower; BAGEL_ATTN_POLY=0/1 forces it off / on
  static const int poly_env = [] { const char* e = getenv("BAGEL_ATTN_POLY"); return e ? (atoi(e) != 0 ? 1 : 0) : -1; }();
  p.poly = poly_env >= 0 ? poly_env : ((causal || max_seqlen_k < 2048) ? 0 : 1);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (head_dim == 128) return launch_attn<128>(tmQ, tmK, tmV, p, batch, max_seqlen_q, s);
  return launch_attn<64>(tmQ, tmK, tmV, p, batch, max_seqlen_q, s);
}
