// Single-query ("decode") attention: every sample contributes at most ONE query token (max_seqlen_q == 1), GQA,
// head_dim 128 — the shape of Bagel.generate_text (reference modeling/bagel/bagel.py:930-1010 ->
// qwen2_navit.py:579-588 with causal=True, one new token against the whole cache).
//
// This is an HBM-bound stream over the K/V cache (2 * len * Hk * 128 * 2 bytes per sample), not a GEMM: the
// wgmma kernel in attn.cu would spend a 128-row query tile (and a whole CTA) on one valid row per q head and
// walk the keys serially. Here instead:
//   * grid = (split, Hk, batch): the keys of one (sample, kv head) are split over the CTAs of a thread-block
//     CLUSTER; each CTA handles all G = Hq/Hk query heads that share the kv head, so K and V are read exactly once;
//   * K/V stream through per-warp cp.async rings (3 stages x 16 keys), ~190 KB in flight per SM;
//   * scores: warp-level m16n8k16 MMAs; the contraction index is permuted identically for q and k, so every lane
//     feeds whole 16-byte chunks as fragments (no transposes, conflict-free swizzled reads);
//   * P*V on the same tensor-core path (P re-packed from the score accumulators, V fragments by ldmatrix.trans);
//   * flash-decoding merge: warps -> CTA through shared memory, CTAs -> rank 0 of the cluster through distributed
//     shared memory, fixed order (deterministic), no workspace, one launch.
#include "common.cuh"
#include "host_util.h"
#include "attn_decode.h"

namespace bagel {

namespace {

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kD = 128;

struct DecodeParams {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* out;
  long long ld_q, ld_k, ld_v, ld_out;
  const int *cu_q, *cu_k, *seqused_k;
  int split;
  float scale_log2;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// m16n8k16 bf16 x bf16 -> fp32 (legacy warp-level tensor-core path; the 7-8 query heads of a GQA group are the M rows)
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int kBlk = 16;        // keys per warp iteration (two 8-key MMA column tiles)
constexpr int kStages = 3;      // per-warp cp.async ring depth
constexpr int kTileBytes = kBlk * kD * 2;            // 4 KB: one K (or V) tile of 16 keys
constexpr int kStageBytes = 2 * kTileBytes;          // K tile then V tile
constexpr int kRingBytes = kWarps * kStages * kStageBytes;   // 96 KB -> two CTAs per SM

__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// K/V stream: every warp owns a 3-stage cp.async ring (16 keys x (256 B K + 256 B V) per stage), so ~24 KB per warp
// (~190 KB per SM) are in flight independent of the register file — this kernel is a latency-bound HBM stream.
// Both contractions run on warp-level tensor cores (m16n8k16, M rows = the G query heads of the group, rows 8-15 idle):
//   S = q K^T : the contraction index d may be permuted freely as long as q and k use the same permutation, so lane
//               (g = lane/4, j = lane%4) takes the 16-byte chunks j, j+4, j+8, j+12 of "its" key row as the B fragments
//               of two MMAs each; the A fragments are the same chunks of the q rows. No transposes.
//   O += P V  : P is the S accumulator re-packed in registers (the FlashAttention-2 fragment identity), V fragments
//               come from ldmatrix.trans on the row-major V tile.
// Both tiles are stored XOR-swizzled by cp.async (16-byte chunk index ^ f(key)) so fragment reads are conflict free.
// A thread owns head g for the softmax AND for its output fragment, so no probabilities cross lanes.
template <int G>
__global__ void __launch_bounds__(kThreads, 2) attn_decode_kernel(const DecodeParams p) {
  extern __shared__ __align__(128) uint8_t ring[];     // [kWarps][kStages][K tile | V tile]; reused for the merge
  __shared__ float s_m[kWarps][G], s_l[kWarps][G];
  __shared__ __align__(16) float part_acc[G][kD];      // this CTA's (un-normalised) partial, read by cluster rank 0
  __shared__ float part_m[G], part_l[G];
  float (*s_acc)[G][kD] = reinterpret_cast<float (*)[G][kD]>(ring);   // [kWarps][G][kD], valid after the key loop

  pdl_launch_dependents();   // the o_proj GEMM behind this kernel may begin prefetching its weights
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = threadIdx.x;
  const int g = lane >> 2, j = lane & 3;
  const int rank = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int q_row = p.cu_q[b];
  const bool active = (p.cu_q[b + 1] - q_row) > 0;
  const int k_begin = p.cu_k[b];
  int len = p.seqused_k ? p.seqused_k[b] : (p.cu_k[b + 1] - k_begin);
  if (!active || len < 0) len = 0;
  const int chunk = (((len + p.split - 1) / p.split) + kBlk - 1) & ~(kBlk - 1);
  const int r0 = min(rank * chunk, len), r1 = min(r0 + chunk, len);

  const __nv_bfloat16* kbase = p.k + (long long)k_begin * p.ld_k + hk * kD;
  const __nv_bfloat16* vbase = p.v + (long long)k_begin * p.ld_v + hk * kD;
  const uint32_t wring = smem_u32(ring) + warp * (kStages * kStageBytes);

  // block i of this warp starts at key r0 + (warp + i*kWarps)*kBlk; rows past r1 are clamped (and masked later)
  auto issue = [&](int i) {
    const int blk = r0 + (warp + i * kWarps) * kBlk;
    if (blk < r1) {
      const uint32_t st = wring + (i % kStages) * kStageBytes;
      const int c = lane & 15;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int kl = (lane >> 4) + 2 * r;                       // key within the block
        const long long key = min(blk + kl, r1 - 1);
        cp_async16(st + kl * 256 + ((c ^ ((kl & 1) << 2)) << 4), kbase + key * p.ld_k + c * 8);
        cp_async16(st + kTileBytes + kl * 256 + ((c ^ (kl & 7)) << 4), vbase + key * p.ld_v + c * 8);
      }
    }
    cp_async_commit();   // always commit: group counting stays uniform
  };
#pragma unroll
  for (int i = 0; i < kStages - 1; ++i) issue(i);

  // A fragments: q row of head g (zero rows for g >= G), chunk (j + 4t) -> k-steps 2t, 2t+1
  uint4 qq[4];
#pragma unroll
  for (int tt = 0; tt < 4; ++tt) qq[tt] = make_uint4(0u, 0u, 0u, 0u);
  if (active && g < G) {
    const uint4* qp = reinterpret_cast<const uint4*>(p.q + (long long)q_row * p.ld_q + (hk * G + g) * kD);
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) qq[tt] = __ldg(qp + j + 4 * tt);
  }

  float m_run = -INFINITY, l_run = 0.f;   // state of head g (replicated over the 4 lanes j; l is a per-lane partial)
  float o[16][4];                         // O fragment: [d tile][c0, c1 = head g, channels 8*tile + 2j, +1 | c2, c3 idle]
#pragma unroll
  for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;

  // ldmatrix lane roles for the V fragments: matrices 0/1 = keys 0-7 / 8-15 of d tile 2x, matrices 2/3 = of d tile 2x+1
  const int lm_key = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int lm_dsel = lane >> 4;

  for (int i = 0;; ++i) {
    const int blk = r0 + (warp + i * kWarps) * kBlk;
    if (blk >= r1) break;
    issue(i + kStages - 1);
    cp_async_wait<kStages - 1>();
    __syncwarp();
    const uint32_t st = wring + (i % kStages) * kStageBytes;

    // ---- S = q k^T: 2 key tiles x 8 k-steps ----
    float sc[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      const int kl = nt * 8 + g;
#pragma unroll
      for (int tt = 0; tt < 4; ++tt) {
        uint4 kk;
        const uint32_t a = st + kl * 256 + (((j + 4 * tt) ^ ((kl & 1) << 2)) << 4);
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(kk.x), "=r"(kk.y), "=r"(kk.z), "=r"(kk.w) : "r"(a));
        mma_bf16_16816(sc[nt], qq[tt].x, 0u, qq[tt].y, 0u, kk.x, kk.y);
        mma_bf16_16816(sc[nt], qq[tt].z, 0u, qq[tt].w, 0u, kk.z, kk.w);
      }
    }

    // ---- online softmax for head g over this block's 16 keys (4 per lane, 4 lanes per head) ----
    float sv[4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        sv[nt * 2 + e] = (blk + nt * 8 + 2 * j + e < r1) ? sc[nt][e] * p.scale_log2 : -INFINITY;
    float mb = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
    const float m_new = fmaxf(m_run, mb);   // finite: the block holds at least one valid key
    const float corr = (m_run == -INFINITY) ? 0.f : ex2f(m_run - m_new);
    float pr[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) pr[e] = ex2f(sv[e] - m_new);   // ex2(-inf) = 0 for masked keys
    // P in bf16 for the tensor cores (as flash-attn does); the row sum uses the same rounded values
    const uint32_t pa0 = pack_bf16x2(pr[0], pr[1]), pa2 = pack_bf16x2(pr[2], pr[3]);
    l_run = l_run * corr + (bf16_lo(pa0) + bf16_hi(pa0)) + (bf16_lo(pa2) + bf16_hi(pa2));
    m_run = m_new;

    // ---- O = O * corr + P V: 16 channel tiles, V fragments by ldmatrix.trans ----
    const uint32_t vt = st + kTileBytes + lm_key * 256;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      uint32_t vb[4];
      ldmatrix_x4_trans(vb, vt + (((2 * x + lm_dsel) ^ (lm_key & 7)) << 4));
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        float (&acc)[4] = o[2 * x + h2];
        acc[0] *= corr; acc[1] *= corr;
        mma_bf16_16816(acc, pa0, 0u, pa2, 0u, vb[2 * h2], vb[2 * h2 + 1]);
      }
    }
    __syncwarp();   // this ring stage is rewritten by a later cp.async
  }
  cp_async_wait<0>();
  __syncthreads();  // every warp is done with its ring: the merge buffers alias it

  // ---- merge: lanes -> warp -> CTA ----
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
  if (g < G) {
    if (j == 0) {
      s_m[warp][g] = m_run;
      s_l[warp][g] = l_run;
    }
#pragma unroll
    for (int n = 0; n < 16; ++n)
      *reinterpret_cast<float2*>(&s_acc[warp][g][n * 8 + 2 * j]) = make_float2(o[n][0], o[n][1]);
  }
  __syncthreads();
#pragma unroll
  for (int h = 0; h < G; ++h) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) M = fmaxf(M, s_m[w][h]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const float wt = (s_m[w][h] == -INFINITY) ? 0.f : ex2f(s_m[w][h] - M);
      L = fmaf(s_l[w][h], wt, L);
      A = fmaf(s_acc[w][h][t], wt, A);
    }
    part_acc[h][t] = A;
    if (t == 0) {
      part_m[h] = M;
      part_l[h] = L;
    }
  }

  // ---- merge: CTAs of the cluster -> rank 0 (distributed shared memory), fixed rank order ----
  if (p.split > 1) cluster_sync_all(); else __syncthreads();
  if (rank == 0 && active) {
    // All distributed-shared-memory reads of a head are issued together (fixed trip count + predicate: with a run-time loop
    // bound every read waited for the previous one, ~300 cycles each, 8 per head on the critical path of every cluster).
    constexpr int kMaxSplit = 8;
#pragma unroll
    for (int h = 0; h < G; ++h) {
      float mr[kMaxSplit], lr[kMaxSplit], ar[kMaxSplit];
#pragma unroll
      for (int r = 0; r < kMaxSplit; ++r) {
        const bool on = r < p.split;
        mr[r] = !on ? -INFINITY : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_m[h]), r) : part_m[h]);
        lr[r] = !on ? 0.f : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_l[h]), r) : part_l[h]);
        ar[r] = !on ? 0.f : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_acc[h][t]), r) : part_acc[h][t]);
      }
      float M = -INFINITY;
#pragma unroll
      for (int r = 0; r < kMaxSplit; ++r) M = fmaxf(M, mr[r]);
      float L = 0.f, A = 0.f;
#pragma unroll
      for (int r = 0; r < kMaxSplit; ++r) {   // fixed rank order: deterministic
        const float wt = (mr[r] == -INFINITY) ? 0.f : ex2f(mr[r] - M);
        L = fmaf(lr[r], wt, L);
        A = fmaf(ar[r], wt, A);
      }
      const float ov = (L > 0.f) ? A / L : 0.f;
      p.out[(long long)q_row * p.ld_out + (hk * G + h) * kD + t] = __float2bfloat16_rn(ov);
    }
  }
  if (p.split > 1) cluster_sync_all();   // peers keep their shared memory alive until rank 0 has read it
}

template <int G>
int launch(const DecodeParams& p, int Hk, int B, cudaStream_t stream) {
  auto kern = attn_decode_kernel<G>;
  static bool attr_done = false;
  if (!attr_done) {
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kRingBytes));
    attr_done = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)p.split, (unsigned)Hk, (unsigned)B);
  cfg.blockDim = dim3(kThreads, 1, 1);
  cfg.dynamicSmemBytes = kRingBytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)p.split;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  BAGEL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

}  // namespace

bool attn_decode_supported(int max_seqlen_q, int head_dim, int Hq, int Hk) {
  static const bool on = [] { const char* e = getenv("BAGEL_ATTN_DECODE"); return !(e && atoi(e) == 0); }();
  if (!on || max_seqlen_q != 1 || head_dim != kD || Hk <= 0 || Hq % Hk) return false;
  const int g = Hq / Hk;
  return g == 1 || g == 2 || g == 4 || g == 7 || g == 8;
}

int attn_decode(const void* q, const void* k, const void* v, void* out, const int* cu_seqlens_q,
                const int* cu_seqlens_k, const int* seqused_k, int batch, int Hq, int Hk, int max_seqlen_k,
                float softmax_scale, long long ld_q, long long ld_k, long long ld_v, long long ld_out,
                cudaStream_t stream) {
  DecodeParams p{};
  p.q = static_cast<const __nv_bfloat16*>(q);
  p.k = static_cast<const __nv_bfloat16*>(k);
  p.v = static_cast<const __nv_bfloat16*>(v);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ld_q = ld_q; p.ld_k = ld_k; p.ld_v = ld_v; p.ld_out = ld_out;
  p.cu_q = cu_seqlens_q; p.cu_k = cu_seqlens_k; p.seqused_k = seqused_k;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  // Two CTAs (8 warps, 8 cp.async rings) fit an SM: aim for one wave of ~2 CTAs per SM, at least 64 keys per CTA,
  // cluster size <= 8 (power of two: odd cluster sizes place badly, see gemm_skinny.cu).
  static const int env_split = [] { const char* e = getenv("BAGEL_DECODE_SPLIT"); const int v = e ? atoi(e) : 0; return v > 8 ? 8 : v; }();
  const long long pairs = (long long)batch * Hk;
  int split = 1;
  while (split < 8 && pairs * split * 2 <= 2LL * sm_count()) split *= 2;
  if (max_seqlen_k > 0)
    while (split > 1 && (max_seqlen_k + split - 1) / split < 64) split >>= 1;
  if (env_split > 0) split = env_split;
  p.split = split;
  switch (Hq / Hk) {
    case 1: return launch<1>(p, Hk, batch, stream);
    case 2: return launch<2>(p, Hk, batch, stream);
    case 4: return launch<4>(p, Hk, batch, stream);
    case 7: return launch<7>(p, Hk, batch, stream);
    case 8: return launch<8>(p, Hk, batch, stream);
    default: return set_error(BAGEL_ERR_SHAPE, "attn_decode: unsupported GQA group %d", Hq / Hk);
  }
}

}  // namespace bagel
