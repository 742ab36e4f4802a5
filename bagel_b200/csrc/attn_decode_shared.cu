// Shared-prefix single-query attention: the decode step of n samples of one prompt (Bagel.generate_text_batch with
// num_samples). The decode rows of a group (the samples of one request) share the group's context ("prefix") K/V
// rows, placed once in the slab, and each row owns its suffix of generated K/V rows. Row r of group g attends, with
// one softmax, to the concatenation of
//   prefix keys [prefix_begin[g], prefix_begin[g] + prefix_len[g]) and
//   suffix keys [suffix_begin[r], suffix_begin[r] + seqused_k[r] - prefix_len[g]).
//
// Same machinery as attn_decode.cu (warp-level m16n8k16 MMAs, per-warp cp.async rings, flash-decoding merge over a
// thread-block cluster), arranged so a prefix tile is read from HBM once for several rows:
//   * one CTA pass serves up to kS = 4 rows of a group. A row is 8 M rows of the MMA (its G <= 8 query heads of one
//     kv head; heads >= G are zero rows), so one 16-row m16n8k16 tile holds two rows and a pass runs two tiles over
//     the same shared-memory K/V tile. Groups of n > kS rows take ceil(n / kS) passes (grid z);
//   * the keys of a pass are segments of 16-key blocks: the prefix, then each row's suffix. A prefix block reaches
//     every row of the pass, a suffix block only its own row (the other rows' scores are masked, which leaves their
//     state bit for bit unchanged; a tile with no row of that suffix is skipped). Each segment is split into equal
//     chunks over the cluster's CTAs, and a CTA deals its chunk of each segment round-robin to the warps starting at
//     warp 0. So which CTA, warp and order a row's keys go through depends only on its prefix and suffix lengths: a
//     row's output does not depend on the other rows of its pass, and equal rows give equal bits;
//   * merge: lanes -> warp -> CTA in shared memory, then the CTAs of the cluster through distributed shared memory in
//     fixed rank order, each (row, head) pair finished by one rank (pair x by rank x % split: a pass holds up to 32
//     pairs, which one rank would read one after another); no atomics, no workspace, so eager runs and graph replays
//     give the same bits.
#include "common.cuh"
#include "host_util.h"

namespace bagel {

namespace {

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kD = 128;
constexpr int kS = 4;                 // decode rows per CTA pass
constexpr int kMT = kS / 2;           // 16-row MMA tiles per pass (two rows each)
constexpr int kBlk = 16;              // keys per warp iteration
constexpr int kStages = 3;
constexpr int kTileBytes = kBlk * kD * 2;
constexpr int kStageBytes = 2 * kTileBytes;
constexpr int kRingBytes = kWarps * kStages * kStageBytes;       // 96 KB -> two CTAs per SM
constexpr int kAccBytes = kWarps * kS * 8 * kD * 4;              // per-warp partials [kWarps][kS*8][kD] after the loop
constexpr int kMaxSplit = 8;
static_assert(kAccBytes + kS * 8 * kD * 4 <= kRingBytes, "merge buffers alias the K/V ring");

struct SharedParams {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* out;
  long long ld_q, ld_k, ld_v, ld_out;
  const int *cu_rows, *prefix_begin, *prefix_len, *suffix_begin, *seqused_k;
  int passes;        // CTA passes per group: ceil(max_group_rows / kS)
  int split;
  float scale_log2;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

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

__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}

// Fragment roles as in attn_decode.cu: lane (g = lane/4, j = lane%4) feeds 16-byte chunks j, j+4, j+8, j+12 of key
// row g (and of query row g) as the B (A) fragments of two MMAs each; the S accumulator is re-packed as the A operand
// of P V; V fragments come from ldmatrix.trans. Tile mt's M rows 0-7 are the heads of pass row 2mt, rows 8-15 of 2mt+1,
// so lane (g, j) owns the softmax state of head g of both rows of every tile.
template <int G>
__global__ void __launch_bounds__(kThreads, 2) attn_decode_shared_kernel(const SharedParams p) {
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ __align__(16) __nv_bfloat16 s_q[kS][8][kD];     // query rows of the pass, 16-byte chunks swizzled
  __shared__ float s_m[kWarps][kS][8], s_l[kWarps][kS][8];
  __shared__ float part_m[kS][8], part_l[kS][8];
  // segment 0: the prefix, 1 + s: the suffix of row s. This CTA's chunk of segment e is blocks [seg_c0, + seg_cnt) of
  // it, at local positions [seg_first[e], seg_first[e] + seg_cnt) (each segment padded to a multiple of kWarps)
  __shared__ int seg_first[kS + 2], seg_c0[kS + 1], seg_cnt[kS + 1], seg_src[kS + 1], seg_len[kS + 1];
  float (*s_acc)[kS * 8][kD] = reinterpret_cast<float (*)[kS * 8][kD]>(ring);
  float (*part_acc)[kD] = reinterpret_cast<float (*)[kD]>(ring + kAccBytes);

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = threadIdx.x;
  const int g = lane >> 2, j = lane & 3;
  const int rank = blockIdx.x, hk = blockIdx.y;
  const int grp = blockIdx.z / p.passes, pass = blockIdx.z % p.passes;
  const int row0 = p.cu_rows[grp] + pass * kS;
  const int nrows = min(kS, p.cu_rows[grp + 1] - row0);
  if (nrows <= 0) return;   // uniform over the cluster (same blockIdx.z): no peer waits for this CTA

  if (t == 0) {
    const int plen = max(p.prefix_len[grp], 0);
    seg_src[0] = p.prefix_begin[grp];
    seg_len[0] = plen;
#pragma unroll
    for (int s = 0; s < kS; ++s) {
      seg_src[1 + s] = s < nrows ? p.suffix_begin[row0 + s] : 0;
      seg_len[1 + s] = s < nrows ? max(p.seqused_k[row0 + s] - plen, 0) : 0;
    }
    seg_first[0] = 0;
#pragma unroll
    for (int e = 0; e <= kS; ++e) {
      const int nb = (seg_len[e] + kBlk - 1) / kBlk, per = (nb + p.split - 1) / p.split;
      const int c0 = min(rank * per, nb);
      seg_c0[e] = c0;
      seg_cnt[e] = min(c0 + per, nb) - c0;
      seg_first[e + 1] = seg_first[e] + ((seg_cnt[e] + kWarps - 1) & ~(kWarps - 1));
    }
  }
  // query rows: head g of pass row s at s_q[s][g], zero for g >= G and s >= nrows
  for (int i = t; i < kS * 8 * 16; i += kThreads) {
    const int s = i >> 7, gg = (i >> 4) & 7, c = i & 15;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (s < nrows && gg < G)
      val = __ldg(reinterpret_cast<const uint4*>(p.q + (long long)(row0 + s) * p.ld_q + (hk * G + gg) * kD) + c);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(&s_q[s][gg][0]) + ((c ^ ((gg & 1) << 2)) << 4)) = val;
  }
  __syncthreads();

  const int nloc = seg_first[kS + 1];
  const uint32_t wring = smem_u32(ring) + warp * (kStages * kStageBytes);

  // local position l -> segment, first key row in the slab, valid keys (1..16; 0 for a padding position)
  auto locate = [&](int l, int& seg, int& src, int& cnt) {
    seg = 0;
#pragma unroll
    for (int e = 1; e <= kS; ++e) seg += (l >= seg_first[e]) ? 1 : 0;
    const int k = l - seg_first[seg];
    const int off = (seg_c0[seg] + k) * kBlk;
    src = seg_src[seg] + off;
    cnt = k < seg_cnt[seg] ? min(kBlk, seg_len[seg] - off) : 0;
  };

  auto issue = [&](int i) {
    const int l = warp + i * kWarps;
    int seg, src, cnt;
    if (l < nloc) locate(l, seg, src, cnt);
    if (l < nloc && cnt > 0) {
      const uint32_t st = wring + (i % kStages) * kStageBytes;
      const int c = lane & 15;
      const __nv_bfloat16* kb = p.k + (long long)src * p.ld_k + hk * kD + c * 8;
      const __nv_bfloat16* vb_ = p.v + (long long)src * p.ld_v + hk * kD + c * 8;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int kl = (lane >> 4) + 2 * r;
        const long long key = min(kl, cnt - 1);   // rows past the segment are clamped (and masked later)
        cp_async16(st + kl * 256 + ((c ^ ((kl & 1) << 2)) << 4), kb + key * p.ld_k);
        cp_async16(st + kTileBytes + kl * 256 + ((c ^ (kl & 7)) << 4), vb_ + key * p.ld_v);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int i = 0; i < kStages - 1; ++i) issue(i);

  float m_run[kMT][2], l_run[kMT][2];
  float o[kMT][16][4];    // [tile][d tile][c0, c1: row 2mt head g | c2, c3: row 2mt+1 head g]
#pragma unroll
  for (int mt = 0; mt < kMT; ++mt) {
    m_run[mt][0] = m_run[mt][1] = -INFINITY;
    l_run[mt][0] = l_run[mt][1] = 0.f;
#pragma unroll
    for (int n = 0; n < 16; ++n) o[mt][n][0] = o[mt][n][1] = o[mt][n][2] = o[mt][n][3] = 0.f;
  }
  const uint32_t qbase = smem_u32(&s_q[0][g][0]);
  const int lm_key = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int lm_dsel = lane >> 4;

  for (int i = 0;; ++i) {
    const int l = warp + i * kWarps;
    if (l >= nloc) break;
    issue(i + kStages - 1);
    int seg, src, cnt;
    locate(l, seg, src, cnt);
    cp_async_wait<kStages - 1>();
    __syncwarp();
    if (cnt <= 0) continue;     // padding: this ring stage was not loaded
    const uint32_t st = wring + (i % kStages) * kStageBytes;
    const uint32_t vt = st + kTileBytes + lm_key * 256;

#pragma unroll
    for (int mt = 0; mt < kMT; ++mt) {
      // rows of this tile that see the block: every row for the prefix, only the suffix's own row otherwise
      const bool on0 = seg == 0 ? (2 * mt < nrows) : (seg - 1 == 2 * mt);
      const bool on1 = seg == 0 ? (2 * mt + 1 < nrows) : (seg - 1 == 2 * mt + 1);
      if (!on0 && !on1) continue;   // warp-uniform

      float sc[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
        const int kl = nt * 8 + g;
#pragma unroll
        for (int tt = 0; tt < 4; ++tt) {
          const uint32_t qoff = ((j + 4 * tt) ^ ((g & 1) << 2)) << 4;
          const uint4 qa = lds128(qbase + (2 * mt) * (8 * kD * 2) + qoff);
          const uint4 qb = lds128(qbase + (2 * mt + 1) * (8 * kD * 2) + qoff);
          const uint4 kk = lds128(st + kl * 256 + (((j + 4 * tt) ^ ((kl & 1) << 2)) << 4));
          mma_bf16_16816(sc[nt], qa.x, qb.x, qa.y, qb.y, kk.x, kk.y);
          mma_bf16_16816(sc[nt], qa.z, qb.z, qa.w, qb.w, kk.z, kk.w);
        }
      }

      uint32_t pa[2][2];     // [row half][key tile] packed bf16 probabilities
      float corr[2];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const bool on = hf ? on1 : on0;
        float sv[4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            sv[nt * 2 + e] = (on && nt * 8 + 2 * j + e < cnt) ? sc[nt][2 * hf + e] * p.scale_log2 : -INFINITY;
        float mb = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
        mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1));
        mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
        const float m_old = m_run[mt][hf];
        const float m_new = fmaxf(m_old, mb);
        // a masked row keeps its state: probabilities 0, corr 1 (or 0 while it has seen no key)
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        corr[hf] = (m_old == -INFINITY) ? 0.f : ex2f(m_old - m_use);
        float pr[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) pr[e] = ex2f(sv[e] - m_use);
        pa[hf][0] = pack_bf16x2(pr[0], pr[1]);
        pa[hf][1] = pack_bf16x2(pr[2], pr[3]);
        l_run[mt][hf] = l_run[mt][hf] * corr[hf] + (bf16_lo(pa[hf][0]) + bf16_hi(pa[hf][0])) +
                        (bf16_lo(pa[hf][1]) + bf16_hi(pa[hf][1]));
        m_run[mt][hf] = m_new;
      }

#pragma unroll
      for (int x = 0; x < 8; ++x) {
        uint32_t vv[4];
        ldmatrix_x4_trans(vv, vt + (((2 * x + lm_dsel) ^ (lm_key & 7)) << 4));
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          float (&acc)[4] = o[mt][2 * x + h2];
          acc[0] *= corr[0]; acc[1] *= corr[0];
          acc[2] *= corr[1]; acc[3] *= corr[1];
          mma_bf16_16816(acc, pa[0][0], pa[1][0], pa[0][1], pa[1][1], vv[2 * h2], vv[2 * h2 + 1]);
        }
      }
    }
    __syncwarp();
  }
  cp_async_wait<0>();
  __syncthreads();   // the merge buffers alias the rings

  // ---- merge: lanes -> warp -> CTA ----
#pragma unroll
  for (int mt = 0; mt < kMT; ++mt)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      float l = l_run[mt][hf];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int s = 2 * mt + hf;
      if (g < G) {
        if (j == 0) {
          s_m[warp][s][g] = m_run[mt][hf];
          s_l[warp][s][g] = l;
        }
#pragma unroll
        for (int n = 0; n < 16; ++n)
          *reinterpret_cast<float2*>(&s_acc[warp][s * 8 + g][n * 8 + 2 * j]) =
              make_float2(o[mt][n][2 * hf], o[mt][n][2 * hf + 1]);
      }
    }
  __syncthreads();
#pragma unroll 1
  for (int s = 0; s < nrows; ++s)
#pragma unroll
    for (int h = 0; h < G; ++h) {
      float M = -INFINITY;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) M = fmaxf(M, s_m[w][s][h]);
      float L = 0.f, A = 0.f;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const float wt = (s_m[w][s][h] == -INFINITY) ? 0.f : ex2f(s_m[w][s][h] - M);
        L = fmaf(s_l[w][s][h], wt, L);
        A = fmaf(s_acc[w][s * 8 + h][t], wt, A);
      }
      part_acc[s * 8 + h][t] = A;
      if (t == 0) {
        part_m[s][h] = M;
        part_l[s][h] = L;
      }
    }

  // ---- merge: CTAs of the cluster, fixed rank order; (row, head) pair x is finished by rank x % split ----
  if (p.split > 1) cluster_sync_all(); else __syncthreads();
#pragma unroll 1
  for (int x = rank; x < nrows * G; x += p.split) {
    const int s = x / G, h = x % G;
    float mr[kMaxSplit], lr[kMaxSplit], ar[kMaxSplit];
#pragma unroll
    for (int r = 0; r < kMaxSplit; ++r) {
      const bool on = r < p.split;
      mr[r] = !on ? -INFINITY : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_m[s][h]), r) : part_m[s][h]);
      lr[r] = !on ? 0.f : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_l[s][h]), r) : part_l[s][h]);
      ar[r] = !on ? 0.f : (p.split > 1 ? ld_dsmem_f32(smem_u32(&part_acc[s * 8 + h][t]), r) : part_acc[s * 8 + h][t]);
    }
    float M = -INFINITY;
#pragma unroll
    for (int r = 0; r < kMaxSplit; ++r) M = fmaxf(M, mr[r]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int r = 0; r < kMaxSplit; ++r) {
      const float wt = (mr[r] == -INFINITY) ? 0.f : ex2f(mr[r] - M);
      L = fmaf(lr[r], wt, L);
      A = fmaf(ar[r], wt, A);
    }
    const float ov = (L > 0.f) ? A / L : 0.f;
    p.out[(long long)(row0 + s) * p.ld_out + (hk * G + h) * kD + t] = __float2bfloat16_rn(ov);
  }
  if (p.split > 1) cluster_sync_all();   // every CTA keeps its shared memory alive until its peers have read it
}

template <int G>
int launch(const SharedParams& p, int Hk, int z, cudaStream_t stream) {
  auto kern = attn_decode_shared_kernel<G>;
  static bool attr_done = false;
  if (!attr_done) {
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kRingBytes));
    attr_done = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)p.split, (unsigned)Hk, (unsigned)z);
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

}  // namespace bagel

using namespace bagel;

extern "C" int bagel_attn_decode_shared_bf16(const void* q, const void* k, const void* v, void* out,
                                             const int* cu_rows, const int* prefix_begin, const int* prefix_len,
                                             const int* suffix_begin, const int* seqused_k, int groups, int rows,
                                             int max_group_rows, int num_heads_q, int num_heads_k, int head_dim,
                                             int max_seqlen_k, float softmax_scale, long long ld_q, long long ld_k,
                                             long long ld_v, long long ld_out, void* stream) {
  if (head_dim != kD)
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_decode_shared_bf16: head_dim must be 128 (got %d)", head_dim);
  if (num_heads_k <= 0 || num_heads_k > 65535 || num_heads_q % num_heads_k)
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_decode_shared_bf16: num_heads_q %% num_heads_k != 0");
  const int G = num_heads_q / num_heads_k;
  if (!(G == 1 || G == 2 || G == 4 || G == 7 || G == 8))
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_decode_shared_bf16: unsupported GQA group %d", G);
  if (groups < 0 || rows < 0 || (groups > 0 && (max_group_rows <= 0 || max_group_rows > rows)))
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_decode_shared_bf16: bad groups / rows / max_group_rows");
  const long long passes = (max_group_rows + kS - 1) / kS;
  if ((long long)groups * passes > 65535)
    return set_error(BAGEL_ERR_SHAPE, "bagel_attn_decode_shared_bf16: too many groups x passes");
  if ((ld_q % 8) || (ld_k % 8) || (ld_v % 8) || (ld_out % 8) ||
      (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15))
    return set_error(BAGEL_ERR_ALIGN, "bagel_attn_decode_shared_bf16: row strides %% 8 and 16-byte aligned pointers required");
  if (ld_q < (long long)num_heads_q * kD || ld_out < (long long)num_heads_q * kD || ld_k < (long long)num_heads_k * kD ||
      ld_v < (long long)num_heads_k * kD)
    return set_error(BAGEL_ERR_ARG, "bagel_attn_decode_shared_bf16: a row stride is shorter than a row");
  if (int rc = require_sm90()) return rc;
  if (groups == 0 || rows == 0) return 0;

  SharedParams p{};
  p.q = static_cast<const __nv_bfloat16*>(q);
  p.k = static_cast<const __nv_bfloat16*>(k);
  p.v = static_cast<const __nv_bfloat16*>(v);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ld_q = ld_q; p.ld_k = ld_k; p.ld_v = ld_v; p.ld_out = ld_out;
  p.cu_rows = cu_rows; p.prefix_begin = prefix_begin; p.prefix_len = prefix_len;
  p.suffix_begin = suffix_begin; p.seqused_k = seqused_k;
  p.passes = (int)passes;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  // attn_decode's split rule over (pass, kv head) pairs: about one wave of two CTAs per SM, >= 64 keys per CTA,
  // power-of-two clusters of at most 8
  const long long pairs = (long long)groups * passes * num_heads_k;
  int split = 1;
  while (split < kMaxSplit && pairs * split * 2 <= 2LL * sm_count()) split *= 2;
  if (max_seqlen_k > 0)
    while (split > 1 && (max_seqlen_k + split - 1) / split < 64) split >>= 1;
  p.split = split;
  const int z = (int)(groups * passes);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (G) {
    case 1: return launch<1>(p, num_heads_k, z, s);
    case 2: return launch<2>(p, num_heads_k, z, s);
    case 4: return launch<4>(p, num_heads_k, z, s);
    case 7: return launch<7>(p, num_heads_k, z, s);
    default: return launch<8>(p, num_heads_k, z, s);
  }
}
