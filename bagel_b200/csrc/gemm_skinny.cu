// Skinny-M GEMM for the token-by-token decode path (and the few und-expert rows of a MoT layer):
//   C[M, N] = epilogue(A[M, K] * W[N, K]^T),  M <= 64.
// With M this small the GEMM is a pure weight stream (HBM bound: 2*N*K bytes), so the tile is built around W:
//   * operands are SWAPPED: a 128-row slab of W is the wgmma "A" operand (two m64 halves), the (padded) tokens are the
//     "B" operand (N = MT in {16, 32, 64}). Of every pipeline stage's bytes 80-94 % are weights; the regular
//     kernel's 128-token tile would spend 80 % of its shared-memory fill on zero padding.
//   * split-K over a thread-block CLUSTER: when N/128 tiles cannot fill the GPU the K range is divided over up to 8
//     CTAs of one cluster; partial accumulators are exchanged through distributed shared memory and summed by the
//     cluster's rank-0 CTA in rank order (deterministic, no atomics, no workspace).
//   * the accumulator [128 features x MT tokens] is parked in shared memory (over the drained operand ring); an epilogue
//     thread owns one output feature, so bias is a scalar and every store instruction of a warp writes 32 consecutive
//     features of one token (64 B).
// Epilogue rounding points are the ones of gemm.cu (the reference's autocast casts).
#include "common.cuh"
#include "host_util.h"
#include "gemm_skinny.h"

namespace bagel {

namespace {

constexpr int kThreads = 256;   // warpgroup 0: TMA (warp 0); warpgroup 1: wgmma + epilogue
constexpr int kBK = 64;         // K elements per pipeline stage (one 128 B swizzle atom)
constexpr int kMaxStages = 12;

enum : int { S_BIAS = 0, S_RESID = 1, S_SWIGLU = 2, S_GELU = 3, S_SILU = 4 };

struct SkinnyParams {
  int M, N, K;
  __nv_bfloat16* C;
  long long ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* resid;
  long long ldr;
  const int* row_map;
  int MT;       // tokens padded to the MMA N size
  int split;    // cluster size along K
  int num_k;    // K blocks in total
  int stages;
};

__device__ __forceinline__ float gelu_tanh_s(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * x * x * x)));
}
__device__ __forceinline__ float silu_s(float x) { return x / (1.0f + __expf(-x)); }

// the 128 threads of the MMA warpgroup only
__device__ __forceinline__ void mma_wg_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// NW = 128-row W slabs per CTA (2 only for SwiGLU: the gate slab and the matching up slab of the interleaved weight).
template <int NW, int EPI, int MT>
__global__ void __launch_bounds__(kThreads, 1)
gemm_skinny_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA,
                   const SkinnyParams p) {
  static_assert((EPI == S_SWIGLU) == (NW == 2), "two W slabs exactly for SwiGLU");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kWBytes = NW * 128 * kBK * 2;
  constexpr int stage_bytes = kWBytes + MT * kBK * 2;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kMaxStages;
  float* part = reinterpret_cast<float*>(smem);  // [NW * MT tokens][128 features] accumulators, over the drained ring

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = (p.split > 1) ? cluster_ctarank() : 0u;
  const int tile = blockIdx.x;
  const int kb_begin = (int)(((long long)rank * p.num_k) / p.split);
  const int kb_end = (int)(((long long)(rank + 1) * p.num_k) / p.split);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmA);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);   // one arrive per MMA warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  pdl_launch_dependents();   // the next PDL kernel may start its own weight prefetch while this one streams

  if (warp == 0) {
    if (elect_one_lane()) {   // not `lane == 0`: see common.cuh
      // The weights do not depend on the kernel in front of this one: fill the (empty) ring with W tiles right away,
      // resolve the grid dependency, then add the token tiles of the same stages (same mbarrier, one expect_tx).
      const int npre = min(p.stages, kb_end - kb_begin);
      for (int i = 0; i < npre; ++i) {
        mbar_expect_tx(&full_bar[i], (uint32_t)stage_bytes);
        tma_load_2d(smem + i * stage_bytes, &tmW, &full_bar[i], (kb_begin + i) * kBK, tile * (NW * 128), kEvictFirst);
      }
      pdl_wait();
      for (int i = 0; i < npre; ++i)
        tma_load_2d(smem + i * stage_bytes + kWBytes, &tmA, &full_bar[i], (kb_begin + i) * kBK, 0, kEvictLast);
      int stage = (npre == p.stages) ? 0 : npre;
      uint32_t phase = (npre == p.stages) ? 1u : 0u;
      for (int kb = kb_begin + npre; kb < kb_end; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
        uint8_t* st = smem + stage * stage_bytes;
        tma_load_2d(st, &tmW, &full_bar[stage], kb * kBK, tile * (NW * 128), kEvictFirst);   // weights: read once
        tma_load_2d(st + kWBytes, &tmA, &full_bar[stage], kb * kBK, 0, kEvictLast);          // tokens: re-read by all
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // MMA warpgroup: acc[w][half] = W slab w, rows [64 half, 64 half + 64) x MT tokens
    float acc[NW][2][MT / 2];
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st = smem_u32(smem + stage * stage_bytes);
      const uint64_t b_desc = gmma_desc_kmajor_sw128(st + kWBytes);
      wgmma_fence();
#pragma unroll
      for (int w = 0; w < NW; ++w) {
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint64_t a_desc = gmma_desc_kmajor_sw128(st + w * (128 * kBK * 2) + hf * (64 * kBK * 2));
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k) wgmma_ss<MT>(acc[w][hf], a_desc + 2 * k, b_desc + 2 * k, (kb > kb_begin) || (k > 0));
        }
      }
      wgmma_commit();
      if (kb > kb_begin) {
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int w = 0; w < NW; ++w)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) gmma_fence_operand(acc[w][hf]);
    mma_wg_sync();   // every warp's wgmma has retired: the operand ring may be overwritten
    const int wq = warp & 3;
    if (kb_end > kb_begin) {
#pragma unroll
      for (int w = 0; w < NW; ++w)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
#pragma unroll
          for (int c = 0; c < MT / 8; ++c)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int r = hf * 64 + wq * 16 + (lane >> 2) + 8 * (i >> 1);    // feature within the slab
              const int m = 8 * c + 2 * (lane & 3) + (i & 1);                  // token
              part[(w * MT + m) * 128 + r] = acc[w][hf][4 * c + i];
            }
    } else {   // empty K range (split > num_k cannot happen, but keep the contract): contributes zeros
      for (int i = threadIdx.x - 128; i < NW * MT * 128; i += 128) part[i] = 0.f;
    }
  }

  // partials visible CTA-wide (and, with a split, cluster-wide)
  if (p.split > 1) cluster_sync_all();
  else __syncthreads();

  if (warp >= 4 && rank == 0) {
    pdl_wait();   // residual reads / output writes below must follow the predecessor kernel
    const int r = threadIdx.x - 128;
    const int n_out = (EPI == S_SWIGLU) ? p.N / 2 : p.N;
    const int n = tile * 128 + r;            // output feature owned by this thread
    const bool n_ok = n < n_out;
    float bias = 0.f;
    if (EPI != S_SWIGLU && p.bias != nullptr && n_ok) bias = __bfloat162float(p.bias[n]);
    const uint32_t part_addr = smem_u32(part + r);
    for (int c = 0; c < p.M; c += 16) {
      float v[16], u[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        v[j] = part[(c + j) * 128 + r];
        if constexpr (EPI == S_SWIGLU) u[j] = part[(MT + c + j) * 128 + r];
      }
      // Output rows and residual values of this chunk: every load is issued here, before the first dependent store (a
      // load -> store -> load chain per token costs one L2 round trip per token).
      long long orow[16];
      float rv[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int m = c + j;
        orow[j] = (p.row_map != nullptr && m < p.M) ? (long long)p.row_map[m] : (long long)m;
      }
      if constexpr (EPI == S_RESID) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          rv[j] = (n_ok && c + j < p.M) ? __bfloat162float(p.resid[orow[j] * p.ldr + n]) : 0.f;
      }
      if constexpr (NW == 1) {
        for (uint32_t pr = 1; pr < (uint32_t)p.split; ++pr) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] += ld_dsmem_f32(part_addr + (uint32_t)((c + j) * 128 * 4), pr);
        }
      }
      if (n_ok) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int m = c + j;
          if (m < p.M) {
            float x = v[j] + bias;
            if constexpr (EPI == S_RESID) {
              x = rv[j] + bf16_round(x);
            } else if constexpr (EPI == S_GELU) {
              x = gelu_tanh_s(bf16_round(x));
            } else if constexpr (EPI == S_SILU) {
              x = silu_s(bf16_round(x));
            } else if constexpr (EPI == S_SWIGLU) {
              x = bf16_round(silu_s(bf16_round(v[j]))) * bf16_round(u[j]);
            }
            p.C[orow[j] * p.ldc + n] = __float2bfloat16_rn(x);
          }
        }
      }
    }
  }

  if (p.split > 1) cluster_sync_all();   // peers stay resident until rank 0 has read their partials
}

template <int NW, int EPI, int MT>
int launch_mt(const CUtensorMap& tmW, const CUtensorMap& tmA, const SkinnyParams& p, int tiles, int smem_bytes,
           cudaStream_t stream) {
  auto kern = gemm_skinny_kernel<NW, EPI, MT>;
  static int attr_bytes = 0;
  if (smem_bytes > attr_bytes) {
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    if (p.split > 8) BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    attr_bytes = smem_bytes;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)tiles, (unsigned)p.split, 1);
  cfg.blockDim = dim3(kThreads, 1, 1);
  cfg.dynamicSmemBytes = (size_t)smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 1;
  at[0].val.clusterDim.y = (unsigned)p.split;
  at[0].val.clusterDim.z = 1;
  // programmatic dependent launch: this kernel's weight prefetch overlaps the tail of whatever runs in front of it
  static const bool pdl = [] { const char* e = getenv("BAGEL_PDL"); return !(e && atoi(e) == 0); }();
  at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 2 : 1;
  BAGEL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmW, tmA, p));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

template <int NW, int EPI>
int launch(const CUtensorMap& tmW, const CUtensorMap& tmA, const SkinnyParams& p, int tiles, int smem_bytes,
           cudaStream_t stream) {
  if (p.MT == 16) return launch_mt<NW, EPI, 16>(tmW, tmA, p, tiles, smem_bytes, stream);
  if (p.MT == 32) return launch_mt<NW, EPI, 32>(tmW, tmA, p, tiles, smem_bytes, stream);
  return launch_mt<NW, EPI, 64>(tmW, tmA, p, tiles, smem_bytes, stream);
}

}  // namespace

bool gemm_skinny_supported(int M, int N, int K, int epilogue) {
  if (M > 64 || N < 256 || K < 64) return false;
  return epilogue == S_BIAS || epilogue == S_RESID || epilogue == S_SWIGLU || epilogue == S_GELU || epilogue == S_SILU;
}

int gemm_skinny(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N, int K,
                const void* bias, const void* resid, long long ldr, const int* row_map, int epilogue,
                cudaStream_t stream) {
  SkinnyParams p{};
  p.M = M; p.N = N; p.K = K;
  p.C = static_cast<__nv_bfloat16*>(C);
  p.ldc = ldc;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.ldr = ldr;
  p.row_map = row_map;
  p.MT = M <= 16 ? 16 : (M <= 32 ? 32 : 64);
  p.num_k = (K + kBK - 1) / kBK;
  const int nw = (epilogue == S_SWIGLU) ? 2 : 1;
  const int tiles = (N + nw * 128 - 1) / (nw * 128);
  const int sms = sm_count();

  // split-K (cluster size): fill the GPU when there are fewer W slabs than SMs
  // portable cluster sizes only (<= 8): larger ones need cudaFuncAttributeNonPortableClusterSizeAllowed and fail at launch
  static const int env_split = [] { const char* e = getenv("BAGEL_SKINNY_SPLIT"); const int v = e ? atoi(e) : 0; return v > 8 ? 8 : v; }();
  static const int env_stages = [] { const char* e = getenv("BAGEL_SKINNY_STAGES"); return e ? atoi(e) : 0; }();
  // What matters: (a) >= ~12 K blocks per CTA, (b) about 1.5 CTAs per SM in total and (c) SMALL shared memory per CTA — a
  // cluster whose CTAs each need a whole SM (deep ring) may not be placeable in one GPC, and the grid then runs in two waves.
  int split = 1;
  if (nw == 1) {
    if (env_split > 0) split = env_split;
    else {
      split = (sms * 8 / 5) / tiles;          // 28 slabs -> 8, 36 -> 6, 1188 -> 0
      if (split > p.num_k / 12) split = p.num_k / 12;   // K=3584 -> 4, K=18944 -> 24
      if (split > 8) split = 8;
      if (split < 1) split = 1;
    }
    if (split > p.num_k) split = p.num_k;
    if (split > 16) split = 16;
  }
  p.split = split;

  const int stage_bytes = nw * 128 * kBK * 2 + p.MT * kBK * 2;
  const long long ctas = (long long)tiles * split;
  // <= ~110 KB per CTA also lets the NEXT kernel's CTAs (PDL weight prefetch) become resident beside this one's
  const int budget = (split > 1) ? 4 * stage_bytes : 110 * 1024;
  int stages = budget / stage_bytes;
  if (env_stages > 0) stages = env_stages;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  const int per_cta_k = (p.num_k + split - 1) / split;
  if (stages > per_cta_k) stages = per_cta_k < 2 ? 2 : per_cta_k;
  // the accumulators [nw * MT][128] fp32 are parked over the ring
  if (stages * stage_bytes < nw * 128 * p.MT * 4) stages = (nw * 128 * p.MT * 4 + stage_bytes - 1) / stage_bytes;
  p.stages = stages;
  const int smem_bytes = stages * stage_bytes + 1024 + 2 * kMaxStages * 8;

  CUtensorMap tmW, tmA;
  if (int rc = make_tmap_2d_bf16(&tmW, W, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, kBK, nw * 128)) return rc;
  if (int rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, kBK, p.MT)) return rc;
  switch (epilogue) {
    case S_BIAS: return launch<1, S_BIAS>(tmW, tmA, p, tiles, smem_bytes, stream);
    case S_RESID: return launch<1, S_RESID>(tmW, tmA, p, tiles, smem_bytes, stream);
    case S_SWIGLU: return launch<2, S_SWIGLU>(tmW, tmA, p, tiles, smem_bytes, stream);
    case S_GELU: return launch<1, S_GELU>(tmW, tmA, p, tiles, smem_bytes, stream);
    case S_SILU: return launch<1, S_SILU>(tmW, tmA, p, tiles, smem_bytes, stream);
    default: return set_error(BAGEL_ERR_ARG, "gemm_skinny: unsupported epilogue %d", epilogue);
  }
}

}  // namespace bagel
