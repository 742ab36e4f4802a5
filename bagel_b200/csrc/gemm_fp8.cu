// Block-scaled FP8 (e4m3) path of the generation expert's MLP (opt-in, `fp8_gen_mlp=True`): the quantiser and the GEMM.
//
// Format (the one place it is defined; bagel_b200/fp8.py and the tests restate it):
//   - a group of values (a 1 x 128 run along K of an activation row, or a 128 x 128 block of a weight) has one fp32 scale
//     s = the smallest power of two with amax <= 448 s, at least 2^-126, and 1 for an all-zero group;
//   - q = e4m3(x / s), round to nearest even. s is a power of two, so x / s is exact, |x / s| <= 448 and q * s is a bf16 value.
//   - GEMM: y[m, n] = sum_kb sa[m, kb] sw[n, kb] (sum_{k in kb} qa[m, k] qw[n, k]); each 128-wide K block's tensor-core sum is
//     scaled and added ("promoted") into a separate fp32 accumulator, so the limited accumulation width of the fp8 wgmma
//     never spans more than 128 products.
//
// The GEMM is the persistent, TMA-fed, warp-specialised design of gemm_bf16_kernel (gemm.cu) with the 2-CTA W multicast:
// a 128-byte swizzle row is 128 e4m3 values, so a stage is a 128 x 128 A box plus a 128 x 128 W box (32 KiB), one K block,
// one scale group. The e4m3 tensors are described to TMA as bf16 tensors of half the width (TMA moves bytes; the box is
// the same 128 bytes wide). The tile is BN = 128 W rows: promotion needs a second 64-column fp32 accumulator per thread,
// and BN = 256 would need 2 x 128.
//
// SwiGLU weight layout (EPI_SWIGLU): W rows interleaved per 128 as 64 gate rows | 64 up rows, so every 128-row tile
// yields 64 output columns. W scales are given per 64-row half tile: w_scales[N / 64, K / 128], so one tile reads two
// scales per K block (gate half, up half; for EPI_RESID both halves repeat the scale of their 128 x 128 block).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "gemm_params.h"
#include "host_util.h"

namespace bagel {

constexpr int kQBK = 128;                    // e4m3 values (= bytes) per K block: one swizzle row and one scale group
constexpr int kQBN = 128;                    // W rows per tile
constexpr int kQABytes = BM * kQBK;          // 16 KiB
constexpr int kQBBytes = kQBN * kQBK;        // 16 KiB
constexpr int kQStageBytes = kQABytes + kQBBytes;
constexpr int kQStages = 6;
constexpr int kQSmemBytes = kQStages * kQStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;

struct Fp8GemmParams {
  int M, N, K, num_kb;
  const float* a_scales;   // [num_kb, ld_as]: the scale of row m, K block kb at kb * ld_as + m
  long long ld_as;
  const float* w_scales;   // [N / 64, num_kb]
  __nv_bfloat16* C;
  long long ldc;
  const __nv_bfloat16* resid;
  long long ldr;
  int num_m, num_n, num_tiles, group_m;
};

// s = 2^k, k = the smallest integer with amax <= 448 * 2^k, from the exponent and mantissa bits of amax:
// amax = 1.f * 2^e and 448 = 1.75 * 2^8, so k = e - 8, plus one when the mantissa is above 1.75's. inv = 1 / s, exactly.
__device__ __forceinline__ float fp8_scale(float amax, float& inv) {
  if (amax == 0.f) {
    inv = 1.f;
    return 1.f;
  }
  const uint32_t b = __float_as_uint(amax);
  int k = (int)((b >> 23) & 0xFF) - 127 - 8 + ((b & 0x7FFFFF) > 0x600000u ? 1 : 0);
  k = max(k, -126);
  inv = __uint_as_float((uint32_t)(127 - k) << 23);
  return __uint_as_float((uint32_t)(k + 127) << 23);
}

__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, __NV_E4M3);
}

// block_rows = 1: a half-warp per (row, K block), 8 values per lane.
__global__ void __launch_bounds__(256) quantize_fp8_rows_kernel(const __nv_bfloat16* __restrict__ X, long long ldx,
                                                                uint8_t* __restrict__ Q, long long ldq,
                                                                float* __restrict__ S, long long lds, int M, int nkb) {
  const long long unit = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  const int l = threadIdx.x & 15;
  const bool ok = unit < (long long)M * nkb;
  const int row = ok ? (int)(unit / nkb) : 0, kb = ok ? (int)(unit % nkb) : 0;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (ok) v = *reinterpret_cast<const uint4*>(X + row * ldx + kb * kQBK + l * 8);
  float x[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y),
                bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(x[i]));
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  float inv;
  const float s = fp8_scale(amax, inv);
  if (!ok) return;
  uint2 q;
  q.x = e4m3x2(x[0] * inv, x[1] * inv) | (e4m3x2(x[2] * inv, x[3] * inv) << 16);
  q.y = e4m3x2(x[4] * inv, x[5] * inv) | (e4m3x2(x[6] * inv, x[7] * inv) << 16);
  *reinterpret_cast<uint2*>(Q + row * ldq + kb * kQBK + l * 8) = q;
  if (l == 0) S[kb * lds + row] = s;
}

// block_rows = 128 (weights, at load time): one CTA of 128 threads per 128 x 128 block, thread t owns column t.
__global__ void __launch_bounds__(128) quantize_fp8_blocks_kernel(const __nv_bfloat16* __restrict__ X, long long ldx,
                                                                  uint8_t* __restrict__ Q, long long ldq,
                                                                  float* __restrict__ S, long long lds, int M) {
  __shared__ float red[4];
  const int t = threadIdx.x, kb = blockIdx.x, rb = blockIdx.y;
  const int r0 = rb * 128, r1 = min(M, r0 + 128);
  const long long col = (long long)kb * kQBK + t;
  float amax = 0.f;
  for (int r = r0; r < r1; ++r) amax = fmaxf(amax, fabsf(__bfloat162float(X[r * ldx + col])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((t & 31) == 0) red[t >> 5] = amax;
  __syncthreads();
  amax = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  float inv;
  const float s = fp8_scale(amax, inv);
  if (t == 0) S[rb * lds + kb] = s;
  for (int r = r0; r < r1; ++r)
    Q[r * ldq + col] = (uint8_t)(e4m3x2(__bfloat162float(X[r * ldx + col]) * inv, 0.f) & 0xFF);
}

template <int EPI, int CLUSTER>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Fp8GemmParams p) {
  static_assert(EPI == EPI_SWIGLU || EPI == EPI_RESID, "fp8 GEMM epilogues: SwiGLU (gate|up) and residual add (down)");
  constexpr int kBSliceRows = kQBN / CLUSTER;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kQStages * kQABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kQStages * kQStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kQStages;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_k = p.num_kb;
  const uint32_t rank = (CLUSTER > 1) ? cluster_ctarank() : 0u;
  const int num_mc = (p.num_m + CLUSTER - 1) / CLUSTER;
  const int first_tile = blockIdx.x / CLUSTER, tile_stride = gridDim.x / CLUSTER;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kQStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CLUSTER * kGemmMmaWarps);
    }
    fence_mbar_init();
  }
  if constexpr (CLUSTER > 1) cluster_sync_all();
  else __syncthreads();

  auto release = [&](int s) {
    if constexpr (CLUSTER == 1) {
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    } else if (lane < CLUSTER) {
      mbar_arrive_cluster(&empty_bar[s], (uint32_t)lane);
    }
  };

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one_lane()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first_tile; tile < p.num_tiles; tile += tile_stride) {
        int m_blk, n_blk;
        tile_coords(tile, num_mc, p.num_n, p.group_m, p.num_n, m_blk, n_blk);
        m_blk = m_blk * CLUSTER + rank;   // past the last M tile (odd count): TMA zero-fills, the epilogue skips the rows
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], kQStageBytes);
          // coordinates in the bf16 view of the e4m3 tensors: 64 "bf16" columns per K block
          tma_load_2d(smem_a + stage * kQABytes, &tmA, &full_bar[stage], kb * (kQBK / 2), m_blk * BM, kEvictNormal);
          uint8_t* b_dst = smem_b + stage * kQBBytes + rank * (kBSliceRows * kQBK);
          const int b_row = n_blk * kQBN + (int)rank * kBSliceRows;
          if constexpr (CLUSTER == 1) tma_load_2d(b_dst, &tmB, &full_bar[stage], kb * (kQBK / 2), b_row, kEvictNormal);
          else tma_load_2d_multicast(b_dst, &tmB, &full_bar[stage], kb * (kQBK / 2), b_row, (1u << CLUSTER) - 1, kEvictNormal);
          if (++stage == kQStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + promotion + epilogue warpgroups (1, 2) =====================
    setmaxnreg_inc<232>();
    const int half = wg - 1;
    const int wq = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first_tile; tile < p.num_tiles; tile += tile_stride) {
      int m_blk, n_blk;
      tile_coords(tile, num_mc, p.num_n, p.group_m, p.num_n, m_blk, n_blk);
      m_blk = m_blk * CLUSTER + rank;
      // this thread's fragment rows r0 and r0 + 8, columns 8c + 2 (lane % 4) + {0, 1} (wgmma.cuh)
      const int r0 = m_blk * BM + half * 64 + wq * 16 + (lane >> 2);
      const bool ok0 = r0 < p.M, ok1 = r0 + 8 < p.M;
      const float* ws = p.w_scales + (long long)(2 * n_blk) * num_k;   // this tile's two 64-row halves
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_k; ++kb) {
        // the scales do not depend on the stage: load them before waiting for it
        const float sa0 = ok0 ? p.a_scales[kb * p.ld_as + r0] : 0.f;
        const float sa1 = ok1 ? p.a_scales[kb * p.ld_as + r0 + 8] : 0.f;
        const float sw0 = ws[kb], sw1 = ws[num_k + kb];
        mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = gmma_desc_kmajor_sw128(smem_u32(smem_a + stage * kQABytes + half * 64 * 128));
        const uint64_t b_desc = gmma_desc_kmajor_sw128(smem_u32(smem_b + stage * kQBBytes));
        float part[64];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kQBK / 32; ++k) wgmma_ss_e4m3_n128(part, a_desc + 2 * k, b_desc + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        gmma_fence_operand(part);
        __syncwarp();
        release(stage);
        // promotion: the 128-deep tensor-core sum, scaled, into the fp32 accumulator
        const float s00 = sa0 * sw0, s01 = sa0 * sw1, s10 = sa1 * sw0, s11 = sa1 * sw1;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float t0 = c < 8 ? s00 : s01, t1 = c < 8 ? s10 : s11;
          acc[4 * c + 0] = fmaf(part[4 * c + 0], t0, acc[4 * c + 0]);
          acc[4 * c + 1] = fmaf(part[4 * c + 1], t0, acc[4 * c + 1]);
          acc[4 * c + 2] = fmaf(part[4 * c + 2], t1, acc[4 * c + 2]);
          acc[4 * c + 3] = fmaf(part[4 * c + 3], t1, acc[4 * c + 3]);
        }
        if (++stage == kQStages) { stage = 0; phase ^= 1; }
      }

      const int cq = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= p.M) continue;
        if constexpr (EPI == EPI_SWIGLU) {
          // columns 0..63 of the tile are gate, 64..127 the matching up rows: output columns n_blk * 64 + [0, 64)
          __nv_bfloat16* crow = p.C + row * p.ldc + n_blk * (kQBN / 2);
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float g0 = bf16_round(acc[4 * c + 2 * h]), g1 = bf16_round(acc[4 * c + 2 * h + 1]);
            const float u0 = bf16_round(acc[4 * (c + 8) + 2 * h]), u1 = bf16_round(acc[4 * (c + 8) + 2 * h + 1]);
            *reinterpret_cast<uint32_t*>(crow + 8 * c + cq) =
                pack_bf16x2(bf16_round(silu_f(g0)) * u0, bf16_round(silu_f(g1)) * u1);
          }
        } else {
          __nv_bfloat16* crow = p.C + row * p.ldc + n_blk * kQBN;
          const __nv_bfloat16* rrow = p.resid + row * p.ldr + n_blk * kQBN;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int n = 8 * c + cq;
            const uint32_t rr = *reinterpret_cast<const uint32_t*>(rrow + n);
            *reinterpret_cast<uint32_t*>(crow + n) =
                pack_bf16x2(bf16_lo(rr) + bf16_round(acc[4 * c + 2 * h]), bf16_hi(rr) + bf16_round(acc[4 * c + 2 * h + 1]));
          }
        }
      }
    }
  }

  if constexpr (CLUSTER > 1) {   // the peer may still arrive on this CTA's empty barriers: leave together
    __syncwarp();
    cluster_sync_all();
  }
}

template <int EPI, int CLUSTER>
static int launch_gemm_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, Fp8GemmParams p, cudaStream_t stream) {
  auto kern = gemm_fp8_kernel<EPI, CLUSTER>;
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kGemmThreads, 1, 1);
  cfg.dynamicSmemBytes = kQSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CLUSTER;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  static int max_ctas = 0;  // per-instantiation; idempotent if raced
  if (max_ctas == 0) {
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kQSmemBytes));
    int n = sm_count();
    if (CLUSTER > 1) {
      cfg.gridDim = dim3(CLUSTER, 1, 1);
      BAGEL_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
      if (n < 1) return set_error(BAGEL_ERR_CUDA, "bagel_gemm_fp8: no %d-CTA cluster fits on this device", CLUSTER);
      n *= CLUSTER;
    }
    max_ctas = n;
  }
  p.num_m = (p.M + BM - 1) / BM;
  p.num_n = p.N / kQBN;
  p.num_tiles = (p.num_m + CLUSTER - 1) / CLUSTER * p.num_n;
  const int group_m = p.num_n >= 64 ? 16 : 32;   // as bagel_gemm_bf16: wide (gate|up) vs narrow (down) outputs
  p.group_m = group_m >= CLUSTER ? group_m / CLUSTER : 1;
  const int grid = p.num_tiles * CLUSTER < max_ctas ? p.num_tiles * CLUSTER : max_ctas;
  cfg.gridDim = dim3((unsigned)grid, 1, 1);
  BAGEL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace bagel

using namespace bagel;

extern "C" int bagel_quantize_fp8_bf16(const void* X, long long ldx, void* Q, long long ldq, float* scales,
                                       long long lds, int M, int K, int block_rows, void* stream) {
  if (M <= 0 || K <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_quantize_fp8_bf16: M and K must be > 0");
  if (K % kQBK) return set_error(BAGEL_ERR_SHAPE, "bagel_quantize_fp8_bf16: K must be a multiple of 128");
  if (block_rows != 1 && block_rows != 128)
    return set_error(BAGEL_ERR_ARG, "bagel_quantize_fp8_bf16: block_rows must be 1 or 128");
  const int nkb = K / kQBK;
  if (lds < (block_rows == 1 ? (long long)M : (long long)nkb))
    return set_error(BAGEL_ERR_ARG, "bagel_quantize_fp8_bf16: lds must be >= %s", block_rows == 1 ? "M" : "K / 128");
  if ((ldx % 8) || (ldq % 16) || (((uintptr_t)X | (uintptr_t)Q) & 15) || ((uintptr_t)scales & 3))
    return set_error(BAGEL_ERR_ALIGN, "bagel_quantize_fp8_bf16: X, Q need 16-byte alignment (ldx %% 8, ldq %% 16)");
  if (ldx < K || ldq < K) return set_error(BAGEL_ERR_ARG, "bagel_quantize_fp8_bf16: ldx and ldq must be >= K");
  if (int rc = require_sm90()) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* x = static_cast<const __nv_bfloat16*>(X);
  uint8_t* q = static_cast<uint8_t*>(Q);
  if (block_rows == 1) {
    const long long threads = (long long)M * nkb * 16;
    quantize_fp8_rows_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(x, ldx, q, ldq, scales, lds, M, nkb);
  } else {
    quantize_fp8_blocks_kernel<<<dim3(nkb, (M + 127) / 128), 128, 0, s>>>(x, ldx, q, ldq, scales, lds, M);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_gemm_fp8(const void* A, long long lda, const float* a_scales, long long ld_as, const void* W,
                              long long ldw, const float* w_scales, void* C, long long ldc, int M, int N, int K,
                              const void* resid, long long ldr, int epilogue, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_fp8: M,N,K must be > 0");
  if ((K % kQBK) || (N % kQBN)) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_fp8: K and N must be multiples of 128");
  if (epilogue != EPI_SWIGLU && epilogue != EPI_RESID)
    return set_error(BAGEL_ERR_ARG, "bagel_gemm_fp8: epilogue %d is not supported (BAGEL_EPI_SWIGLU or BAGEL_EPI_RESID)",
                     epilogue);
  if (ld_as < M) return set_error(BAGEL_ERR_ARG, "bagel_gemm_fp8: ld_as must be >= M");
  if ((lda % 16) || (ldw % 16) || (ldc % 8))
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_fp8: lda, ldw must be multiples of 16 and ldc of 8");
  if (((uintptr_t)A | (uintptr_t)W | (uintptr_t)C | (uintptr_t)resid) & 15)
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_fp8: A, W, C and resid must be 16-byte aligned");
  if (((uintptr_t)a_scales | (uintptr_t)w_scales) & 3)
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_fp8: scales must be 4-byte aligned");
  if (epilogue == EPI_RESID && (resid == nullptr || (ldr % 8)))
    return set_error(BAGEL_ERR_ARG, "bagel_gemm_fp8: BAGEL_EPI_RESID needs resid with ldr %% 8 == 0");
  const int n_out = epilogue == EPI_SWIGLU ? N / 2 : N;
  if (lda < K || ldw < K || ldc < n_out || (epilogue == EPI_RESID && ldr < N))
    return set_error(BAGEL_ERR_ARG, "bagel_gemm_fp8: lda, ldw must be >= K, ldc >= the output width (%d), ldr >= N",
                     n_out);
  if (a_scales == nullptr || w_scales == nullptr) return set_error(BAGEL_ERR_ARG, "bagel_gemm_fp8: scales are required");
  if (int rc = require_sm90()) return rc;

  Fp8GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.num_kb = K / kQBK;
  p.a_scales = a_scales; p.ld_as = ld_as; p.w_scales = w_scales;
  p.C = static_cast<__nv_bfloat16*>(C); p.ldc = ldc;
  p.resid = static_cast<const __nv_bfloat16*>(resid); p.ldr = ldr;
  const int cluster = (M + BM - 1) / BM >= 2 ? 2 : 1;
  CUtensorMap tmA, tmB;   // e4m3 [rows, K] viewed as bf16 [rows, K / 2]
  if (int rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K / 2, (uint64_t)M, (uint64_t)lda / 2, kQBK / 2, BM)) return rc;
  if (int rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)K / 2, (uint64_t)N, (uint64_t)ldw / 2, kQBK / 2, kQBN / cluster))
    return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (epilogue == EPI_SWIGLU)
    return cluster == 2 ? launch_gemm_fp8<EPI_SWIGLU, 2>(tmA, tmB, p, s) : launch_gemm_fp8<EPI_SWIGLU, 1>(tmA, tmB, p, s);
  return cluster == 2 ? launch_gemm_fp8<EPI_RESID, 2>(tmA, tmB, p, s) : launch_gemm_fp8<EPI_RESID, 1>(tmA, tmB, p, s);
}
