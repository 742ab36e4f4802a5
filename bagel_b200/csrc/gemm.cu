// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epilogue( A[M,K] * W[N,K]^T )
//
// Replaces every nn.Linear on BAGEL's forward path (reference: modeling/bagel/qwen2_navit.py:515-517,
// 529-536, 589-594; modeling/qwen2/modeling_qwen2.py:200-201; modeling/bagel/bagel.py:801-833), which
// the reference runs as cuBLASLt GEMM + separate ATen elementwise launches.
//
//   warpgroup 0    : TMA producer (one elected lane: cp.async.bulk.tensor 2D, 128B swizzle, kStages-deep smem ring)
//   warpgroups 1-2 : MMA + epilogue, 64 rows of the 128 x BN tile each (wgmma m64nBNk16, fp32 accumulators in
//                    registers, one wgmma group kept in flight), fused epilogue straight from the accumulator fragments
//
// The producer runs ahead into the next tile of the persistent loop while the MMA warpgroups are in their epilogue.
// A and W are both K-major ("TN" GEMM: nn.Linear weight layout), fp32 accumulation, bf16 output.
//
// CLUSTER = 2 (every GEMM with two or more M tiles, not the convolution): the two CTAs of a cluster compute M tiles
// 2i and 2i + 1 of the same N tile, so they need the same W tile. Each producer loads its own A tile and one half
// (BN / 2 rows) of W, multicast into the same place of the stage in both CTAs: per K block a CTA reads 16 KiB of A and
// BN * 64 B of W from L2 instead of 16 KiB + BN * 128 B. A stage is refilled only when the MMA warps of BOTH CTAs are
// done with it (each releases it in both CTAs), so the two CTAs walk the same tiles with their rings in lockstep.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "host_util.h"
#include "gemm_skinny.h"
#include "gemm_params.h"

namespace bagel {

template <int BN>
struct GemmCfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BN == 256) ? 4 : (BN == 128 ? 6 : (BN == 64 ? 8 : 10));
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN, int EPI, bool CONV = false, int CLUSTER = 1>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  static_assert(EPI != EPI_SWIGLU || BN == 256, "SwiGLU epilogue pairs 128 gate + 128 up columns");
  static_assert(CLUSTER == 1 || (CLUSTER == 2 && !CONV), "CTA pairs for the plain GEMM only");
  constexpr int kBSliceRows = BN / CLUSTER;   // W rows one producer loads per stage (tmB's box)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * Cfg::kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;                  // [kStages]  TMA -> MMA: the local producer's arrive + the stage's bytes
  uint64_t* empty_bar = bars + kStages;       // [kStages]  MMA -> TMA: one arrive per MMA warp of every CTA of the cluster

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_k = CONV ? p.ksize * p.ksize * p.cin_chunks : (p.K + BK - 1) / BK;
  // persistent loop over cluster tiles (CLUSTER M tiles x one N tile); this CTA takes M tile CLUSTER * m + rank
  const uint32_t rank = (CLUSTER > 1) ? cluster_ctarank() : 0u;
  const int num_mc = (p.num_m + CLUSTER - 1) / CLUSTER;
  const int first_tile = blockIdx.x / CLUSTER, tile_stride = gridDim.x / CLUSTER;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CLUSTER * kGemmMmaWarps);
    }
    fence_mbar_init();
  }
  if constexpr (CLUSTER > 1) cluster_sync_all();   // the peer's barriers exist before any remote arrive or multicast
  else __syncthreads();

  // A consumed stage is released (once per MMA warp) in every CTA whose producer writes into it: lane r arrives in rank r.
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
      const uint64_t hint_a = (p.hints & 2) ? kEvictFirst : ((p.hints & 8) ? kEvictLast : kEvictNormal);
      const uint64_t hint_w = (p.hints & 1) ? kEvictLast : ((p.hints & 16) ? kEvictFirst : kEvictNormal);
      for (int tile = first_tile; tile < p.num_tiles; tile += tile_stride) {
        int m_blk, n_blk;
        tile_coords(tile, num_mc, p.num_n, p.group_m, p.group_n, m_blk, n_blk);
        m_blk = m_blk * CLUSTER + rank;   // past the last M tile (odd count): TMA zero-fills, the epilogue skips the rows
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (CONV) {
            // m_blk -> (image, tile row, tile col); K block -> (tap, channel chunk). Out-of-image coordinates
            // (the conv's zero padding, ragged tile edges) are zero-filled by TMA.
            const int tiles_img = p.tiles_w * p.tiles_h;
            const int img = m_blk / tiles_img, t_in = m_blk - img * tiles_img;
            const int h0 = (t_in / p.tiles_w) * p.th, w0 = (t_in % p.tiles_w) * p.tw;
            const int tap = kb / p.cin_chunks, cc = kb - tap * p.cin_chunks;
            const int kh = tap / p.ksize, kw = tap - kh * p.ksize;
            tma_load_4d(smem_a + stage * Cfg::kABytes, &tmA, &full_bar[stage], cc * BK, w0 * p.stride + kw - p.pad,
                        h0 * p.stride + kh - p.pad, img, hint_a);
          } else {
            tma_load_2d(smem_a + stage * Cfg::kABytes, &tmA, &full_bar[stage], kb * BK, m_blk * BM, hint_a);
          }
          // W rows [n_blk * BN + rank * kBSliceRows, + kBSliceRows) into the same rows of the stage in every CTA of the
          // cluster; 128B-swizzled K-major slices of a multiple of 8 rows put together are byte-identical to one BN-row box
          uint8_t* b_dst = smem_b + stage * Cfg::kBBytes + rank * (kBSliceRows * BK * 2);
          const int b_row = n_blk * BN + (int)rank * kBSliceRows;
          if constexpr (CLUSTER == 1) tma_load_2d(b_dst, &tmB, &full_bar[stage], kb * BK, b_row, hint_w);
          else tma_load_2d_multicast(b_dst, &tmB, &full_bar[stage], kb * BK, b_row, (1u << CLUSTER) - 1, hint_w);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue warpgroups (1, 2) =====================
    setmaxnreg_inc<232>();
    const int half = wg - 1;                      // rows [64 * half, 64 * half + 64) of every tile
    const int wq = warp & 3;                      // warp within the warpgroup: fragment rows 16 wq .. 16 wq + 15
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first_tile; tile < p.num_tiles; tile += tile_stride) {
      int m_blk, n_blk;
      tile_coords(tile, num_mc, p.num_n, p.group_m, p.group_n, m_blk, n_blk);
      m_blk = m_blk * CLUSTER + rank;
      float acc[BN / 2];
      int prev = 0;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = gmma_desc_kmajor_sw128(smem_u32(smem_a + stage * Cfg::kABytes + half * 64 * 128));
        const uint64_t b_desc = gmma_desc_kmajor_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WGMMA_K; ++k) wgmma_ss<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wgmma_commit();
        if (kb > 0) {   // the previous k block's MMAs have retired: its smem slot may be refilled
          wgmma_wait<1>();
          __syncwarp();
          release(prev);
        }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      gmma_fence_operand(acc);
      __syncwarp();
      release(prev);

      // epilogue: this thread holds rows r0 = 16 wq + lane / 4 and r0 + 8 (of its 64-row half), columns 8c + 2 (lane % 4) + {0, 1}
      const int cq = 2 * (lane & 3);
      if constexpr (EPI == EPI_QKV) {
        static_assert(BN == 256, "fused QKV epilogue: two 128-wide heads per tile");
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m_blk * BM + half * 64 + wq * 16 + (lane >> 2) + 8 * h;
          const bool row_ok = row < p.M;
          const long long out_row = (row_ok && p.row_map != nullptr) ? (long long)p.row_map[row] : (long long)row;
          qkv_epilogue_rows(p, acc, h, cq, n_blk, row_ok, out_row);
        }
      } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row_in_tile = half * 64 + wq * 16 + (lane >> 2) + 8 * h;
        bool row_ok;
        long long out_row;
        if constexpr (CONV) {
          const int tiles_img = p.tiles_w * p.tiles_h;
          const int img = m_blk / tiles_img, t_in = m_blk - img * tiles_img;
          const int ho = (t_in / p.tiles_w) * p.th + row_in_tile / p.tw;
          const int wo = (t_in % p.tiles_w) * p.tw + row_in_tile % p.tw;
          row_ok = (ho < p.Ho) && (wo < p.Wo);
          out_row = (long long)(img * p.Ho + ho) * p.Wo + wo;
        } else {
          const int row = m_blk * BM + row_in_tile;
          row_ok = row < p.M;
          out_row = row;
          if (p.row_map != nullptr && row_ok) out_row = p.row_map[row];
        }
        if (!row_ok) continue;
        if constexpr (EPI == EPI_SWIGLU) {
          const int n_out0 = n_blk * (BN / 2);
          __nv_bfloat16* crow = p.C + out_row * p.ldc + n_out0;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int n = 8 * c + cq;
            if (n_out0 + n >= p.N / 2) continue;
            const float g0 = bf16_round(acc[4 * c + 2 * h]), g1 = bf16_round(acc[4 * c + 2 * h + 1]);
            const float u0 = bf16_round(acc[4 * (c + 16) + 2 * h]), u1 = bf16_round(acc[4 * (c + 16) + 2 * h + 1]);
            store4(crow + n, pack_bf16x2(bf16_round(silu_f(g0)) * u0, bf16_round(silu_f(g1)) * u1), p.hints & 4);
          }
        } else {
          const int n0_tile = n_blk * BN;
          __nv_bfloat16* crow = p.C + out_row * p.ldc + n0_tile;
          const __nv_bfloat16* rrow = (EPI == EPI_RESID) ? p.resid + out_row * p.ldr + n0_tile : nullptr;
          const float* rrow32 = (EPI == EPI_RESID_F32) ? p.resid32 + out_row * p.ldr + n0_tile : nullptr;
          float* crow32 = (EPI == EPI_F32 || EPI == EPI_RESID_F32) ? p.C32 + out_row * p.ldc + n0_tile : nullptr;
          // The row's residuals are all loaded before its first store: C may alias resid, so the compiler cannot move a
          // load above an earlier store, and loads interleaved with the stores would be BN / 8 dependent round trips.
          uint32_t rres[EPI == EPI_RESID ? BN / 8 : 1];
          if constexpr (EPI == EPI_RESID) {
#pragma unroll
            for (int c = 0; c < BN / 8; ++c)
              if (n0_tile + 8 * c + cq < p.N) rres[c] = *reinterpret_cast<const uint32_t*>(rrow + 8 * c + cq);
          }
#pragma unroll
          for (int c = 0; c < BN / 8; ++c) {
            const int n = 8 * c + cq;              // N % 8 == 0: a column pair is in or out together
            if (n0_tile + n >= p.N) continue;
            float x0 = acc[4 * c + 2 * h], x1 = acc[4 * c + 2 * h + 1];
            if (p.bias != nullptr) {
              const uint32_t bb = *reinterpret_cast<const uint32_t*>(p.bias + n0_tile + n);
              x0 += bf16_lo(bb);
              x1 += bf16_hi(bb);
            }
            if constexpr (EPI == EPI_RESID) {
              const uint32_t rr = rres[c];
              x0 = bf16_lo(rr) + bf16_round(x0);
              x1 = bf16_hi(rr) + bf16_round(x1);
            } else if constexpr (EPI == EPI_RESID_F32) {
              const float2 r2 = *reinterpret_cast<const float2*>(rrow32 + n);
              x0 = __fadd_rn(r2.x, bf16_round(x0));
              x1 = __fadd_rn(r2.y, bf16_round(x1));
            } else if constexpr (EPI == EPI_GELU) {
              x0 = gelu_tanh_f(bf16_round(x0));
              x1 = gelu_tanh_f(bf16_round(x1));
            } else if constexpr (EPI == EPI_SILU) {
              x0 = silu_f(bf16_round(x0));
              x1 = silu_f(bf16_round(x1));
            }
            if constexpr (EPI == EPI_F32 || EPI == EPI_RESID_F32) {
              *reinterpret_cast<float2*>(crow32 + n) = make_float2(x0, x1);
            } else {
              store4(crow + n, pack_bf16x2(x0, x1), p.hints & 4);
            }
          }
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

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// Cluster size of a (non-convolution) GEMM over M rows: CTA pairs sharing the W tile as soon as there are two M tiles.
// tmB's box is BN / cluster rows.
static int gemm_cluster(int M) { return (M + BM - 1) / BM >= 2 ? 2 : 1; }

template <int BN, int EPI, bool CONV, int CLUSTER>
static int launch_gemm_cluster(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_kernel<BN, EPI, CONV, CLUSTER>;
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kGemmThreads, 1, 1);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
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
    BAGEL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    int n = sm_count();
    if (CLUSTER > 1) {   // how many pairs fit at once depends on how the SMs are spread over the GPCs
      cfg.gridDim = dim3(CLUSTER, 1, 1);
      BAGEL_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
      if (n < 1) return set_error(BAGEL_ERR_CUDA, "bagel_gemm_bf16: no %d-CTA cluster fits on this device", CLUSTER);
      n *= CLUSTER;
    }
    max_ctas = n;
  }
  if (!CONV) p.num_m = (p.M + BM - 1) / BM;  // CONV: set by the caller (images x tiles per image)
  p.num_n = (p.N + BN - 1) / BN;
  p.num_tiles = (p.num_m + CLUSTER - 1) / CLUSTER * p.num_n;   // cluster tiles
  // Raster group: group_m M-tiles share one sweep over the N tiles: 16 for wide outputs (gate|up: 148 N-tiles), 32 for
  // narrow ones (14-18 N-tiles: qkv, o_proj, down_proj). The kernel counts it in cluster tiles.
  {
    static const int env_g = [] { const char* e = getenv("BAGEL_GEMM_GROUP_M"); return e ? atoi(e) : 0; }();
    static const int env_n = [] { const char* e = getenv("BAGEL_GEMM_GROUP_N"); return e ? atoi(e) : -1; }();
    static const int env_h = [] { const char* e = getenv("BAGEL_GEMM_HINTS"); return e ? atoi(e) : -1; }();
    const int group_m = env_g > 0 ? env_g : (p.num_n >= 64 ? 16 : 32);
    p.group_m = group_m >= CLUSTER ? group_m / CLUSTER : 1;
    // N super-tiles only where W does not fit the L2 beside the streams (gate|up: 272 MB); 0 / >= num_n = one sweep
    int gn = env_n >= 0 ? env_n : 0;
    if (gn <= 0 || gn > p.num_n) gn = p.num_n;
    p.group_n = gn;
    p.hints = env_h >= 0 ? env_h : 0;
  }
  const int grid = p.num_tiles * CLUSTER < max_ctas ? p.num_tiles * CLUSTER : max_ctas;
  if (CLUSTER == 1) {
    kern<<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(tmA, tmB, p);
  } else {
    cfg.gridDim = dim3((unsigned)grid, 1, 1);
    BAGEL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p));
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <int BN, int EPI, bool CONV = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream,
                       int cluster) {
  if constexpr (!CONV) {
    if (cluster == 2) return launch_gemm_cluster<BN, EPI, CONV, 2>(tmA, tmB, p, stream);
  }
  return launch_gemm_cluster<BN, EPI, CONV, 1>(tmA, tmB, p, stream);
}

template <int BN>
static int dispatch_epi(int epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p,
                        cudaStream_t s, int cluster) {
  switch (epi) {
    case EPI_BIAS: return launch_gemm<BN, EPI_BIAS>(tmA, tmB, p, s, cluster);
    case EPI_RESID: return launch_gemm<BN, EPI_RESID>(tmA, tmB, p, s, cluster);
    case EPI_GELU: return launch_gemm<BN, EPI_GELU>(tmA, tmB, p, s, cluster);
    case EPI_SILU: return launch_gemm<BN, EPI_SILU>(tmA, tmB, p, s, cluster);
    case EPI_F32: return launch_gemm<BN, EPI_F32>(tmA, tmB, p, s, cluster);
    case EPI_RESID_F32: return launch_gemm<BN, EPI_RESID_F32>(tmA, tmB, p, s, cluster);
    default: return set_error(BAGEL_ERR_ARG, "bagel_gemm_bf16: unknown epilogue %d", epi);
  }
}

}  // namespace bagel

using namespace bagel;

extern "C" int bagel_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc,
                               int M, int N, int K, const void* bias, const void* resid, long long ldr,
                               const int* row_map, int epilogue, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_bf16: M,N,K must be > 0");
  if ((lda % 8) || (ldw % 8) || (ldc % 8) || (K % 8) || (N % 8))
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_bf16: K, N and leading dims must be multiples of 8 (16 B)");
  if (((uintptr_t)A | (uintptr_t)W | (uintptr_t)C | (uintptr_t)bias | (uintptr_t)resid) & 15)
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_bf16: pointers must be 16-byte aligned");
  if ((epilogue == EPI_RESID || epilogue == EPI_RESID_F32) && (resid == nullptr || (ldr % 8)))
    return set_error(BAGEL_ERR_ARG, "bagel_gemm_bf16: the residual epilogues need resid with ldr %% 8 == 0");
  if (int rc = require_sm90()) return rc;

  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.C = static_cast<__nv_bfloat16*>(C);
  p.ldc = ldc;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.resid32 = static_cast<const float*>(resid);   // BAGEL_EPI_RESID_F32: resid and C are fp32 [*, ldr] / [*, ldc]
  p.ldr = ldr;
  p.row_map = row_map;
  p.C32 = static_cast<float*>(C);  // used by the fp32-output epilogues (C is then an fp32 [M, ldc] buffer)
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  if (epilogue == EPI_SWIGLU && (N % 256))
    return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_bf16: SwiGLU needs N (=2*I, interleaved) %% 256 == 0");
  // token-by-token decode / und-expert text rows: weight-streaming kernel with swapped operands and cluster split-K
  static const bool skinny_on = [] { const char* e = getenv("BAGEL_GEMM_SKINNY"); return !(e && atoi(e) == 0); }();
  if (skinny_on && gemm_skinny_supported(M, N, K, epilogue))
    return gemm_skinny(A, lda, W, ldw, C, ldc, M, N, K, bias, resid, ldr, row_map, epilogue, s);

  int bn;
  if (epilogue == EPI_SWIGLU) {
    if (N % 256) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_bf16: SwiGLU needs N (=2*I, interleaved) %% 256 == 0");
    bn = 256;
  } else {
    bn = (N % 256 == 0 || N >= 1024) ? 256 : (N > 64 ? 128 : 64);
    // skinny M (text decode, und-expert rows of a MoT layer): the GEMM is a weight stream, so use narrow tiles to put
    // 4x more CTAs (and TMA pipelines) on the W matrix
    if (M <= BM && N >= 1024) bn = (N <= 8192) ? 32 : 64;  // >= 112 CTAs on the 3584/4608-wide projections
  }
  const int cluster = gemm_cluster(M);
  CUtensorMap tmA, tmB;
  if (int rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM)) return rc;
  if (int rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, BK, bn / cluster)) return rc;

  if (epilogue == EPI_SWIGLU) return launch_gemm<256, EPI_SWIGLU>(tmA, tmB, p, s, cluster);
  if (bn == 256) return dispatch_epi<256>(epilogue, tmA, tmB, p, s, cluster);
  if (bn == 128) return dispatch_epi<128>(epilogue, tmA, tmB, p, s, cluster);
  if (bn == 32) return dispatch_epi<32>(epilogue, tmA, tmB, p, s, cluster);
  return dispatch_epi<64>(epilogue, tmA, tmB, p, s, cluster);
}


// ---------------------------------------------------------------------------------------------
// Implicit-GEMM 2-D convolution on NHWC bf16 activations (FLUX VAE: modeling/autoencoder.py:76-80, 102-108,
// 114-119, 139, 170, 221, 248 — the reference runs these as cuDNN NCHW convolutions).
//   out[b, ho, wo, :] = epilogue( sum_{kh,kw,c} x[b, ho*s + kh - pad, wo*s + kw - pad, c] * w[:, kh, kw, c] )
// No im2col buffer: each (tap, 64-channel chunk) K-slice of the A tile is one 4-D TMA box whose signed
// coordinates fall outside the image exactly where the convolution pads with zeros.
// ---------------------------------------------------------------------------------------------
extern "C" int bagel_conv2d_nhwc_bf16(const void* x, int B, int Hi, int Wi, int Cin, const void* w, int Cout, int ksize,
                                      int stride, int pad, const void* bias, const void* resid, void* out, int Ho,
                                      int Wo, void* stream) {
  if (ksize != 1 && ksize != 3) return set_error(BAGEL_ERR_ARG, "bagel_conv2d_nhwc_bf16: ksize must be 1 or 3");
  if (stride != 1 && stride != 2) return set_error(BAGEL_ERR_ARG, "bagel_conv2d_nhwc_bf16: stride must be 1 or 2");
  if (Cin % 64) return set_error(BAGEL_ERR_SHAPE, "bagel_conv2d_nhwc_bf16: Cin must be a multiple of 64 (pad channels)");
  if (Cout % 8) return set_error(BAGEL_ERR_SHAPE, "bagel_conv2d_nhwc_bf16: Cout must be a multiple of 8 (pad filters)");
  if (B <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_conv2d_nhwc_bf16: bad sizes");
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)out | (uintptr_t)bias | (uintptr_t)resid) & 15)
    return set_error(BAGEL_ERR_ALIGN, "bagel_conv2d_nhwc_bf16: pointers must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;

  GemmParams p{};
  p.Ho = Ho; p.Wo = Wo;
  int tw = 128;
  while (tw > Wo) tw >>= 1;  // largest power of two <= min(Wo, 128)
  if (tw < 1) tw = 1;
  p.tw = tw; p.th = 128 / tw;
  p.tiles_w = (Wo + p.tw - 1) / p.tw;
  p.tiles_h = (Ho + p.th - 1) / p.th;
  p.ksize = ksize; p.pad = pad; p.stride = stride; p.cin_chunks = Cin / 64;
  p.M = B * Ho * Wo; p.N = Cout; p.K = ksize * ksize * Cin;
  p.num_m = B * p.tiles_w * p.tiles_h;
  p.C = static_cast<__nv_bfloat16*>(out);
  p.ldc = Cout;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.ldr = Cout;
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  CUtensorMap tmA, tmB;
  if (int rc = make_tmap_4d_nhwc_bf16(&tmA, x, B, Hi, Wi, Cin, 64, p.tw, p.th, stride)) return rc;
  const int bn = (Cout % 256 == 0 || Cout >= 1024) ? 256 : (Cout > 64 ? 128 : 64);
  if (int rc = make_tmap_2d_bf16(&tmB, w, (uint64_t)p.K, (uint64_t)Cout, (uint64_t)p.K, BK, bn)) return rc;
  const bool res = resid != nullptr;
  if (bn == 256) return res ? launch_gemm<256, EPI_RESID, true>(tmA, tmB, p, s, 1) : launch_gemm<256, EPI_BIAS, true>(tmA, tmB, p, s, 1);
  if (bn == 128) return res ? launch_gemm<128, EPI_RESID, true>(tmA, tmB, p, s, 1) : launch_gemm<128, EPI_BIAS, true>(tmA, tmB, p, s, 1);
  return res ? launch_gemm<64, EPI_RESID, true>(tmA, tmB, p, s, 1) : launch_gemm<64, EPI_BIAS, true>(tmA, tmB, p, s, 1);
}


// QKV projection with the whole pre-attention tail fused into the epilogue (head_dim 128):
//   [q|k|v] = A W^T + b ; per-head RMSNorm(q,k) with expert-routed weights ; RoPE ; bf16 ; q -> q_out,
//   k/v -> merged KV buffers at kv_rows[row]. Replaces bagel_gemm_bf16 + bagel_qk_norm_rope (and the [N, 4608]
//   round trip through HBM between them).
extern "C" int bagel_gemm_qkv_norm_rope(const void* A, long long lda, const void* W, long long ldw, const void* bias,
                                        int M, int K, const int* row_map, const void* q_w0, const void* k_w0,
                                        const void* q_w1, const void* k_w1, const uint8_t* expert, const float* cos_t,
                                        const float* sin_t, void* q_out, long long ld_q, void* k_out, void* v_out,
                                        long long ld_kv, const int* kv_rows, int Hq, int Hk, float eps, int fp32_flow,
                                        void* stream) {
  const int N = (Hq + 2 * Hk) * 128;
  if (M <= 0 || K <= 0 || Hq <= 0 || Hk <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_qkv_norm_rope: bad sizes");
  if (N % 256) return set_error(BAGEL_ERR_SHAPE, "bagel_gemm_qkv_norm_rope: Hq + 2*Hk must be even (two heads per tile)");
  if ((lda % 8) || (ldw % 8) || (K % 8) || (ld_q % 8) || (ld_kv % 8))
    return set_error(BAGEL_ERR_ALIGN, "bagel_gemm_qkv_norm_rope: K and leading dims must be multiples of 8");
  if (bias == nullptr || q_w0 == nullptr || k_w0 == nullptr || cos_t == nullptr || sin_t == nullptr)
    return set_error(BAGEL_ERR_ARG, "bagel_gemm_qkv_norm_rope: bias, norm weights and RoPE tables are required");
  if (int rc = require_sm90()) return rc;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.row_map = row_map;
  if (fp32_flow < 0 || fp32_flow > 3) return set_error(BAGEL_ERR_ARG, "bagel_gemm_qkv_norm_rope: flow must be 0..3");
  p.qkv.qw0 = q_w0; p.qkv.kw0 = k_w0;
  p.qkv.qw1 = q_w1; p.qkv.kw1 = k_w1;
  p.qkv.expert = expert; p.qkv.cos_t = cos_t; p.qkv.sin_t = sin_t;
  p.qkv.q_out = static_cast<__nv_bfloat16*>(q_out); p.qkv.k_out = static_cast<__nv_bfloat16*>(k_out);
  p.qkv.v_out = static_cast<__nv_bfloat16*>(v_out);
  p.qkv.ld_q = ld_q; p.qkv.ld_kv = ld_kv; p.qkv.kv_rows = kv_rows;
  p.qkv.Hq = Hq; p.qkv.Hk = Hk; p.qkv.eps = eps; p.qkv.fp32_flow = fp32_flow;
  const int cluster = gemm_cluster(M);
  CUtensorMap tmA, tmB;
  if (int rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM)) return rc;
  if (int rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, BK, 256 / cluster)) return rc;
  return launch_gemm<256, EPI_QKV>(tmA, tmB, p, static_cast<cudaStream_t>(stream), cluster);
}
