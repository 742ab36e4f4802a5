// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
// Everything here is a device-side primitive used by gemm.cu / gemm_skinny.cu / attn.cu; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace bagel {

// ---------------------------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trap (-> cudaErrorLaunchFailure on the host), never as a
// hung GPU. ~4e9 cycles is seconds of wall clock, far beyond any legitimate wait in these kernels.
// The diagnostic message is a debug build only (-DBAGEL_MBAR_TRACE, see tools/build_variant.py): printf is a call
// (vprintf), and a call anywhere on a path that runs while a wgmma group is in flight makes ptxas serialize every
// wgmma of the kernel (C7510 "wgmma pipeline crossing function boundary").
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
#ifdef BAGEL_MBAR_TRACE
      printf("bagel_b200: mbarrier wait timed out (block %d thread %d bar %u parity %u)\n", blockIdx.x,
             threadIdx.x, smem_u32(bar), parity);
#endif
      __trap();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// thread-block clusters: rank, cluster-wide barrier, distributed shared memory
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// Every thread of every CTA of the cluster (aligned: each warp converged).
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Address of the same shared-memory offset in the CTA of rank `rank` of this cluster.
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local_addr, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_addr), "r"(rank));
  return remote;
}
__device__ __forceinline__ float ld_dsmem_f32(uint32_t local_addr, uint32_t rank) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(mapa_shared(local_addr, rank)) : "memory");
  return v;
}
// Arrive on the mbarrier at the same offset in the CTA of rank `rank` (default semantics: release at CTA scope). Meant for
// handing back a slot whose readers were async-proxy operations that have already completed (wgmma after
// wgmma.wait_group): a .release.cluster arrive would put a MEMBAR.GPU in front of every arrive.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(mapa_shared(smem_u32(bar), rank)) : "memory");
}

// Exactly one lane of a CONVERGED warp (elect.sync): guards single-thread TMA issue; with it ptxas knows that one thread
// runs the region, behind `lane == 0` it has to assume divergence.
__device__ __forceinline__ bool elect_one_lane() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor is still running; it must execute pdl_wait() before touching anything the predecessor
// produces (or writing anything it reads). pdl_launch_dependents() lets the NEXT such kernel start early.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// L2 cache-policy words (same encodings CUTLASS uses for TMA cache hints)
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1,
                                            uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}
// The box lands at the same shared-memory offset in every CTA of `cta_mask` (bit r = cluster rank r), and each of those
// CTAs' mbarrier at the offset of `bar` receives the complete_tx of the bytes written into that CTA.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma: shared-memory matrix descriptors, fences, the M = 64 warpgroup MMA
// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (PTX "matrix-descriptor", sm_90 wgmma flavour):
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base_offset | [62,64) layout (1 = SWIZZLE_128B)
// K-major SWIZZLE_128B operand tile: rows are 128 B apart, 8-row groups are 1024 B apart (SBO); LBO unused (1).
// Advancing 16 elements (32 B) along K inside the 128 B swizzle atom is +2 in the start field.
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// MN-major SWIZZLE_128B operand tile (V in P*V): along MN 64 elements (128 B) are contiguous and the next 64-element
// block is LBO bytes away; along K rows are 128 B apart, 8-row groups SBO (= 1024) apart.
__device__ __forceinline__ uint64_t gmma_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// Register operands of an in-flight wgmma must not be touched (or moved) by the compiler until wgmma_wait retires it.
template <int N>
__device__ __forceinline__ void gmma_fence_operand(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands in shared memory; issued by all 128 threads of a warpgroup.
template <int N, int kTnspB = 0>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (N == 16) wgmma_ss_n16<kTnspB>(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 32) wgmma_ss_n32<kTnspB>(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 64) wgmma_ss_n64<kTnspB>(d, a_desc, b_desc, scale_d);
  else if constexpr (N == 128) wgmma_ss_n128<kTnspB>(d, a_desc, b_desc, scale_d);
  else {
    static_assert(N == 256, "wgmma_ss: N in {16, 32, 64, 128, 256}");
    wgmma_ss_n256<kTnspB>(d, a_desc, b_desc, scale_d);
  }
}
// D[64 x N] (+)= A[64 x 16] (registers) * B[16 x N] (shared memory)
template <int N, int kTnspB>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  if constexpr (N == 64) wgmma_rs_n64<kTnspB>(d, a, b_desc, scale_d);
  else {
    static_assert(N == 128, "wgmma_rs: N in {64, 128}");
    wgmma_rs_n128<kTnspB>(d, a, b_desc, scale_d);
  }
}

// Warp-specialised kernels: the producer warpgroup gives registers back, the MMA warpgroups take them.
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// ---------------------------------------------------------------------------------------------
// numerics helpers: explicit bf16 rounding points (the reference's autocast casts, SURVEY.md §8a)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

}  // namespace bagel
