// Host-side helpers shared by the C-ABI translation units: error reporting, device queries, TMA descriptors.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/bagel_b200.h"

namespace bagel {

extern std::atomic<long long> g_launches;       // kernels launched by this library (bagel_launch_count)
int set_error(int code, const char* fmt, ...);  // records thread-local message, returns `code`
int sm_count();                                 // SMs of the current device (cached per device)
int require_sm90();                             // 0 if current device is sm_90, else BAGEL_ERR_ARCH
// 2D bf16 tensor map: global [rows, cols] with row pitch `ld` elements; box [box_rows, box_cols];
// 128-byte swizzle; out-of-bounds reads are zero-filled.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld,
                      uint32_t box_cols, uint32_t box_rows);

// 2D bf16 tensor map for TMA STORES of [box_rows, box_cols] sub-tiles (box_cols * 2 = 64 bytes, 64-byte swizzle).
int make_tmap_2d_bf16_store(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld,
                            uint32_t box_cols, uint32_t box_rows);

// 4-D bf16 tensor map over an NHWC activation [B, H, W, C]: box [1, box_h, box_w, box_c] output pixels, traversal
// stride `stride` along W and H (strided convolutions), 128-byte swizzle, zero fill outside the tensor.
int make_tmap_4d_nhwc_bf16(CUtensorMap* out, const void* base, int B, int H, int W, int C, uint32_t box_c,
                           uint32_t box_w, uint32_t box_h, uint32_t stride);

// Launch with (optionally) the programmatic-dependent-launch attribute: the kernel may become resident while its predecessor
// in the stream is still running; it must execute griddepcontrol.wait (pdl_wait()) before touching the predecessor's data.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_maybe_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                                    Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// BAGEL_PDL_SMALL=1: also launch the small glue kernels of a decode step (RMSNorm, q/k-norm + RoPE) with the PDL attribute
bool pdl_small_enabled();

#define BAGEL_CUDA_CHECK(expr)                                                                       \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return ::bagel::set_error(BAGEL_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                __FILE__, __LINE__);                                                 \
  } while (0)

}  // namespace bagel
