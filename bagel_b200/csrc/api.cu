// C-ABI plumbing: error reporting, device queries, TMA descriptor encoding.
#include <atomic>
#include <mutex>

#include "host_util.h"

namespace bagel {

static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

struct DevInfo {
  bool known = false;
  int sms = 0;
  int major = 0;
};
static DevInfo g_dev[64];
static std::mutex g_dev_mu;

static const DevInfo& dev_info() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  DevInfo& d = g_dev[dev];
  if (!d.known) {
    cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&d.major, cudaDevAttrComputeCapabilityMajor, dev);
    d.known = true;
  }
  return d;
}

int sm_count() { return dev_info().sms; }

bool pdl_small_enabled() {
  static const bool on = [] { const char* e = getenv("BAGEL_PDL_SMALL"); return e && atoi(e) != 0; }();
  return on;
}

int require_sm90() {
  const DevInfo& d = dev_info();
  if (d.major != 9)
    return set_error(BAGEL_ERR_ARCH, "bagel_b200 kernels are sm_90a only; current device is sm_%d*", d.major * 10);
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld,
                      uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) base=%p cols=%llu rows=%llu ld=%llu box=%ux%u",
                     (int)r, base, (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld,
                     box_cols, box_rows);
  return 0;
}

// Store-side map: box [box_rows, box_cols] with box_cols * 2 == 64 bytes and 64-byte swizzle (the epilogue warps stage
// 32 x 32 bf16 sub-tiles: the 16-byte chunk index of a row is XORed with (row >> 1) & 3, which makes their 16-byte
// shared-memory writes conflict-free). Rows / columns beyond the tensor are clipped by the TMA unit.
int make_tmap_2d_bf16_store(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld,
                            uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled(store) failed (%d) base=%p cols=%llu rows=%llu ld=%llu", (int)r,
                     base, (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld);
  return 0;
}

int make_tmap_4d_nhwc_bf16(CUtensorMap* out, const void* base, int B, int H, int W, int C, uint32_t box_c,
                           uint32_t box_w, uint32_t box_h, uint32_t stride) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  // with an element stride s the box spans box*s source elements and copies every s-th one
  cuuint32_t box[4] = {box_c, box_w * stride, box_h * stride, 1};
  cuuint32_t estr[4] = {1, stride, stride, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(BAGEL_ERR_CUDA, "cuTensorMapEncodeTiled(4d) failed (%d) dims=[%d,%d,%d,%d] box=[%u,%u,%u] stride=%u",
                     (int)r, C, W, H, B, box_c, box_w, box_h, stride);
  return 0;
}

}  // namespace bagel

extern "C" const char* bagel_last_error(void) { return bagel::g_err; }
extern "C" int bagel_abi_version(void) { return 3; }
extern "C" long long bagel_launch_count(void) { return bagel::g_launches.load(); }
