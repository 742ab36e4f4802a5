// Batched image generation of independent requests (Bagel.generate_image_batch): the fused CFG + renorm + Euler step of
// bagel_cfg_euler_step with every request as its own segment. Per-request scales, renorm types and the per-step CFG
// switch are read from device memory, so one captured denoising-step graph serves every step of a run.
// No tensor-core code in this translation unit.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "host_util.h"

namespace bagel {

namespace {

__device__ __forceinline__ float rbf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct CfgBatchArgs {
  const __nv_bfloat16* v;
  long long ldv;
  const int *seg, *row_main, *row_text, *row_img;
  float* x;
  int M, C, R;
  const float *sT, *sI, *renorm_min;
  const int *renorm_type, *cfg_on;
  const float* dt_dev;
  float* part;   // [M, 2] per-row sums of v^2 and w^2 (global-renorm rows only)
  float* scale;  // [R] global-renorm scale per request
  int* begin;    // [R] first row of each request (written by pass 1 for every request that has rows)
};

// The branch set a latent row actually uses at this step: text CFG when its request has CFG on, a text-dropped row and
// sT > 1; image CFG inside that when it also has an image-dropped row and sI > 1 (Bagel._cfg_update's rule).
struct RowCfg {
  int q, use_cfg, img, type;
  float sT, sI;
  long long src, srcT, srcI;
};

__device__ __forceinline__ RowCfg row_cfg(const CfgBatchArgs& a, int r) {
  RowCfg c;
  c.q = a.seg[r];
  const int rt = a.row_text[r], ri = a.row_img[r];
  c.sT = a.sT[c.q];
  c.sI = a.sI[c.q];
  c.type = a.renorm_type[c.q];
  c.use_cfg = (a.cfg_on[c.q] != 0 && rt >= 0 && c.sT > 1.0f) ? 1 : 0;
  c.img = (c.use_cfg && ri >= 0 && c.sI > 1.0f) ? 1 : 0;
  c.src = (long long)a.row_main[r] * a.ldv;
  c.srcT = c.use_cfg ? (long long)rt * a.ldv : 0;
  c.srcI = c.img ? (long long)ri * a.ldv : 0;
  return c;
}

// cfg_combine of elementwise.cu with the row's own scales: every op rounds to bf16
__device__ __forceinline__ float combine(const RowCfg& c, float v, float vT, float vI) {
  const float u = rbf16(vT + rbf16(c.sT * rbf16(v - vT)));
  return c.img ? rbf16(vI + rbf16(c.sI * rbf16(u - vI))) : u;
}

}  // namespace

// A request's rows form one run of seg, so a row starts its request iff the row before it belongs to another one.
__device__ __forceinline__ bool run_start(const CfgBatchArgs& a, int r) { return r == 0 || a.seg[r - 1] != a.seg[r]; }

// Pass 1: one warp per latent row. The first row of each request records itself in begin[]; a row of a global-renorm
// request with CFG on writes part[r] = (sum v^2, sum w^2) over the row.
__global__ void __launch_bounds__(128) cfg_batch_rownorm_kernel(const CfgBatchArgs a) {
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= a.M) return;
  if (lane == 0 && run_start(a, r)) a.begin[a.seg[r]] = r;
  const RowCfg c = row_cfg(a, r);
  if (!c.use_cfg || c.type != 0) return;
  float sv = 0.f, sw = 0.f;
  for (int ch = lane; ch < a.C; ch += 32) {
    const float v = __bfloat162float(a.v[c.src + ch]);
    const float vT = __bfloat162float(a.v[c.srcT + ch]);
    const float vI = c.img ? __bfloat162float(a.v[c.srcI + ch]) : 0.f;
    const float w = combine(c, v, vT, vI);
    sv += v * v;
    sw += w * w;
  }
  sv = wsum(sv);
  sw = wsum(sw);
  if (lane == 0) {
    a.part[2LL * r] = sv;
    a.part[2LL * r + 1] = sw;
  }
}

// Pass 2: one block per request, over that request's rows only. Its rows' partials are summed in a fixed order that
// depends only on the request's own rows (thread t takes rows begin + t, begin + t + 256, ... of its run; then a fixed
// tree), so the scale is bit-reproducible and no other request can change it. No atomics. begin[q] is trusted only if
// it is the start of a run of q: a request without rows keeps whatever an earlier launch left there, and that entry
// then fails the test.
constexpr int kNormThreads = 256;
__global__ void __launch_bounds__(kNormThreads) cfg_batch_scale_kernel(const CfgBatchArgs a) {
  const int q = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ float sh[2][kNormThreads / 32];
  const int first = a.begin[q];
  const bool active = a.renorm_type[q] == 0 && a.cfg_on[q] != 0 && first >= 0 && first < a.M && a.seg[first] == q &&
                      run_start(a, first);   // block-uniform
  if (!active) {
    if (tid == 0) a.scale[q] = 1.0f;
    return;
  }
  float sv = 0.f, sw = 0.f;
  for (int r = first + tid; r < a.M; r += kNormThreads) {
    if (a.seg[r] != q) break;        // past the end of the request's run
    const RowCfg c = row_cfg(a, r);
    if (!c.use_cfg) continue;        // a row without a text-dropped branch takes no CFG and adds nothing to the norms
    sv += a.part[2LL * r];
    sw += a.part[2LL * r + 1];
  }
  sv = wsum(sv);
  sw = wsum(sw);
  if (lane == 0) { sh[0][warp] = sv; sh[1][warp] = sw; }
  __syncthreads();
  if (tid == 0) {
    float nv2 = 0.f, nw2 = 0.f;
    for (int w = 0; w < kNormThreads / 32; ++w) { nv2 += sh[0][w]; nw2 += sh[1][w]; }
    const float nv = rbf16(sqrtf(nv2)), nw = rbf16(sqrtf(nw2));
    a.scale[q] = fminf(fmaxf(rbf16(nv / rbf16(nw + 1e-8f)), a.renorm_min[q]), 1.0f);
  }
}

// Pass 3: one warp per latent row (up to 4 channels per lane), the arithmetic of cfg_apply_kernel with the row's
// request parameters.
__global__ void __launch_bounds__(128) cfg_batch_apply_kernel(const CfgBatchArgs a) {
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= a.M) return;
  const RowCfg c = row_cfg(a, r);
  const float rmin = a.renorm_min[c.q];
  const float gscale = (c.use_cfg && c.type == 0) ? a.scale[c.q] : 1.f;
  float ww[4];
  float sv = 0.f, sw = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {   // channels lane, lane + 32, ... (C <= 128): a fixed trip count keeps ww in registers
    const int ch = lane + 32 * k;
    if (ch >= a.C) break;
    const float v = __bfloat162float(a.v[c.src + ch]);
    float w = v;
    if (c.use_cfg) {
      const float vT = __bfloat162float(a.v[c.srcT + ch]);
      const float vI = c.img ? __bfloat162float(a.v[c.srcI + ch]) : 0.f;
      if (c.type == 2) {
        w = rbf16(vT + rbf16(c.sT * rbf16(v - vT)));  // u; image CFG applied after renorm
      } else {
        w = combine(c, v, vT, vI);
      }
    }
    ww[k] = w;
    sv += v * v;
    sw += w * w;
  }
  const float dt = *a.dt_dev;
  float scale = gscale;
  if (c.use_cfg && c.type != 0) {
    sv = wsum(sv);
    sw = wsum(sw);
    const float nv = rbf16(sqrtf(sv)), nw = rbf16(sqrtf(sw));
    scale = fminf(fmaxf(rbf16(nv / rbf16(nw + 1e-8f)), rmin), 1.0f);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int ch = lane + 32 * k;
    if (ch >= a.C) break;
    float w = ww[k];
    if (c.use_cfg) {
      w = rbf16(w * scale);
      if (c.type == 2 && c.img) {
        const float vI = __bfloat162float(a.v[c.srcI + ch]);
        w = rbf16(vI + rbf16(c.sI * rbf16(w - vI)));
      }
    }
    float* xp = a.x + (long long)r * a.C + ch;
    *xp = *xp - rbf16(w * dt);
  }
}

}  // namespace bagel

using namespace bagel;

#define COUNT_LAUNCH() g_launches.fetch_add(1, std::memory_order_relaxed)

extern "C" int bagel_cfg_euler_step_batch(const void* v, long long ldv, const int* seg, const int* row_main,
                                          const int* row_text, const int* row_img, float* x, int M, int C, int R,
                                          const float* cfg_text_scale, const float* cfg_img_scale,
                                          const float* renorm_min, const int* renorm_type, const int* cfg_on,
                                          const float* dt_dev, float* workspace, void* stream) {
  if (M <= 0) return 0;
  if (C <= 0 || C > 128) return set_error(BAGEL_ERR_SHAPE, "bagel_cfg_euler_step_batch: C must be in [1, 128]");
  if (R <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_cfg_euler_step_batch: R must be > 0");
  if (ldv < C) return set_error(BAGEL_ERR_SHAPE, "bagel_cfg_euler_step_batch: ldv must be >= C");
  if (!v || !seg || !row_main || !row_text || !row_img || !x || !cfg_text_scale || !cfg_img_scale || !renorm_min ||
      !renorm_type || !cfg_on || !dt_dev || !workspace)
    return set_error(BAGEL_ERR_ARG, "bagel_cfg_euler_step_batch: every pointer argument is required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CfgBatchArgs a{};
  a.v = static_cast<const __nv_bfloat16*>(v);
  a.ldv = ldv; a.seg = seg; a.row_main = row_main; a.row_text = row_text; a.row_img = row_img;
  a.x = x; a.M = M; a.C = C; a.R = R;
  a.sT = cfg_text_scale; a.sI = cfg_img_scale; a.renorm_min = renorm_min; a.renorm_type = renorm_type;
  a.cfg_on = cfg_on; a.dt_dev = dt_dev;
  a.part = workspace;
  a.scale = workspace + 2LL * M;
  a.begin = reinterpret_cast<int*>(workspace + 2LL * M + R);
  // the renorm types and the CFG switch live on the device: the two norm passes always run and skip rows and requests
  // that take no global renorm at this step (a fixed launch sequence whatever the step and the mix of requests)
  cfg_batch_rownorm_kernel<<<(M + 3) / 4, 128, 0, s>>>(a);
  COUNT_LAUNCH();
  cfg_batch_scale_kernel<<<R, kNormThreads, 0, s>>>(a);
  COUNT_LAUNCH();
  cfg_batch_apply_kernel<<<(M + 3) / 4, 128, 0, s>>>(a);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}
