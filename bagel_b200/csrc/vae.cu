// HBM-bound kernels of the FLUX VAE (modeling/autoencoder.py): GroupNorm(32)+swish on NHWC activations,
// nearest 2x upsampling, row softmax for the single-head d=512 mid attention, bf16 transpose.
// The convolutions themselves are the implicit-GEMM wgmma kernel in gemm.cu (bagel_conv2d_nhwc_bf16).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "host_util.h"

namespace bagel {

// ---------------------------------------------------------------------------------------------
// GroupNorm statistics, pass 1: partial (sum, sum of squares) per (image, slab, group).
// x: [B, HW, C] bf16 (NHWC), G groups of C/G consecutive channels. Deterministic: no atomics, the slabs are
// reduced in a fixed order by pass 2. HBM-bound: the grid is sized so that every SM holds several CTAs and every
// thread keeps four 16-byte loads in flight (round 1 launched 64 CTAs with one load per thread in flight per image:
// 0.24 TB/s at 1024^2 x 128 channels, a third of the whole VAE decode).
// ---------------------------------------------------------------------------------------------
constexpr int kGnMaxSlabs = 1024;

__global__ void __launch_bounds__(256)
gn_partial_kernel(const __nv_bfloat16* __restrict__ x, float2* __restrict__ partial, long long HW, int C, int G,
                  int slabs) {
  const int b = blockIdx.y, slab = blockIdx.x;
  const int cpg = C / G;
  const int vec_per_pix = C >> 3;  // 16-byte vectors per pixel
  const long long pix0 = HW * slab / slabs, pix1 = HW * (slab + 1) / slabs;
  const long long nvec = (pix1 - pix0) * vec_per_pix;
  const uint4* base = reinterpret_cast<const uint4*>(x + ((long long)b * HW + pix0) * C);
  __shared__ float4 part[256];  // per-thread (s0, q0, s1, q1); reduced in a fixed order -> deterministic
  // a thread always visits the same vector slot of a pixel (blockDim % vec_per_pix == 0 is guaranteed by the host:
  // vec_per_pix in {16,32,64}), so its channels -> groups mapping is fixed
  const int slot = threadIdx.x % vec_per_pix;
  const int c0 = slot * 8;
  float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
  const int g0 = c0 / cpg;  // a vector of 8 channels spans 1 or 2 groups when cpg >= 4
  float m0[4];              // 1 if channel pair e belongs to the vector's first group, else 0 (no dynamic register indexing)
#pragma unroll
  for (int e = 0; e < 4; ++e) m0[e] = ((c0 + 2 * e) / cpg == g0) ? 1.0f : 0.0f;
  auto acc = [&](const uint4& v) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a = bf16_lo(u[e]), c = bf16_hi(u[e]);
      const float sm = a + c, sq = fmaf(a, a, c * c);
      s0 = fmaf(m0[e], sm, s0); q0 = fmaf(m0[e], sq, q0);
      s1 = fmaf(1.0f - m0[e], sm, s1); q1 = fmaf(1.0f - m0[e], sq, q1);
    }
  };
  long long i = threadIdx.x;
  for (; i + 3 * 256 < nvec; i += 4 * 256) {   // four independent loads in flight per thread
    const uint4 v0 = base[i], v1 = base[i + 256], v2 = base[i + 512], v3 = base[i + 768];
    acc(v0); acc(v1); acc(v2); acc(v3);
  }
  for (; i < nvec; i += 256) acc(base[i]);
  part[threadIdx.x] = make_float4(s0, q0, s1, q1);
  __syncthreads();
  if (threadIdx.x < G) {
    const int g = threadIdx.x;
    float ss = 0.f, qq = 0.f;
    for (int t = 0; t < (int)blockDim.x; ++t) {
      const int tc0 = (t % vec_per_pix) * 8;
      const int tg0 = tc0 / cpg, tg1 = (tc0 + 7) / cpg;
      const float4 v = part[t];
      if (tg0 == g) { ss += v.x; qq += v.y; }
      if (tg1 == g && tg1 != tg0) { ss += v.z; qq += v.w; }
    }
    partial[((long long)b * slabs + slab) * G + g] = make_float2(ss, qq);
  }
}

// pass 2: reduce slabs -> (mean, rstd) per (image, group). One CTA per (group, image): thread t sums slabs t, t+256, ...
// (all its loads in flight at once), then a fixed-order tree over the 256 partial sums in shared memory: deterministic.
// (The previous version walked up to 1024 slabs with 8 threads per group in ONE CTA: 32 dependent rounds of loads = 20 us
// per GroupNorm, 0.6 ms per VAE decode.)
__global__ void __launch_bounds__(256)
gn_finalize_kernel(const float2* __restrict__ partial, float2* __restrict__ stats, int G, int slabs, float count,
                   float eps) {
  const int g = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  __shared__ double sh_s[256], sh_q[256];
  const float2* base = partial + (long long)b * slabs * G + g;
  double s = 0.0, q = 0.0;
  int i = t;
  if (i + 768 < slabs) {   // the common case (1024 slabs): four independent loads in flight
    const float2 p0 = base[(long long)i * G], p1 = base[(long long)(i + 256) * G];
    const float2 p2 = base[(long long)(i + 512) * G], p3 = base[(long long)(i + 768) * G];
    s = ((double)p0.x + p1.x) + ((double)p2.x + p3.x);
    q = ((double)p0.y + p1.y) + ((double)p2.y + p3.y);
    i += 1024;
  }
  for (; i < slabs; i += 256) {
    const float2 p = base[(long long)i * G];
    s += p.x;
    q += p.y;
  }
  sh_s[t] = s;
  sh_q[t] = q;
  __syncthreads();
#pragma unroll
  for (int w = 128; w > 0; w >>= 1) {
    if (t < w) {
      sh_s[t] += sh_s[t + w];
      sh_q[t] += sh_q[t + w];
    }
    __syncthreads();
  }
  if (t == 0) {
    const double mean = sh_s[0] / count;
    const double var = fmax(sh_q[0] / count - mean * mean, 0.0);
    stats[b * G + g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

// pass 3: y = bf16( act( (x - mean) * rstd * w + b ) ), act = swish (x * sigmoid(x)) or identity. A thread owns one
// 8-channel slot of the pixel (grid stride is a multiple of the vectors per pixel), so its affine parameters and group
// statistics are loaded ONCE; the loop is load / 8 FMA (+ swish) / store with four vectors in flight.
__global__ void __launch_bounds__(256)
gn_apply_kernel(const __nv_bfloat16* __restrict__ x, const float2* __restrict__ stats, const float* __restrict__ w,
                const float* __restrict__ bias, __nv_bfloat16* __restrict__ y, long long HW, int C, int G,
                int swish, long long vec_per_image) {
  const int cpg = C / G;
  const int vec_per_pix = C >> 3;
  const int b = blockIdx.y;
  const long long stride = (long long)gridDim.x * blockDim.x;          // multiple of vec_per_pix (256 % vpp == 0)
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c0 = (int)(i % vec_per_pix) * 8;
  float sc[8], sh[8];   // y = x * sc + sh  with sc = rstd * w, sh = b - mean * rstd * w  (same value, fewer ops per element:
                        // (x - mean) * rstd * w + b evaluated as one FMA; fp32, far below the bf16 output rounding)
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float2 st = stats[b * G + (c0 + e) / cpg];
    const float ww = w[c0 + e];
    sc[e] = st.y * ww;
    sh[e] = bias[c0 + e] - st.x * st.y * ww;
  }
  const uint4* xi = reinterpret_cast<const uint4*>(x) + (long long)b * vec_per_image;
  uint4* yo = reinterpret_cast<uint4*>(y) + (long long)b * vec_per_image;
  auto one = [&](const uint4& v) -> uint4 {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float a = fmaf(bf16_lo(u[e]), sc[2 * e], sh[2 * e]);
      float c = fmaf(bf16_hi(u[e]), sc[2 * e + 1], sh[2 * e + 1]);
      if (swish) {
        a = __fdividef(a, 1.0f + __expf(-a));
        c = __fdividef(c, 1.0f + __expf(-c));
      }
      o[e] = pack_bf16x2(a, c);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  for (; i + 3 * stride < vec_per_image; i += 4 * stride) {
    const uint4 v0 = xi[i], v1 = xi[i + stride], v2 = xi[i + 2 * stride], v3 = xi[i + 3 * stride];
    yo[i] = one(v0); yo[i + stride] = one(v1); yo[i + 2 * stride] = one(v2); yo[i + 3 * stride] = one(v3);
  }
  for (; i < vec_per_image; i += stride) yo[i] = one(xi[i]);
}

// nearest-neighbour 2x upsample, NHWC: y[b, 2h+i, 2w+j, :] = x[b, h, w, :]
__global__ void __launch_bounds__(256)
upsample2x_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int H, int W, int C,
                  long long total_vec) {
  const int vpp = C >> 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpp);
    long long pix = i / vpp;
    const int wo = (int)(pix % (2 * W));
    pix /= 2 * W;
    const int ho = (int)(pix % (2 * H));
    const long long b = pix / (2 * H);
    const long long src = ((b * H + (ho >> 1)) * W + (wo >> 1)) * vpp + v;
    reinterpret_cast<uint4*>(y)[i] = reinterpret_cast<const uint4*>(x)[src];
  }
}

// P[r, :] = bf16(softmax(S[r, :] * scale)) — one block per row, fp32 logits (VAE mid attention, d = 512).
// kPer > 0: the row (L <= 256 * kPer) is read ONCE into registers (max, sum and output from the same values: 1 read +
// 1 bf16 write instead of three fp32 passes); kPer = 0: any L, three passes.
template <int kPer>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ S, long long lds, __nv_bfloat16* __restrict__ P, long long ldp, int L,
                    float scale_log2) {
  const long long r = blockIdx.x;
  const float* s = S + r * lds;
  __shared__ float red[8];
  float v[kPer > 0 ? kPer : 1];
  float mx = -INFINITY;
  if constexpr (kPer > 0) {
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = threadIdx.x + k * 256;
      v[k] = (i < L) ? s[i] : -INFINITY;
      mx = fmaxf(mx, v[k]);
    }
  } else {
    for (int i = threadIdx.x; i < L; i += blockDim.x) mx = fmaxf(mx, s[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  if constexpr (kPer > 0) {
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      v[k] = exp2f((v[k] - mx) * scale_log2);     // -inf padding -> 0
      sum += v[k];
    }
  } else {
    for (int i = threadIdx.x; i < L; i += blockDim.x) sum += exp2f((s[i] - mx) * scale_log2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  __nv_bfloat16* p = P + r * ldp;
  if constexpr (kPer > 0) {
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = threadIdx.x + k * 256;
      if (i < L) p[i] = __float2bfloat16_rn(v[k] * inv);
    }
  } else {
    for (int i = threadIdx.x; i < L; i += blockDim.x) p[i] = __float2bfloat16_rn(exp2f((s[i] - mx) * scale_log2) * inv);
  }
}

// y[c, r] = x[r, c]  (bf16, 32x32 smem tiles)
__global__ void __launch_bounds__(256)
transpose_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ y, long long ldy,
                 int R, int Cc) {
  __shared__ __nv_bfloat16 t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    t[i][threadIdx.x] = (r < R && c < Cc) ? x[(long long)r * ldx + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < Cc && r < R) y[(long long)c * ldy + r] = t[threadIdx.x][i];
  }
}

}  // namespace bagel

using namespace bagel;
#define COUNT_LAUNCH() g_launches.fetch_add(1, std::memory_order_relaxed)

extern "C" long long bagel_groupnorm_workspace_bytes(int B, int groups) {
  return (long long)B * kGnMaxSlabs * groups * sizeof(float2) + (long long)B * groups * sizeof(float2);
}

extern "C" int bagel_groupnorm_nhwc_bf16(const void* x, const void* w, const void* b, void* y, void* workspace, int B,
                                         long long HW, int C, int groups, float eps, int swish, void* stream) {
  if (B <= 0 || HW <= 0) return 0;
  if (groups != 32) return set_error(BAGEL_ERR_ARG, "bagel_groupnorm_nhwc_bf16: groups must be 32");
  const int vpp = C / 8;
  if (C % 128 || (256 % vpp) != 0) return set_error(BAGEL_ERR_SHAPE, "bagel_groupnorm_nhwc_bf16: C must be 128, 256 or 512");
  if (workspace == nullptr) return set_error(BAGEL_ERR_ARG, "bagel_groupnorm_nhwc_bf16: workspace required");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // enough slabs for ~4 CTAs per SM over the batch, at least 64 pixels per slab, at most kGnMaxSlabs (workspace size)
  long long want = (148LL * 4 + B - 1) / B;
  if (want > HW / 64) want = HW / 64;
  if (want > kGnMaxSlabs) want = kGnMaxSlabs;
  if (want < 1) want = 1;
  const int slabs = (int)want;
  float2* partial = static_cast<float2*>(workspace);
  float2* stats = partial + (long long)B * kGnMaxSlabs * groups;
  auto X = static_cast<const __nv_bfloat16*>(x);
  gn_partial_kernel<<<dim3(slabs, B), 256, 0, s>>>(X, partial, HW, C, groups, slabs);
  COUNT_LAUNCH();
  gn_finalize_kernel<<<dim3(groups, B), 256, 0, s>>>(partial, stats, groups, slabs, (float)((double)HW * (C / groups)), eps);
  COUNT_LAUNCH();
  const long long vec_per_image = HW * vpp;
  long long blocks = (vec_per_image + 256 * 4 - 1) / (256 * 4);
  const long long cap = (148LL * 16 + B - 1) / B;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  gn_apply_kernel<<<dim3((unsigned)blocks, B), 256, 0, s>>>(X, stats, static_cast<const float*>(w), static_cast<const float*>(b),
                                                            static_cast<__nv_bfloat16*>(y), HW, C, groups, swish, vec_per_image);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_upsample2x_nhwc_bf16(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  if (C % 8) return set_error(BAGEL_ERR_SHAPE, "bagel_upsample2x_nhwc_bf16: C %% 8");
  const long long total_vec = (long long)B * 4 * H * W * (C / 8);
  if (total_vec <= 0) return 0;
  long long blocks = (total_vec + 255) / 256;
  if (blocks > 148 * 16) blocks = 148 * 16;
  upsample2x_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), H, W, C, total_vec);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_softmax_rows_f32(const float* S, long long lds, void* P, long long ldp, int rows, int L,
                                      float scale, void* stream) {
  if (rows <= 0 || L <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto Pb = static_cast<__nv_bfloat16*>(P);
  const float sl2 = scale * 1.4426950408889634f;
  if (L <= 256 * 8) softmax_rows_kernel<8><<<rows, 256, 0, st>>>(S, lds, Pb, ldp, L, sl2);
  else if (L <= 256 * 32) softmax_rows_kernel<32><<<rows, 256, 0, st>>>(S, lds, Pb, ldp, L, sl2);
  else if (L <= 256 * 64) softmax_rows_kernel<64><<<rows, 256, 0, st>>>(S, lds, Pb, ldp, L, sl2);
  else softmax_rows_kernel<0><<<rows, 256, 0, st>>>(S, lds, Pb, ldp, L, sl2);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_transpose_bf16(const void* x, long long ldx, void* y, long long ldy, int R, int Cc, void* stream) {
  if (R <= 0 || Cc <= 0) return 0;
  transpose_kernel<<<dim3((Cc + 31) / 32, (R + 31) / 32), dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), ldx, static_cast<__nv_bfloat16*>(y), ldy, R, Cc);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}
