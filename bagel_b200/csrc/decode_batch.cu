// Batched text decode of independent requests (Bagel.generate_text_batch): on-device sampling and per-request stopping.
// Both kernels keep their state in device memory, so a whole decode step stays one replayable CUDA graph.
// No tensor-core code in this translation unit.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "host_util.h"

namespace bagel {

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), counter-based: the draw for
// (key, counter) needs no state and no sequence position, so every logit of every row gets its own uniform.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// Gumbel-perturbed score of one logit: l / T - log(-log u), u = (top 23 bits of x + 0.5) * 2^-23. The sum needs at
// most 24 significant bits, so it is exact in fp32 and u lies in [2^-24, 1 - 2^-24], strictly inside (0, 1). (With 24
// bits, x >> 8 = 2^24 - 1 would round 2^24 - 0.5 up to 2^24: u = 1, score +inf, a pick that ignores the logits.)
// logf (not __logf): -log(u) is ~6e-8 for u next to 1, where an absolute-error log would lose every digit.
__device__ __forceinline__ float gumbel_score(float logit, float inv_t, uint32_t x) {
  const float u = (static_cast<float>(x >> 9) + 0.5f) * 1.1920928955078125e-7f;
  return logit * inv_t - logf(-logf(u));
}

__device__ __forceinline__ float bf16_lo_f(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi_f(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

// One block per row, like argmax_rows_kernel: the argmax of the Gumbel-perturbed scores is a draw from
// softmax(logits / T) (Gumbel-max). Counter of logit j at decode step s: (s, j / 4, 0, 0), word j % 4; key = the row's
// 64-bit key split (low, high) = (seed, request id). Ties go to the lowest index.
// kSample = false scores each logit by its own value: argmax_rows_kernel's pick (first maximum, same NaN / -inf
// handling), for the greedy rows of a mixed batch.
constexpr int kSampleThreads = 1024;
template <bool kSample>
__device__ __forceinline__ void pick_row(const __nv_bfloat16* __restrict__ logits, long long ld, int V, float inv_t,
                                         const long long* __restrict__ keys, const int* __restrict__ step_dev,
                                         long long* __restrict__ tokens, int* __restrict__ tokens32) {
  const __nv_bfloat16* row = logits + (long long)blockIdx.x * ld;
  uint32_t k0 = 0, k1 = 0, step = 0;
  if constexpr (kSample) {
    const unsigned long long key = static_cast<unsigned long long>(keys[blockIdx.x]);
    k0 = static_cast<uint32_t>(key);
    k1 = static_cast<uint32_t>(key >> 32);
    step = static_cast<uint32_t>(step_dev[0]);
  }
  float best = -INFINITY;
  int bi = 0x7fffffff;
  auto take = [&](float v, int i) {
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
  };
  int vec_end = 0;
  if ((ld % 8) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    vec_end = V & ~7;
    for (int i = threadIdx.x * 8; i < vec_end; i += kSampleThreads * 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(row + i);
      if constexpr (kSample) {
        const uint4 r0 = philox4x32_10(make_uint4(step, (uint32_t)i >> 2, 0u, 0u), k0, k1);
        const uint4 r1 = philox4x32_10(make_uint4(step, ((uint32_t)i >> 2) + 1u, 0u, 0u), k0, k1);
        take(gumbel_score(bf16_lo_f(u.x), inv_t, r0.x), i);     take(gumbel_score(bf16_hi_f(u.x), inv_t, r0.y), i + 1);
        take(gumbel_score(bf16_lo_f(u.y), inv_t, r0.z), i + 2); take(gumbel_score(bf16_hi_f(u.y), inv_t, r0.w), i + 3);
        take(gumbel_score(bf16_lo_f(u.z), inv_t, r1.x), i + 4); take(gumbel_score(bf16_hi_f(u.z), inv_t, r1.y), i + 5);
        take(gumbel_score(bf16_lo_f(u.w), inv_t, r1.z), i + 6); take(gumbel_score(bf16_hi_f(u.w), inv_t, r1.w), i + 7);
      } else {
        take(bf16_lo_f(u.x), i);     take(bf16_hi_f(u.x), i + 1);
        take(bf16_lo_f(u.y), i + 2); take(bf16_hi_f(u.y), i + 3);
        take(bf16_lo_f(u.z), i + 4); take(bf16_hi_f(u.z), i + 5);
        take(bf16_lo_f(u.w), i + 6); take(bf16_hi_f(u.w), i + 7);
      }
    }
  }
  for (int i = vec_end + threadIdx.x; i < V; i += kSampleThreads) {
    if constexpr (kSample) {
      const uint4 r = philox4x32_10(make_uint4(step, (uint32_t)i >> 2, 0u, 0u), k0, k1);
      const int w = i & 3;
      const uint32_t x = w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
      take(gumbel_score(__bfloat162float(row[i]), inv_t, x), i);
    } else {
      take(__bfloat162float(row[i]), i);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  __shared__ float sv[kSampleThreads / 32];
  __shared__ int si[kSampleThreads / 32];
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x];
    bi = si[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) {
      if (bi == 0x7fffffff) bi = 0;   // all-NaN / all -inf row: an in-range index, as argmax_rows
      tokens[blockIdx.x] = bi;
      if (tokens32) tokens32[blockIdx.x] = bi;
    }
  }
}

__global__ void __launch_bounds__(kSampleThreads)
sample_rows_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, float inv_t,
                   const long long* __restrict__ keys, const int* __restrict__ step_dev, long long* __restrict__ tokens,
                   int* __restrict__ tokens32) {
  pick_row<true>(logits, ld, V, inv_t, keys, step_dev, tokens, tokens32);
}

// Per-row settings: row b is greedy when inv_temperature[b] == 0, else sampled at inv_t = inv_temperature[b]. The branch
// is uniform over the block, so each row runs exactly the code of the single-setting kernel it matches.
__global__ void __launch_bounds__(kSampleThreads)
sample_rows_mixed_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V,
                         const float* __restrict__ inv_temperature, const long long* __restrict__ keys,
                         const int* __restrict__ step_dev, long long* __restrict__ tokens, int* __restrict__ tokens32) {
  const float inv_t = inv_temperature[blockIdx.x];
  if (inv_t == 0.0f) pick_row<false>(logits, ld, V, 0.0f, keys, step_dev, tokens, tokens32);
  else pick_row<true>(logits, ld, V, inv_t, keys, step_dev, tokens, tokens32);
}

// Per-request stopping. A live request records its current token, then either takes next[b] (seq_len / pos advance)
// or finishes: next[b] is the end token, or its history is full. A finished request keeps its token, seq_len and pos,
// so the step it keeps running rewrites its own last K/V slot with the same values and never leaves its slab.
__global__ void decode_advance_stop_kernel(int* __restrict__ seq_len, long long* __restrict__ pos,
                                           long long* __restrict__ tokens, int* __restrict__ tokens32,
                                           const long long* __restrict__ next, long long* __restrict__ history,
                                           int* __restrict__ step_dev, int* __restrict__ finished,
                                           int* __restrict__ unfinished, long long end_token_id, int max_length,
                                           long long pad, int B) {
  const int b = threadIdx.x;
  const int step = step_dev[0];
  int live = 0;
  if (b < B) {
    long long* h = step < max_length ? history + (long long)step * B + b : nullptr;
    if (finished[b]) {
      if (h) *h = pad;
    } else {
      if (h) *h = tokens[b];
      const long long nt = next[b];
      if (nt == end_token_id || step + 1 >= max_length) {
        finished[b] = 1;
      } else {
        seq_len[b] += 1;
        pos[b] += 1;
        tokens[b] = nt;
        tokens32[b] = static_cast<int>(nt);
        live = 1;
      }
    }
  }
  const int n = __syncthreads_count(live);
  if (b == 0) {
    unfinished[0] = n;
    step_dev[0] = step + 1;
  }
}

// decode_advance_stop_kernel with a limit per request: request b finishes at step max_length[b] - 1 at the latest, and
// history has history_rows rows (rows at step >= history_rows are not written).
__global__ void decode_advance_stop_limits_kernel(int* __restrict__ seq_len, long long* __restrict__ pos,
                                                  long long* __restrict__ tokens, int* __restrict__ tokens32,
                                                  const long long* __restrict__ next, long long* __restrict__ history,
                                                  int* __restrict__ step_dev, int* __restrict__ finished,
                                                  int* __restrict__ unfinished, long long end_token_id,
                                                  const int* __restrict__ max_length, int history_rows, long long pad,
                                                  int B) {
  const int b = threadIdx.x;
  const int step = step_dev[0];
  int live = 0;
  if (b < B) {
    long long* h = step < history_rows ? history + (long long)step * B + b : nullptr;
    if (finished[b]) {
      if (h) *h = pad;
    } else {
      if (h) *h = tokens[b];
      const long long nt = next[b];
      if (nt == end_token_id || step + 1 >= max_length[b]) {
        finished[b] = 1;
      } else {
        seq_len[b] += 1;
        pos[b] += 1;
        tokens[b] = nt;
        tokens32[b] = static_cast<int>(nt);
        live = 1;
      }
    }
  }
  const int n = __syncthreads_count(live);
  if (b == 0) {
    unfinished[0] = n;
    step_dev[0] = step + 1;
  }
}

}  // namespace bagel

using namespace bagel;

#define COUNT_LAUNCH() g_launches.fetch_add(1, std::memory_order_relaxed)

extern "C" int bagel_sample_rows_bf16(const void* logits, long long ld, int B, int V, float temperature,
                                      const long long* keys, const int* step_dev, long long* tokens, int* tokens32,
                                      void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (!(temperature > 0.0f) || isinf(temperature))
    return set_error(BAGEL_ERR_ARG, "bagel_sample_rows_bf16: temperature must be finite and > 0 (greedy: bagel_argmax_rows_bf16)");
  if (ld < V) return set_error(BAGEL_ERR_SHAPE, "bagel_sample_rows_bf16: ld must be >= V");
  if (keys == nullptr || step_dev == nullptr || tokens == nullptr)
    return set_error(BAGEL_ERR_ARG, "bagel_sample_rows_bf16: keys, step_dev and tokens are required");
  sample_rows_kernel<<<B, kSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(logits), ld, V, 1.0f / temperature, keys, step_dev, tokens, tokens32);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_decode_advance_stop(int* seq_len, long long* pos, long long* tokens, int* tokens32,
                                         const long long* next, long long* history, int* step_dev, int* finished,
                                         int* unfinished, long long end_token_id, int max_length, long long pad, int B,
                                         void* stream) {
  if (B <= 0) return 0;
  if (B > 1024) return set_error(BAGEL_ERR_SHAPE, "bagel_decode_advance_stop: B must be <= 1024");
  if (max_length <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_decode_advance_stop: max_length must be > 0");
  decode_advance_stop_kernel<<<1, ((B + 31) / 32) * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      seq_len, pos, tokens, tokens32, next, history, step_dev, finished, unfinished, end_token_id, max_length, pad, B);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_sample_rows_mixed_bf16(const void* logits, long long ld, int B, int V, const float* inv_temperature,
                                            const long long* keys, const int* step_dev, long long* tokens, int* tokens32,
                                            void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (ld < V) return set_error(BAGEL_ERR_SHAPE, "bagel_sample_rows_mixed_bf16: ld must be >= V");
  if (inv_temperature == nullptr || keys == nullptr || step_dev == nullptr || tokens == nullptr)
    return set_error(BAGEL_ERR_ARG, "bagel_sample_rows_mixed_bf16: inv_temperature, keys, step_dev and tokens are required");
  sample_rows_mixed_kernel<<<B, kSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(logits), ld, V, inv_temperature, keys, step_dev, tokens, tokens32);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_decode_advance_stop_limits(int* seq_len, long long* pos, long long* tokens, int* tokens32,
                                                const long long* next, long long* history, int* step_dev, int* finished,
                                                int* unfinished, long long end_token_id, const int* max_length,
                                                int history_rows, long long pad, int B, void* stream) {
  if (B <= 0) return 0;
  if (B > 1024) return set_error(BAGEL_ERR_SHAPE, "bagel_decode_advance_stop_limits: B must be <= 1024");
  if (history_rows <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_decode_advance_stop_limits: history_rows must be > 0");
  if (max_length == nullptr) return set_error(BAGEL_ERR_ARG, "bagel_decode_advance_stop_limits: max_length is required");
  decode_advance_stop_limits_kernel<<<1, ((B + 31) / 32) * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      seq_len, pos, tokens, tokens32, next, history, step_dev, finished, unfinished, end_token_id, max_length,
      history_rows, pad, B);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}
