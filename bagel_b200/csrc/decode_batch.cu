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
// kFloor = true (sample_rows_filtered_kernel) makes a sampled row treat every logit below `lfloor` as NaN, which is never
// picked: the draw is restricted to l >= lfloor with each kept logit's uniform unchanged, and the uniforms of logits
// below it are not computed. A greedy row ignores it.
constexpr int kSampleThreads = 1024;
template <bool kSample, bool kFloor = false>
__device__ __forceinline__ void pick_row(const __nv_bfloat16* __restrict__ logits, long long ld, int V, float inv_t,
                                         const long long* __restrict__ keys, const int* __restrict__ step_dev,
                                         long long* __restrict__ tokens, int* __restrict__ tokens32,
                                         float lfloor = -INFINITY) {
  const __nv_bfloat16* row = logits + (long long)blockIdx.x * ld;
  auto lf = [&](float l) {
    if constexpr (kFloor) return l >= lfloor ? l : __int_as_float(0x7fffffff);
    else return l;
  };
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
      if constexpr (kSample && kFloor) {      // no logit of the group is kept: its uniforms are not needed
        const float m = fmaxf(fmaxf(fmaxf(bf16_lo_f(u.x), bf16_hi_f(u.x)), fmaxf(bf16_lo_f(u.y), bf16_hi_f(u.y))),
                              fmaxf(fmaxf(bf16_lo_f(u.z), bf16_hi_f(u.z)), fmaxf(bf16_lo_f(u.w), bf16_hi_f(u.w))));
        if (!(m >= lfloor)) continue;
      }
      if constexpr (kSample) {
        const uint4 r0 = philox4x32_10(make_uint4(step, (uint32_t)i >> 2, 0u, 0u), k0, k1);
        const uint4 r1 = philox4x32_10(make_uint4(step, ((uint32_t)i >> 2) + 1u, 0u, 0u), k0, k1);
        take(gumbel_score(lf(bf16_lo_f(u.x)), inv_t, r0.x), i);
        take(gumbel_score(lf(bf16_hi_f(u.x)), inv_t, r0.y), i + 1);
        take(gumbel_score(lf(bf16_lo_f(u.y)), inv_t, r0.z), i + 2);
        take(gumbel_score(lf(bf16_hi_f(u.y)), inv_t, r0.w), i + 3);
        take(gumbel_score(lf(bf16_lo_f(u.z)), inv_t, r1.x), i + 4);
        take(gumbel_score(lf(bf16_hi_f(u.z)), inv_t, r1.y), i + 5);
        take(gumbel_score(lf(bf16_lo_f(u.w)), inv_t, r1.z), i + 6);
        take(gumbel_score(lf(bf16_hi_f(u.w)), inv_t, r1.w), i + 7);
      } else {
        take(bf16_lo_f(u.x), i);     take(bf16_hi_f(u.x), i + 1);
        take(bf16_lo_f(u.y), i + 2); take(bf16_hi_f(u.y), i + 3);
        take(bf16_lo_f(u.z), i + 4); take(bf16_hi_f(u.z), i + 5);
        take(bf16_lo_f(u.w), i + 6); take(bf16_hi_f(u.w), i + 7);
      }
    }
  }
  for (int i = vec_end + threadIdx.x; i < V; i += kSampleThreads) {
    if constexpr (kSample && kFloor) {
      if (!(__bfloat162float(row[i]) >= lfloor)) continue;
    }
    if constexpr (kSample) {
      const uint4 r = philox4x32_10(make_uint4(step, (uint32_t)i >> 2, 0u, 0u), k0, k1);
      const int w = i & 3;
      const uint32_t x = w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
      take(gumbel_score(lf(__bfloat162float(row[i])), inv_t, x), i);
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

// ---------------------------------------------------------------------------------------------
// Truncated sampling (top-k, top-p, min-p). Each filter keeps the logits at or above some value, so together they keep
// l >= floor for one floor per row. bf16 values map to monotone 16-bit keys, so the floor is an exact radix select: a
// histogram of the high 11 key bits, then one of the low 5 bits inside one high bin. Counts are integers and the top-p
// mass is fixed point (each fp32 e_j rounded to a multiple of 2^-40), so every sum is exact and its bits do not depend
// on the order in which threads add: replay, eager runs and every batch position agree. e_j depends on the key alone,
// so a low-bit histogram needs counts only; its mass is count * e(key).
// ---------------------------------------------------------------------------------------------
constexpr int kLoBits = 5, kLoBins = 1 << kLoBits, kHiBins = 1 << (16 - kLoBits);
constexpr float kMassScale = 1099511627776.0f;      // 2^40: e_j <= 1
constexpr int kFilteredMaxV = 262144;               // a high bin's 14-bit mass chunks then sum below 2^32

// Key of a bf16 value: larger value, larger key; -0 takes +0's key. -1 for +-inf and NaN (never counted).
__device__ __forceinline__ int bf16_key(uint32_t bits) {
  if ((bits & 0x7F80u) == 0x7F80u) return -1;
  if (bits == 0x8000u) bits = 0;
  return (bits & 0x8000u) ? static_cast<int>(~bits & 0xFFFFu) : static_cast<int>(bits | 0x8000u);
}

__device__ __forceinline__ float key_value(int key) {
  const uint32_t bits = (key & 0x8000) ? (key & 0x7FFF) : (~key & 0xFFFF);
  return __uint_as_float(bits << 16);
}

// e of a logit value v: fp32 exp((v - l_max) * inv_t) in units of 2^-40 (at most 2^40).
__device__ __forceinline__ unsigned long long mass_of(float v, float mx, float inv_t) {
  return __float2ull_rn(expf((v - mx) * inv_t) * kMassScale);
}

// Calls f(key, value) for every element of the row (elements past V come as NaN, key -1). Each thread loads four
// 8-element groups before it uses them, so that enough of the row is in flight from L2.
template <typename F>
__device__ __forceinline__ void for_each_logit(const __nv_bfloat16* __restrict__ row, int V, bool vec, F&& f) {
  constexpr int kGroups = 4;
  const uint16_t* r16 = reinterpret_cast<const uint16_t*>(row);
  for (int g0 = 0; g0 < V; g0 += kSampleThreads * 8 * kGroups) {
    uint4 w[kGroups];
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      const int j = g0 + (g * kSampleThreads + threadIdx.x) * 8;
      if (vec && j + 8 <= V) {
        w[g] = *reinterpret_cast<const uint4*>(row + j);
      } else {
        uint32_t x[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t lo = j + 2 * q < V ? r16[j + 2 * q] : 0x7FFFu;
          const uint32_t hi = j + 2 * q + 1 < V ? r16[j + 2 * q + 1] : 0x7FFFu;
          x[q] = lo | (hi << 16);
        }
        w[g] = make_uint4(x[0], x[1], x[2], x[3]);
      }
    }
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      const uint32_t x[4] = {w[g].x, w[g].y, w[g].z, w[g].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        f(bf16_key(x[q] & 0xFFFFu), bf16_lo_f(x[q]));
        f(bf16_key(x[q] >> 16), bf16_hi_f(x[q]));
      }
    }
  }
}

// Warp 0: the bin at which the sum of h[0..NB) taken from the top bin down first reaches target, i.e.
// sum(h[bin+1..]) < target <= sum(h[bin..]); *above = sum(h[bin+1..]). -1 when the whole sum stays below target.
// Lane l owns the NB / 32 bins below NB - 1 - l * NB / 32 (inclusive). Integer sums: exact in any order.
template <typename T, int NB>
__device__ __forceinline__ int find_from_top(const T* h, T target, T* above) {
  constexpr int kPer = NB / 32;
  const int lane = threadIdx.x & 31;
  const int top = NB - 1 - kPer * lane;
  T s = 0;
#pragma unroll 8
  for (int q = 0; q < kPer; ++q) s += h[top - q];
  T incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  const unsigned hit = __ballot_sync(0xffffffffu, incl >= target);
  if (hit == 0) return -1;
  const int owner = __ffs(hit) - 1;
  int bin = -1;
  T acc = incl - s;
  if (lane == owner) {
    for (int q = 0; q < kPer; ++q) {
      if (acc + h[top - q] >= target) { bin = top - q; break; }
      acc += h[top - q];
    }
  }
  *above = __shfl_sync(0xffffffffu, acc, owner);
  return __shfl_sync(0xffffffffu, bin, owner);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Warp 0: lo_mass[i] = lo_cnt[i] * e(key of low bin i of high bin hi) for i >= lo_min, else 0; returns their sum.
__device__ __forceinline__ unsigned long long low_bin_masses(const unsigned* lo_cnt, unsigned long long* lo_mass, int hi,
                                                            int lo_min, float mx, float inv_t) {
  const int i = threadIdx.x & 31;
  const unsigned long long m =
      i >= lo_min && lo_cnt[i] ? lo_cnt[i] * mass_of(key_value((hi << kLoBits) | i), mx, inv_t) : 0ull;
  lo_mass[i] = m;
  __syncwarp();
  return warp_sum(m);
}

// The floor of one sampled row: the largest of the top-k, top-p and min-p thresholds that are set (see
// include/bagel_b200.h). -inf when the row has no finite logit.
__device__ __noinline__ float row_floor(const __nv_bfloat16* __restrict__ row, int V, bool vec, float inv_t, int k,
                                        float p, float min_p) {
  __shared__ unsigned cnt_hi[kHiBins];
  // top-p mass of each high bin: three 14-bit chunk sums while counting (native 32-bit shared atomics), then the
  // same memory read as one 64-bit sum per bin
  __shared__ unsigned long long mass_buf[3 * kHiBins / 2];
  __shared__ unsigned lo_cnt[kLoBins];
  __shared__ unsigned long long lo_mass[kLoBins];
  __shared__ float red[kSampleThreads / 32];
  __shared__ int s_hk, s_rem, s_hp, s_key;
  __shared__ unsigned long long s_rem_p;
  unsigned* chunk = reinterpret_cast<unsigned*>(mass_buf);
  unsigned long long* mass_hi = mass_buf;
  const bool has_k = k > 0 && k < V, has_p = p < 1.0f, has_min = min_p > 0.0f;
  for (int i = threadIdx.x; i < kHiBins; i += kSampleThreads) {
    cnt_hi[i] = 0;
    chunk[i] = chunk[kHiBins + i] = chunk[2 * kHiBins + i] = 0;
  }
  if (threadIdx.x < kLoBins) lo_cnt[threadIdx.x] = 0;
  __syncthreads();

  // pass 1: the largest finite logit; the count of every high bin
  float mx = -INFINITY;
  for_each_logit(row, V, vec, [&](int key, float v) {
    mx = fmaxf(mx, key >= 0 ? v : -INFINITY);
    if (has_k && key >= 0) atomicAdd(&cnt_hi[key >> kLoBits], 1u);
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (mx == -INFINITY) return -INFINITY;            // no finite logit: nothing to truncate
  if (threadIdx.x < 32) {
    int hk = -1;
    unsigned above = 0;
    if (has_k) hk = find_from_top<unsigned, kHiBins>(cnt_hi, static_cast<unsigned>(k), &above);
    if (threadIdx.x == 0) { s_hk = hk; s_rem = static_cast<int>(k - above); }
  }
  __syncthreads();
  const int hk = s_hk;                               // -1: fewer than k finite logits, top-k keeps them all
  int floor_key = 0;                                 // below every finite key (the smallest is 0x0080)
  if (hk >= 0 || has_p) {
    // pass 2: the counts inside top-k's high bin; the top-p mass of every high bin
    for_each_logit(row, V, vec, [&](int key, float v) {
      if (key < 0) return;
      if ((key >> kLoBits) == hk) atomicAdd(&lo_cnt[key & (kLoBins - 1)], 1u);
      if (has_p) {
        const unsigned long long e = mass_of(v, mx, inv_t);
        const int h = key >> kLoBits;
        if (e & 0x3FFFu) atomicAdd(&chunk[h], static_cast<unsigned>(e & 0x3FFFu));
        if ((e >> 14) & 0x3FFFu) atomicAdd(&chunk[kHiBins + h], static_cast<unsigned>((e >> 14) & 0x3FFFu));
        if (e >> 28) atomicAdd(&chunk[2 * kHiBins + h], static_cast<unsigned>(e >> 28));
      }
    });
    __syncthreads();
    if (has_p) {
      unsigned long long m[kHiBins / kSampleThreads];
#pragma unroll
      for (int q = 0; q < kHiBins / kSampleThreads; ++q) {
        const int i = threadIdx.x + q * kSampleThreads;
        m[q] = chunk[i] + (static_cast<unsigned long long>(chunk[kHiBins + i]) << 14) +
               (static_cast<unsigned long long>(chunk[2 * kHiBins + i]) << 28);
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < kHiBins / kSampleThreads; ++q) mass_hi[threadIdx.x + q * kSampleThreads] = m[q];
      __syncthreads();
    }
    if (threadIdx.x < 32) {
      int lo_k = 0;
      if (hk >= 0) {
        unsigned above;
        lo_k = find_from_top<unsigned, kLoBins>(lo_cnt, static_cast<unsigned>(s_rem), &above);
        floor_key = (hk << kLoBits) | lo_k;
      }
      int hp = -1;
      unsigned long long rem_p = 0;
      if (has_p) {
        if (hk >= 0) {             // restrict the mass to the logits top-k keeps
          const unsigned long long part = low_bin_masses(lo_cnt, lo_mass, hk, lo_k, mx, inv_t);
          for (int i = threadIdx.x; i < hk; i += 32) mass_hi[i] = 0;
          if (threadIdx.x == 0) mass_hi[hk] = part;
          __syncwarp();
        }
        unsigned long long total = 0;
        for (int i = threadIdx.x; i < kHiBins; i += 32) total += mass_hi[i];
        total = warp_sum(total);
        // the smallest integer mass >= p * total, at least 1 (p <= 0 keeps the maximum's ties only)
        const double t = ceil(static_cast<double>(p) * static_cast<double>(total));
        const unsigned long long target = t > 1.0 ? static_cast<unsigned long long>(t) : 1ull;
        unsigned long long above;
        hp = find_from_top<unsigned long long, kHiBins>(mass_hi, target, &above);
        rem_p = target - above;
        if (hp == hk) {            // top-k's bin: its low-bin masses are already there
          const int lo_p = find_from_top<unsigned long long, kLoBins>(lo_mass, rem_p, &above);
          floor_key = max(floor_key, (hp << kLoBits) | lo_p);
          hp = -1;
        }
      }
      if (threadIdx.x == 0) { s_hp = hp; s_rem_p = rem_p; s_key = floor_key; }
    }
    __syncthreads();
    floor_key = s_key;
    if (s_hp >= 0) {
      // pass 3: the counts inside top-p's high bin, when it is not top-k's
      const int hp = s_hp;
      if (threadIdx.x < kLoBins) lo_cnt[threadIdx.x] = 0;
      __syncthreads();
      for_each_logit(row, V, vec, [&](int key, float) {
        if (key >= 0 && (key >> kLoBits) == hp) atomicAdd(&lo_cnt[key & (kLoBins - 1)], 1u);
      });
      __syncthreads();
      if (threadIdx.x < 32) {
        low_bin_masses(lo_cnt, lo_mass, hp, 0, mx, inv_t);
        unsigned long long above;
        const int lo_p = find_from_top<unsigned long long, kLoBins>(lo_mass, s_rem_p, &above);
        if (threadIdx.x == 0) s_key = max(floor_key, (hp << kLoBits) | lo_p);
      }
      __syncthreads();
      floor_key = s_key;
    }
  }
  // min-p: the smallest key whose value passes the fp32 test. The test is monotone in the value, so a binary search
  // over the keys up to the maximum's finds it; the maximum itself always passes when min_p <= 1.
  if (has_min) {
    const float lmp = logf(min_p);
    int lo = 0x0080, hi = bf16_key(__float_as_uint(mx) >> 16);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((key_value(mid) - mx) * inv_t >= lmp) hi = mid;
      else lo = mid + 1;
    }
    floor_key = max(floor_key, lo);
  }
  return key_value(max(floor_key, 0x0080));
}

// Per-row settings as sample_rows_mixed_kernel, plus per-row top_k (<= 0: off), top_p (>= 1: off) and min_p (<= 0:
// off) for the sampled rows. A sampled row draws exactly as sample_rows_kernel would, among the logits at or above its
// floor only; with every filter off that is sample_rows_kernel's pick.
__global__ void __launch_bounds__(kSampleThreads)
sample_rows_filtered_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V,
                            const float* __restrict__ inv_temperature, const int* __restrict__ top_k,
                            const float* __restrict__ top_p, const float* __restrict__ min_p,
                            const long long* __restrict__ keys, const int* __restrict__ step_dev,
                            long long* __restrict__ tokens, int* __restrict__ tokens32) {
  const int b = blockIdx.x;
  const float inv_t = inv_temperature[b];
  if (inv_t == 0.0f) {
    // argmax: the floor only applies to sampled rows. An instantiation of its own keeps the shared-memory layout, and
    // so the SASS, of sample_rows_mixed_kernel unchanged.
    pick_row<false, true>(logits, ld, V, 0.0f, keys, step_dev, tokens, tokens32);
    return;
  }
  const int k = top_k[b];
  const float p = top_p[b], mp = min_p[b];
  float lfloor = -INFINITY;
  if ((k > 0 && k < V) || p < 1.0f || mp > 0.0f) {
    const bool vec = (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0;
    lfloor = row_floor(logits + (long long)b * ld, V, vec, inv_t, k, p, mp);
  }
  pick_row<true, true>(logits, ld, V, inv_t, keys, step_dev, tokens, tokens32, lfloor);
}

// ---------------------------------------------------------------------------------------------
// Repetition, frequency and presence penalties on the tokens a request has generated (see include/bagel_b200.h). The
// state of row b is seen[b] = {n, tok[cap], cnt[cap]}: the n distinct tokens fed so far (step >= 1, while unfinished)
// and how often each was fed, in order of first appearance. A step adds the token fed at it (tokens[b], chosen at the
// previous step) with one thread, then rewrites each distinct token's logit once from the row it reads: O(n) work, no
// atomics, and nothing depends on the order in which threads run.
// ---------------------------------------------------------------------------------------------
constexpr int kPenaltyThreads = 256;

__global__ void __launch_bounds__(kPenaltyThreads)
apply_penalties_kernel(__nv_bfloat16* __restrict__ logits, long long ld, int V, const float* __restrict__ repetition,
                       const float* __restrict__ frequency, const float* __restrict__ presence,
                       const long long* __restrict__ tokens, const int* __restrict__ finished,
                       const int* __restrict__ step_dev, int* __restrict__ seen, int cap) {
  const int b = blockIdx.x;
  const float rp = repetition[b], fp = frequency[b], pp = presence[b];
  if (rp == 1.0f && fp == 0.0f && pp == 0.0f) return;     // penalties off: the row is not touched
  int* st = seen + (long long)b * (1 + 2 * (long long)cap);
  int* tok = st + 1;
  int* cnt = tok + cap;
  __shared__ int s_hit;
  int n = st[0];
  const long long t = tokens[b];
  if (step_dev[0] >= 1 && !finished[b] && t >= 0 && t < V) {
    if (threadIdx.x == 0) s_hit = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kPenaltyThreads)
      if (tok[i] == static_cast<int>(t)) s_hit = i;         // the list is distinct: at most one thread writes
    __syncthreads();
    const int hit = s_hit;
    if (hit < 0 && n < cap) {
      if (threadIdx.x == 0) { tok[n] = static_cast<int>(t); cnt[n] = 1; st[0] = n + 1; }
      ++n;
    } else if (hit >= 0 && threadIdx.x == 0) {
      cnt[hit] += 1;
    }
    __syncthreads();
  }
  __nv_bfloat16* row = logits + (long long)b * ld;
  for (int i = threadIdx.x; i < n; i += kPenaltyThreads) {
    const int j = tok[i];
    const float l = __bfloat162float(row[j]);
    if (isnan(l)) continue;                                   // NaN keeps its bits
    // one rounding per operation, in this order (the intrinsics are never contracted into an FMA)
    float r = l < 0.0f ? __fmul_rn(l, rp) : __fdiv_rn(l, rp);
    r = __fsub_rn(r, __fmul_rn(fp, static_cast<float>(cnt[i])));
    r = __fsub_rn(r, pp);
    row[j] = __float2bfloat16_rn(r);
  }
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

extern "C" int bagel_sample_rows_filtered_bf16(const void* logits, long long ld, int B, int V,
                                               const float* inv_temperature, const int* top_k, const float* top_p,
                                               const float* min_p, const long long* keys, const int* step_dev,
                                               long long* tokens, int* tokens32, void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (B > 1024) return set_error(BAGEL_ERR_SHAPE, "bagel_sample_rows_filtered_bf16: B must be <= 1024");
  if (V > kFilteredMaxV) return set_error(BAGEL_ERR_SHAPE, "bagel_sample_rows_filtered_bf16: V must be <= 262144");
  if (ld < V) return set_error(BAGEL_ERR_SHAPE, "bagel_sample_rows_filtered_bf16: ld must be >= V");
  if (inv_temperature == nullptr || top_k == nullptr || top_p == nullptr || min_p == nullptr || keys == nullptr ||
      step_dev == nullptr || tokens == nullptr)
    return set_error(BAGEL_ERR_ARG, "bagel_sample_rows_filtered_bf16: every pointer but tokens32 is required");
  sample_rows_filtered_kernel<<<B, kSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(logits), ld, V, inv_temperature, top_k, top_p, min_p, keys, step_dev, tokens,
      tokens32);
  COUNT_LAUNCH();
  BAGEL_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int bagel_apply_penalties_bf16(void* logits, long long ld, int B, int V, const float* repetition,
                                          const float* frequency, const float* presence, const long long* tokens,
                                          const int* finished, const int* step_dev, int* seen, int capacity,
                                          void* stream) {
  if (B <= 0 || V <= 0) return 0;
  if (ld < V) return set_error(BAGEL_ERR_SHAPE, "bagel_apply_penalties_bf16: ld must be >= V");
  if (capacity <= 0) return set_error(BAGEL_ERR_SHAPE, "bagel_apply_penalties_bf16: capacity must be > 0");
  if (logits == nullptr || repetition == nullptr || frequency == nullptr || presence == nullptr || tokens == nullptr ||
      finished == nullptr || step_dev == nullptr || seen == nullptr)
    return set_error(BAGEL_ERR_ARG, "bagel_apply_penalties_bf16: every pointer is required");
  apply_penalties_kernel<<<B, kPenaltyThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<__nv_bfloat16*>(logits), ld, V, repetition, frequency, presence, tokens, finished, step_dev, seen,
      capacity);
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
