// Token sampling on the device: temperature -> top-k -> top-p -> draw, on one fp32 logits row, written to device memory.
// HF's warpers (sampling.warp_logits) without a sort: both thresholds come from radix selects on the order-preserving
// 32-bit key of the scaled scores, and the draw is an index-order inverse CDF.  See DESIGN.md section 3.
//
// Every weight is held in 2^-40 fixed point relative to the maximum (w = rint(exp(s - max) * 2^40), at most 2^58 summed
// over 2^18 tokens), so all sums - the top-p bin masses, the kept total and the draw's running sum - are integer sums:
// exact, and the same whatever order the threads add them in.  A token whose weight rounds to 0 (below 2^-41 of the
// maximum's) is never drawn.
#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

constexpr int kSampleThreads = 1024;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kSampleMaxV = 262144;
constexpr int kSampleBins = 2048;           // radix digits of 11, 11 and 10 bits (shifts 21, 10, 0)
constexpr int kSampleSmemV = 49152;         // rows up to this many keys (192 KB) stay in shared memory

__device__ __forceinline__ uint32_t philox4x32_10_x0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                     uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// s = l / T rounded like torch's `scores / temperature`; NaN counts as -inf and -0 as +0, so that the key order below is
// the float order of the scores (and key_score inverts score_key exactly).
__device__ __forceinline__ float clean_score(float s) { return s != s ? -INFINITY : (s == 0.f ? 0.f : s); }

__device__ __forceinline__ float sample_score(const float* row, int i, float T) {
  return clean_score(__fdiv_rn(__ldg(row + i), T));
}

__device__ __forceinline__ uint32_t score_key(float s) {
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Fixed-point weight exp(s - mx) * 2^40: 0 for -inf, exactly 2^40 for the maximum (also when it is +inf).
__device__ __forceinline__ unsigned long long sample_weight(float s, float mx) {
  if (s == -INFINITY) return 0ull;
  const float w = s == mx ? 1.f : expf(s - mx);
  return __float2ull_rn(w * 0x1p40f);
}

__device__ __forceinline__ unsigned long long warp_scan_incl(unsigned long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// sum_{lane' >= lane} v(lane') within the warp.
__device__ __forceinline__ unsigned long long warp_suffix_incl(unsigned long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v += t;
  }
  return v;
}

// sum_{t' >= tid} v(t') over the block.  Starts and ends with a block barrier.
__device__ __forceinline__ unsigned long long block_suffix_sum(unsigned long long v, unsigned long long* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  unsigned long long incl = warp_suffix_incl(v, lane);
  if (lane == 0) red[w] = incl;
  __syncthreads();
  if (threadIdx.x < 32) red[threadIdx.x] = warp_suffix_incl(red[threadIdx.x], threadIdx.x);
  __syncthreads();
  if (w + 1 < kSampleWarps) incl += red[w + 1];
  __syncthreads();
  return incl;
}

// f(i, key) for every index of the row, this thread's share.  SMEM: the keys pass 1 left in shared memory; otherwise
// recomputed from the logits with 8 independent loads in flight per thread (the passes are latency-bound on L2).
template <bool SMEM, typename F>
__device__ __forceinline__ void for_keys(const float* __restrict__ row, int V, float T, const uint32_t* keys, F&& f) {
  if (SMEM) {
    for (int i = threadIdx.x; i < V; i += kSampleThreads) f(i, keys[i]);
  } else {
    for (int base = threadIdx.x; base < V; base += 8 * kSampleThreads) {
      float l[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = base + u * kSampleThreads;
        l[u] = i < V ? __ldg(row + i) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = base + u * kSampleThreads;
        if (i < V) f(i, score_key(clean_score(__fdiv_rn(l[u], T))));
      }
    }
  }
}

// One radix level: with hist[b] = the count or mass of the region's tokens whose digit is b, find the highest digit b*
// whose inclusive-from-the-top sum c(b*) reaches `need` (c(b) = sum of hist[b' >= b]).  Every thread returns b* and
// above = c(b* + 1), the amount strictly above it inside the region.  If no digit reaches `need`, b* = 0.
__device__ __forceinline__ void radix_pick(const unsigned long long* hist, int nbins, unsigned long long need,
                                           unsigned long long* red, uint32_t* pick_bin, unsigned long long* pick_above,
                                           uint32_t& bin, unsigned long long& above) {
  const int per = nbins / kSampleThreads;            // 2 or 1 digits per thread, thread t owns [t*per, t*per + per)
  const int b0 = threadIdx.x * per;
  unsigned long long loc = 0;
  for (int j = 0; j < per; ++j) loc += hist[b0 + j];
  if (threadIdx.x == 0) {
    *pick_bin = 0;
    *pick_above = 0;
  }
  unsigned long long c = block_suffix_sum(loc, red) - loc;   // sum of the digits above this thread's
  for (int j = per - 1; j >= 0; --j) {
    const unsigned long long a = c;
    c += hist[b0 + j];
    if (c >= need && a < need) {                     // exactly one digit when the region's total reaches `need`
      *pick_bin = (uint32_t)(b0 + j);
      *pick_above = a;
    }
  }
  __syncthreads();
  bin = *pick_bin;
  above = *pick_above;
}

// SMEM: the row's keys stay in dynamic shared memory after pass 1 (V <= kSampleSmemV); otherwise every pass recomputes
// them from the logits (an L2-resident re-read).  SCORED: once the thresholds are known, one more pass writes the warped
// row (l / T where kept, -inf elsewhere) to slot n of rec->scores; without it `rec` is not read.
template <bool SMEM, bool SCORED>
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_token_kernel(const float* __restrict__ logits, int V, const vl2_sample_params* __restrict__ params,
                    const int64_t* __restrict__ counter_dev, int64_t counter_add, int64_t* __restrict__ out,
                    const vl2_score_record_params* __restrict__ rec) {
  extern __shared__ uint32_t keys[];
  __shared__ unsigned long long hist[kSampleBins];
  __shared__ unsigned long long red[kSampleWarps];
  __shared__ unsigned long long seg[kSampleWarps];
  __shared__ unsigned long long pick_above;
  __shared__ uint32_t pick_bin;
  pdl_launch_dependents();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int b = tid; b < kSampleBins; b += kSampleThreads) hist[b] = 0;
  pdl_wait();
  const float T = params->temperature, top_p = params->top_p;
  const int top_k = params->top_k;
  const uint64_t seed = params->seed;
  const uint64_t n = (uint64_t)*counter_dev + (uint64_t)counter_add;
  const bool topk_on = top_k > 1 && top_k < V;       // k == 1: t_k is the maximum; k <= 0 or k >= V: no top-k
  const bool topp_on = !(top_p >= 1.f);               // NaN / <= 0 keep the maximum's tie group only (need = 1 below)
  __syncthreads();

  // pass 1: the keys, the maximum key with its first index (the token when nothing is drawable), top-k's first digit
  unsigned long long best = 0;
  for_keys<false>(logits, V, T, keys, [&](int i, uint32_t k) {
    if (SMEM) keys[i] = k;
    best = max(best, ((unsigned long long)k << 32) | (0xffffffffu - (uint32_t)i));
    if (topk_on) atomicAdd(&hist[k >> 21], 1ull);
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) red[warp] = best;
  __syncthreads();
  if (tid < 32) {
    best = red[tid];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (tid == 0) seg[0] = best;
  }
  __syncthreads();
  best = seg[0];
  const uint32_t max_key = (uint32_t)(best >> 32);
  const int first_max = (int)(0xffffffffu - (uint32_t)best);
  const float mx = key_score(max_key);

  // top-k: t_k = the k-th largest key counting duplicates (radix select over exact counts)
  uint32_t thr = top_k == 1 ? max_key : 0u;
  if (topk_on) {
    unsigned long long need = (unsigned long long)top_k;
    uint32_t prefix = 0;
    for (int level = 0; level < 3; ++level) {
      const int shift = level == 0 ? 21 : (level == 1 ? 10 : 0);
      const int bits = level == 2 ? 10 : 11;
      if (level > 0) {
        __syncthreads();
        for (int b = tid; b < kSampleBins; b += kSampleThreads) hist[b] = 0;
        __syncthreads();
        for_keys<SMEM>(logits, V, T, keys, [&](int, uint32_t k) {
          if ((uint32_t)((uint64_t)k >> (shift + bits)) == prefix)
            atomicAdd(&hist[(k >> shift) & ((1u << bits) - 1)], 1ull);
        });
      }
      __syncthreads();
      uint32_t bin;
      unsigned long long above;
      radix_pick(hist, 1 << bits, need, red, &pick_bin, &pick_above, bin, above);
      need -= above;
      prefix = (prefix << bits) | bin;
    }
    thr = prefix;
  }

  // top-p: the lowest key tau whose kept mass strictly above it is below top_p * Z; kept = key >= tau.  A tie group has
  // one key, so it is kept or dropped whole; the maximum's group (mass above = 0) always stays.
  if (topp_on) {
    __syncthreads();
    for (int b = tid; b < kSampleBins; b += kSampleThreads) hist[b] = 0;
    __syncthreads();
    unsigned long long z = 0;
    for_keys<SMEM>(logits, V, T, keys, [&](int, uint32_t k) {
      if (k < thr) return;
      const unsigned long long w = sample_weight(key_score(k), mx);
      if (w == 0) return;
      z += w;
      atomicAdd(&hist[k >> 21], w);
    });
    z = block_suffix_sum(z, red);                    // thread 0 holds the block total
    if (tid == 0) seg[0] = z;
    __syncthreads();
    z = seg[0];
    const double pz = (double)top_p * (double)z;
    unsigned long long need = pz >= 1.0 ? (unsigned long long)ceil(pz) : 1ull;
    uint32_t prefix = 0;
    for (int level = 0; level < 3; ++level) {
      const int shift = level == 0 ? 21 : (level == 1 ? 10 : 0);
      const int bits = level == 2 ? 10 : 11;
      if (level > 0) {
        __syncthreads();
        for (int b = tid; b < kSampleBins; b += kSampleThreads) hist[b] = 0;
        __syncthreads();
        for_keys<SMEM>(logits, V, T, keys, [&](int, uint32_t k) {
          if (k < thr || (uint32_t)((uint64_t)k >> (shift + bits)) != prefix) return;
          const unsigned long long w = sample_weight(key_score(k), mx);
          if (w != 0) atomicAdd(&hist[(k >> shift) & ((1u << bits) - 1)], w);
        });
      }
      __syncthreads();
      uint32_t bin;
      unsigned long long above;
      radix_pick(hist, 1 << bits, need, red, &pick_bin, &pick_above, bin, above);
      need -= above;
      prefix = (prefix << bits) | bin;
    }
    thr = max(thr, prefix);
  }

  if (SCORED) {
    const int64_t slot = (int64_t)n;
    float* dst = rec->scores;
    if (dst != nullptr && rec->V == V && slot >= 0 && slot < rec->capacity) {
      dst += slot * (int64_t)V;
      for (int i = tid; i < V; i += kSampleThreads) {
        const float s = __fdiv_rn(__ldg(logits + i), T);          // unclean: -0.0 and NaN stay as torch leaves them
        dst[i] = (SMEM ? keys[i] : score_key(clean_score(s))) >= thr ? s : -INFINITY;
      }
    }
  }

  // draw: warp w owns the index range [w * L, (w + 1) * L); the kept mass of each range, then one warp walks the range
  // that holds the target in index order
  auto weight_at = [&](int i) -> unsigned long long {
    const uint32_t k = SMEM ? keys[i] : score_key(sample_score(logits, i, T));
    return k >= thr ? sample_weight(key_score(k), mx) : 0ull;
  };
  const int L = (V + kSampleWarps - 1) / kSampleWarps;
  const int lo = min(V, warp * L), hi = min(V, lo + L);
  unsigned long long part = 0;
  for (int base = lo + lane; base < hi; base += 4 * 32) {
    unsigned long long w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) w[u] = base + 32 * u < hi ? weight_at(base + 32 * u) : 0ull;
#pragma unroll
    for (int u = 0; u < 4; ++u) part += w[u];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  __syncthreads();
  if (lane == 0) seg[warp] = part;
  __syncthreads();
  if (warp == 0) {
    const unsigned long long mine = seg[lane];
    const unsigned long long incl = warp_scan_incl(mine, lane);
    const unsigned long long zk = __shfl_sync(0xffffffffu, incl, 31);
    const uint32_t a = philox4x32_10_x0((uint32_t)n, (uint32_t)(n >> 32), 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32)) >> 8;
    // target = floor(u * zk) with u = a * 2^-24: the token is the first index whose running sum exceeds it
    const unsigned long long plo = (unsigned long long)a * zk, phi = __umul64hi((unsigned long long)a, zk);
    const unsigned long long target = (phi << 40) | (plo >> 24);
    const unsigned int owner = __ballot_sync(0xffffffffu, incl > target && incl - mine <= target);
    const int ow = owner ? __ffs(owner) - 1 : 0;
    const unsigned long long before = __shfl_sync(0xffffffffu, incl - mine, ow);
    if (lane == 0) {
      red[0] = zk;
      red[1] = target;
      red[2] = (unsigned long long)ow;
      red[3] = before;
    }
  }
  __syncthreads();
  if (red[0] == 0) {                                 // nothing drawable (every score -inf or NaN)
    if (tid == 0) *out = first_max;
    return;
  }
  if (warp != (int)red[2]) return;
  const unsigned long long target = red[1];
  unsigned long long run = red[3];
  for (int base = lo; base < hi; base += 4 * 32) {
    unsigned long long w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + 32 * u + lane;
      w[u] = i < hi ? weight_at(i) : 0ull;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const unsigned long long incl = run + warp_scan_incl(w[u], lane);
      const unsigned int hit = __ballot_sync(0xffffffffu, incl > target);
      if (hit) {
        if (lane == __ffs(hit) - 1) *out = base + 32 * u + lane;
        return;
      }
      run = __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  if (lane == 0) *out = first_max;                   // unreachable: the range's mass covers the target
}

}  // namespace vl2

using namespace vl2;

template <bool SCORED>
static int sample_token_launch(const char* fn, const float* logits, int V, const vl2_sample_params* params,
                               const int64_t* counter_dev, int64_t counter_add, int64_t* token_out,
                               const vl2_score_record_params* rec, void* stream) {
  VL2_REQUIRE(V > 0 && V <= kSampleMaxV, VL2_E_BADSHAPE, "%s: V = %d outside [1, %d]", fn, V, kSampleMaxV);
  VL2_REQUIRE(logits && params && counter_dev && token_out && (rec || !SCORED), VL2_E_BADALIGN, "%s: null pointer", fn);
  VL2_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 3) == 0 && (reinterpret_cast<uintptr_t>(params) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(counter_dev) & 7) == 0 && (reinterpret_cast<uintptr_t>(token_out) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(rec) & 7) == 0,
              VL2_E_BADALIGN, "%s: logits need 4-byte, params / counter / token / record 8-byte alignment", fn);
  if (V <= kSampleSmemV) {
    VL2_SMEM_OPT_IN((sample_token_kernel<true, SCORED>), kSampleSmemV * 4);
    launch_kernel(sample_token_kernel<true, SCORED>, dim3(1), dim3(kSampleThreads), (size_t)V * 4, (cudaStream_t)stream,
                  1, logits, V, params, counter_dev, counter_add, token_out, rec);
  } else {
    launch_kernel(sample_token_kernel<false, SCORED>, dim3(1), dim3(kSampleThreads), 0, (cudaStream_t)stream, 1, logits,
                  V, params, counter_dev, counter_add, token_out, rec);
  }
  VL2_CHECK_LAUNCH("sample_token_kernel");
  return VL2_OK;
}

extern "C" int vl2_sample_token(const float* logits, int V, const vl2_sample_params* params, const int64_t* counter_dev,
                                int64_t counter_add, int64_t* token_out, void* stream) {
  return sample_token_launch<false>("vl2_sample_token", logits, V, params, counter_dev, counter_add, token_out, nullptr,
                                    stream);
}

extern "C" int vl2_sample_token_scored(const float* logits, int V, const vl2_sample_params* params,
                                       const int64_t* counter_dev, int64_t counter_add, int64_t* token_out,
                                       const vl2_score_record_params* record, void* stream) {
  return sample_token_launch<true>("vl2_sample_token_scored", logits, V, params, counter_dev, counter_add, token_out,
                                   record, stream);
}
