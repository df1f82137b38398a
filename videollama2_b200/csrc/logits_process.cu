// HF's logits processors on the device, in place on one fp32 logits row: repetition penalty, then the bans (no-repeat
// n-grams, bad words, minimum new tokens, suppressed tokens).  The statement in torch is sampling.process_logits; see
// DESIGN.md section 3.
//
// Only listed indices are touched: the history's tokens, the n-gram and bad-word completions and the EOS / suppress
// tables.  One CTA; the cost per token is O(n * N + table sizes) with no pass over the row.  A token hit by several
// rules ends as -inf if any ban hits it (a barrier orders the penalty's writes before the bans'), else penalised once;
// threads that ban the same token all store -inf.
#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

constexpr int kProcThreads = 1024;
constexpr int kProcMaxV = 262144;

__device__ __forceinline__ bool in_vocab(int64_t t, int V) { return t >= 0 && t < V; }

__global__ void __launch_bounds__(kProcThreads, 1)
logits_process_kernel(float* __restrict__ logits, int V, const vl2_logits_process_params* __restrict__ P,
                      const int64_t* __restrict__ hist, const int64_t* __restrict__ n_dev, int64_t n_add) {
  __shared__ uint32_t seen[kProcMaxV / 32];          // one bit per vocabulary id: which history tokens are penalised
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x;
  const int64_t n = max((int64_t)0, *n_dev + n_add);
  const float pen = P->repetition_penalty;
  const int N = P->no_repeat_ngram_size;

  // repetition penalty: the first thread to set a token's bit owns it, so a repeated token is penalised once.  Only
  // the bits of history tokens are cleared (no pass over the vocabulary).
  if (pen != 1.f && n > 0) {
    for (int64_t j = tid; j < n; j += kProcThreads) {
      const int64_t t = hist[j];
      if (in_vocab(t, V)) atomicAnd(&seen[t >> 5], ~(1u << (t & 31)));
    }
    __syncthreads();
    for (int64_t j = tid; j < n; j += kProcThreads) {
      const int64_t t = hist[j];
      if (!in_vocab(t, V)) continue;
      const uint32_t bit = 1u << (t & 31);
      if (atomicOr(&seen[t >> 5], bit) & bit) continue;
      const float s = logits[t];
      logits[t] = s < 0.f ? __fmul_rn(s, pen) : __fdiv_rn(s, pen);
    }
  }
  __syncthreads();                                   // every ban below lands after every penalised store

  // no-repeat n-grams: the n-gram starting at i is h[i .. i + N); its last token is banned when h[i .. i + N - 1) equals
  // the history's last N - 1 tokens
  if (N > 0 && n >= N) {
    const int64_t tail = n - (N - 1);
    for (int64_t i = tid; i + N <= n; i += kProcThreads) {
      bool match = true;
      for (int k = 0; k < N - 1 && match; ++k) match = hist[i + k] == hist[tail + k];
      if (match && in_vocab(hist[i + N - 1], V)) logits[hist[i + N - 1]] = -INFINITY;
    }
  }

  // bad words: a single id always; a sequence of L ids bans its last one when the history (at least L long, as HF
  // requires) ends with its first L - 1
  const int n_bad = P->n_bad;
  if (n_bad > 0) {
    const int64_t* off = P->bad_offsets;
    const int64_t* ids = P->bad_ids;
    for (int q = tid; q < n_bad; q += kProcThreads) {
      const int64_t a = off[q], L = off[q + 1] - a;
      if (L < 1 || (L > 1 && n < L)) continue;
      bool match = true;
      for (int64_t k = 0; k < L - 1 && match; ++k) match = hist[n - (L - 1) + k] == ids[a + k];
      if (match && in_vocab(ids[a + L - 1], V)) logits[ids[a + L - 1]] = -INFINITY;
    }
  }

  // minimum new tokens: EOS is banned while fewer than min_new_tokens ids have been generated
  if (n < P->min_new_tokens) {
    for (int e = tid; e < P->n_eos; e += kProcThreads)
      if (in_vocab(P->eos_ids[e], V)) logits[P->eos_ids[e]] = -INFINITY;
  }
  for (int e = tid; e < P->n_suppress; e += kProcThreads)
    if (in_vocab(P->suppress_ids[e], V)) logits[P->suppress_ids[e]] = -INFINITY;
}

}  // namespace vl2

using namespace vl2;

extern "C" int vl2_process_logits(float* logits, int V, const vl2_logits_process_params* params, const int64_t* history,
                                  const int64_t* n_dev, int64_t n_add, void* stream) {
  VL2_REQUIRE(V > 0 && V <= kProcMaxV, VL2_E_BADSHAPE, "vl2_process_logits: V = %d outside [1, %d]", V, kProcMaxV);
  VL2_REQUIRE(logits && params && history && n_dev, VL2_E_BADALIGN, "vl2_process_logits: null pointer");
  VL2_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 3) == 0 && (reinterpret_cast<uintptr_t>(params) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(history) & 7) == 0 && (reinterpret_cast<uintptr_t>(n_dev) & 7) == 0,
              VL2_E_BADALIGN, "vl2_process_logits: logits need 4-byte, params / history / n 8-byte alignment");
  launch_kernel(logits_process_kernel, dim3(1), dim3(kProcThreads), 0, (cudaStream_t)stream, 1, logits, V, params,
                history, n_dev, n_add);
  VL2_CHECK_LAUNCH("logits_process_kernel");
  return VL2_OK;
}
