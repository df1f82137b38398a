// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,Nout] = epi(A[M,K] * W[N,K]^T).
//
//   warpgroup 0   TMA producer (one thread): cp.async.bulk.tensor A/B tiles -> 128B-swizzled smem ring;
//                 epilogue operands (epilogue variants only), during the k-loop: warp 1 loads the tile's residual /
//                 RoPE-table slots by TMA into a small smem ring, warps 2-3 compute its 128 row factors into smem
//   warpgroups 1, 2  consumers: wgmma.mma_async m64 x BN x k16 from the ring (rows 0..63 / 64..127 of the 128-row tile),
//                 fp32 accumulators in registers, then the epilogue from the accumulator fragments:
//                 row_scale / folded RMSNorm or LayerNorm / bias / activation / SwiGLU / RoPE / residual / statistics.
//                 A variant writes each 16 x 32 slot of a warp into a swizzled smem staging tile that one lane stores by
//                 TMA; the generic epilogue stores to global directly (optionally also to peer buffers or an NVSwitch
//                 multicast address)
//
// Tiles are 128 x BN, BN in {64,...,256} step 32 chosen per launch by a wave / operand-traffic cost model (choose_tile);
// BLOCK_K = 64 bf16 = one 128-byte swizzle atom; the grid is persistent (<= #SMs CTAs, static round-robin over tiles,
// M fastest so that a wave shares W tiles through L2).  M/N/K tails: TMA zero-fills out-of-bounds reads; TMA stores clip
// at the output's bounds, the generic epilogue's stores are predicated.
#include <stdlib.h>
#include <string.h>

#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int kConsumerThreads = 256;              // two consumer warpgroups
static constexpr int kGemmThreads = 128 + kConsumerThreads;
static constexpr int kConvLine = 16;                      // Conv3d front end: output lines and columns per time step are padded to 16

// Shared memory of the epilogue variants, carved out of the 227 KB next to the A/B ring:
//   output staging: per consumer warp two 16-row x 32-column 16-bit tiles (64-byte rows, SWIZZLE_64B; SwiGLU: 16 columns,
//                   32-byte rows, SWIZZLE_32B), each written by the warp and stored by one TMA store;
//   operand ring:   kOpSlots 128-row x 32-column slots of the residual or of the RoPE table (64-byte rows, SWIZZLE_64B);
//   row factors:    the tile's 128 row factors, double-buffered (tile t / t + 1).
static constexpr int kOpSlots = 2;
static constexpr int kOpSlotBytes = 128 * 64;
static constexpr int kStageTileBytes = 16 * 64;
static constexpr int kEpiOutBytes = (kConsumerThreads / 32) * 2 * kStageTileBytes;
static constexpr int kEpiSmemBytes = kEpiOutBytes + kOpSlots * kOpSlotBytes + 2 * 128 * 4;
static constexpr int kSmemLimit = 227 * 1024;

// PAIR = true: the two CTAs of a cluster compute a 256 x BN tile (128 rows each) and share its B tile: each CTA loads
// HALF of the B rows and the TMA unit multicasts them into both CTAs' shared memory, so a k-block costs
// 16 KB + BN*64 B of L2 traffic per CTA instead of 16 KB + BN*128 B.  A ring slot is free once the consumers of BOTH
// CTAs have read it (the peer's multicast writes into it), so every consumer warp releases it in both CTAs.
template <int BN, bool PAIR>
struct GemmCfg {
  static_assert(BN % 32 == 0 && BN >= 64 && BN <= 256, "BN must be a multiple of 32 in [64,256]");
  static_assert(!PAIR || BN >= 128, "a pair tile is at least 128 columns wide");
  static constexpr int kStageBytesA = BM * BK * 2;
  static constexpr int kStageBytesB = BN * BK * 2;
  static constexpr int kHalfBytesB = BN / 2 * BK * 2;     // pair: the half of B one CTA loads (1024-byte multiple)
  static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
  static constexpr int kExtraBytes = 1024;               // barriers
  static constexpr int kMaxStages = (kSmemLimit - kExtraBytes - kEpiSmemBytes) / kStageBytes;
  static constexpr int kStages = kMaxStages > 8 ? 8 : kMaxStages;
  static_assert(kStages >= 4, "the ring must keep at least 4 stages next to the epilogue's shared memory");
  static constexpr int kSmemBytes = kStages * kStageBytes + kEpiSmemBytes + kExtraBytes;
  static constexpr int kAcc = BN / 2;                     // fp32 accumulators per consumer thread
  static constexpr int kEmptyArrivals = (PAIR ? 2 : 1) * (kConsumerThreads / 32);
  static_assert(!PAIR || kHalfBytesB % 1024 == 0, "the peer's half of B must start on a swizzle-atom boundary");
};

struct GemmParams {
  void* C;
  const float* bias;
  const void* residual;
  const float* row_scale;
  int64_t ldc, ldr;
  int M, N, K;
  int act;
  int out_f32;
  int num_m_tiles, num_n_tiles;
  // epilogue-fused all-gather: peers' copies of C (NVLink P2P stores) or one NVSwitch multicast address
  __nv_bfloat16* bcast[8];
  __nv_bfloat16* mc;
  int n_bcast;
  // folded RMSNorm / LayerNorm (see vl2.h)
  const float* rms_sumsq_in;
  const float* ln_sum_in;
  const float* ln_colsum;
  float* rowsum_out;
  float* sumsq_out;
  int rms_nparts;
  float rms_inv_dim, rms_eps;
  // split-K of the last, partial round (see launch_gemm): items >= split_first are K-slices of the remaining tiles
  int split_first, split_s, num_items;
  float* ws_partial;      // [tiles past split_first][split_s - 1][tile rows][BN] fp32 partial accumulators
  unsigned* ws_flags;     // [tiles past split_first][2] arrival counters (self-resetting)
  // implicit-GEMM Conv3d(k = s = 2) front end (see vl2.h: conv_C > 0).  A rows are the output positions in a padded
  // enumeration (to, ho16, wo16): 16 x 16 rows per output time step, so that one 128-row tile is 8 whole output lines of
  // one time step and a k-block (one tap x 64 channels) of the tile is ONE 5-D TMA box over x viewed as
  // [T, H/2, 2, W/2, 2C] (the stride-2 walks along H and W become unit walks over the coarse indices at a fixed parity);
  // the spatial zero padding and the padded rows are TMA out-of-bounds fill.
  int conv_C, conv_pad, conv_Ho, conv_Wo, conv_To;
  // RoPE in the QKV epilogue (see vl2.h): adjacent output columns (2i, 2i+1) of a head are a rotation pair
  const uint32_t* rope_tab;
  int rope_cols, rope_D, rope_pos0;
  int trace;   // debug: CTA 0 records clock64() at item boundaries of its first consumer thread (vl2_debug_gemm_trace)
  int epi;     // epilogue variant (kEpi*), the same for every tile of the launch
};

// [0] items traced; per item t (<= 7), at 8*t + 4: consumer starts the item, 8*t + 5: accumulator complete,
// 8*t + 6: its part of the tile is stored (a variant: its last TMA store issued and done reading shared memory).  Inside
// the item's first 32-column slot (generic epilogue): 8*t + 1: its accumulators selected, 8*t + 2: its residuals loaded
// (both -1 in a variant), 8*t + 3: the slot stored (every epilogue; a variant: its TMA store issued); 8*t + 7 is scratch.
__device__ long long g_gemm_trace[128];

// one 4-byte store replicated by the NVSwitch to every GPU of the multicast group
__device__ __forceinline__ void multimem_st32(void* mc_addr, uint32_t v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc_addr), "f"(__uint_as_float(v)) : "memory");
}

__device__ __forceinline__ float fast_sigmoid_mul(float x, float k_log2e) {
  // x * sigmoid(k x) = x / (1 + 2^(-k*log2e*x)); approximate reciprocal on the MUFU pipe
  return __fdividef(x, 1.f + fast_exp2(-k_log2e * x));
}
__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5 x (1 + tanh(u)) = x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3)      (HF "gelu_pytorch_tanh", SigLIP MLP)
  const float u2 = x * fmaf(0.0356774081f * x, x, 0.7978845608f) * 2.885390082f;   // 2 u log2(e)
  return __fdividef(x, 1.f + fast_exp2(-u2));
}
__device__ __forceinline__ float act_apply(float x, int act) {
  switch (act) {
    case VL2_ACT_QUICK_GELU: return fast_sigmoid_mul(x, 1.702f * 1.4426950408889634f);
    case VL2_ACT_SILU: return fast_sigmoid_mul(x, 1.4426950408889634f);
    case VL2_ACT_GELU_ERF: return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
    case VL2_ACT_GELU_TANH: return gelu_tanh(x);
    default: return x;
  }
}

// One unit of the persistent loop: a whole output tile (part = -1), or - for the tiles of the last, partial round - one
// K-slice of a tile: part 0 owns the tile (adds the other slices' partials and runs the epilogue), parts > 0 dump their
// fp32 accumulators to the workspace.  Every role (producer, consumers) decodes the same sequence.
constexpr size_t kSplitFlagBytes = 65536;  // arrival counters at the head of the split-K workspace, one 128-byte line each
constexpr int kSplitFlagStride = 32;       // (zero at first use, self-resetting)
constexpr double kSplitOverheadCycles = 16000.0;   // dump + fence + flag + owner's partial reads
struct WorkItem { int tile, kb0, kb1, part; };
__device__ __forceinline__ WorkItem decode_item(int item, const GemmParams& p, int nkb) {
  WorkItem w;
  if (item < p.split_first) {
    w.tile = item; w.kb0 = 0; w.kb1 = nkb; w.part = -1;
  } else {
    const int j = item - p.split_first;
    w.tile = p.split_first + j / p.split_s;
    w.part = j % p.split_s;
    w.kb0 = (int)((long long)w.part * nkb / p.split_s);
    w.kb1 = (int)((long long)(w.part + 1) * nkb / p.split_s);
  }
  return w;
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// A consumer warp hands a ring slot back to the producer(s).  A pair releases it in both CTAs, since the peer's multicast
// also writes into it.  No memory fence is needed: the slot holds only wgmma operands, whose (async-proxy) reads are
// complete once wgmma.wait_group has returned, and the next write into the slot is a TMA load that the producer issues only
// after its mbarrier wait has observed this arrival.  So the arrival publishes no data and needs no release at cluster
// scope; mbar_arrive_cluster (release.cluster) would put a GPU-scope MEMBAR in every consumer warp's k-loop.
template <bool PAIR>
__device__ __forceinline__ void release_slot(uint64_t* empty_bar, uint32_t rank) {
  mbar_arrive(empty_bar);
  if (PAIR) mbar_arrive_peer(empty_bar, rank ^ 1u);
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }

// sum the producer's per-32-column partials of one row in a fixed order (deterministic: no atomics anywhere).  kRolled
// keeps the vector loop rolled (the same sums in the same order): for the row-factor warps, which run with 40 registers.
template <bool kRolled>
__device__ __forceinline__ float sum_parts(const float* pp, int nparts) {
  const int nvec = (nparts % 4 == 0) ? nparts : 0;   // rows are 16-byte aligned only then
  float q = 0.f;
  int i = 0;
  if (kRolled) {
#pragma unroll 1
    for (; i + 4 <= nvec; i += 4) {
      const float4 t4 = *reinterpret_cast<const float4*>(pp + i);
      q += (t4.x + t4.y) + (t4.z + t4.w);
    }
  } else {
    for (; i + 4 <= nvec; i += 4) {
      const float4 t4 = *reinterpret_cast<const float4*>(pp + i);
      q += (t4.x + t4.y) + (t4.z + t4.w);
    }
  }
  for (; i < nparts; ++i) q += pp[i];
  return q;
}

// ---------------------------------------------------------------------------------------------------------------------
// Epilogue of one consumer thread.  wgmma accumulator layout (m64 x BN, warp w of the warpgroup, lane = 4 g + t):
//   acc[4 j + 0, 1] = rows 16 w + g,     columns 8 j + 2 t, 8 j + 2 t + 1
//   acc[4 j + 2, 3] = rows 16 w + g + 8, the same columns
// so a thread holds two rows and, per 8-column group, an adjacent column pair: exactly a SwiGLU (gate, up) pair and a
// RoPE rotation pair.  The four threads of a quad (same g) together hold a row's 8 columns of every group; the
// per-32-column statistics are reduced over the quad.
// ---------------------------------------------------------------------------------------------------------------------
// The two output rows of a consumer thread and their per-row factors, shared by every epilogue.
struct EpiRows {
  int rows[2];    // output row (p.M = none)
  float rs[2];    // row factor: row_scale x folded-norm rstd
  float mu[2];    // folded LayerNorm mean
  bool ok[2];
};
// The row factor of output row `row` (1 past p.M) and its folded LayerNorm mean (0 without).  The consumers of the generic
// epilogue compute it for their own rows; for a variant the epilogue-operand warp computes the tile's rows into shared
// memory during the k-loop.
template <bool kRolled>
__device__ __forceinline__ float row_factor(const GemmParams& p, int row, float& mu) {
  float rs = (p.row_scale != nullptr && row < p.M) ? p.row_scale[row] : 1.f;
  mu = 0.f;
  if (p.rms_sumsq_in != nullptr && row < p.M) {
    float q = sum_parts<kRolled>(p.rms_sumsq_in + (int64_t)row * p.rms_nparts, p.rms_nparts) * p.rms_inv_dim;   // E[x^2]
    if (p.ln_sum_in != nullptr) {
      mu = sum_parts<kRolled>(p.ln_sum_in + (int64_t)row * p.rms_nparts, p.rms_nparts) * p.rms_inv_dim;
      q = fmaxf(q - mu * mu, 0.f);                                                                      // variance
    }
    rs *= rsqrtf(q + p.rms_eps);
  }
  return rs;
}
__device__ __forceinline__ EpiRows epi_rows(const GemmParams& p, int m0, int rloc) {
  EpiRows r;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m0 + rloc + 8 * h;
    r.ok[h] = row < p.M;
    r.rs[h] = row_factor<false>(p, row, r.mu[h]);
    int gr = row;
    if (p.conv_C > 0) {   // padded (to, ho16, wo16) row -> real output row, or nothing for the padding positions
      const int wo = gr % kConvLine, ho = (gr / kConvLine) % kConvLine, to = gr / (kConvLine * kConvLine);
      gr = (wo < p.conv_Wo && ho < p.conv_Ho && to < p.conv_To) ? (to * p.conv_Ho + ho) * p.conv_Wo + wo : p.M;
      r.ok[h] = gr < p.M;
    }
    r.rows[h] = gr;
  }
  return r;
}

// Trace points inside the first 32-column slot of an epilogue (see g_gemm_trace); `tr` is null when not traced.
__device__ __forceinline__ void trace_point(long long* tr, int i) {
  if (tr != nullptr) tr[i] = clock64();
}

// The generic epilogue: every feature tested at run time, one 32-column slot per iteration.  It serves the launches no
// specialised variant covers (fp32 output, the conv front end, peer / multicast copies, folded LayerNorm, split-K).
template <int BN>
__device__ __forceinline__ void gemm_epilogue(float (&acc)[BN / 2], const GemmParams& p, const EpiRows& r, int n0,
                                              long long* tr) {
  const int lane = threadIdx.x & 31, t = lane & 3;
  const bool swiglu = p.act == VL2_ACT_SWIGLU;
  const bool ln = p.ln_sum_in != nullptr;
  const int* rows = r.rows;
  const float* rs = r.rs;
  const float* mu = r.mu;
  const bool* ok = r.ok;
  const __nv_bfloat16* res = reinterpret_cast<const __nv_bfloat16*>(p.residual);
  __nv_bfloat16* cb = reinterpret_cast<__nv_bfloat16*>(p.C);
  // 32-column slots, one per iteration and NOT unrolled.  A slot's code carries every epilogue feature, about 340
  // instructions per column pair.  Unrolled over all BN / 32 slots it made a ~400 KB kernel, far more than the SM's
  // instruction caches hold, and the epilogue of a 128 x 256 tile took ~200 k cycles in the kernel's trace; rolled here
  // and over the 8-column groups below, the kernel is ~3.5 k instructions and the same epilogue takes ~50 k.  Registers
  // cannot be indexed at run time, so each iteration first selects its slot's 16 accumulators into v[] with compile-time
  // indices.
#pragma unroll 1
  for (int s = 0; s < BN / 32; ++s) {
    if (n0 + 32 * s >= p.N) break;         // uniform over the warpgroup
    float v[16];
#pragma unroll
    for (int k = 0; k < BN / 32; ++k) {
      if (k == s) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = acc[16 * k + i];
      }
    }
    if (s == 0) trace_point(tr, 1);
    // the slot's residuals in one batch of loads: one L2 round trip per slot instead of one per column pair.  A residual
    // that aliases the output is read at this thread's own output positions only, before the thread writes them.
    uint32_t rv[4][2] = {};
    if (res != nullptr) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int c = n0 + 8 * (4 * s + jj) + 2 * t;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (n0 + 8 * (4 * s + jj) < p.N && ok[h]) rv[jj][h] = *reinterpret_cast<const uint32_t*>(res + (int64_t)rows[h] * p.ldr + c);
      }
    }
    if (s == 0 && tr != nullptr) {   // the store consumes two of the loads: the clock after it is their round trip
      tr[7] = rv[0][0] ^ rv[3][1];
      trace_point(tr, 2);
    }
    float ssq[2] = {0.f, 0.f}, ssum[2] = {0.f, 0.f};
#pragma unroll 1
    for (int jj = 0; jj < 4; ++jj) {   // 8-column groups, not unrolled either: the loop body is two column pairs
      float vj[4] = {v[0], v[1], v[2], v[3]};
      uint32_t rj[2] = {rv[0][0], rv[0][1]};
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        if (k == jj) {
#pragma unroll
          for (int i = 0; i < 4; ++i) vj[i] = v[4 * k + i];
          rj[0] = rv[k][0];
          rj[1] = rv[k][1];
        }
      }
      const int j = 4 * s + jj;
      const int c = n0 + 8 * j + 2 * t;    // this thread's column pair
      const bool col_ok = n0 + 8 * j < p.N;   // N % 8 == 0: the whole 8-column group is in or out
      float2 bq = make_float2(0.f, 0.f), cs = make_float2(0.f, 0.f);
      if (col_ok && p.bias != nullptr) bq = __ldg(reinterpret_cast<const float2*>(p.bias + c));
      if (col_ok && ln) cs = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + c));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float x0 = vj[2 * h], x1 = vj[2 * h + 1];
        if (ln) { x0 = fmaf(-mu[h], cs.x, x0); x1 = fmaf(-mu[h], cs.y, x1); }
        x0 = x0 * rs[h] + bq.x;
        x1 = x1 * rs[h] + bq.y;
        const bool st_ok = col_ok && ok[h];
        if (swiglu) {
          // (gate, up) -> one output at column c / 2; the even lane of a lane pair stores both lanes' outputs
          const float o = fast_sigmoid_mul(x0, 1.4426950408889634f) * x1;
          const float o_next = __shfl_down_sync(0xffffffffu, o, 1);
          if (st_ok && (t & 1) == 0) {
            *reinterpret_cast<uint32_t*>(cb + (int64_t)rows[h] * p.ldc + (c >> 1)) = pack_bf16(o, o_next);
          }
          continue;
        }
        x0 = act_apply(x0, p.act);
        x1 = act_apply(x1, p.act);
        if (p.rope_tab != nullptr && c < p.rope_cols && st_ok) {
          const uint32_t e = __ldg(p.rope_tab + (int64_t)(p.rope_pos0 + rows[h]) * (p.rope_D >> 1) + ((c % p.rope_D) >> 1));
          const float co = bf16_lo(e), sn = bf16_hi(e);
          const float a = x0, b = x1;
          x0 = a * co - b * sn;
          x1 = b * co + a * sn;
        }
        if (res != nullptr && st_ok) {
          x0 += bf16_lo(rj[h]);
          x1 += bf16_hi(rj[h]);
        }
        if (p.out_f32) {
          if (st_ok) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + (int64_t)rows[h] * p.ldc + c) = make_float2(x0, x1);
          continue;
        }
        const uint32_t pk = pack_bf16(x0, x1);
        if (st_ok) {
          const int64_t off = (int64_t)rows[h] * p.ldc + c;
          *reinterpret_cast<uint32_t*>(cb + off) = pk;
          if (p.mc != nullptr) {
            multimem_st32(p.mc + off, pk);
          } else {
            for (int pi = 0; pi < p.n_bcast; ++pi) *reinterpret_cast<uint32_t*>(p.bcast[pi] + off) = pk;
          }
        }
        const float a0 = bf16_lo(pk), a1 = bf16_hi(pk);   // statistics of what the consumer will read
        ssq[h] += a0 * a0 + a1 * a1;
        ssum[h] += a0 + a1;
      }
    }
    if (p.sumsq_out != nullptr) {   // one slot per 32 output columns (N % 32 == 0), reduced over the quad
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float q = ssq[h], sm = ssum[h];
        q += __shfl_xor_sync(0xffffffffu, q, 1);
        q += __shfl_xor_sync(0xffffffffu, q, 2);
        sm += __shfl_xor_sync(0xffffffffu, sm, 1);
        sm += __shfl_xor_sync(0xffffffffu, sm, 2);
        if (t == 0 && ok[h]) {
          const int64_t slot = (int64_t)rows[h] * (p.N >> 5) + ((n0 >> 5) + s);
          p.sumsq_out[slot] = q;
          if (p.rowsum_out != nullptr) p.rowsum_out[slot] = sm;
        }
      }
    }
    if (s == 0) trace_point(tr, 3);
  }
}

// Epilogue variants, one per launch (GemmParams::epi, chosen by classify_epilogue on the host).  A variant has its
// features fixed at compile time; the arithmetic is the generic epilogue's, operation for operation, so the results are
// bit-identical to it.
enum : int {
  kEpiGeneric = 0,
  kEpiNone,          // row factor only (row_scale / folded RMSNorm)
  kEpiBias,
  kEpiBiasSigmoid,   // bias + x * sigmoid(k x): quick-GELU (k = 1.702) or SiLU (k = 1)
  kEpiBiasGeluErf,
  kEpiBiasGeluTanh,
  kEpiBiasRes,
  kEpiResSumsq,      // residual + per-32-column sums of squares (decoder o_proj / down)
  kEpiRope,          // (+ bias, run-time) + RoPE (fused QKV)
  kEpiSwiglu,        // SwiGLU (gate-up)
};

// Does 32-column slot c0 of a variant's tile have an operand slot (residual or RoPE table entries) in the operand ring?
// The epilogue-operand warp and the consumers walk the same sequence.
__device__ __forceinline__ bool slot_has_operand(const GemmParams& p, int c0) {
  return p.epi == kEpiBiasRes || p.epi == kEpiResSumsq || (p.epi == kEpiRope && c0 < p.rope_cols);
}
template <int BN>
__device__ __forceinline__ int epi_slots(const GemmParams& p, int n0) { return min(BN / 32, (p.N - n0 + 31) / 32); }

// Byte offset of 4-byte word `word` of 16-byte chunk `chunk` in row r of a shared-memory tile of 64-byte rows that TMA
// reads or writes with SWIZZLE_64B (the chunk index XOR bits 1-2 of the row), and the same for 32-byte rows with
// SWIZZLE_32B (XOR bit 2 of the row).  The eight rows of a warp's fragment access then fall on distinct banks.
__device__ __forceinline__ uint32_t swz64(int r, int chunk, int word) { return r * 64 + ((chunk ^ ((r >> 1) & 3)) << 4) + 4 * word; }
__device__ __forceinline__ uint32_t swz32(int r, int chunk, int byte) { return r * 32 + ((chunk ^ ((r >> 2) & 1)) << 4) + byte; }

// The epilogue variants' shared memory (see kEpiSmemBytes) and, right behind it, their barriers.  One base pointer: the
// roles that use it run with few registers.
static constexpr int kEpiBarriers = 4 + 2 * kOpSlots;
struct EpiSmem {
  uint8_t* base;
  __device__ uint8_t* out(int cw, int i) const { return base + (2 * cw + i) * kStageTileBytes; }   // warp cw's tile i
  __device__ uint8_t* op(int k) const { return base + kEpiOutBytes + k * kOpSlotBytes; }
  __device__ float* rs(int b) const { return reinterpret_cast<float*>(base + kEpiOutBytes + kOpSlots * kOpSlotBytes) + b * 128; }
  __device__ uint64_t* bar(int i) const { return reinterpret_cast<uint64_t*>(base + kEpiSmemBytes) + i; }
  __device__ uint64_t* rs_full(int b) const { return bar(b); }                   // row-factor warps -> consumers
  __device__ uint64_t* rs_empty(int b) const { return bar(2 + b); }              // consumer warps -> row-factor warps
  __device__ uint64_t* op_full(int k) const { return bar(4 + k); }               // TMA -> consumers
  __device__ uint64_t* op_empty(int k) const { return bar(4 + kOpSlots + k); }   // consumer warps -> operand warp
};

// bias of one 32-column slot (zero past N or without bias), loaded one slot ahead of its use
__device__ __forceinline__ void load_bias(float2 (&b)[4], const GemmParams& p, int n0, int s) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int c = n0 + 8 * (4 * s + jj) + 2 * t;
    b[jj] = make_float2(0.f, 0.f);
    if (p.bias != nullptr && n0 + 8 * (4 * s + jj) < p.N) b[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + c));
  }
}

// One 32-column slot s of a variant, from the slot's 16 accumulators v[], its operand words op[] (residual or RoPE table
// entries, read from the operand ring) and bias, into the warp's staging tile at shared address `stage`.  Every value is
// written; the TMA store clips rows and columns outside the output.
template <int V>
__device__ __forceinline__ void epilogue_slot(const float* v, const uint32_t (&op)[4][2], const float2 (&bias)[4],
                                              const GemmParams& p, const EpiRows& r, int n0, int s, float k_log2e,
                                              uint32_t stage) {
  constexpr bool kRes = V == kEpiBiasRes || V == kEpiResSumsq;
  constexpr bool kSumsq = V == kEpiResSumsq;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  float ssq[2] = {0.f, 0.f};
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * s + jj;
    const int c = n0 + 8 * j + 2 * t;
    const bool col_ok = n0 + 8 * j < p.N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float x0 = v[4 * jj + 2 * h], x1 = v[4 * jj + 2 * h + 1];
      x0 = x0 * r.rs[h] + bias[jj].x;   // a launch without bias adds 0, as the generic epilogue does
      x1 = x1 * r.rs[h] + bias[jj].y;
      const bool st_ok = col_ok && r.ok[h];
      if (V == kEpiSwiglu) {
        // output columns 4 jj + t, 4 jj + t + 1 of the slot's 16: the even lane of a lane pair writes both lanes' outputs
        const float o = fast_sigmoid_mul(x0, 1.4426950408889634f) * x1;
        const float o_next = __shfl_down_sync(0xffffffffu, o, 1);
        if ((t & 1) == 0) sts32(stage + swz32(g + 8 * h, jj >> 1, 8 * (jj & 1) + 2 * t), pack_bf16(o, o_next));
        continue;
      }
      if (V == kEpiBiasSigmoid) { x0 = fast_sigmoid_mul(x0, k_log2e); x1 = fast_sigmoid_mul(x1, k_log2e); }
      if (V == kEpiBiasGeluErf) { x0 = act_apply(x0, VL2_ACT_GELU_ERF); x1 = act_apply(x1, VL2_ACT_GELU_ERF); }
      if (V == kEpiBiasGeluTanh) { x0 = gelu_tanh(x0); x1 = gelu_tanh(x1); }
      if (V == kEpiRope && c < p.rope_cols && st_ok) {
        const uint32_t e = op[jj][h];
        const float co = bf16_lo(e), sn = bf16_hi(e);
        const float a = x0, b = x1;
        x0 = a * co - b * sn;
        x1 = b * co + a * sn;
      }
      if (kRes && st_ok) {
        x0 += bf16_lo(op[jj][h]);
        x1 += bf16_hi(op[jj][h]);
      }
      const uint32_t pk = pack_bf16(x0, x1);
      sts32(stage + swz64(g + 8 * h, jj, t), pk);
      if (kSumsq) {
        const float a0 = bf16_lo(pk), a1 = bf16_hi(pk);
        ssq[h] += a0 * a0 + a1 * a1;
      }
    }
  }
  if (kSumsq) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float q = ssq[h];
      q += __shfl_xor_sync(0xffffffffu, q, 1);
      q += __shfl_xor_sync(0xffffffffu, q, 2);
      if (t == 0 && r.ok[h]) p.sumsq_out[(int64_t)r.rows[h] * (p.N >> 5) + ((n0 >> 5) + s)] = q;
    }
  }
}

// The epilogue of a consumer thread.  `it` counts the CTA's items (row-factor buffer), `op_idx` the operand slots so far.
//
// A variant takes its row factors from shared memory and loops over 32-column slots without unrolling: unrolled over a
// 128 x 256 tile, the nine of them made a ~20 k-instruction kernel.  Each iteration works on acc[0..15], indices fixed at
// compile time, and then moves the array down by one slot (register moves; no run-time select of the slot's
// accumulators).  Per slot a warp reads its operand words from the ring, writes its 16 x 32 piece into one of its two
// staging tiles and one lane stores that by TMA without waiting for it; a staging tile is rewritten once the store that
// read it two slots ago has finished reading (the previous tile's stores, a k-loop ago, before the first slot).  A residual that aliases the output is in shared memory before the tile's
// stores of the same positions are issued.
template <int BN>
__device__ __forceinline__ void run_epilogue(float (&acc)[BN / 2], const GemmParams& p, const CUtensorMap* tmap_c,
                                             const EpiSmem& sm, int m0, int n0, int rloc, int it, uint32_t& op_idx,
                                             long long* tr) {
  if (p.epi == kEpiGeneric) {
    gemm_epilogue<BN>(acc, p, epi_rows(p, m0, rloc), n0, tr);
    return;
  }
  if (tr != nullptr) { tr[1] = -1; tr[2] = -1; }   // generic-only trace points: not recorded by this launch
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int cw = (threadIdx.x - 128) >> 5;         // consumer warp 0..7: rows [16 cw, 16 cw + 16) of the tile
  EpiRows r;
  {
    const int b = it & 1;
    mbar_wait(sm.rs_full(b), (it >> 1) & 1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      r.rows[h] = m0 + rloc + 8 * h;
      r.ok[h] = r.rows[h] < p.M;
      r.rs[h] = sm.rs(b)[rloc + 8 * h];
      r.mu[h] = 0.f;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(sm.rs_empty(b));
  }
  const float k_log2e = p.act == VL2_ACT_QUICK_GELU ? 1.702f * 1.4426950408889634f : 1.4426950408889634f;
  const int nslots = epi_slots<BN>(p, n0);
  const bool swiglu = p.epi == kEpiSwiglu;
  float2 bias[4], bias_next[4];
  load_bias(bias, p, n0, 0);
  if (lane == 0) bulk_wait_read<0>();
#pragma unroll 1
  for (int s = 0; s < nslots; ++s) {
    if (s + 1 < nslots) load_bias(bias_next, p, n0, s + 1);
    uint32_t op[4][2] = {};
    if (slot_has_operand(p, n0 + 32 * s)) {
      const int k = op_idx % kOpSlots;
      mbar_wait(sm.op_full(k), (op_idx / kOpSlots) & 1);
      const uint32_t base = smem_u32(sm.op(k));
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) op[jj][h] = lds32(base + swz64(rloc + 8 * h, jj, t));
      __syncwarp();
      if (lane == 0) mbar_arrive(sm.op_empty(k));
      ++op_idx;
    }
    uint8_t* stage = sm.out(cw, s & 1);
    if (lane == 0 && s >= 2) bulk_wait_read<1>();   // the store that read this staging tile (slot s - 2) is done reading it
    __syncwarp();
    const uint32_t st = smem_u32(stage);
    switch (p.epi) {   // uniform over the launch
      case kEpiNone: epilogue_slot<kEpiNone>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiBias: epilogue_slot<kEpiBias>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiBiasSigmoid: epilogue_slot<kEpiBiasSigmoid>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiBiasGeluErf: epilogue_slot<kEpiBiasGeluErf>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiBiasGeluTanh: epilogue_slot<kEpiBiasGeluTanh>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiBiasRes: epilogue_slot<kEpiBiasRes>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiResSumsq: epilogue_slot<kEpiResSumsq>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      case kEpiRope: epilogue_slot<kEpiRope>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
      default: epilogue_slot<kEpiSwiglu>(acc, op, bias, p, r, n0, s, k_log2e, st); break;
    }
    fence_proxy_async_smem();   // the warp's writes -> visible to the TMA store
    __syncwarp();
    if (lane == 0) {
      tma_store_2d(tmap_c, stage, swiglu ? (n0 >> 1) + 16 * s : n0 + 32 * s, m0 + 16 * cw);
      bulk_commit_group();
    }
#pragma unroll
    for (int i = 0; i + 16 < BN / 2; ++i) acc[i] = acc[i + 16];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) bias[jj] = bias_next[jj];
    if (s == 0) trace_point(tr, 3);
  }
}

template <int BN, bool PAIR>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_op,
                       const GemmParams p) {
  using Cfg = GemmCfg<BN, PAIR>;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int tile0 = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;        // persistent tile loop start / stride
  const int tile_stride = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  constexpr int kTileM = PAIR ? 2 * BM : BM;
  // SWIZZLE_128B operands need 1024-byte aligned stage bases: the kernel has no static smem, so the dynamic window
  // starts at offset 0 of the CTA's shared memory (checked below; a misaligned base traps instead of corrupting).
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) { asm volatile("trap;"); }
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kStageBytesA;
  const EpiSmem es{smem + Cfg::kStages * Cfg::kStageBytes};   // 1024-byte aligned: stage sizes are multiples of 1 KB
  uint64_t* bars = es.bar(kEpiBarriers);
  uint64_t* full_bar = bars;                        // [kStages]  TMA -> consumers
  uint64_t* empty_bar = bars + Cfg::kStages;        // [kStages]  consumers (of both CTAs of a pair) -> TMA

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_k_blocks = (p.K + BK - 1) / BK;

  pdl_launch_dependents();   // let the next kernel's CTAs take the SMs this kernel's last wave leaves idle
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], Cfg::kEmptyArrivals);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(es.rs_full(i), 64);
      mbar_init(es.rs_empty(i), kConsumerThreads / 32);
    }
    for (int i = 0; i < kOpSlots; ++i) {
      mbar_init(es.op_full(i), 1);
      mbar_init(es.op_empty(i), kConsumerThreads / 32);
    }
    if (p.epi != kEpiGeneric) {
      tma_prefetch_desc(&tmap_c);
      if (p.residual != nullptr || p.rope_tab != nullptr) tma_prefetch_desc(&tmap_op);
    }
    fence_barrier_init();
  }
  pdl_wait();                // predecessors complete + visible: nothing above touched global memory
  if (PAIR) cluster_sync_all(); else __syncthreads();   // barrier inits visible (cluster-wide for a pair)

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      const bool conv = p.conv_C > 0;
      const int slabs = conv ? p.conv_C / BK : 1;
      for (int item = tile0; item < p.num_items; item += tile_stride) {
        const WorkItem w = decode_item(item, p, num_k_blocks);
        const int m0 = (w.tile % p.num_m_tiles) * kTileM + (int)rank * BM;
        const int n0 = (w.tile / p.num_m_tiles) * BN;
        // conv: this 128-row tile = output lines ho_base .. ho_base + 7 of time step `to`
        const int line0 = m0 / kConvLine, to = line0 / kConvLine, ho_base = line0 % kConvLine;
        int tap = w.kb0 / slabs, slab = w.kb0 - tap * slabs;
        for (int kb = w.kb0; kb < w.kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);   // a pair: own A + both halves of B land here
          uint8_t* dst_a = smem_a + stage * Cfg::kStageBytesA;
          if (conv) {
            // implicit im2col: k-block = (tap, 64-channel slab).  Input index along each axis = 2 * out + e, e = d - pad in
            // {-1, 0, 1}: parity e & 1, coarse index out + floor(e / 2)  (-1 = the zero-padded border -> out of bounds)
            const int et = (tap >> 2) - p.conv_pad, eh = ((tap >> 1) & 1) - p.conv_pad, ew = (tap & 1) - p.conv_pad;
            const int ph = eh & 1, pw = ew & 1;
            const int c0 = pw * p.conv_C + slab * BK, wc0 = (ew - pw) / 2, hc0 = ho_base + (eh - ph) / 2, t = 2 * to + et;
            tma_load_5d(dst_a, &tmap_a, &full_bar[stage], c0, wc0, ph, hc0, t);
            if (++slab == slabs) { slab = 0; ++tap; }
          } else {
            tma_load_2d(dst_a, &tmap_a, &full_bar[stage], kb * BK, m0);
          }
          uint8_t* dst_b = smem_b + stage * Cfg::kStageBytesB;
          if (PAIR) tma_load_2d_mc(dst_b + rank * Cfg::kHalfBytesB, &tmap_b, &full_bar[stage], kb * BK, n0 + (int)rank * (BN / 2), 3);
          else tma_load_2d(dst_b, &tmap_b, &full_bar[stage], kb * BK, n0);
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    } else if (warp == 1 && lane == 0 && p.epi != kEpiGeneric && (p.residual != nullptr || p.rope_tab != nullptr)) {
      // ===================== epilogue operands of a variant: residual / RoPE-table slots =====================
      // The tile's operand slots into the ring by TMA, the first ones while the tile's k-loop runs.  Independent of the
      // A/B producer, so the A/B ring never waits on epilogue buffers.
      uint32_t op_idx = 0;
      for (int item = tile0; item < p.num_items; item += tile_stride) {
        const WorkItem w = decode_item(item, p, num_k_blocks);   // a variant's launch is not split: item = tile
        const int m0 = (w.tile % p.num_m_tiles) * kTileM + (int)rank * BM;
        const int n0 = (w.tile / p.num_m_tiles) * BN;
        const int nslots = epi_slots<BN>(p, n0);
        for (int s = 0; s < nslots; ++s) {
          const int c0 = n0 + 32 * s;
          if (!slot_has_operand(p, c0)) continue;
          const int k = op_idx % kOpSlots;
          mbar_wait_parked(es.op_empty(k), ((op_idx / kOpSlots) & 1) ^ 1);
          mbar_arrive_expect_tx(es.op_full(k), kOpSlotBytes);
          // the RoPE table [pos][D / 2] of (cos, sin) pairs is mapped as 16-bit pairs: entry e = columns 2 e, 2 e + 1
          if (p.epi == kEpiRope) tma_load_2d(es.op(k), &tmap_op, es.op_full(k), c0 % p.rope_D, p.rope_pos0 + m0);
          else tma_load_2d(es.op(k), &tmap_op, es.op_full(k), c0, m0);
          ++op_idx;
        }
      }
    } else if (warp >= 2 && p.epi != kEpiGeneric) {
      // ===================== epilogue operands of a variant: row factors =====================
      // The tile's 128 row factors (rows i and i + 64 of thread i), with the generic epilogue's arithmetic, into the
      // tile's half of the row-factor buffer while its k-loop runs: the consumers' epilogue starts without a row prologue.
      int it = 0;
      for (int tile = tile0; tile < p.num_items; tile += tile_stride, ++it) {   // a variant's launch is not split
        const int m0 = (tile % p.num_m_tiles) * kTileM + (int)rank * BM;
        const int b = it & 1;
        mbar_wait_parked(es.rs_empty(b), ((it >> 1) & 1) ^ 1);
#pragma unroll 1
        for (int r = threadIdx.x - 64; r < BM; r += 64) {
          float mu;
          es.rs(b)[r] = row_factor<true>(p, m0 + r, mu);
        }
        mbar_arrive(es.rs_full(b));
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== consumers: wgmma main loop + epilogue =====================
    const int wg = (warp >> 2) - 1;              // 0 / 1: rows [64 wg, 64 wg + 64) of the CTA's 128-row block
    const int ctid = threadIdx.x - 128;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's two accumulator rows
    const uint64_t da0 = gmma_desc_sw128(smem_u32(smem_a) + wg * 64 * 128, 16, 1024);
    const uint64_t db0 = gmma_desc_sw128(smem_u32(smem_b), 16, 1024);
    const bool tr = p.trace && blockIdx.x == 0 && ctid == 0;
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    uint32_t op_idx = 0;
    float acc[Cfg::kAcc];
    for (int item = tile0; item < p.num_items; item += tile_stride, ++it) {
      const WorkItem w = decode_item(item, p, num_k_blocks);
      const int tile = w.tile;
      if (tr && it < 7) g_gemm_trace[8 * it + 4] = clock64();
      const int m0 = (tile % p.num_m_tiles) * kTileM + (int)rank * BM;
      const int n0 = (tile / p.num_m_tiles) * BN;
      int prev = -1;
      for (int kb = w.kb0; kb < w.kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        const uint64_t da = da0 + (uint64_t)((stage * Cfg::kStageBytesA) >> 4);
        const uint64_t db = db0 + (uint64_t)((stage * Cfg::kStageBytesB) >> 4);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) Wgmma<BN, 0>::ss(acc, da + 2 * k, db + 2 * k, (kb != w.kb0 || k != 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();            // the previous k-block's MMAs are complete: its ring slot can be refilled
        if (prev >= 0 && lane == 0) release_slot<PAIR>(&empty_bar[prev], rank);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_keep(acc);
      if (lane == 0) release_slot<PAIR>(&empty_bar[prev], rank);
      if (tr && it < 7) g_gemm_trace[8 * it + 5] = clock64();
      const int slot = (tile - p.split_first) * (p.split_s - 1);   // workspace slot of a split tile's slices
      // partials layout per CTA: [accumulator quad][consumer thread][4 floats] (every warp access is one 512-byte piece)
      if (w.part > 0) {
        // ---- K-slice of a split tile: dump the fp32 accumulators, then signal the owner
        float* dst = p.ws_partial + ((size_t)slot + (w.part - 1)) * ((size_t)kTileM * BN) + (size_t)rank * (BM * BN) + ctid * 4;
#pragma unroll
        for (int q = 0; q < Cfg::kAcc / 4; ++q)
          __stcg(reinterpret_cast<float4*>(dst + q * (kConsumerThreads * 4)),
                 make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]));
        __threadfence();
        consumer_sync();   // every thread's partials are fenced
        if (ctid == 0) atomicAdd(p.ws_flags + ((tile - p.split_first) * 2 + (int)rank) * kSplitFlagStride, 1u);
        continue;
      }
      if (w.part == 0) {
        // owner of a split tile: the other K-slices run concurrently on other CTAs of this (last) round.  ONE thread polls
        // (a line of its own per counter): hundreds of pollers on one L2 line starve the arriving atomics
        unsigned* flag = p.ws_flags + ((tile - p.split_first) * 2 + (int)rank) * kSplitFlagStride;
        if (ctid == 0) {
          unsigned spins = 0;
          while (ld_acquire_gpu(flag) < (unsigned)(p.split_s - 1)) {
            if (++spins > (1u << 24)) { asm volatile("trap;"); }
            __nanosleep(200);
          }
        }
        consumer_sync();
        const float* src = p.ws_partial + (size_t)slot * ((size_t)kTileM * BN) + (size_t)rank * (BM * BN) + ctid * 4;
        for (int pp = 0; pp < p.split_s - 1; ++pp) {   // fixed order: deterministic
#pragma unroll
          for (int q = 0; q < Cfg::kAcc / 4; ++q) {
            const float4 t4 = __ldcg(reinterpret_cast<const float4*>(src + (size_t)pp * ((size_t)kTileM * BN) + q * (kConsumerThreads * 4)));
            acc[4 * q] += t4.x; acc[4 * q + 1] += t4.y; acc[4 * q + 2] += t4.z; acc[4 * q + 3] += t4.w;
          }
        }
        consumer_sync();   // every thread has consumed the partials: re-arm the counter for the next launch
        if (ctid == 0) *flag = 0u;
      }
      run_epilogue<BN>(acc, p, &tmap_c, es, m0, n0, rloc, it, op_idx, (tr && it < 7) ? g_gemm_trace + 8 * it : nullptr);
      // the warp's TMA stores are complete before the CTA's shared memory goes away (inside the loop: placed after it, the
      // wait made ptxas hold the consumers to the launch's 168 registers)
      if (item + tile_stride >= p.num_items && lane == 0) bulk_wait_all();
      if (tr && it < 7) {
        bulk_wait_read_all();   // the variants' stores: issued by this thread, done reading shared memory
        g_gemm_trace[8 * it + 6] = clock64();
        g_gemm_trace[0] = it + 1;
      }
    }
  }
  if (PAIR) cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

static bool splitk_enabled();

// Tile choice: a launch costs waves x tile time + one epilogue; a tile costs k-blocks x kb_cycles.  A k-block of a
// 128 x BN tile is bound by the larger of
//   * the tensor pipe: 128 x BN x 64 MACs at ~1024 dense bf16 MACs per clock per SM (the H100 SXM data sheet's
//     989 TFLOP/s over 132 SMs at 1.83 GHz), i.e. 8 x BN cycles, plus ~200 cycles per k-block of barrier hand-over
//     and issue that a wider tile amortises over more columns;
//   * operand ingest from L2: 16 KB of A + the CTA's B bytes (all BN rows, or BN / 2 for a pair) at ~64 B/clk;
//   * the ring's latency cover: ~2000 cycles of L2/HBM latency over the ring's stages.
struct TileChoice { int bn; bool pair; };
static constexpr double kIngestBytesPerClk = 64.0;

static double kb_cycles(int bn, bool pair) {
  const double stage_bytes = 16384.0 + bn * 128.0;
  int stages = (int)((kSmemLimit - 1024 - kEpiSmemBytes) / stage_bytes);   // GemmCfg::kStages
  if (stages > 8) stages = 8;
  const double mma = 128.0 * bn * 64.0 / 1024.0 + 200.0;
  const double ingest = (16384.0 + (pair ? bn / 2 : bn) * 128.0) / kIngestBytesPerClk;
  const double lat = 2000.0 / stages;
  double c = mma > ingest ? mma : ingest;
  return c > lat ? c : lat;
}


// How many persistent units (CTAs, or CTA pairs) of this instantiation the current device can run at once, or a negative
// VL2_E_* code.  A pair needs two free SMs of one GPC, so fewer than sm_count() / 2 pairs may fit; on an H100 SXM
// (132 SMs) all 66 pairs of every width fit, which the persistent grid of launch_gemm assumes.
template <int BN, bool PAIR>
static int coresident_units() {
  using Cfg = GemmCfg<BN, PAIR>;
  VL2_SMEM_OPT_IN((gemm_bf16_wgmma_kernel<BN, PAIR>), Cfg::kSmemBytes);
  int n = 0;
  if (PAIR) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(sm_count() & ~1);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    VL2_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, gemm_bf16_wgmma_kernel<BN, PAIR>, &cfg));
  } else {
    VL2_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gemm_bf16_wgmma_kernel<BN, PAIR>, kGemmThreads,
                                                                 Cfg::kSmemBytes));
    n *= sm_count();
  }
  return n;
}

// The epilogue variant of a launch, from the fields of its arguments that are set.  Launches no variant covers take the
// generic epilogue: fp32 output, the conv front end, peer / multicast copies, folded LayerNorm (ln_sum_in, rowsum_out).
static int classify_epilogue(const vl2_gemm_args* a) {
  if (a->out_f32 || a->conv_C > 0 || a->n_bcast > 0 || a->mc_out != nullptr || a->ln_sum_in != nullptr ||
      a->rowsum_out != nullptr)
    return kEpiGeneric;
  const bool bias = a->bias != nullptr, res = a->residual != nullptr, sumsq = a->sumsq_out != nullptr;
  if (a->act == VL2_ACT_SWIGLU) return bias ? kEpiGeneric : kEpiSwiglu;    // validated: no residual, no statistics
  if (a->rope_tab != nullptr) return sumsq ? kEpiGeneric : kEpiRope;       // validated: no activation, no residual
  if (sumsq) return (res && !bias && a->act == VL2_ACT_NONE) ? kEpiResSumsq : kEpiGeneric;
  if (res) return (bias && a->act == VL2_ACT_NONE) ? kEpiBiasRes : kEpiGeneric;
  if (a->act == VL2_ACT_NONE) return bias ? kEpiBias : kEpiNone;
  if (!bias) return kEpiGeneric;
  switch (a->act) {
    case VL2_ACT_QUICK_GELU:
    case VL2_ACT_SILU: return kEpiBiasSigmoid;
    case VL2_ACT_GELU_ERF: return kEpiBiasGeluErf;
    case VL2_ACT_GELU_TANH: return kEpiBiasGeluTanh;
    default: return kEpiGeneric;
  }
}

template <int BN, bool PAIR>
static int launch_gemm(const vl2_gemm_args* a, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, PAIR>;
  CUtensorMap ta, tb;
  const bool conv = a->conv_C > 0;
  int conv_To = 0, conv_Ho = 0, conv_Wo = 0;
  if (conv) {
    // x [T,H,W,C] viewed as [T, H/2, 2, W/2, 2C]: a tap's stride-2 walks along H and W are unit walks over the coarse
    // indices at fixed parities (the W parity is folded into the channel coordinate: offset parity*C of the merged 2C axis).
    // Box = 64 channels x 16 coarse columns (one padded output line) x 8 coarse rows (the tile's 8 output lines).
    const int p_ = a->conv_pad;
    conv_To = (a->conv_T + 2 * p_ - 2) / 2 + 1;
    conv_Ho = (a->conv_H + 2 * p_ - 2) / 2 + 1;
    conv_Wo = (a->conv_W + 2 * p_ - 2) / 2 + 1;
    // odd H / W without padding (SigLIP 27 x 27, stc_connector_v35): the last coarse index would pair the last pixel with
    // the first one of the next row / frame; no stored output needs it, so it is declared out of bounds (zero fill)
    const uint64_t wcols = (a->conv_W % 2 == 1 && p_ == 0) ? (uint64_t)a->conv_W / 2 : (uint64_t)(a->conv_W + 1) / 2;
    const uint64_t hrows = (a->conv_H % 2 == 1 && p_ == 0) ? (uint64_t)a->conv_H / 2 : (uint64_t)(a->conv_H + 1) / 2;
    const uint64_t C_ = (uint64_t)a->conv_C, W_ = (uint64_t)a->conv_W, H_ = (uint64_t)a->conv_H;
    uint64_t dims[5] = {2 * C_, wcols, 2, hrows, (uint64_t)a->conv_T};
    uint64_t str[4] = {2 * C_ * 2, W_ * C_ * 2, 2 * W_ * C_ * 2, H_ * W_ * C_ * 2};
    uint32_t box[5] = {BK, (uint32_t)kConvLine, 1, (uint32_t)(BM / kConvLine), 1};
    int rc = make_tmap_bf16(&ta, a->A, 5, dims, str, box);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
    uint64_t str[1] = {(uint64_t)a->lda * 2};
    uint32_t box[2] = {BK, BM};
    int rc = make_tmap_bf16(&ta, a->A, 2, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
    uint64_t str[1] = {(uint64_t)a->ldw * 2};
    uint32_t box[2] = {BK, (uint32_t)(PAIR ? BN / 2 : BN)};
    int rc = make_tmap_bf16(&tb, a->W, 2, dims, str, box);
    if (rc) return rc;
  }
  GemmParams p;
  p.C = a->C; p.bias = a->bias; p.residual = a->residual; p.row_scale = a->row_scale;
  p.ldc = a->ldc; p.ldr = a->ldr; p.M = a->M; p.N = a->N; p.K = a->K; p.act = a->act; p.out_f32 = a->out_f32;
  p.rms_sumsq_in = a->rms_sumsq_in; p.sumsq_out = a->sumsq_out; p.rms_nparts = a->rms_nparts;
  p.ln_sum_in = a->ln_sum_in; p.ln_colsum = a->ln_colsum; p.rowsum_out = a->rowsum_out;
  p.rms_inv_dim = a->rms_inv_dim; p.rms_eps = a->rms_eps;
  // reserved2: 777 traces the launch, 778 forces the generic epilogue (tests compare it with the variants), 779 both
  p.trace = (a->reserved2 == 777 || a->reserved2 == 779) ? 1 : 0;
  p.n_bcast = a->n_bcast;
  p.mc = reinterpret_cast<__nv_bfloat16*>(a->mc_out);
  for (int i = 0; i < 8; ++i) p.bcast[i] = reinterpret_cast<__nv_bfloat16*>(i < a->n_bcast ? a->bcast_out[i] : nullptr);
  const int tile_m = PAIR ? 2 * BM : BM;
  p.rope_tab = a->rope_tab; p.rope_cols = a->rope_cols; p.rope_D = a->rope_D; p.rope_pos0 = a->rope_pos0;
  p.conv_C = conv ? a->conv_C : 0; p.conv_pad = a->conv_pad; p.conv_Ho = conv_Ho; p.conv_Wo = conv_Wo; p.conv_To = conv_To;
  const int m_rows = conv ? conv_To * kConvLine * kConvLine : a->M;     // rows of the (padded) A enumeration
  p.num_m_tiles = (m_rows + tile_m - 1) / tile_m;
  p.num_n_tiles = (a->N + BN - 1) / BN;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int slots = PAIR ? sm_count() / 2 : sm_count();
  // Split-K of the last, partial round (wave quantisation): the `rem` tiles left for `slots` CTAs (pairs) are cut into s
  // K-slices each, so the round costs a fraction of a tile time.  Slice 0 owns the tile: it adds the other slices' fp32
  // partials (workspace, fixed order -> deterministic) and runs the epilogue.  Needs the caller's workspace (splitk_ws).
  p.split_first = tiles;
  p.split_s = 1;
  p.ws_flags = nullptr;
  p.ws_partial = nullptr;
  {
    const int num_kb = (a->K + BK - 1) / BK;
    const int rem = tiles % slots;
    // s slices per remaining tile; the rem * s items may need more than one sub-round: pick the s with the shortest tail
    // ceil(rem * s / slots) / s (in tile times; 1.0 = unsplit).  Items are dealt out in index order, an owner only waits for
    // higher-numbered items and an item is only queued behind a lower-numbered one, so the waits cannot form a cycle.
    int s = 1;
    if (rem > 0) {
      // a split must beat the unsplit round by 10 % after paying for the partials' round trip through L2
      const double tile_cycles = kb_cycles(BN, PAIR) * num_kb;
      double best = 0.9 * tile_cycles;
      for (int c = 2; c <= 4; ++c) {
        if (num_kb / c < 8) break;
        const double tail = (double)((rem * c + slots - 1) / slots) / c;
        const double cost = tail * tile_cycles + kSplitOverheadCycles;
        if (cost < best) { best = cost; s = c; }
      }
    }
    const bool forced = rem > 0 && a->reserved3 >= 2 && a->reserved3 <= 4 && num_kb >= a->reserved3;   // test hook
    if (forced) s = a->reserved3;
    const size_t need = kSplitFlagBytes + (size_t)rem * (s > 1 ? s - 1 : 0) * tile_m * BN * sizeof(float);
    if (s > 1 && (splitk_enabled() || forced) && a->splitk_ws != nullptr && (size_t)a->splitk_ws_bytes >= need &&
        (size_t)2 * rem * kSplitFlagStride * 4 <= kSplitFlagBytes && aligned16(a->splitk_ws)) {
      p.split_first = tiles - rem;
      p.split_s = s;
      p.ws_flags = reinterpret_cast<unsigned*>(a->splitk_ws);
      p.ws_partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a->splitk_ws) + kSplitFlagBytes);
    }
  }
  p.num_items = p.split_first + (tiles - p.split_first) * p.split_s;
  p.epi = (p.split_s > 1 || a->reserved2 == 778 || a->reserved2 == 779) ? kEpiGeneric : classify_epilogue(a);
  // A variant's output leaves by TMA stores of 16-row slots whose map clips the M and N tails (and keeps a strided view's
  // columns past N untouched); its residual or RoPE table arrives by TMA loads of 128-row slots.  vl2_gemm_bf16 requires
  // 16-byte aligned pointers and leading dimensions that are multiples of 8 elements, so every such launch has the maps.
  CUtensorMap tc, top;
  memset(&tc, 0, sizeof(tc));
  memset(&top, 0, sizeof(top));
  if (p.epi != kEpiGeneric) {
    const bool swiglu = p.epi == kEpiSwiglu;
    uint64_t dims[2] = {(uint64_t)(swiglu ? a->N / 2 : a->N), (uint64_t)a->M};
    uint64_t str[1] = {(uint64_t)a->ldc * 2};
    uint32_t box[2] = {swiglu ? 16u : 32u, 16u};
    int rc = make_tmap_bf16(&tc, a->C, 2, dims, str, box, swiglu ? 32 : 64);
    if (rc) return rc;
    if (p.epi == kEpiRope) {
      uint64_t rdims[2] = {(uint64_t)a->rope_D, (uint64_t)a->rope_pos0 + (uint64_t)a->M};   // the positions it reads
      uint64_t rstr[1] = {(uint64_t)a->rope_D * 2};
      uint32_t rbox[2] = {32u, (uint32_t)BM};
      rc = make_tmap_bf16(&top, a->rope_tab, 2, rdims, rstr, rbox, 64);
    } else if (a->residual != nullptr) {
      uint64_t rdims[2] = {(uint64_t)a->N, (uint64_t)a->M};
      uint64_t rstr[1] = {(uint64_t)a->ldr * 2};
      uint32_t rbox[2] = {32u, (uint32_t)BM};
      rc = make_tmap_bf16(&top, a->residual, 2, rdims, rstr, rbox, 64);
    }
    if (rc) return rc;
  }
  const int units = p.num_items < slots ? p.num_items : slots;
  const dim3 grid(PAIR ? 2 * units : units), block(kGemmThreads);
  VL2_SMEM_OPT_IN((gemm_bf16_wgmma_kernel<BN, PAIR>), Cfg::kSmemBytes);
  VL2_CHECK_CUDA(launch_kernel(gemm_bf16_wgmma_kernel<BN, PAIR>, grid, block, Cfg::kSmemBytes, stream, PAIR ? 2 : 1, ta, tb, tc, top,
                                 p));
  VL2_CHECK_LAUNCH("gemm_bf16_wgmma_kernel");
  return VL2_OK;
}

static TileChoice choose_tile(int M, int N, int K, int sms, bool allow_pair, bool allow_split) {
  const int kb = (K + BK - 1) / BK;
  static const int cands[7] = {256, 224, 192, 160, 128, 96, 64};
  TileChoice best = {256, false};
  double best_cost = -1;
  for (int pair = (allow_pair ? 1 : 0); pair >= 0; --pair) {
    for (int i = 0; i < 7; ++i) {
      const int bn = cands[i];
      if (pair && bn < 128) continue;
      if (bn > 64 && N <= bn - 32) continue;  // do not pick a tile much wider than the matrix
      const int tile_m = pair ? 256 : 128;
      const long tiles = (long)((M + tile_m - 1) / tile_m) * ((N + bn - 1) / bn);
      const long slots = pair ? sms / 2 : sms;
      const long full = tiles / slots, rem = tiles % slots;
      const double per_kb = kb_cycles(bn, pair != 0);
      // the last, partial round costs a whole tile time, or a fraction of it when launch_gemm can split it along K
      double tail = rem > 0 ? 1.0 : 0.0;
      if (allow_split && rem > 0) {
        for (int c = 2; c <= 4 && kb / c >= 8; ++c) {
          const double t = (double)((rem * c + slots - 1) / slots) / c + kSplitOverheadCycles / (per_kb * kb);
          if (t < tail * 0.9) tail = t;
        }
      }
      const double cost = ((double)full + tail) * (kb * per_kb + 600.0) + 2000.0 + bn * 16.0;
      if (best_cost < 0 || cost < best_cost * 0.98) { best_cost = cost; best.bn = bn; best.pair = pair != 0; }
    }
  }
  return best;
}

// VL2_GEMM_SPLITK=1 enables the split-K tail round (needs the caller's workspace).  Default OFF: it makes a GEMM's
// rounding depend on M (how many tiles land in the last round), which would end the bit-exact frame-sharding /
// frame-independence properties of the vision tower (tests/test_fullsize_gpu.py).
static bool splitk_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VL2_GEMM_SPLITK");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

static bool pair_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VL2_GEMM_PAIR");
    v = (e == nullptr || e[0] != '0') ? 1 : 0;
  }
  return v == 1;
}

}  // namespace vl2

// Host-side planning only (no launch, no device work): which tile the cost model picks for a problem and how the
// persistent grid will be filled.  Lets tests pin the scheduler's decisions for the shapes of the path on a CPU box.
extern "C" int vl2_gemm_plan(int M, int N, int K, int with_splitk_ws, int32_t* out6) {
  using namespace vl2;
  VL2_REQUIRE(M > 0 && N > 0 && K > 0 && out6 != nullptr, VL2_E_BADSHAPE, "vl2_gemm_plan: bad arguments");
  const int sms = sm_count();
  const TileChoice t = choose_tile(M, N, K, sms, pair_enabled(), splitk_enabled() && with_splitk_ws != 0);
  const int tile_m = t.pair ? 2 * BM : BM;
  const int tiles = ((M + tile_m - 1) / tile_m) * ((N + t.bn - 1) / t.bn);
  const int slots = t.pair ? sms / 2 : sms;
  out6[0] = t.bn;
  out6[1] = t.pair ? 1 : 0;
  out6[2] = tiles;
  out6[3] = slots;
  out6[4] = (tiles + slots - 1) / slots;   // rounds of the persistent loop
  out6[5] = sms;
  return VL2_OK;
}

// How many CTAs (pair = 0) or CTA pairs (pair = 1) of the BN-wide GEMM kernel the current device runs at once, from the
// occupancy API at the kernel's shared-memory size.
extern "C" int vl2_gemm_coresident(int bn, int pair, int32_t* out) {
  using namespace vl2;
  VL2_REQUIRE(out != nullptr && bn >= 64 && bn <= 256 && bn % 32 == 0 && (pair == 0 || bn >= 128), VL2_E_BADSHAPE,
              "vl2_gemm_coresident: bad arguments (bn %d, pair %d)", bn, pair);
  int n;
  if (pair) {
    switch (bn) {
      case 256: n = coresident_units<256, true>(); break;
      case 224: n = coresident_units<224, true>(); break;
      case 192: n = coresident_units<192, true>(); break;
      case 160: n = coresident_units<160, true>(); break;
      default: n = coresident_units<128, true>(); break;
    }
  } else {
    switch (bn) {
      case 256: n = coresident_units<256, false>(); break;
      case 224: n = coresident_units<224, false>(); break;
      case 192: n = coresident_units<192, false>(); break;
      case 160: n = coresident_units<160, false>(); break;
      case 128: n = coresident_units<128, false>(); break;
      case 96: n = coresident_units<96, false>(); break;
      default: n = coresident_units<64, false>(); break;
    }
  }
  if (n < 0) return n;
  *out = n;
  return VL2_OK;
}

// Debug: copy the item-boundary cycle trace of the last traced launch (args->reserved2 == 777 or 779) to host memory.
extern "C" int vl2_debug_gemm_trace(long long* host_out128) {
  VL2_REQUIRE(host_out128 != nullptr, VL2_E_BADSHAPE, "vl2_debug_gemm_trace: null output");
  VL2_CHECK_CUDA(cudaDeviceSynchronize());
  VL2_CHECK_CUDA(cudaMemcpyFromSymbol(host_out128, vl2::g_gemm_trace, 128 * sizeof(long long)));
  return VL2_OK;
}

extern "C" int vl2_gemm_bf16(const vl2_gemm_args* a, void* stream) {
  using namespace vl2;
  VL2_REQUIRE(a != nullptr, VL2_E_BADSHAPE, "vl2_gemm_bf16: null args");
  VL2_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, VL2_E_BADSHAPE, "vl2_gemm_bf16: M,N,K must be positive (%d,%d,%d)",
              a->M, a->N, a->K);
  VL2_REQUIRE(a->K % 8 == 0 && a->N % 8 == 0, VL2_E_BADSHAPE, "vl2_gemm_bf16: K and N must be multiples of 8 (%d,%d)",
              a->K, a->N);
  VL2_REQUIRE(a->lda % 8 == 0 && a->ldw % 8 == 0 && a->ldc % 8 == 0 && (a->residual == nullptr || a->ldr % 8 == 0),
              VL2_E_BADALIGN, "vl2_gemm_bf16: leading dimensions must be multiples of 8 elements");
  VL2_REQUIRE(a->lda >= a->K && a->ldw >= a->K, VL2_E_BADSHAPE, "vl2_gemm_bf16: lda/ldw smaller than K");
  VL2_REQUIRE(aligned16(a->A) && aligned16(a->W) && aligned16(a->C) && aligned16(a->residual) && aligned16(a->bias),
              VL2_E_BADALIGN, "vl2_gemm_bf16: pointers must be 16-byte aligned");
  VL2_REQUIRE(a->act >= VL2_ACT_NONE && a->act <= VL2_ACT_GELU_TANH, VL2_E_UNSUPPORTED, "vl2_gemm_bf16: unknown act %d",
              a->act);
  VL2_REQUIRE(a->sumsq_out == nullptr || (!a->out_f32 && a->act != VL2_ACT_SWIGLU && a->N % 32 == 0), VL2_E_UNSUPPORTED,
              "vl2_gemm_bf16: sumsq_out supports bf16, non-SwiGLU outputs with N %% 32 == 0 only");
  VL2_REQUIRE(a->rms_sumsq_in == nullptr || a->rms_nparts > 0, VL2_E_BADSHAPE, "vl2_gemm_bf16: rms_nparts must be positive");
  VL2_REQUIRE(a->ln_sum_in == nullptr || (a->rms_sumsq_in != nullptr && a->ln_colsum != nullptr), VL2_E_BADSHAPE,
              "vl2_gemm_bf16: ln_sum_in needs rms_sumsq_in (sums of squares) and ln_colsum");
  VL2_REQUIRE(a->rowsum_out == nullptr || a->sumsq_out != nullptr, VL2_E_UNSUPPORTED,
              "vl2_gemm_bf16: rowsum_out is written together with sumsq_out");
  VL2_REQUIRE(a->n_bcast >= 0 && a->n_bcast <= 8, VL2_E_BADSHAPE, "vl2_gemm_bf16: n_bcast must be in [0,8]");
  if (a->n_bcast > 0 || a->mc_out != nullptr) {
    VL2_REQUIRE(!a->out_f32 && a->act != VL2_ACT_SWIGLU, VL2_E_UNSUPPORTED,
                "vl2_gemm_bf16: the broadcast epilogue supports bf16, non-SwiGLU outputs only");
    for (int i = 0; i < a->n_bcast; ++i)
      VL2_REQUIRE(a->bcast_out[i] != nullptr && aligned16(a->bcast_out[i]), VL2_E_BADALIGN,
                  "vl2_gemm_bf16: broadcast target %d must be a 16-byte aligned device pointer", i);
  }
  if (a->act == VL2_ACT_SWIGLU) {
    VL2_REQUIRE(a->residual == nullptr && !a->out_f32 && a->N % 16 == 0, VL2_E_UNSUPPORTED,
                "vl2_gemm_bf16: SWIGLU epilogue needs N %% 16 == 0, bf16 output and no residual");
  }
  if (a->rope_tab != nullptr) {
    VL2_REQUIRE(a->rope_D >= 32 && a->rope_D % 32 == 0 && a->rope_cols > 0 && a->rope_cols % a->rope_D == 0 &&
                    a->rope_cols <= a->N && a->rope_pos0 >= 0 && aligned16(a->rope_tab),
                VL2_E_BADSHAPE, "vl2_gemm_bf16: rope epilogue needs head width %% 32 == 0, rope_cols a multiple of it (<= N)");
    VL2_REQUIRE(!a->out_f32 && a->act == VL2_ACT_NONE && a->residual == nullptr, VL2_E_UNSUPPORTED,
                "vl2_gemm_bf16: the rope epilogue supports bf16 output without activation / residual");
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int m_plan = a->M;
  if (a->conv_C > 0) {
    const int p_ = a->conv_pad;
    VL2_REQUIRE(a->conv_T > 0 && a->conv_H > 0 && a->conv_W > 0 && (p_ == 0 || p_ == 1) && a->conv_C % 64 == 0,
                VL2_E_BADSHAPE, "vl2_gemm_bf16: conv front end needs T,H,W > 0, pad in {0,1}, C %% 64 == 0");
    const int To = (a->conv_T + 2 * p_ - 2) / 2 + 1, Ho = (a->conv_H + 2 * p_ - 2) / 2 + 1, Wo = (a->conv_W + 2 * p_ - 2) / 2 + 1;
    VL2_REQUIRE((a->conv_W % 2 == 0 && a->conv_H % 2 == 0) || p_ == 0, VL2_E_UNSUPPORTED,
                "vl2_gemm_bf16: conv front end: odd H / W needs pad 0");
    VL2_REQUIRE(To > 0 && Ho > 0 && Wo > 0 && Wo <= kConvLine && Ho <= kConvLine, VL2_E_UNSUPPORTED,
                "vl2_gemm_bf16: conv front end supports up to %d x %d output positions per time step (got %d x %d)", kConvLine,
                kConvLine, Ho, Wo);
    VL2_REQUIRE(a->K == 8 * a->conv_C && a->M == To * Ho * Wo, VL2_E_BADSHAPE,
                "vl2_gemm_bf16: conv front end needs K == 8*C and M == To*Ho*Wo (M=%d, expected %d)", a->M, To * Ho * Wo);
    VL2_REQUIRE(a->residual == nullptr && a->row_scale == nullptr && a->rms_sumsq_in == nullptr && a->sumsq_out == nullptr &&
                    !a->out_f32 && a->act != VL2_ACT_SWIGLU && a->n_bcast == 0 && a->mc_out == nullptr,
                VL2_E_UNSUPPORTED, "vl2_gemm_bf16: the conv front end supports bias + activation epilogues, bf16 output");
    m_plan = To * kConvLine * kConvLine;
  }
  const bool split_ok = splitk_enabled() && a->splitk_ws != nullptr && a->conv_C == 0;
  TileChoice t = choose_tile(m_plan, a->N, a->K, sm_count(), pair_enabled(), split_ok);
  // test hook: reserved = BN forces a single-CTA tile width, 1000 + BN forces the two-CTA (cluster pair) kernel
  if (a->reserved >= 64 && a->reserved <= 256 && a->reserved % 32 == 0) { t.bn = a->reserved; t.pair = false; }
  if (a->reserved >= 1128 && a->reserved <= 1256 && (a->reserved - 1000) % 32 == 0) { t.bn = a->reserved - 1000; t.pair = true; }
  if (t.pair) {
    switch (t.bn) {
      case 256: return launch_gemm<256, true>(a, st);
      case 224: return launch_gemm<224, true>(a, st);
      case 192: return launch_gemm<192, true>(a, st);
      case 160: return launch_gemm<160, true>(a, st);
      default: return launch_gemm<128, true>(a, st);
    }
  }
  switch (t.bn) {
    case 256: return launch_gemm<256, false>(a, st);
    case 224: return launch_gemm<224, false>(a, st);
    case 192: return launch_gemm<192, false>(a, st);
    case 160: return launch_gemm<160, false>(a, st);
    case 128: return launch_gemm<128, false>(a, st);
    case 96: return launch_gemm<96, false>(a, st);
    default: return launch_gemm<64, false>(a, st);
  }
}
