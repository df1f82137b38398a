// FlashAttention-style fused attention for sm_90a (non-causal ViT heads and causal GQA decoder heads).
//
// Work item = one 128-row query tile of one (batch, head); one CTA per item, 384 threads:
//   warpgroup 0     TMA producer (one thread): Q once, then the K and V rings (2 stages each, 128 keys x D per stage)
//   warpgroups 1, 2 query rows [0, 64) / [64, 128) of the tile, each:
//                     S_j  = Q K_j^T   wgmma m64 x 128 x k16, A = Q and B = K_j both K-major SW128 from smem
//                     online softmax on the S fragments in registers (a row lives in the four threads of a quad)
//                     O   += P_j V_j   wgmma m64 x D x k16, A = P_j from REGISTERS (the S accumulator layout is the A
//                                      fragment layout), B = V_j as an MN-major SW128 operand (no transpose pass)
// O accumulates in registers and is rescaled per tile by exp2(m_old - m_new); the final 1 / l is applied at the store.
#include <stdlib.h>

#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

static constexpr int kAttnThreads = 384;
static constexpr int BQ = 128;
static constexpr int BKV = 128;

template <int D>
struct AttnCfg {
  static constexpr int kAtoms = D / 64;                 // 64-column (128-byte) swizzle atoms per row
  static constexpr int kAtomBytes = 128 * 128;          // 128 rows x 128 B
  static constexpr int kTileBytes = BKV * D * 2;        // one Q / K / V tile
  static constexpr int kOffQ = 0;
  static constexpr int kOffK = kTileBytes;              // 2 stages
  static constexpr int kOffV = 3 * kTileBytes;          // 2 stages
  static constexpr int kOffBar = 5 * kTileBytes;
  static constexpr int kSmemBytes = kOffBar + 128;
};

// Debug cycle trace (vl2_attn_args.reserved == 777): CTA (0,0,0), consumer thread 0 accumulates the cycles of each phase
// of its key-tile loop: [0] waiting for K_j, [1] Q K^T + softmax, [2] waiting for V_j + P V; [7] key tiles, [8] items.
__device__ long long g_attn_trace[16];

struct AttnParams {
  int trace;
  void* out;
  int64_t ldo;
  int S, Hq, group;  // group = Hq / Hkv
  int d_true;        // real head width (<= D); columns beyond it are TMA zero fill
  int causal;
  float scale_log2;  // softmax scale * log2(e)
};

template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  using Cfg = AttnCfg<D>;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) { asm volatile("trap;"); }
  uint8_t* sQ = smem + Cfg::kOffQ;
  uint8_t* sK = smem + Cfg::kOffK;
  uint8_t* sV = smem + Cfg::kOffV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kOffBar);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;    // [2]
  uint64_t* k_empty = bars + 3;   // [2]
  uint64_t* v_full = bars + 5;    // [2]
  uint64_t* v_empty = bars + 7;   // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // Non-causal: x = query tile, y = head (consecutive CTAs share a head's K/V in L2).  Causal: x = head, y = query-tile
  // rank, heaviest (latest) tile first: the hardware hands CTAs out in x-fastest order, so every head's longest CTA is
  // scheduled before any shorter one - longest-processing-time-first list scheduling over the SMs (and the query heads of
  // a GQA group, adjacent in x, read the same K/V tiles at the same time).
  const int qt = p.causal ? (int)(gridDim.y - 1 - blockIdx.y) : (int)blockIdx.x;
  const int head = p.causal ? (int)blockIdx.x : (int)blockIdx.y;
  const int b = blockIdx.z;
  const int kvh = head / p.group;
  const int q0 = qt * BQ;
  const int n_kv = p.causal ? (qt + 1) : (p.S + BKV - 1) / BKV;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);   // the 8 consumer warps
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
  }
  pdl_wait();
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ===================== TMA producer: Q, then K_j / V_j in key-tile order =====================
      mbar_arrive_expect_tx(q_full, Cfg::kTileBytes);
#pragma unroll
      for (int a = 0; a < Cfg::kAtoms; ++a) tma_load_4d(sQ + a * Cfg::kAtomBytes, &tmap_q, q_full, a * 64, head, q0, b);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j & 1;
        const uint32_t ph = ((j >> 1) & 1) ^ 1;
        mbar_wait(&k_empty[st], ph);
        mbar_arrive_expect_tx(&k_full[st], Cfg::kTileBytes);
#pragma unroll
        for (int a = 0; a < Cfg::kAtoms; ++a)
          tma_load_4d(sK + st * Cfg::kTileBytes + a * Cfg::kAtomBytes, &tmap_k, &k_full[st], a * 64, kvh, j * BKV, b);
        mbar_wait(&v_empty[st], ph);
        mbar_arrive_expect_tx(&v_full[st], Cfg::kTileBytes);
#pragma unroll
        for (int a = 0; a < Cfg::kAtoms; ++a)
          tma_load_4d(sV + st * Cfg::kTileBytes + a * Cfg::kAtomBytes, &tmap_v, &v_full[st], a * 64, kvh, j * BKV, b);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== consumers: 64 query rows per warpgroup =====================
    const int wg = (warp >> 2) - 1;
    const int g = lane >> 2, t = lane & 3;
    const int rloc = wg * 64 + (warp & 3) * 16 + g;   // this thread's rows: rloc, rloc + 8 (of the query tile)
    const int qi[2] = {q0 + rloc, q0 + rloc + 8};
    // Q: K-major, this warpgroup's 64 rows start 64 x 128 B into every atom; k-step kk = atom kk / 4, +32 B per step
    const uint64_t dq = gmma_desc_sw128(smem_u32(sQ) + wg * 64 * 128, 16, 1024);
    const uint64_t dk0 = gmma_desc_sw128(smem_u32(sK), 16, 1024);
    // V: MN-major (d contiguous): 16 keys = two 8-row groups (SBO 1024 B), the next 64-wide d atom is LBO = one atom away
    const uint64_t dv0 = gmma_desc_sw128(smem_u32(sV), Cfg::kAtomBytes, 1024);
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const bool tr = p.trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 128;
    long long t0 = 0, acc_t[3] = {0, 0, 0};
#define VL2_TR(i) do { if (tr) { const long long t1 = clock64(); acc_t[i] += t1 - t0; t0 = t1; } } while (0)
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_kv; ++j) {
      if (tr) t0 = clock64();
      const int st = j & 1;
      const uint32_t ph = (j >> 1) & 1;
      mbar_wait(&k_full[st], ph);
      VL2_TR(0);
      float s[BKV / 2];
      wgmma_fence();
      const uint64_t dk = dk0 + (uint64_t)((st * Cfg::kTileBytes) >> 4);
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t off = ((kk >> 2) * Cfg::kAtomBytes + (kk & 3) * 32) >> 4;
        Wgmma<BKV, 0>::ss(s, dq + off, dk + off, kk != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_keep(s);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[st]);   // K_j has been read
      // ---- online softmax.  s[4 c + 2 h + e] = row qi[h], key j * BKV + 8 c + 2 t + e
      const bool need_mask = (j * BKV + BKV > p.S) || (p.causal && (j * BKV + BKV - 1 > q0));
      if (need_mask) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int lim = p.causal ? min(p.S - 1, qi[h]) : (p.S - 1);   // last visible key of the row
#pragma unroll
          for (int c = 0; c < BKV / 8; ++c)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (j * BKV + 8 * c + 2 * t + e > lim) s[4 * c + 2 * h + e] = -INFINITY;
        }
      }
      float alpha[2], m_use[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < BKV / 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[h], mx * p.scale_log2);
        m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;   // fully masked rows stay finite
        alpha[h] = (m[h] == -INFINITY) ? 0.f : fast_exp2(m[h] - m_use[h]);
        m[h] = m_new;
      }
      uint32_t pa[BKV / 16][4];   // P_j as the A fragments of the P V k-steps (16 keys each)
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int c = 0; c < BKV / 8; ++c) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float p0 = fast_exp2(fmaf(s[4 * c + 2 * h], p.scale_log2, -m_use[h]));
          const float p1 = fast_exp2(fmaf(s[4 * c + 2 * h + 1], p.scale_log2, -m_use[h]));
          rs[h] += p0 + p1;
          pa[c >> 1][(c & 1) * 2 + h] = pack_bf16(p0, p1);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l[h] = l[h] * alpha[h] + rs[h];
#pragma unroll
      for (int c = 0; c < D / 8; ++c)
#pragma unroll
        for (int h = 0; h < 2; ++h) { o[4 * c + 2 * h] *= alpha[h]; o[4 * c + 2 * h + 1] *= alpha[h]; }
      VL2_TR(1);
      mbar_wait(&v_full[st], ph);
      wgmma_fence();
      const uint64_t dv = dv0 + (uint64_t)((st * Cfg::kTileBytes) >> 4);
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) Wgmma<D, 1>::rs(o, pa[kk], dv + (uint64_t)((kk * 2048) >> 4), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_keep(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[st]);   // V_j has been read
      VL2_TR(2);
    }
    if (tr) {
      for (int i = 0; i < 3; ++i) g_attn_trace[i] = acc_t[i];
      g_attn_trace[7] = n_kv;
      g_attn_trace[8] = 1;
    }
#undef VL2_TR
    // ---- normalise and store: the row sum is spread over the quad
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = 1.f / lt;
      if (qi[h] >= p.S) continue;
      __nv_bfloat16* orow = reinterpret_cast<__nv_bfloat16*>(p.out) + ((int64_t)b * p.S + qi[h]) * p.ldo + head * p.d_true;
#pragma unroll
      for (int c = 0; c < D / 8; ++c) {
        if (8 * c >= p.d_true) break;   // head_dim < D: the zero-padded columns are not stored
        *reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * t) = pack_bf16(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
      }
    }
  }
}

template <int D>
static int launch_attn(const vl2_attn_args* a, cudaStream_t stream) {
  using Cfg = AttnCfg<D>;
  CUtensorMap tq, tk, tv;
  // 4-D maps (d, head, row, batch): a head narrower than the kernel's D (e.g. SigLIP's 72) is zero-filled by the TMA
  // unit beyond its true width, so QK^T and PV simply see zero columns.
  const uint32_t box[4] = {64, 1, 128, 1};
  const uint64_t dt = (uint64_t)a->D;
  {
    uint64_t dims[4] = {dt, (uint64_t)a->Hq, (uint64_t)a->S, (uint64_t)a->B};
    uint64_t str[3] = {dt * 2, (uint64_t)a->ldq * 2, (uint64_t)a->ldq * 2 * a->S};
    int rc = make_tmap_bf16(&tq, a->q, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {dt, (uint64_t)a->Hkv, (uint64_t)a->S, (uint64_t)a->B};
    uint64_t str[3] = {dt * 2, (uint64_t)a->ldk * 2, (uint64_t)a->ldk * 2 * a->S};
    int rc = make_tmap_bf16(&tk, a->k, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {dt, (uint64_t)a->Hkv, (uint64_t)a->S, (uint64_t)a->B};
    uint64_t str[3] = {dt * 2, (uint64_t)a->ldv * 2, (uint64_t)a->ldv * 2 * a->S};
    int rc = make_tmap_bf16(&tv, a->v, 4, dims, str, box);
    if (rc) return rc;
  }
  AttnParams p;
  p.trace = (a->reserved == 777) ? 1 : 0;
  p.out = a->out; p.ldo = a->ldo; p.d_true = a->D; p.S = a->S; p.Hq = a->Hq; p.group = a->Hq / a->Hkv; p.causal = a->causal;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  VL2_SMEM_OPT_IN(attn_fwd_kernel<D>, Cfg::kSmemBytes);
  const int n_qt = (a->S + BQ - 1) / BQ;
  dim3 grid(a->causal ? a->Hq : n_qt, a->causal ? n_qt : a->Hq, a->B);
  VL2_CHECK_CUDA(launch_kernel(attn_fwd_kernel<D>, grid, dim3(kAttnThreads), Cfg::kSmemBytes, stream, 1, tq, tk, tv, p));
  VL2_CHECK_LAUNCH("attn_fwd_kernel");
  return VL2_OK;
}

}  // namespace vl2

extern "C" int vl2_attention(const vl2_attn_args* a, void* stream) {
  using namespace vl2;
  VL2_REQUIRE(a != nullptr, VL2_E_BADSHAPE, "vl2_attention: null args");
  VL2_REQUIRE(a->B > 0 && a->S > 0 && a->Hq > 0 && a->Hkv > 0 && a->Hq % a->Hkv == 0, VL2_E_BADSHAPE,
              "vl2_attention: bad B/S/heads (%d,%d,%d,%d)", a->B, a->S, a->Hq, a->Hkv);
  VL2_REQUIRE(a->D >= 8 && a->D <= 128 && a->D % 8 == 0, VL2_E_UNSUPPORTED,
              "vl2_attention: head_dim %d unsupported (multiple of 8, <= 128)", a->D);
  VL2_REQUIRE(a->ldq % 8 == 0 && a->ldk % 8 == 0 && a->ldv % 8 == 0 && a->ldo % 8 == 0, VL2_E_BADALIGN,
              "vl2_attention: row strides must be multiples of 8 elements");
  VL2_REQUIRE(aligned16(a->q) && aligned16(a->k) && aligned16(a->v) && aligned16(a->out), VL2_E_BADALIGN,
              "vl2_attention: pointers must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (a->D <= 64) return launch_attn<64>(a, st);
  return launch_attn<128>(a, st);
}

// Debug: copy the cycle trace of the last traced vl2_attention launch (see g_attn_trace) to host memory.
extern "C" int vl2_debug_attn_trace(long long* host_out16) {
  VL2_CHECK_CUDA(cudaDeviceSynchronize());
  VL2_CHECK_CUDA(cudaMemcpyFromSymbol(host_out16, vl2::g_attn_trace, 16 * sizeof(long long)));
  return VL2_OK;
}
