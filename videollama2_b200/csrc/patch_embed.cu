// ViT patch embedding as ONE implicit-GEMM kernel on wgmma (HF CLIPVisionEmbeddings.forward, HF:clip/modeling_clip.py:202-218,
// followed by CLIPVisionTransformer.pre_layrnorm :739-741; HF SiglipVisionEmbeddings for the VideoLLaMA2.1 tower):
//
//   tok[f, 1+p, :] = LN( conv_PxP_strideP(pixels[f])[p, :] + pos[1+p, :] ),   tok[f, 0, :] = LN( cls + pos[0, :] )     (CLIP)
//   tok[f, p, :]   =     conv_PxP_strideP(pixels[f])[p, :] + bias + pos[p, :]                                          (SigLIP)
//
// No im2col matrix exists: the A operand (128 patches x K = 3 P^2 pixel values) is gathered from the NCHW frames by all
// threads straight into the 128-byte-swizzled shared-memory layout wgmma reads, once per CTA and for the whole K
// (10 k-blocks = 160 KB).  A 128-patch row block is split along the output channels over a CLUSTER of NS CTAs
// (NS <= 8; C / NS <= 256 columns each), so a 16-frame video fills the SMs; each consumer thread keeps its rows' part of
// the CTA's whole column range in registers (up to two 128-column accumulators) while the conv weight streams through a
// 2-stage TMA ring.
// Epilogue: + position row (+ bias).  CLIP: the row's x and x^2 over this CTA's columns (reduced over the quad of threads
// that hold a row); the partial statistics of the NS CTAs are exchanged through distributed shared memory
// (st.shared::cluster + remote mbarrier arrives, summed in rank order); then normalise and store.  Nothing un-normalised
// ever leaves the SM.  One launch replaces vl2_patch_im2col + vl2_gemm_bf16 + vl2_clip_embed_finish.
#include "host_common.h"
#include "ptx.cuh"
#include "row_common.cuh"

namespace vl2 {

static constexpr int kPeBM = 128, kPeBN = 128, kPeBK = 64;
static constexpr int kPeMaxKB = 10;                           // K padded to at most 640 (3 * 14 * 14 = 588)
static constexpr int kPeMaxCols = 256;                        // columns per CTA: two 128-column accumulators per thread
static constexpr int kPeStagesB = 2;
static constexpr int kPeThreads = 384;                        // warpgroup 0: TMA; 1, 2: wgmma + epilogue; all gather A
static constexpr int kPeStageB = kPeBN * kPeBK * 2;           // 16 KB
static constexpr int kPeOffB = kPeMaxKB * kPeBM * kPeBK * 2;  // 160 KB of A
static constexpr int kPeMaxStatTiles = 16;                    // 128-column tiles of a whole row (C <= 2048 in the LayerNorm form)
static constexpr int kPeOffStats = kPeOffB + kPeStagesB * kPeStageB;       // [16 tiles][128 rows] float2
static constexpr int kPeOffBar = kPeOffStats + kPeMaxStatTiles * 128 * 8;
static constexpr int kPeSmem = kPeOffBar + 256;

struct PatchEmbedParams {
  const __nv_bfloat16* px;      // [F, 3, H, W]
  const __nv_bfloat16* pos;     // [np + has_cls, C]
  const __nv_bfloat16* cls;     // [C] or NULL
  const __nv_bfloat16* gamma;   // pre-LN (CLIP) or NULL
  const __nv_bfloat16* beta;
  const float* bias;            // conv bias (SigLIP) or NULL
  __nv_bfloat16* out;           // [F * (np + has_cls), C]
  int F, H, W, P, G, np, C, K, nkb, M;
  int ns, cols, n_tiles;        // CTAs per row block (cluster size), columns per CTA, 128-column B tiles per CTA
  float eps;
};

__device__ __forceinline__ void st_cluster_f32x2(uint32_t local_addr, uint32_t rank, float a, float b) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.v2.f32 [ra], {%2, %3};\n\t}"
      ::"r"(local_addr), "r"(rank), "f"(a), "f"(b)
      : "memory");
}

__global__ void __launch_bounds__(kPeThreads, 1)
patch_embed_kernel(const __grid_constant__ CUtensorMap tmap_w, const PatchEmbedParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) { asm volatile("trap;"); }
  uint8_t* sA = smem;                                              // [nkb][128 rows][128 B], swizzled
  uint8_t* sB = smem + kPeOffB;                                    // [2][128 rows][128 B]
  float2* sStats = reinterpret_cast<float2*>(smem + kPeOffStats);  // [global 128-column tile][row] partial (sum, sum of squares)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kPeOffBar);
  uint64_t* b_full = bars;            // [2]   TMA -> MMA
  uint64_t* b_empty = bars + 2;       // [2]   MMA (8 consumer warps) -> TMA
  uint64_t* stat_bar = bars + 4;      //       64 * ns arrivals: every CTA's partial statistics have landed here

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = p.ns > 1 ? cluster_ctarank() : 0u;
  const int m0 = (int)(blockIdx.x / p.ns) * kPeBM;
  const int n_begin = (int)rank * p.cols;
  const bool clip = p.gamma != nullptr;
  const int has_cls = p.cls != nullptr ? 1 : 0;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_w);
    for (int i = 0; i < kPeStagesB; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], 8);
    }
    mbar_init(stat_bar, 64 * p.ns);
    fence_barrier_init();
  }
  pdl_wait();
  // ===================== A gather by every thread: (patch row, k-block) pairs =====================
  // The 28-byte pixel runs of a 14 x 14 patch break TMA's 16-byte rule, so this is plain LDG straight into the
  // 128-byte-swizzled K-major layout wgmma reads.
  {
    const int pp2 = p.P * p.P;
    const int64_t cstride = (int64_t)p.H * p.W;
    for (int idx = threadIdx.x; idx < kPeBM * p.nkb; idx += kPeThreads) {
      const int r = idx & (kPeBM - 1), kb = idx / kPeBM;
      const int m = m0 + r;
      const bool valid = m < p.M;
      const int f = valid ? m / p.np : 0, pp = valid ? m % p.np : 0;
      const int ph = pp / p.G, pw = pp % p.G;
      const __nv_bfloat16* src0 = p.px + ((int64_t)f * 3 * p.H + (int64_t)ph * p.P) * p.W + pw * p.P;   // (c = 0, i = 0, j = 0)
      int c = (kb * 64) / pp2, rem = (kb * 64) % pp2;   // decomposition of the running k (advances by 2: P is even)
      int i = rem / p.P, j = rem % p.P;
      const uint32_t row_base = smem_u32(sA) + kb * (kPeBM * 128) + r * 128;
#pragma unroll
      for (int ch = 0; ch < 8; ++ch) {
        uint32_t w4[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = kb * 64 + ch * 8 + e * 2;
          uint32_t v = 0;
          if (valid && k < p.K) v = *reinterpret_cast<const uint32_t*>(src0 + c * cstride + (int64_t)i * p.W + j);
          w4[e] = v;
          j += 2;
          if (j == p.P) { j = 0; if (++i == p.P) { i = 0; ++c; } }
        }
        sts128(row_base + ((ch ^ (r & 7)) << 4), make_uint4(w4[0], w4[1], w4[2], w4[3]));
      }
    }
  }
  fence_proxy_async_smem();       // generic-proxy smem writes -> visible to the tensor core's async proxy
  if (p.ns > 1) cluster_sync_all(); else __syncthreads();      // A complete; peers' barriers exist before remote arrivals

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ===================== TMA: conv weight tiles [128 output channels x 64 k] of this CTA's column range =====================
      int st = 0;
      uint32_t ph = 0;
      for (int jn = 0; jn < p.n_tiles; ++jn)
        for (int kb = 0; kb < p.nkb; ++kb) {
          mbar_wait(&b_empty[st], ph ^ 1);
          mbar_arrive_expect_tx(&b_full[st], kPeStageB);
          tma_load_2d(sB + st * kPeStageB, &tmap_w, &b_full[st], kb * kPeBK, n_begin + jn * kPeBN);
          if (++st == kPeStagesB) { st = 0; ph ^= 1; }
        }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== wgmma: accumulator tile jn (columns [128 jn, 128 jn + 128) of the range) =====================
    const int wg = (warp >> 2) - 1;
    const int t = lane & 3;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: rloc, rloc + 8
    const uint64_t da0 = gmma_desc_sw128(smem_u32(sA) + wg * 64 * 128, 16, 1024);
    const uint64_t db0 = gmma_desc_sw128(smem_u32(sB), 16, 1024);
    float acc[2][64];
    int st = 0;
    uint32_t ph = 0;
#pragma unroll
    for (int jn = 0; jn < 2; ++jn) {
      if (jn >= p.n_tiles) break;
      for (int kb = 0; kb < p.nkb; ++kb) {
        mbar_wait(&b_full[st], ph);
        wgmma_fence();
        const uint64_t da = da0 + (uint64_t)((kb * kPeBM * 128) >> 4);
        const uint64_t db = db0 + (uint64_t)((st * kPeStageB) >> 4);
#pragma unroll
        for (int k = 0; k < kPeBK / 16; ++k) Wgmma<kPeBN, 0>::ss(acc[jn], da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(acc[jn]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[st]);
        if (++st == kPeStagesB) { st = 0; ph ^= 1; }
      }
    }
    // ===================== epilogue.  acc[jn][4 c + 2 h + e] = row rloc + 8 h, column 128 jn + 8 c + 2 t + e =====================
    int out_row[2];
    bool valid[2];
    const __nv_bfloat16* pos_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + rloc + 8 * h;
      valid[h] = m < p.M;
      const int f = valid[h] ? m / p.np : 0, pp = valid[h] ? m % p.np : 0;
      out_row[h] = f * (p.np + has_cls) + has_cls + pp;
      pos_row[h] = p.pos + (int64_t)(has_cls + pp) * p.C + n_begin;
    }
    // x of one column pair: accumulator (+ bias) + position row, exactly as both passes must see it
    auto load_pair = [&](int jn, int c, int h, float& x0, float& x1) {
      const int col = jn * kPeBN + 8 * c + 2 * t;
      const uint32_t pv = valid[h] ? __ldg(reinterpret_cast<const uint32_t*>(pos_row[h] + col)) : 0u;
      const float a0 = acc[jn][4 * c + 2 * h], a1 = acc[jn][4 * c + 2 * h + 1];
      // CLIP: the conv output is rounded to 16 bits (HF's conv returns the activation dtype) before the fp32 position
      // add + LayerNorm; SigLIP: conv + bias + position in fp32, one rounding at the store
      if (clip) {
        x0 = __bfloat162float(__float2bfloat16_rn(a0)) + bf16_lo(pv);
        x1 = __bfloat162float(__float2bfloat16_rn(a1)) + bf16_hi(pv);
      } else {
        const float2 bq = p.bias != nullptr ? __ldg(reinterpret_cast<const float2*>(p.bias + n_begin + col)) : make_float2(0.f, 0.f);
        x0 = a0 + bq.x + bf16_lo(pv);
        x1 = a1 + bq.y + bf16_hi(pv);
      }
    };
    float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
    if (clip) {
      // ---- the row statistics of this CTA's columns, ONE partial per 128-column tile.  The tiles are the same whatever
      // the cluster size (column ranges are multiples of 128 whenever the split can vary), and the final sum below runs
      // over the row's tiles in global order: the result does not depend on how many CTAs shared the row, which keeps the
      // tower bit-identical for any number of frames per launch (frame sharding).
      const int tile0 = n_begin / kPeBN;
#pragma unroll
      for (int jn = 0; jn < 2; ++jn) {
        if (jn >= p.n_tiles) break;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = 0.f, sq = 0.f;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            if (jn * kPeBN + 8 * c >= p.cols) break;
            float x0, x1;
            load_pair(jn, c, h, x0, x1);
            s += x0 + x1;
            sq = fmaf(x0, x0, fmaf(x1, x1, sq));
          }
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          sq += __shfl_xor_sync(0xffffffffu, sq, 1);
          sq += __shfl_xor_sync(0xffffffffu, sq, 2);
          // ---- hand the partial to every CTA of the cluster (distributed shared memory)
          const int r = rloc + 8 * h;
          if (t == 0) {
            if (p.ns > 1) {
              const uint32_t slot = smem_u32(sStats + (tile0 + jn) * 128 + r);
              for (uint32_t rr = 0; rr < (uint32_t)p.ns; ++rr) st_cluster_f32x2(slot, rr, s, sq);
            } else {
              sStats[(tile0 + jn) * 128 + r] = make_float2(s, sq);
            }
          }
        }
      }
      if (t == 0) {
        for (uint32_t rr = 0; rr < (uint32_t)p.ns; ++rr) {
          if (p.ns > 1) mbar_arrive_cluster(stat_bar, rr);   // release.cluster: the stores above are visible to whoever acquires
          else mbar_arrive(stat_bar);
        }
      }
      mbar_wait_cluster(stat_bar, 0);                // acquire.cluster: pairs with the peers' release arrivals
      const int row_tiles = (p.C + kPeBN - 1) / kPeBN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float ts = 0.f, tq = 0.f;
        for (int tt = 0; tt < row_tiles; ++tt) { const float2 v2 = sStats[tt * 128 + rloc + 8 * h]; ts += v2.x; tq += v2.y; }
        mean[h] = ts / (float)p.C;
        rstd[h] = rsqrtf(fmaxf(tq / (float)p.C - mean[h] * mean[h], 0.f) + p.eps);
      }
    }
    // ---- normalise / finish and store
#pragma unroll
    for (int jn = 0; jn < 2; ++jn) {
      if (jn >= p.n_tiles) break;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const int col = jn * kPeBN + 8 * c + 2 * t;
        if (jn * kPeBN + 8 * c >= p.cols) break;
        float gm0 = 1.f, gm1 = 1.f, bt0 = 0.f, bt1 = 0.f;
        if (clip) {
          const uint32_t gv = __ldg(reinterpret_cast<const uint32_t*>(p.gamma + n_begin + col));
          const uint32_t bv = __ldg(reinterpret_cast<const uint32_t*>(p.beta + n_begin + col));
          gm0 = bf16_lo(gv); gm1 = bf16_hi(gv); bt0 = bf16_lo(bv); bt1 = bf16_hi(bv);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float x0, x1;
          load_pair(jn, c, h, x0, x1);
          if (clip) {
            x0 = (x0 - mean[h]) * rstd[h] * gm0 + bt0;
            x1 = (x1 - mean[h]) * rstd[h] * gm1 + bt1;
          }
          if (valid[h]) *reinterpret_cast<uint32_t*>(p.out + (int64_t)out_row[h] * p.C + n_begin + col) = pack_bf16(x0, x1);
        }
      }
    }
    // the class-token row is the same for every frame: LN(cls + pos[0]); the CTAs of row block 0 write their column range
    if (clip && m0 == 0 && warp == 4) {
      float cs = 0.f, cq = 0.f;
      for (int c0 = lane * 8; c0 < p.C; c0 += 256) {
        float a[8], b[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.cls + c0)), a);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.pos + c0)), b);
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float xv = a[e] + b[e]; cs += xv; cq = fmaf(xv, xv, cq); }
      }
      cs = warp_sum(cs);
      cq = warp_sum(cq);
      const float mu = cs / (float)p.C;
      const float rs = rsqrtf(fmaxf(cq / (float)p.C - mu * mu, 0.f) + p.eps);
      for (int c0 = n_begin + lane * 8; c0 < n_begin + p.cols; c0 += 256) {
        float a[8], b[8], gm[8], bt[8], o8[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.cls + c0)), a);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.pos + c0)), b);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.gamma + c0)), gm);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.beta + c0)), bt);
#pragma unroll
        for (int e = 0; e < 8; ++e) o8[e] = (a[e] + b[e] - mu) * rs * gm[e] + bt[e];
        const uint4 pk = pack8(o8);
        for (int ff = 0; ff < p.F; ++ff) *reinterpret_cast<uint4*>(p.out + (int64_t)ff * (p.np + 1) * p.C + c0) = pk;
      }
    }
  }
  if (p.ns > 1) cluster_sync_all();   // no CTA leaves while a peer may still write its statistics into it
}

}  // namespace vl2

using namespace vl2;

extern "C" int vl2_patch_embed(const vl2_patch_embed_args* a, void* stream) {
  VL2_REQUIRE(a != nullptr, VL2_E_BADSHAPE, "vl2_patch_embed: null args");
  VL2_REQUIRE(a->F > 0 && a->P > 0 && a->P % 2 == 0 && a->H >= a->P && a->W >= a->P && a->W % 2 == 0, VL2_E_BADSHAPE,
              "vl2_patch_embed: need F > 0, even patch size, even W, H/W >= P (F=%d P=%d H=%d W=%d)", a->F, a->P, a->H, a->W);
  const int K = 3 * a->P * a->P;
  VL2_REQUIRE(a->Kpad % 64 == 0 && a->Kpad >= K && a->Kpad <= kPeMaxKB * 64, VL2_E_UNSUPPORTED,
              "vl2_patch_embed: Kpad must be a multiple of 64 in [3*P*P, %d] (Kpad=%d)", kPeMaxKB * 64, a->Kpad);
  VL2_REQUIRE(a->C > 0 && a->C % 32 == 0, VL2_E_BADSHAPE, "vl2_patch_embed: C %% 32 == 0 required (C=%d)", a->C);
  VL2_REQUIRE(a->pixels && a->weight && a->pos && a->out, VL2_E_BADSHAPE, "vl2_patch_embed: null pointer");
  const bool clip = a->gamma != nullptr;
  VL2_REQUIRE(!clip || (a->beta != nullptr && a->cls != nullptr), VL2_E_BADSHAPE,
              "vl2_patch_embed: the CLIP form needs cls, gamma and beta");
  VL2_REQUIRE(clip || a->cls == nullptr, VL2_E_UNSUPPORTED, "vl2_patch_embed: a class token without pre-LN is not a tower of the path");
  VL2_REQUIRE(aligned16(a->pixels) && aligned16(a->weight) && aligned16(a->pos) && aligned16(a->out) && aligned16(a->gamma) &&
                  aligned16(a->beta) && aligned16(a->cls),
              VL2_E_BADALIGN, "vl2_patch_embed: pointers must be 16-byte aligned");
  PatchEmbedParams p;
  p.px = (const __nv_bfloat16*)a->pixels; p.pos = (const __nv_bfloat16*)a->pos; p.cls = (const __nv_bfloat16*)a->cls;
  p.gamma = (const __nv_bfloat16*)a->gamma; p.beta = (const __nv_bfloat16*)a->beta; p.bias = a->bias;
  p.out = (__nv_bfloat16*)a->out;
  p.F = a->F; p.H = a->H; p.W = a->W; p.P = a->P; p.G = a->W / a->P; p.np = (a->H / a->P) * (a->W / a->P); p.C = a->C;
  p.K = K; p.nkb = a->Kpad / 64; p.M = a->F * p.np; p.eps = a->eps;
  // Columns per CTA: at most 256 (two 128-column register accumulators per consumer thread), a multiple of 32; prefer the
  // split that fills the SMs.  The split is a cluster of up to 8 CTAs (the CLIP form exchanges LayerNorm statistics over
  // it, so its column ranges are whole 128-column tiles); 3 and 6 suit SigLIP's 1152 and 288-wide test towers.
  const int blocks_m = (p.M + kPeBM - 1) / kPeBM;
  int ns = 0;
  const int cands_clip[4] = {1, 2, 4, 8}, cands_any[6] = {1, 2, 3, 4, 6, 8};
  const int* cands = clip ? cands_clip : cands_any;
  const int ncand = clip ? 4 : 6;
  for (int i = 0; i < ncand; ++i) {
    const int s = cands[i];
    if (a->C % s != 0 || (a->C / s) % 32 != 0 || a->C / s > kPeMaxCols) continue;
    if (clip && s > 1 && (a->C / s) % kPeBN != 0) continue;            // statistics tiles must line up with global 128-column tiles
    if (ns == 0) ns = s;
    else if (blocks_m * s <= sm_count() && a->C / s >= 128) ns = s;      // a finer split only while it still is one wave
  }
  VL2_REQUIRE(!clip || (a->C + kPeBN - 1) / kPeBN <= kPeMaxStatTiles, VL2_E_UNSUPPORTED, "vl2_patch_embed: C <= %d with a LayerNorm",
              kPeMaxStatTiles * kPeBN);
  VL2_REQUIRE(ns > 0, VL2_E_UNSUPPORTED, "vl2_patch_embed: C = %d cannot be split into <= 8 column ranges of <= 256", a->C);
  p.ns = ns; p.cols = a->C / ns; p.n_tiles = (p.cols + kPeBN - 1) / kPeBN;
  CUtensorMap tw;
  {
    uint64_t dims[2] = {(uint64_t)a->Kpad, (uint64_t)a->C};
    uint64_t str[1] = {(uint64_t)a->Kpad * 2};
    uint32_t box[2] = {kPeBK, kPeBN};
    int rc = make_tmap_bf16(&tw, a->weight, 2, dims, str, box);
    if (rc) return rc;
  }
  VL2_SMEM_OPT_IN(patch_embed_kernel, kPeSmem);
  VL2_CHECK_CUDA(launch_kernel(patch_embed_kernel, dim3(blocks_m * ns), dim3(kPeThreads), kPeSmem, (cudaStream_t)stream, ns, tw, p));
  VL2_CHECK_LAUNCH("patch_embed_kernel");
  return VL2_OK;
}
