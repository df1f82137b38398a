// HBM-bound row kernels: LayerNorm(+SiLU,+residual), RMSNorm, CLIP embedding assembly, depthwise 3x3 + LN + SiLU
// (+ SE pooling), SE scaling, im2col front-ends, RoPE, embedding gather.  bf16 storage, fp32 math, 16-byte accesses.
#include "row_common.cuh"

namespace vl2 {


// ---------------------------------------------------------------------------------------------------------
// LayerNorm (+ residual, + SiLU) and RMSNorm (HF rounding order: y = gamma * bf16(x * rstd)), one warp per row,
// 8 rows per CTA, no block barriers.  Narrow rows (C <= 1024) stay in registers as packed bf16 (two-pass centred
// variance); wide rows use the streaming kernels further down.
// ---------------------------------------------------------------------------------------------------------


template <int NV>
__global__ void __launch_bounds__(256, (NV >= 16 ? 2 : 1))
layernorm_warp_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                      const __nv_bfloat16* __restrict__ beta, const __nv_bfloat16* __restrict__ residual,
                      __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps, int act) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = C / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  uint4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    v[i] = (vi < nvec) ? xr[vi] : make_uint4(0, 0, 0, 0);
    float f[8];
    unpack8(v[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j];
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (lane + i * 32 < nvec) {
      float f[8];
      unpack8(v[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; q += d * d; }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  const uint4* br = reinterpret_cast<const uint4*>(beta);
  const uint4* rr = residual ? reinterpret_cast<const uint4*>(residual + row * C) : nullptr;
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float f[8], g[8], b[8], o[8];
      unpack8(v[i], f);
      unpack8(__ldg(gr + vi), g);
      unpack8(__ldg(br + vi), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (f[j] - mean) * rstd * g[j] + b[j];
      if (rr) {
        float r[8];
        unpack8(rr[vi], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      if (act == VL2_ACT_SILU) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = silu(o[j]);
      }
      yr[vi] = pack8(o);
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(256)
rmsnorm_warp_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                    __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = C / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  uint4 v[NV];
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    v[i] = (vi < nvec) ? xr[vi] : make_uint4(0, 0, 0, 0);
    float f[8];
    unpack8(v[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) q += f[j] * f[j];
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float f[8], g[8], o[8];
      unpack8(v[i], f);
      unpack8(__ldg(gr + vi), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j] * __bfloat162float(__float2bfloat16_rn(f[j] * rstd));
      yr[vi] = pack8(o);
    }
  }
}

// Wide rows (C > 1024): keep nothing in registers -> full occupancy; pass 1 accumulates sum / sum of squares
// (fp32), pass 2 re-reads the row (L2-resident: it was streamed microseconds ago) and writes the result.
__global__ void __launch_bounds__(256)
layernorm_stream_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                        const __nv_bfloat16* __restrict__ beta, const __nv_bfloat16* __restrict__ residual,
                        __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps, int act) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = C / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  float s = 0.f, q = 0.f;
#pragma unroll 4
  for (int vi = lane; vi < nvec; vi += 32) {
    float f[8];
    unpack8(xr[vi], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s += f[j]; q = fmaf(f[j], f[j], q); }
  }
  const float mean = warp_sum(s) / (float)C;
  const float var = fmaxf(warp_sum(q) / (float)C - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  const uint4* br = reinterpret_cast<const uint4*>(beta);
  const uint4* rr = residual ? reinterpret_cast<const uint4*>(residual + row * C) : nullptr;
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll 2
  for (int vi = lane; vi < nvec; vi += 32) {
    float f[8], g[8], b[8], o[8];
    unpack8(xr[vi], f);
    unpack8(__ldg(gr + vi), g);
    unpack8(__ldg(br + vi), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (f[j] - mean) * rstd * g[j] + b[j];
    if (rr) {
      float r[8];
      unpack8(rr[vi], r);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += r[j];
    }
    if (act == VL2_ACT_SILU) {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = silu(o[j]);
    }
    yr[vi] = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
rmsnorm_stream_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                      __nv_bfloat16* __restrict__ y, int64_t rows, int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = C / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  float q = 0.f;
#pragma unroll 4
  for (int vi = lane; vi < nvec; vi += 32) {
    float f[8];
    unpack8(xr[vi], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) q = fmaf(f[j], f[j], q);
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll 2
  for (int vi = lane; vi < nvec; vi += 32) {
    float f[8], g[8], o[8];
    unpack8(xr[vi], f);
    unpack8(__ldg(gr + vi), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = g[j] * __bfloat162float(__float2bfloat16_rn(f[j] * rstd));
    yr[vi] = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
row_sumsq_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, float* __restrict__ sum_out, int64_t rows,
                 int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  float q = 0.f, s = 0.f;
#pragma unroll 4
  for (int vi = lane; vi < C / 8; vi += 32) {
    float f[8];
    unpack8(xr[vi], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { q = fmaf(f[j], f[j], q); s += f[j]; }
  }
  q = warp_sum(q);
  s = warp_sum(s);
  if (lane == 0) {
    out[row] = q;
    if (sum_out != nullptr) sum_out[row] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------
// CLIP embeddings: tok[f,0] = cls + pos[0]; tok[f,1+p] = patch[f,p] + pos[1+p]; then pre_layrnorm.
// ---------------------------------------------------------------------------------------------------------
__global__ void clip_embed_finish_kernel(const __nv_bfloat16* __restrict__ patch, const __nv_bfloat16* __restrict__ cls,
                                         const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ gamma,
                                         const __nv_bfloat16* __restrict__ beta, __nv_bfloat16* __restrict__ tok, int np,
                                         int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[64];
  const int t = blockIdx.x % (np + 1);
  const int f = blockIdx.x / (np + 1);
  const int nvec = C / 8;
  const uint4* src = (t == 0) ? reinterpret_cast<const uint4*>(cls)
                              : reinterpret_cast<const uint4*>(patch + ((int64_t)f * np + (t - 1)) * C);
  const uint4* pr = reinterpret_cast<const uint4*>(pos + (int64_t)t * C);
  float v[kMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      float a[8], b[8];
      unpack8(src[vi], a);
      unpack8(__ldg(pr + vi), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[i][j] = a[j] + b[j];
        s += v[i][j];
      }
    }
  }
  const float mean = block_sum2(s, 0.f, red).x / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
    }
  }
  const float rstd = rsqrtf(block_sum2(q, 0.f, red).x / (float)C + eps);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  const uint4* br = reinterpret_cast<const uint4*>(beta);
  uint4* yr = reinterpret_cast<uint4*>(tok + (int64_t)blockIdx.x * C);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = threadIdx.x + i * blockDim.x;
    if (vi < nvec) {
      float g[8], b[8], o[8];
      unpack8(__ldg(gr + vi), g);
      unpack8(__ldg(br + vi), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      yr[vi] = pack8(o);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Patch im2col: pixels [F,3,H,W] -> A [F*(H/P)*(W/P), Kpad]; column = c*P*P + i*P + j.  One thread per bf16 pair.
// ---------------------------------------------------------------------------------------------------------
__global__ void patch_im2col_kernel(const __nv_bfloat16* __restrict__ px, __nv_bfloat16* __restrict__ A, int F, int H,
                                    int W, int P, int Kpad) {
  pdl_launch_dependents();
  pdl_wait();
  const int gw = W / P, gh = H / P;
  const int K = 3 * P * P;
  const int64_t total = (int64_t)F * gh * gw * (Kpad / 2);
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int col = (int)(idx % (Kpad / 2)) * 2;
    const int64_t row = idx / (Kpad / 2);
    uint32_t out = 0;
    if (col < K) {
      const int pw = (int)(row % gw), ph = (int)((row / gw) % gh), f = (int)(row / ((int64_t)gw * gh));
      const int c = col / (P * P), r = col % (P * P), i = r / P, j = r % P;
      const __nv_bfloat16* s = px + (((int64_t)f * 3 + c) * H + (ph * P + i)) * W + pw * P + j;
      out = *reinterpret_cast<const uint32_t*>(s);  // P, W and j even => 4-byte aligned, (j, j+1) in one image row
    }
    *reinterpret_cast<uint32_t*>(A + row * Kpad + col) = out;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Depthwise 3x3 (zero pad 1, per frame) + LayerNorm over C + SiLU, channels-last.  One CTA per (frame, image row);
// the 3x3 window slides along W in registers (3 new 16-byte loads per pixel per thread); per-(f,h) channel sums of the
// output go to `pool_partial[f, h, C]` (deterministic SE pooling: reduced by se_pool_reduce_kernel).
// Thread t owns channels [8t, 8t+8) => C <= 8 * blockDim.x.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512)
dwconv3x3_ln_silu_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w9c,
                         const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                         __nv_bfloat16* __restrict__ y, float* __restrict__ pool_partial, int H, int W, int C,
                         float eps, int Cl) {
  // Cl = channels this CTA owns (C, or C / 2 when the row is split over a 2-CTA cluster: 8192-wide connector of the 72B
  // model).  The LayerNorm runs over all C channels: with a split the two CTAs exchange their partial (sum, sum of squares)
  // of every pixel pair through distributed shared memory and add them in rank order.
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t dw_smem[];   // [9][Cl] bf16 weights (registers are spent on the pixel window)
  __shared__ float red[128];
  __shared__ float4 xchg[2][2];                        // [pair parity][source rank] partial statistics of a pixel pair
  __shared__ uint64_t xbar[2];                         // [pair parity] both ranks' partials have landed (2 arrivals)
  const int split = C / Cl;
  const uint32_t crank = split > 1 ? cluster_ctarank() : 0u;
  const int row_id = split > 1 ? (int)(blockIdx.x / split) : (int)blockIdx.x;
  const int h = row_id % H;
  const int f = row_id / H;
  const int cb = (int)crank * Cl;                      // first channel of this CTA
  const int c0 = cb + threadIdx.x * 8;
  const bool active = (int)threadIdx.x * 8 < Cl;
  const uint4 zero4 = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 9 * (Cl / 8); i += blockDim.x) {
    const int tap = i / (Cl / 8), v = i - tap * (Cl / 8);
    reinterpret_cast<uint4*>(dw_smem)[i] = __ldg(reinterpret_cast<const uint4*>(w9c + (int64_t)tap * C + cb) + v);
  }
  uint4 gp = zero4, bp = zero4;
  if (active) {
    gp = __ldg(reinterpret_cast<const uint4*>(gamma + c0));
    bp = __ldg(reinterpret_cast<const uint4*>(beta + c0));
  }
  if (split > 1 && threadIdx.x == 0) {
    mbar_init(&xbar[0], 2);
    mbar_init(&xbar[1], 2);
    fence_barrier_init();
  }
  if (split > 1) cluster_sync_all(); else __syncthreads();
  const uint32_t wbase = smem_u32(dw_smem) + threadIdx.x * 16;
  const __nv_bfloat16* xf = x + (int64_t)f * H * W * C;
  auto load_col = [&](int wcol, uint4 (&col)[3]) {
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int hh = h + dh - 1;
      if (active && hh >= 0 && hh < H && wcol >= 0 && wcol < W)
        col[dh] = *reinterpret_cast<const uint4*>(xf + ((int64_t)hh * W + wcol) * C + c0);
      else
        col[dh] = zero4;
    }
  };
  // TWO output pixels per iteration: one block-wide reduction (4 values) serves both LayerNorms, every tap weight is read
  // from shared memory once per pair, and the two columns of the next pair are prefetched a full iteration ahead.
  // Window slots 0..3 = columns wc-1 .. wc+2, slots 4..5 = the prefetch.
  uint4 win[6][3];  // [column slot][dh], packed 16-bit
  load_col(-1, win[0]);
  load_col(0, win[1]);
  load_col(1, win[2]);
  load_col(2, win[3]);
  float pool[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) pool[j] = 0.f;
  float g[8], bta[8];
  unpack8(gp, g);
  unpack8(bp, bta);
  for (int wc = 0; wc < W; wc += 2) {
    load_col(wc + 3, win[4]);
    load_col(wc + 4, win[5]);
    float acc0[8], acc1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
#pragma unroll
    for (int dw = 0; dw < 3; ++dw) {
#pragma unroll
      for (int dh = 0; dh < 3; ++dh) {
        float x0[8], x1[8], wv[8];
        unpack8(active ? lds128(wbase + (dh * 3 + dw) * Cl * 2) : zero4, wv);
        unpack8(win[dw][dh], x0);
        unpack8(win[dw + 1][dh], x1);
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc0[j] = fmaf(x0[j], wv[j], acc0[j]); acc1[j] = fmaf(x1[j], wv[j], acc1[j]); }
      }
    }
    // one fused block reduction per pixel PAIR (sum, sum of squares of both): conv outputs are O(1), fp32 E[x^2]-mean^2 is safe
    float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {   // inactive threads hold zeros
      s0 += acc0[j]; q0 = fmaf(acc0[j], acc0[j], q0);
      s1 += acc1[j]; q1 = fmaf(acc1[j], acc1[j], q1);
    }
    float4 sq = block_sum4(s0, q0, s1, q1, red);
    if (split > 1) {
      // exchange the pair's partial statistics with the other half of the channels; parity-indexed slots and barriers, so
      // the next pair's exchange can start before everybody has read this one (a slot is rewritten two pairs later, after a
      // full cluster-wide barrier phase in between)
      const int par = (wc >> 1) & 1;
      const uint32_t phase = (uint32_t)((wc >> 2) & 1);
      if (threadIdx.x == 0) {
        for (uint32_t rr = 0; rr < 2; ++rr) {
          const uint32_t slot = smem_u32(&xchg[par][crank]);
          asm volatile(
              "{\n\t.reg .b32 ra;\n\t"
              "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
              "st.shared::cluster.v4.f32 [ra], {%2, %3, %4, %5};\n\t}"
              ::"r"(slot), "r"(rr), "f"(sq.x), "f"(sq.y), "f"(sq.z), "f"(sq.w)
              : "memory");
          mbar_arrive_cluster(&xbar[par], rr);
        }
      }
      mbar_wait_cluster(&xbar[par], phase);
      const float4 a = xchg[par][0], b = xchg[par][1];
      sq = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    const bool second = wc + 1 < W;
    if (active) {
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        if (px == 1 && !second) break;
        const float mean = (px == 0 ? sq.x : sq.z) / (float)C;
        const float rstd = rsqrtf(fmaxf((px == 0 ? sq.y : sq.w) / (float)C - mean * mean, 0.f) + eps);
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = silu(((px == 0 ? acc0[j] : acc1[j]) - mean) * rstd * g[j] + bta[j]);
        const uint4 packed = pack8(o);
        *reinterpret_cast<uint4*>(y + (((int64_t)f * H + h) * W + wc + px) * C + c0) = packed;
        float r[8];
        unpack8(packed, r);  // pool what the next op will actually read (16-bit rounded)
#pragma unroll
        for (int j = 0; j < 8; ++j) pool[j] += r[j];
      }
    }
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      win[0][dh] = win[2][dh]; win[1][dh] = win[3][dh]; win[2][dh] = win[4][dh]; win[3][dh] = win[5][dh];
    }
  }
  if (active && pool_partial != nullptr) {
    float* pp = pool_partial + ((int64_t)f * H + h) * C + c0;
    *reinterpret_cast<float4*>(pp) = make_float4(pool[0], pool[1], pool[2], pool[3]);
    *reinterpret_cast<float4*>(pp + 4) = make_float4(pool[4], pool[5], pool[6], pool[7]);
  }
}

// pooled[f,c] = (sum_h partial[f,h,c]) / (H*W)
__global__ void se_pool_reduce_kernel(const float* __restrict__ partial, float* __restrict__ pooled, int H, int C,
                                      float inv_hw) {
  pdl_launch_dependents();
  pdl_wait();
  const int f = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int h = 0; h < H; ++h) s += partial[((int64_t)f * H + h) * C + c];
  pooled[(int64_t)f * C + c] = s * inv_hw;
}

__global__ void se_scale_kernel(__nv_bfloat16* __restrict__ y, const float* __restrict__ s, int HW, int C,
                                int64_t total_vec) {
  pdl_launch_dependents();
  pdl_wait();
  const int cv = C / 8;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total_vec;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % cv) * 8;
    const int64_t pix = idx / cv;
    const int f = (int)(pix / HW);
    uint4* p = reinterpret_cast<uint4*>(y) + idx;
    float v[8];
    unpack8(*p, v);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(s + (int64_t)f * C + c0));
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(s + (int64_t)f * C + c0 + 4));
    v[0] *= s0.x; v[1] *= s0.y; v[2] *= s0.z; v[3] *= s0.w;
    v[4] *= s1.x; v[5] *= s1.y; v[6] *= s1.z; v[7] *= s1.w;
    *p = pack8(v);
  }
}

// ---------------------------------------------------------------------------------------------------------
// Conv3d (k = s = 2) im2col, channels-last: A[(to,ho,wo), tap*C + c] = x[2to-pad+dt, 2ho-pad+dh, 2wo-pad+dw, c].
// ---------------------------------------------------------------------------------------------------------
__global__ void conv3d_im2col_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ A, int T, int H,
                                     int W, int C, int pad, int To, int Ho, int Wo) {
  pdl_launch_dependents();
  pdl_wait();
  const int cv = C / 8;
  const int64_t total = (int64_t)To * Ho * Wo * 8 * cv;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % cv) * 8;
    const int tap = (int)((idx / cv) % 8);
    const int64_t row = idx / ((int64_t)cv * 8);
    const int wo = (int)(row % Wo), ho = (int)((row / Wo) % Ho), to = (int)(row / ((int64_t)Wo * Ho));
    const int dt = tap >> 2, dh = (tap >> 1) & 1, dw = tap & 1;
    const int t = 2 * to - pad + dt, hh = 2 * ho - pad + dh, ww = 2 * wo - pad + dw;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (t >= 0 && t < T && hh >= 0 && hh < H && ww >= 0 && ww < W)
      v = *reinterpret_cast<const uint4*>(x + (((int64_t)t * H + hh) * W + ww) * C + c0);
    *reinterpret_cast<uint4*>(A + row * (8 * (int64_t)C) + (int64_t)tap * C + c0) = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// RoPE (rotate-half pairing i <-> i + D/2) applied in place to the q and k heads of a fused QKV buffer.
// One thread per (token, i); loops over heads.  cos/sin from fp32 inv_freq (HF computes them in fp32).
// ---------------------------------------------------------------------------------------------------------
// One CTA per token: cos/sin of the D/2 frequencies go through smem once, then each thread rotates 8 pairs of one
// head with 16-byte accesses.
__global__ void rope_kernel(__nv_bfloat16* __restrict__ qkv, int64_t ld, int S, int Hq, int Hkv, int D, int q_off,
                            int k_off, int pos0, const float* __restrict__ inv_freq, const int* __restrict__ pos_ptr,
                            __nv_bfloat16* __restrict__ append_base, int64_t append_ld, int append_width, int interleaved) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float cs[];  // [D/2] cos, [D/2] sin
  const int half = D / 2;
  const int s = blockIdx.x;
  if (pos_ptr != nullptr) pos0 = *pos_ptr;   // graph-replayed decode step: the position lives in device memory
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    float sn, c;
    sincosf((float)(pos0 + s) * inv_freq[i], &sn, &c);
    // HF casts cos/sin to the activation dtype before use
    cs[i] = __bfloat162float(__float2bfloat16_rn(c));
    cs[half + i] = __bfloat162float(__float2bfloat16_rn(sn));
  }
  __syncthreads();
  const int vph = half / 8;  // 16-byte vectors per half head
  __nv_bfloat16* row = qkv + (int64_t)s * ld;
  for (int t = threadIdx.x; t < (Hq + Hkv) * vph; t += blockDim.x) {
    const int h = t / vph, i0 = (t % vph) * 8;
    __nv_bfloat16* p = row + (h < Hq ? q_off + h * D : k_off + (h - Hq) * D) + i0;
    if (interleaved) {
      // pairs are adjacent columns (2i, 2i+1): this thread's 8 frequencies i0..i0+7 cover 16 consecutive elements
      __nv_bfloat16* pi = row + (h < Hq ? q_off + h * D : k_off + (h - Hq) * D) + 2 * i0;
      float lo[8], hi[8];
      unpack8(*reinterpret_cast<const uint4*>(pi), lo);
      unpack8(*reinterpret_cast<const uint4*>(pi + 8), hi);
      float o0[8], o1[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float c0 = cs[i0 + j], s0 = cs[half + i0 + j];
        o0[2 * j] = lo[2 * j] * c0 - lo[2 * j + 1] * s0;
        o0[2 * j + 1] = lo[2 * j + 1] * c0 + lo[2 * j] * s0;
        const float c1 = cs[i0 + 4 + j], s1 = cs[half + i0 + 4 + j];
        o1[2 * j] = hi[2 * j] * c1 - hi[2 * j + 1] * s1;
        o1[2 * j + 1] = hi[2 * j + 1] * c1 + hi[2 * j] * s1;
      }
      *reinterpret_cast<uint4*>(pi) = pack8(o0);
      *reinterpret_cast<uint4*>(pi + 8) = pack8(o1);
      continue;
    }
    float a[8], b[8], oa[8], ob[8];
    unpack8(*reinterpret_cast<const uint4*>(p), a);
    unpack8(*reinterpret_cast<const uint4*>(p + half), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float c = cs[i0 + j], sn = cs[half + i0 + j];
      oa[j] = a[j] * c - b[j] * sn;
      ob[j] = b[j] * c + a[j] * sn;
    }
    *reinterpret_cast<uint4*>(p) = pack8(oa);
    *reinterpret_cast<uint4*>(p + half) = pack8(ob);
  }
  if (append_base != nullptr) {
    // decode: append the (rotated) fused row to the KV cache at row `pos0 + s`
    __syncthreads();
    const uint4* src = reinterpret_cast<const uint4*>(row);
    uint4* dst = reinterpret_cast<uint4*>(append_base + (int64_t)(pos0 + s) * append_ld);
    for (int v = threadIdx.x; v < append_width / 8; v += blockDim.x) dst[v] = src[v];
  }
}

// out[dst_row[i], :] = table[ids[i], :]
__global__ void embed_splice_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ dst_row,
                                    const __nv_bfloat16* __restrict__ table, int64_t vocab,
                                    __nv_bfloat16* __restrict__ out, int H) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x;
  int64_t id = ids[i];
  if (id < 0 || id >= vocab) return;  // modal placeholder or invalid id: row is written by the connector
  const uint4* src = reinterpret_cast<const uint4*>(table + id * H);
  uint4* dst = reinterpret_cast<uint4*>(out + (int64_t)dst_row[i] * H);
  for (int v = threadIdx.x; v < H / 8; v += blockDim.x) dst[v] = __ldg(src + v);
}

// ---------------------------------------------------------------------------------------------------------
// Skinny GEMM: C[M,N] = act(A[M,K] W[N,K]^T + bias), M <= 32.  One warp per output column n; W streams once from
// HBM (16-byte loads), A (tiny) is re-read from L1/L2.
// ---------------------------------------------------------------------------------------------------------
// Skinny GEMM on the legacy tensor path (mma.sync m16n8k16, bf16 -> fp32): the whole A matrix (M <= 16 rows) is one
// m16 tile, so a warp streams W rows with 16-byte loads and multiplies them against A fragments it reads straight from
// L2 (A is a few hundred KB).  CTA = 16 output columns; its 8 warps split K and reduce through smem.  The k index is
// permuted consistently for A and B so that one 16-byte load supplies two k16 steps (lane quad q holds physical
// k = 32*kb + 8q .. 8q+7).  HBM-bound on W; this is the SE excitation MLP and every linear layer of a decode step.
static constexpr int kSkinnyNT8 = 2;  // n8 tiles per CTA
static constexpr int kSkinnyBatch = 4;  // k-blocks whose loads are in flight together (per warp)

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." VL2_MMA_SYNC_TYPES ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// raw 16 (fp32 A: 32) bytes of A row `row`, elements k .. k+7; the caller guarantees a valid address (indices are clamped,
// results of clamped loads are discarded) so that the loads of several k-blocks can be in flight together
// (volatile: ptxas otherwise sinks each load next to the mma that consumes it, i.e. one DRAM round trip per k-block; volatile
// asm statements keep their source order, and the mma wrapper is volatile too, so a batch's loads all precede its mmas)
__device__ __forceinline__ uint4 ldg_nc_v4_ordered(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
template <bool A_F32>
struct SkinnyA { uint4 lo, hi; };
template <bool A_F32>
__device__ __forceinline__ SkinnyA<A_F32> skinny_load_a(const void* A, int row, int64_t K, int k) {
  SkinnyA<A_F32> r;
  if (A_F32) {
    const uint4* ar = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(A) + (int64_t)row * K + k);
    r.lo = ldg_nc_v4_ordered(ar);
    r.hi = ldg_nc_v4_ordered(ar + 1);
  } else {
    r.lo = ldg_nc_v4_ordered(reinterpret_cast<const __nv_bfloat16*>(A) + (int64_t)row * K + k);
    r.hi = make_uint4(0, 0, 0, 0);
  }
  return r;
}
template <bool A_F32>
__device__ __forceinline__ uint4 skinny_pack_a(const SkinnyA<A_F32>& r, bool keep) {
  if (!keep) return make_uint4(0, 0, 0, 0);
  if (A_F32)
    return make_uint4(pack_bf16(__uint_as_float(r.lo.x), __uint_as_float(r.lo.y)), pack_bf16(__uint_as_float(r.lo.z), __uint_as_float(r.lo.w)),
                      pack_bf16(__uint_as_float(r.hi.x), __uint_as_float(r.hi.y)), pack_bf16(__uint_as_float(r.hi.z), __uint_as_float(r.hi.w)));
  return r.lo;
}

template <bool A_F32>
__global__ void __launch_bounds__(256)
gemm_skinny_kernel(const void* __restrict__ Av, const __nv_bfloat16* __restrict__ Wt, const float* __restrict__ bias,
                   const __nv_bfloat16* __restrict__ residual, void* __restrict__ Cv, int out_f32, int M, int N, int K,
                   int act) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8][kSkinnyNT8][4][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, q = lane & 3;
  const int n_base = blockIdx.x * (8 * kSkinnyNT8);
  const int nkb = (K + 31) / 32;
  for (int m0 = 0; m0 < M; m0 += 16) {
    float acc[kSkinnyNT8][4];
#pragma unroll
    for (int t = 0; t < kSkinnyNT8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[t][e] = 0.f;
    // kSkinnyBatch k-blocks per trip: ALL their loads (branch-free: out-of-range indices are clamped to a valid address and
    // the values dropped) are issued before the first mma, so a warp keeps kSkinnyBatch x 1.5 KB in flight instead of one
    // dependent DRAM round trip per k-block (38 -> us per 8 MB weight matrix at M = 16; profiles/r02_skinny_gemm.txt)
    const int row_lo = min(m0 + g, M - 1), row_hi = min(m0 + g + 8, M - 1);
    const bool lo_ok = m0 + g < M, hi_ok = m0 + g + 8 < M;
    const uint32_t zero = (act == 0x7fffffff) ? 0xffffffffu : 0u;   // no such activation: 0, but only at run time
    for (int kb0 = warp; kb0 < nkb; kb0 += 8 * kSkinnyBatch) {
      SkinnyA<A_F32> ra_lo[kSkinnyBatch], ra_hi[kSkinnyBatch];
      uint4 rw[kSkinnyBatch][kSkinnyNT8];
      bool okk[kSkinnyBatch];
#pragma unroll
      for (int u = 0; u < kSkinnyBatch; ++u) {
        const int k = (kb0 + 8 * u) * 32 + q * 8;
        okk[u] = k < K;
        const int kc = okk[u] ? k : 0;
        ra_lo[u] = skinny_load_a<A_F32>(Av, row_lo, K, kc);
        ra_hi[u] = skinny_load_a<A_F32>(Av, row_hi, K, kc);
#pragma unroll
        for (int t = 0; t < kSkinnyNT8; ++t) {
          const int n = min(n_base + t * 8 + g, N - 1);
          rw[u][t] = ldg_nc_v4_ordered(Wt + (int64_t)n * K + kc);
        }
      }
      // ptxas sinks each load next to the mma that consumes it (one DRAM round trip per k-block, whatever the source order);
      // making the FIRST mma depend on every load of the batch keeps them all in flight together.  `zero` is 0 at run time
      // but not at compile time.
      uint32_t dep = 0;
#pragma unroll
      for (int u = 0; u < kSkinnyBatch; ++u) {
        dep ^= ra_lo[u].lo.x ^ ra_hi[u].lo.x ^ (A_F32 ? (ra_lo[u].hi.x ^ ra_hi[u].hi.x) : 0u);
#pragma unroll
        for (int t = 0; t < kSkinnyNT8; ++t) dep ^= rw[u][t].x;
      }
      dep &= zero;
#pragma unroll
      for (int u = 0; u < kSkinnyBatch; ++u) {
        uint4 a_lo = skinny_pack_a<A_F32>(ra_lo[u], okk[u] && lo_ok);
        if (u == 0) a_lo.x ^= dep;
        const uint4 a_hi = skinny_pack_a<A_F32>(ra_hi[u], okk[u] && hi_ok);
#pragma unroll
        for (int t = 0; t < kSkinnyNT8; ++t) {
          // (columns n >= N read row N-1: they are never stored; a k block past K has zero A)
          const uint4 bw = rw[u][t];
          mma_bf16_16816(acc[t], a_lo.x, a_hi.x, a_lo.y, a_hi.y, bw.x, bw.y);
          mma_bf16_16816(acc[t], a_lo.z, a_hi.z, a_lo.w, a_hi.w, bw.z, bw.w);
        }
      }
    }
    __syncthreads();  // red[] is reused across m0 passes
#pragma unroll
    for (int t = 0; t < kSkinnyNT8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) red[warp][t][e][lane] = acc[t][e];
    __syncthreads();
    if (warp < kSkinnyNT8) {
      const int t = warp;
      float c[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += red[w][t][e][lane];
        c[e] = v;
      }
      const int n = n_base + t * 8 + q * 2;  // c0,c1: (row g, cols n, n+1); c2,c3: (row g+8, cols n, n+1)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + g + 8 * h;
        if (row < M && n < N) {
          float r0 = c[2 * h], r1 = c[2 * h + 1];
          if (bias) { r0 += bias[n]; if (n + 1 < N) r1 += bias[n + 1]; }
          if (act == VL2_ACT_SWIGLU) {  // (n, n+1) is a (gate, up) pair -> output column n/2 of N/2
            const float o = silu(r0) * r1;
            const int64_t oi = (int64_t)row * (N / 2) + (n >> 1);
            if (out_f32) reinterpret_cast<float*>(Cv)[oi] = o;
            else reinterpret_cast<__nv_bfloat16*>(Cv)[oi] = __float2bfloat16_rn(o);
          } else {
            float r[2] = {r0, r1};
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              if (n + j < N) {
                float o = r[j];
                if (act == VL2_ACT_SILU) o = silu(o);
                else if (act == 100) o = 1.f / (1.f + __expf(-o));
                const int64_t oi = (int64_t)row * N + n + j;
                if (residual) o += __bfloat162float(residual[oi]);
                if (out_f32) reinterpret_cast<float*>(Cv)[oi] = o;
                else reinterpret_cast<__nv_bfloat16*>(Cv)[oi] = __float2bfloat16_rn(o);
              }
            }
          }
        }
      }
    }
  }
}



}  // namespace vl2

using namespace vl2;
typedef __nv_bfloat16 bf16;

extern "C" int vl2_layernorm(const void* x, const void* gamma, const void* beta, const void* residual, void* y,
                             int64_t rows, int C, float eps, int act, void* stream) {
  VL2_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, VL2_E_BADSHAPE,
              "vl2_layernorm: rows=%lld C=%d unsupported (C %% 8 == 0)", (long long)rows, C);
  VL2_REQUIRE(act == VL2_ACT_NONE || act == VL2_ACT_SILU, VL2_E_UNSUPPORTED, "vl2_layernorm: act %d unsupported", act);
  VL2_REQUIRE(aligned16(x) && aligned16(y) && aligned16(gamma) && aligned16(beta) && aligned16(residual), VL2_E_BADALIGN,
              "vl2_layernorm: pointers must be 16-byte aligned");
  const unsigned wgrid = (unsigned)((rows + 7) / 8);
  const int nv = (C / 8 + 31) / 32;
#define VL2_LN_WARP(NV)                                                                                   \
  launch_kernel(layernorm_warp_kernel<NV>, dim3(wgrid), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, (const bf16*)gamma, \
      (const bf16*)beta, (const bf16*)residual, (bf16*)y, rows, C, eps, act)
  if (nv <= 1) VL2_LN_WARP(1);
  else if (nv <= 2) VL2_LN_WARP(2);
  else if (nv <= 4) VL2_LN_WARP(4);
  else if (nv <= 6) VL2_LN_WARP(6);     // C <= 1536: SigLIP-so400m rows (1152) stay in registers
  else if (nv <= 16) VL2_LN_WARP(16);   // C <= 4096 (the connector's RegStage rows): 64 registers of packed row per lane, ONE
                                        // pass over global memory with all 16 loads in flight (the two-pass stream kernel took
                                        // 55-64 us on 9216 x 4096 and 23-26 us on 1521 x 4096: latency, not bandwidth)
  else
    launch_kernel(layernorm_stream_kernel, dim3(wgrid), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, (const bf16*)gamma, (const bf16*)beta,
                                                                   (const bf16*)residual, (bf16*)y, rows, C, eps, act);
#undef VL2_LN_WARP
  VL2_CHECK_LAUNCH("layernorm_kernel");
  return VL2_OK;
}

extern "C" int vl2_rmsnorm(const void* x, const void* gamma, void* y, int64_t rows, int C, float eps, void* stream) {
  VL2_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, VL2_E_BADSHAPE,
              "vl2_rmsnorm: rows=%lld C=%d unsupported", (long long)rows, C);
  VL2_REQUIRE(aligned16(x) && aligned16(y) && aligned16(gamma), VL2_E_BADALIGN, "vl2_rmsnorm: 16-byte alignment");
  const unsigned wgrid = (unsigned)((rows + 7) / 8);
  const int nv = (C / 8 + 31) / 32;
#define VL2_RMS_WARP(NV) \
  launch_kernel(rmsnorm_warp_kernel<NV>, dim3(wgrid), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, (const bf16*)gamma, (bf16*)y, rows, C, eps)
  if (nv <= 1) VL2_RMS_WARP(1);
  else if (nv <= 2) VL2_RMS_WARP(2);
  else if (nv <= 4) VL2_RMS_WARP(4);
  else
    launch_kernel(rmsnorm_stream_kernel, dim3(wgrid), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, (const bf16*)gamma, (bf16*)y, rows, C, eps);
#undef VL2_RMS_WARP
  VL2_CHECK_LAUNCH("rmsnorm_kernel");
  return VL2_OK;
}

extern "C" int vl2_row_sumsq(const void* x, float* out, int64_t rows, int C, void* stream) {
  VL2_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, VL2_E_BADSHAPE, "vl2_row_sumsq: rows=%lld C=%d unsupported", (long long)rows, C);
  VL2_REQUIRE(aligned16(x), VL2_E_BADALIGN, "vl2_row_sumsq: 16-byte alignment");
  launch_kernel(row_sumsq_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, out,
                (float*)nullptr, rows, C);
  VL2_CHECK_LAUNCH("row_sumsq_kernel");
  return VL2_OK;
}

extern "C" int vl2_row_stats(const void* x, float* sum_out, float* sumsq_out, int64_t rows, int C, void* stream) {
  VL2_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && sum_out != nullptr && sumsq_out != nullptr, VL2_E_BADSHAPE,
              "vl2_row_stats: rows=%lld C=%d unsupported", (long long)rows, C);
  VL2_REQUIRE(aligned16(x), VL2_E_BADALIGN, "vl2_row_stats: 16-byte alignment");
  launch_kernel(row_sumsq_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x,
                sumsq_out, sum_out, rows, C);
  VL2_CHECK_LAUNCH("row_sumsq_kernel");
  return VL2_OK;
}

extern "C" int vl2_patch_im2col(const void* pixels, void* A, int F, int H, int W, int P, int Kpad, void* stream) {
  VL2_REQUIRE(F > 0 && P > 0 && H >= P && W >= P, VL2_E_BADSHAPE, "vl2_patch_im2col: H,W must be at least P");
  VL2_REQUIRE(Kpad % 8 == 0 && Kpad >= 3 * P * P && W % 2 == 0 && P % 2 == 0, VL2_E_BADSHAPE,
              "vl2_patch_im2col: Kpad %% 8 == 0, Kpad >= 3*P*P, even W and even P required (P=%d)", P);
  VL2_REQUIRE((reinterpret_cast<uintptr_t>(pixels) & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 3) == 0, VL2_E_BADALIGN,
              "vl2_patch_im2col: pixels and A must be 4-byte aligned (pixel pairs are copied as one word)");
  const int64_t total = (int64_t)F * (H / P) * (W / P) * (Kpad / 2);
  launch_kernel(patch_im2col_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)pixels, (bf16*)A, F, H, W, P,
                                                                             Kpad);
  VL2_CHECK_LAUNCH("patch_im2col_kernel");
  return VL2_OK;
}

extern "C" int vl2_clip_embed_finish(const void* patch, const void* cls, const void* pos, const void* gamma,
                                     const void* beta, void* tok, int F, int np, int C, float eps, void* stream) {
  VL2_REQUIRE(F > 0 && np > 0 && C % 8 == 0 && C <= 512 * 8 * kMaxVec, VL2_E_BADSHAPE, "vl2_clip_embed_finish: bad shape");
  VL2_REQUIRE(aligned16(patch) && aligned16(cls) && aligned16(pos) && aligned16(gamma) && aligned16(beta) && aligned16(tok),
              VL2_E_BADALIGN,
              "vl2_clip_embed_finish: 16-byte alignment");
  launch_kernel(clip_embed_finish_kernel, dim3((unsigned)(F * (np + 1))), dim3(row_threads(C)), 0, (cudaStream_t)stream, 1, 
      (const bf16*)patch, (const bf16*)cls, (const bf16*)pos, (const bf16*)gamma, (const bf16*)beta, (bf16*)tok, np, C,
      eps);
  VL2_CHECK_LAUNCH("clip_embed_finish_kernel");
  return VL2_OK;
}

extern "C" int vl2_dwconv3x3_ln_silu(const void* x, const void* w9c, const void* gamma, const void* beta, void* y,
                                     float* pooled, int F, int H, int W, int C, float eps, void* stream) {
  VL2_REQUIRE(F > 0 && H > 0 && W > 0 && C % 8 == 0 && (C <= 8 * 512 || (C <= 16 * 512 && C % 16 == 0)), VL2_E_BADSHAPE,
              "vl2_dwconv3x3_ln_silu: C %% 8 == 0 and C <= 4096, or C %% 16 == 0 and C <= 8192 (C=%d)", C);
  VL2_REQUIRE(aligned16(x) && aligned16(w9c) && aligned16(y) && aligned16(gamma) && aligned16(beta) && aligned16(pooled),
              VL2_E_BADALIGN, "vl2_dwconv3x3_ln_silu: 16-byte alignment");
  // `pooled` layout: [F*C] pooled means followed by [F*H*C] per-row partial sums (workspace); see vl2.h.
  const int split = C > 8 * 512 ? 2 : 1;       // wide rows: two CTAs (a cluster) share a pixel row, half the channels each
  const int Cl = C / split;
  int threads = (Cl / 8 + 31) / 32 * 32;
  float* partial = pooled ? pooled + (int64_t)F * C : nullptr;
  const size_t dw_smem = (size_t)9 * Cl * sizeof(bf16);
  if (dw_smem > 48 * 1024) {
    VL2_SMEM_OPT_IN(dwconv3x3_ln_silu_kernel, 9 * 4096 * 2);
  }
  launch_kernel(dwconv3x3_ln_silu_kernel, dim3((unsigned)(F * H * split)), dim3(threads), dw_smem, (cudaStream_t)stream, split,
      (const bf16*)x, (const bf16*)w9c, (const bf16*)gamma, (const bf16*)beta, (bf16*)y, partial, H, W, C, eps, Cl);
  VL2_CHECK_LAUNCH("dwconv3x3_ln_silu_kernel");
  if (pooled) {
    dim3 grid((C + 255) / 256, F);
    launch_kernel(se_pool_reduce_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 1, partial, pooled, H, C, 1.f / (float)(H * W));
    VL2_CHECK_LAUNCH("se_pool_reduce_kernel");
  }
  return VL2_OK;
}

extern "C" int vl2_se_scale(void* y, const float* s, int F, int HW, int C, void* stream) {
  VL2_REQUIRE(F > 0 && HW > 0 && C % 8 == 0, VL2_E_BADSHAPE, "vl2_se_scale: bad shape");
  VL2_REQUIRE(aligned16(y) && aligned16(s), VL2_E_BADALIGN, "vl2_se_scale: 16-byte alignment");
  const int64_t total = (int64_t)F * HW * (C / 8);
  launch_kernel(se_scale_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, 1, (bf16*)y, s, HW, C, total);
  VL2_CHECK_LAUNCH("se_scale_kernel");
  return VL2_OK;
}

extern "C" int vl2_conv3d_im2col(const void* x, void* A, int T, int H, int W, int C, int pad, int To, int Ho, int Wo,
                                 void* stream) {
  VL2_REQUIRE(T > 0 && H > 0 && W > 0 && C % 8 == 0 && To > 0 && Ho > 0 && Wo > 0 && (pad == 0 || pad == 1),
              VL2_E_BADSHAPE, "vl2_conv3d_im2col: bad shape");
  VL2_REQUIRE(aligned16(x) && aligned16(A), VL2_E_BADALIGN, "vl2_conv3d_im2col: 16-byte alignment");
  const int64_t total = (int64_t)To * Ho * Wo * 8 * (C / 8);
  launch_kernel(conv3d_im2col_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, 1, (const bf16*)x, (bf16*)A, T, H, W, C, pad,
                                                                              To, Ho, Wo);
  VL2_CHECK_LAUNCH("conv3d_im2col_kernel");
  return VL2_OK;
}

extern "C" int vl2_rope_inplace(void* qkv, int64_t ld, int S, int Hq, int Hkv, int D, int q_off, int k_off, int pos0,
                                const float* inv_freq, int interleaved, void* stream) {
  VL2_REQUIRE(S > 0 && D % 2 == 0 && Hq > 0 && Hkv >= 0 && inv_freq != nullptr, VL2_E_BADSHAPE, "vl2_rope_inplace: bad shape");
  VL2_REQUIRE(D % 16 == 0 && ld % 8 == 0 && q_off % 8 == 0 && k_off % 8 == 0 && aligned16(qkv), VL2_E_BADALIGN,
              "vl2_rope_inplace: D %% 16 == 0 and 16-byte aligned heads required");
  int threads = (Hq + Hkv) * (D / 16);
  threads = threads > 512 ? 512 : ((threads + 31) / 32 * 32);
  launch_kernel(rope_kernel, dim3(S), dim3(threads), D * sizeof(float), (cudaStream_t)stream, 1, (bf16*)qkv, ld, S, Hq, Hkv, D, q_off, k_off, pos0,
                inv_freq, (const int*)nullptr, (bf16*)nullptr, (int64_t)0, 0, interleaved);
  VL2_CHECK_LAUNCH("rope_kernel");
  return VL2_OK;
}

extern "C" int vl2_embed_splice(const int64_t* ids, const int32_t* dst_row, int n, const void* table, int64_t vocab,
                                void* out, int H, void* stream) {
  VL2_REQUIRE(n > 0 && H % 8 == 0, VL2_E_BADSHAPE, "vl2_embed_splice: bad shape");
  VL2_REQUIRE(aligned16(table) && aligned16(out), VL2_E_BADALIGN, "vl2_embed_splice: 16-byte alignment");
  launch_kernel(embed_splice_kernel, dim3(n), dim3(128), 0, (cudaStream_t)stream, 1, ids, dst_row, (const bf16*)table, vocab, (bf16*)out, H);
  VL2_CHECK_LAUNCH("embed_splice_kernel");
  return VL2_OK;
}


extern "C" int vl2_gemm_skinny(const void* A, int a_f32, const void* W, const float* bias, const void* residual, void* C,
                               int out_f32, int M, int N, int K, int act, void* stream) {
  VL2_REQUIRE(M > 0 && M <= 32 && N > 0 && K > 0 && K % 8 == 0, VL2_E_BADSHAPE,
              "vl2_gemm_skinny: need 0 < M <= 32 and K %% 8 == 0 (M=%d K=%d)", M, K);
  VL2_REQUIRE(aligned16(A) && aligned16(W), VL2_E_BADALIGN, "vl2_gemm_skinny: 16-byte alignment");
  VL2_REQUIRE(act == VL2_ACT_NONE || act == VL2_ACT_SILU || act == 100 || act == VL2_ACT_SWIGLU, VL2_E_UNSUPPORTED,
              "vl2_gemm_skinny: act %d", act);
  VL2_REQUIRE(act != VL2_ACT_SWIGLU || (N % 2 == 0 && residual == nullptr), VL2_E_UNSUPPORTED,
              "vl2_gemm_skinny: SWIGLU needs even N and no residual");
  if (M == 1 && !a_f32) return launch_gemv(A, W, bias, residual, C, out_f32, N, K, act, 0.f, (cudaStream_t)stream);
  const int blocks = (N + 8 * kSkinnyNT8 - 1) / (8 * kSkinnyNT8);
  if (a_f32)
    launch_kernel(gemm_skinny_kernel<true>, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, 1, A, (const bf16*)W, bias, (const bf16*)residual, C, out_f32, M, N, K, act);
  else
    launch_kernel(gemm_skinny_kernel<false>, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, 1, A, (const bf16*)W, bias, (const bf16*)residual, C, out_f32, M, N, K, act);
  VL2_CHECK_LAUNCH("gemm_skinny_kernel");
  return VL2_OK;
}

// ---- graph-replayable decode step: the token position is read from device memory ------------------------------
extern "C" int vl2_decode_rope_append(void* qkv_row, void* cache, int64_t cache_ld, const int32_t* pos_dev, int Hq, int Hkv,
                                      int D, const float* inv_freq, int interleaved, void* stream) {
  VL2_REQUIRE(qkv_row && cache && pos_dev && inv_freq && D % 16 == 0 && cache_ld % 8 == 0, VL2_E_BADSHAPE,
              "vl2_decode_rope_append: bad arguments");
  VL2_REQUIRE(aligned16(qkv_row) && aligned16(cache), VL2_E_BADALIGN, "vl2_decode_rope_append: 16-byte alignment");
  const int width = (Hq + 2 * Hkv) * D;
  int threads = (Hq + Hkv) * (D / 16);
  threads = threads > 512 ? 512 : ((threads + 31) / 32 * 32);
  launch_kernel(rope_kernel, dim3(1), dim3(threads), D * sizeof(float), (cudaStream_t)stream, 1, (bf16*)qkv_row, (int64_t)width, 1,
                Hq, Hkv, D, 0, Hq * D, 0, inv_freq, (const int*)pos_dev, (bf16*)cache, cache_ld, width, interleaved);
  VL2_CHECK_LAUNCH("rope_kernel");
  return VL2_OK;
}
