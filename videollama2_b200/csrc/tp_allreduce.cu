// Tensor-parallel all-reduce fused with the residual stream's RMSNorm statistics, over NVLink 5 / NVSwitch, as ONE kernel:
//   x[S,H] = sum over ranks of part_r[S,H]   (bf16 partial outputs of a row-parallel GEMM; rank 0's partial carries the residual)
//   ss[S]  = sum_h x[s,h]^2                  (what the next folded RMSNorm reads: vl2_gemm_args.rms_sumsq_in, one part per row)
// Every rank owns a contiguous block of rows: it reduces them (peer loads over NVLink in rank order, fp32 accumulation, one
// rounding; optionally one multimem.ld_reduce through the switch), squares what it will store, and writes rows + statistics
// into EVERY rank's buffers (one multimem.st through the NVSwitch, or peer stores) - the two-shot all-reduce, nothing else
// on the wire.
// Cross-GPU ordering is inside the kernel: a start barrier (every rank's partial is complete) and an end barrier (every
// rank's rows have landed everywhere; nobody still reads a partial) over symmetric-memory signal pads, so the stream needs
// no collective library call and no extra launches.  The reference has no counterpart (no tensor parallelism).
#include "row_common.cuh"

namespace vl2 {

struct TpArParams {
  const __nv_bfloat16* part[8];   // every rank's partial buffer (symmetric memory, peer-mapped); part[rank] is local
  __nv_bfloat16* xout[8];         // every rank's result buffer
  float* stats[8];                // every rank's row statistics
  uint32_t* pads[8];              // every rank's signal pad: [0..7] start arrivals, [8..15] done arrivals, [16] local block counter
  const __nv_bfloat16* part_mc;   // multicast addresses of the same buffers (NULL = no NVLS: peer loads / stores)
  __nv_bfloat16* xout_mc;
  float* stats_mc;
  int rank, world, S, H;
  uint32_t epoch;                 // 1, 2, 3, ... per call (same on every rank)
};

__device__ __forceinline__ void signal_add_sys(uint32_t* p) {
  asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void wait_ge(const uint32_t* p, uint32_t want) {
  uint32_t spins = 0;
  while ((int32_t)(ld_acquire_sys(p) - want) < 0) {
    if (++spins > (1u << 26)) { asm volatile("trap;"); }   // a lost peer must not hang the box
    __nanosleep(64);
  }
}
// in-switch reduction of one 16-byte vector (8 bf16) over all ranks of the multicast group, fp32 accumulation
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_addr) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4." VL2_MULTIMEM_TYPE " {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc_addr)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_v4(void* mc_addr, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_addr), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}
__device__ __forceinline__ void multimem_st_f32(float* mc_addr, float v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc_addr), "f"(v) : "memory");
}

// RED_MC: reduce inside the NVSwitch (multimem.ld_reduce).  Checked with scripts/tp_allreduce_check.py: the switch does
// NOT round the bf16 result to nearest - ~19 % of the elements differ by one bf16 ulp from the correctly rounded fp32 sum
// (which NCCL and the peer-load path both produce bit for bit) - so it is opt-in; the default reduces with peer loads in
// rank order (exact fp32 accumulation, one rounding) and uses the switch only to BROADCAST (ST_MC: multimem.st, an exact copy).
template <bool RED_MC, bool ST_MC>
__global__ void __launch_bounds__(256)
tp_allreduce_stats_kernel(const TpArParams p) {
  __shared__ float red[64];
  const int tid = threadIdx.x;
  uint32_t* my_pad = p.pads[p.rank];
  // the producing GEMM / GEMV precedes this kernel in its stream, but under PDL it triggers before its stores: wait for
  // it before signalling that this rank's partial is complete
  pdl_wait();
  // ---- start barrier: every rank's partial is complete
  if (blockIdx.x == 0 && tid < p.world) signal_add_sys(p.pads[tid] + p.rank);
  if (tid < p.world) wait_ge(my_pad + tid, p.epoch);
  __syncthreads();

  const int rows_per = (p.S + p.world - 1) / p.world;
  const int r0 = p.rank * rows_per;
  const int r1 = min(p.S, r0 + rows_per);
  const int nvec = p.H / 8;
  for (int row = r0 + (int)blockIdx.x; row < r1; row += (int)gridDim.x) {
    const int64_t base = (int64_t)row * p.H;
    float q = 0.f;
    for (int v = tid; v < nvec; v += blockDim.x) {
      uint4 out;
      if (RED_MC) {
        out = multimem_ld_reduce_bf16x8(p.part_mc + base + v * 8);
      } else {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int r = 0; r < p.world; ++r) {              // fixed order: the same bits whoever owns the row
          float f[8];
          unpack8(*reinterpret_cast<const uint4*>(p.part[r] + base + v * 8), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
        out = pack8(acc);
      }
      float f[8];
      unpack8(out, f);                                     // statistics of what the consumers will read (bf16-rounded)
#pragma unroll
      for (int j = 0; j < 8; ++j) q = fmaf(f[j], f[j], q);
      if (ST_MC) {
        multimem_st_v4(p.xout_mc + base + v * 8, out);
      } else {
        for (int r = 0; r < p.world; ++r) *reinterpret_cast<uint4*>(p.xout[r] + base + v * 8) = out;
      }
    }
    const float tot = block_sum2(q, 0.f, red).x;
    if (tid == 0) {
      if (ST_MC) multimem_st_f32(p.stats_mc + row, tot);
      else for (int r = 0; r < p.world; ++r) p.stats[r][row] = tot;
    }
  }
  // ---- end barrier: this rank's rows are visible everywhere, and no peer still reads this rank's partial
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    const uint32_t arrived = atomicAdd(my_pad + 16, 1u);
    if (arrived == gridDim.x - 1) {                        // last block of this rank
      my_pad[16] = 0u;                                     // re-arm for the next launch (ordered before the signals below)
      __threadfence_system();
      for (int r = 0; r < p.world; ++r) signal_add_sys(p.pads[r] + 8 + p.rank);
      for (int r = 0; r < p.world; ++r) wait_ge(my_pad + 8 + r, p.epoch);
    }
  }
}

}  // namespace vl2

using namespace vl2;

extern "C" int vl2_tp_allreduce_stats(const vl2_tp_allreduce_args* a, void* stream) {
  VL2_REQUIRE(a != nullptr, VL2_E_BADSHAPE, "vl2_tp_allreduce_stats: null args");
  VL2_REQUIRE(a->world >= 1 && a->world <= 8 && a->rank >= 0 && a->rank < a->world && a->S > 0 && a->H > 0 && a->H % 8 == 0 &&
                  a->epoch > 0,
              VL2_E_BADSHAPE, "vl2_tp_allreduce_stats: bad rank/world/shape/epoch (%d/%d, %d x %d, %u)", a->rank, a->world,
              a->S, a->H, a->epoch);
  const bool mc = a->part_mc != nullptr;
  VL2_REQUIRE(!mc || (a->xout_mc != nullptr && a->stats_mc != nullptr), VL2_E_BADSHAPE,
              "vl2_tp_allreduce_stats: all three multicast addresses or none");
  TpArParams p;
  for (int r = 0; r < 8; ++r) {
    const bool used = r < a->world;
    p.part[r] = used ? reinterpret_cast<const __nv_bfloat16*>(a->part[r]) : nullptr;
    p.xout[r] = used ? reinterpret_cast<__nv_bfloat16*>(a->xout[r]) : nullptr;
    p.stats[r] = used ? a->stats[r] : nullptr;
    p.pads[r] = used ? a->pads[r] : nullptr;
    if (used) {
      VL2_REQUIRE(a->pads[r] != nullptr && a->part[r] != nullptr && (mc || (a->xout[r] && a->stats[r])), VL2_E_BADSHAPE,
                  "vl2_tp_allreduce_stats: missing buffer of rank %d", r);
      VL2_REQUIRE(aligned16(a->part[r]) && aligned16(a->xout[r]), VL2_E_BADALIGN, "vl2_tp_allreduce_stats: 16-byte alignment");
    }
  }
  p.part_mc = reinterpret_cast<const __nv_bfloat16*>(a->part_mc);
  p.xout_mc = reinterpret_cast<__nv_bfloat16*>(a->xout_mc);
  p.stats_mc = a->stats_mc;
  p.rank = a->rank; p.world = a->world; p.S = a->S; p.H = a->H; p.epoch = a->epoch;
  const int rows_per = (a->S + a->world - 1) / a->world;
  int blocks = rows_per < 2 * sm_count() ? rows_per : 2 * sm_count();
  if (blocks < 1) blocks = 1;
  cudaStream_t st = (cudaStream_t)stream;
  const bool inswitch = mc && a->inswitch_reduce != 0;
  if (inswitch) launch_kernel(tp_allreduce_stats_kernel<true, true>, dim3(blocks), dim3(256), 0, st, 1, p);
  else if (mc) launch_kernel(tp_allreduce_stats_kernel<false, true>, dim3(blocks), dim3(256), 0, st, 1, p);
  else launch_kernel(tp_allreduce_stats_kernel<false, false>, dim3(blocks), dim3(256), 0, st, 1, p);
  VL2_CHECK_LAUNCH("tp_allreduce_stats_kernel");
  return VL2_OK;
}
