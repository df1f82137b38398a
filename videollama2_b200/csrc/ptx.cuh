// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), clusters, wgmma (see also wgmma.cuh).
// Everything here is device-only and header-only.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

// ----------------------------------------------------------------------------------------------
// 16-bit storage type of the library.  The same sources build twice: libvl2.so stores activations / weights as bf16,
// libvl2_f16.so (-DVL2_HALF) as IEEE fp16 - the reference's own inference dtype (videollama2/__init__.py:60,
// model/__init__.py:71 load everything with torch_dtype=float16).  Every kernel moves 16-bit elements through the helpers
// below (pack_bf16 / bf16_lo / bf16_hi / unpack8 / pack8) and the CUDA conversion intrinsics, so the half build only
// re-targets those names; accumulation is fp32 either way and wgmma takes both input formats.
// ----------------------------------------------------------------------------------------------
#ifdef VL2_HALF
#define __nv_bfloat16 __half
#define __nv_bfloat162 __half2
#define __float2bfloat16_rn __float2half_rn
#define __bfloat162float __half2float
#define __floats2bfloat162_rn __floats2half2_rn
#define __bfloat16_as_ushort __half_as_ushort
#define VL2_WGMMA_TYPES "f16.f16"
#define VL2_MMA_SYNC_TYPES "f16.f16"
#define VL2_MULTIMEM_TYPE "f16x2"
#define VL2_STORAGE_DTYPE 1
#else
#define VL2_WGMMA_TYPES "bf16.bf16"
#define VL2_MMA_SYNC_TYPES "bf16.bf16"
#define VL2_MULTIMEM_TYPE "bf16x2"
#define VL2_STORAGE_DTYPE 0
#endif

namespace vl2 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL, opt-in with VL2_PDL=1): every kernel of the library can be launched with the
// programmatic-stream-serialization attribute and starts with  pdl_launch_dependents(); ...local setup...; pdl_wait();
// so the NEXT kernel's CTAs are scheduled (and run their prologue) while this kernel's last wave drains, and a kernel
// never touches global memory before all of its predecessors have completed and flushed.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin on try_wait (HW-suspending). A bounded spin count turns a protocol bug into a trap instead of a hang,
// which matters on a GPU box we cannot attach to: a hung kernel costs the whole gpurun lease.
#ifndef VL2_MBAR_SPIN_LIMIT
#define VL2_MBAR_SPIN_LIMIT (1u << 24)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // First poll outside the loop: ptxas puts a YIELD in front of a polling LOOP's try_wait, and a warp that yields next to
  // a sibling warp with a long run of ready instructions (the other half-row's exp2 pass, an epilogue) is not picked
  // again for ~200 cycles - even when the barrier was complete all along.  The straight-line poll carries no YIELD.
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > VL2_MBAR_SPIN_LIMIT) { asm volatile("trap;"); }
  }
}

// Wait that PARKS the thread: try_wait with a suspend-time hint, so the hardware keeps the thread asleep until the phase
// completes (or the hint expires) instead of returning to a polling loop after the short default limit.  For the roles
// that wait LONG by design (a producer for a free ring slot, the MMA issuer for the softmax warps, epilogue warps for a
// whole mainloop): their polling loops kept the SM's barrier unit so busy that every other thread's poll - even one that
// is satisfied at once - took ~200 cycles instead of ~40 (attention trace: "repeated (satisfied) S poll").
__device__ __forceinline__ bool mbar_try_wait_parked(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait_parked(bar, parity)) {
    if (++spins > VL2_MBAR_SPIN_LIMIT) { asm volatile("trap;"); }
  }
}

// Wait for two barriers at once: both polls are in flight together, so a wait that is already satisfied costs one barrier
// round trip instead of two (each poll is a few hundred cycles when eight warps hit the barrier unit at the same time).
__device__ __forceinline__ void mbar_wait2(uint64_t* bar_a, uint32_t parity_a, uint64_t* bar_b, uint32_t parity_b) {
  {   // first pair of polls outside the loop (no YIELD in front of it: see mbar_wait)
    const bool a = mbar_try_wait(bar_a, parity_a);
    const bool b = mbar_try_wait(bar_b, parity_b);
    if (a && b) return;
  }
  uint32_t spins = 0;
  for (;;) {
    const bool a = mbar_try_wait(bar_a, parity_a);
    const bool b = mbar_try_wait(bar_b, parity_b);
    if (a && b) break;
    if (++spins > VL2_MBAR_SPIN_LIMIT) { asm volatile("trap;"); }
  }
}

// wait whose acquire has CLUSTER scope: for barriers other CTAs of the cluster arrive on (release.cluster) after writing
// this CTA's shared memory through DSMEM
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0, ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!ok && ++spins > VL2_MBAR_SPIN_LIMIT) { asm volatile("trap;"); }
  }
}


// ----------------------------------------------------------------------------------------------
// Proxy fence: generic-proxy shared-memory writes -> visible to the async proxy (TMA, wgmma operands)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// TMA store of one box from shared to global memory (bulk async-group completion).  The writers of the smem box must
// have executed fence.proxy.async (fence_proxy_async_smem) and synchronised with the issuing thread first; parts of the
// box outside the tensor are not written.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the issuing thread's bulk groups have finished READING shared memory (the source buffers may be rewritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// at most N of the issuing thread's bulk groups are still reading shared memory (the older groups' sources may be rewritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// the issuing thread's bulk groups are complete, their global writes included
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// Hint a 2-D tile of a tensor map into L2 (no smem, no barrier): issued a few k-blocks ahead of the real load so that the
// HBM latency is off the smem-stage round trip.
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* m, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1)
               : "memory");
}
// 1-D bulk copy global -> shared (no tensor map): size and both addresses multiples of 16 bytes.
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA load of one box, written to the same shared-memory offset in every CTA of `cta_mask` (cluster multicast); each
// destination CTA's mbarrier at the offset of `bar` receives the bytes it got.
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                               uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// Clusters
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same smem offset in CTA `rank` of the cluster, releasing this thread's prior writes at
// cluster scope: for an arrival that publishes data written through DSMEM.  ptxas puts a GPU-scope MEMBAR in front of it.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar_local, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar_local)), "r"(rank)
      : "memory");
}
// The same arrival without the cluster-scope release (default semantics: release at CTA scope), which compiles to a bare
// SYNCS.ARRIVE with no memory barrier.  Enough for a signal that publishes no data of its own, e.g. "I have finished
// reading this ring slot" when the reads were async-proxy (wgmma) reads already complete at wgmma.wait_group.
__device__ __forceinline__ void mbar_arrive_peer(uint64_t* bar_local, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar_local)), "r"(rank)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// Warpgroup MMA (wgmma).  Shared-memory matrix descriptor (64 bit), sm_90 flavour:
//   [0,14) start address >> 4   [16,30) leading-dim byte offset >> 4   [32,46) stride-dim byte offset >> 4
//   [49,52) base offset          [62,64) layout type (1 = 128B swizzle)
// K-major, SWIZZLE_128B (what TMA writes for a {64 x rows} 16-bit box with CU_TENSOR_MAP_SWIZZLE_128B):
//   row r lives at r*128 B, its 16-byte chunks XOR-ed with (r & 7); 8-row groups are 1024 B apart => SBO = 1024;
//   LBO is unused.  Stepping K by 16 elements inside the 128-B atom is start address += 32 B.
// MN-major, SWIZZLE_128B (a {64 x k-rows} box whose contiguous dim is M/N):
//   element (mn, k) lives at k*128 B + mn*2 B (swizzled by k & 7); 8-k groups 1024 B apart => SBO = 1024;
//   the next 64-wide MN atom is LBO bytes away.  Stepping K by 16 is start address += 2048 B.
// Stage bases are 1024-byte aligned, so the base offset field stays 0.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
// order this thread's register / shared-memory accesses before the wgmma that follow (accumulators, register A operands)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accumulator reads / writes across a wgmma that is still in flight
template <int N>
__device__ __forceinline__ void wgmma_keep(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup role (all warps of the warpgroup execute it)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// 2^x on the MUFU pipe (single instruction; inputs here are <= ~8, flush-to-zero is fine for probabilities)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// explicit shared-space 16-byte accesses on 32-bit shared addresses (keeps the compiler from emitting generic LD/ST)
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------------------------
// small numeric helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
#ifdef VL2_HALF
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu))); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u >> 16))); }
#else
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
#endif

}  // namespace vl2

#include "wgmma.cuh"
