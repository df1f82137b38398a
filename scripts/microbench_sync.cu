// Latency of the synchronisation primitives the attention kernel's softmax warps use, measured in isolation:
// successful mbarrier try_wait / test_wait (1 warp vs 8 warps polling the same barrier), bar.sync over 256 / 64 threads,
// __syncwarp, st.shared + ld.shared exchange.  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.u32 %0, 1, 0, P1;\n\t}\n"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ bool test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.u32 %0, 1, 0, P1;\n\t}\n"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__global__ void k(long long* out, int active_warps) {
  __shared__ uint64_t bar;
  __shared__ float xch[256];
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&bar)) : "memory");
  __syncthreads();
  long long t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  constexpr int N = 32;
  if (warp < active_warps) {
    long long t0 = clock64();
    for (int i = 0; i < N; ++i) while (!try_wait(&bar, 0)) {}
    long long t1 = clock64(); t[0] = t1 - t0; t0 = t1;
    for (int i = 0; i < N; ++i) while (!test_wait(&bar, 0)) {}
    t1 = clock64(); t[1] = t1 - t0; t0 = t1;
    for (int i = 0; i < N; ++i) __syncwarp();
    t1 = clock64(); t[2] = t1 - t0; t0 = t1;
    for (int i = 0; i < N; ++i) { if ((threadIdx.x & 31) == 0) while (!try_wait(&bar, 0)) {} __syncwarp(); }
    t1 = clock64(); t[3] = t1 - t0; t0 = t1;
    float v = threadIdx.x;
    for (int i = 0; i < N; ++i) {   // the max exchange: st.shared, named barrier over the active warps, 2 x ld.shared
      xch[threadIdx.x] = v;
      asm volatile("bar.sync 1, %0;" ::"r"(active_warps * 32) : "memory");
      v = fmaxf(xch[threadIdx.x ^ 128 % (active_warps * 32)], xch[threadIdx.x]) + 1.f;
    }
    t1 = clock64(); t[4] = t1 - t0; t0 = t1;
    if (active_warps == 8) {
      for (int i = 0; i < N; ++i) {   // the same exchange over pair barriers (warp w and w + 4: 64 threads)
        xch[threadIdx.x] = v;
        asm volatile("bar.sync %0, 64;" ::"r"(2 + (warp & 3)) : "memory");
        v = fmaxf(xch[threadIdx.x ^ 128], xch[threadIdx.x]) + 1.f;
      }
      t1 = clock64(); t[5] = t1 - t0; t0 = t1;
    }
    for (int i = 0; i < N; ++i) { long long c = clock64(); t[7] += c & 1; }
    t1 = clock64(); t[6] = t1 - t0;
    if (v == -1.f) t[6] = 0;
  }
  if (threadIdx.x == 0) for (int i = 0; i < 8; ++i) out[i] = t[i] / N;
}
int main() {
  long long* d; cudaMalloc(&d, 64);
  for (int aw : {1, 8}) {
    k<<<1, 256>>>(d, aw); k<<<1, 256>>>(d, aw);
    long long h[8]; cudaMemcpy(h, d, 64, cudaMemcpyDeviceToHost);
    printf("active warps %d: try_wait(success) %lld, test_wait(success) %lld, __syncwarp %lld, lane0 try_wait + __syncwarp %lld, "
           "sts + bar.sync(all) + 2 lds %lld, sts + bar.sync(64) + 2 lds %lld, clock64 %lld cycles each\n",
           aw, h[0], h[1], h[2], h[3], h[4], h[5], h[6]);
  }
  return 0;
}
