// Per-step score rows for generate(output_scores / output_logits): one fp32 row [V] copied into slot *step_dev + add of
// a per-call buffer described by a device parameter block (vl2_score_record_params), so one captured decode graph
// records into buffers of any size.  See DESIGN.md section 3.
//
// A row is 128 KB (V = 32000) to 608 KB (V = 152064): the copy is spread over ceil(V / 1024) CTAs with four independent
// loads in flight per thread.
#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

constexpr int kRecordThreads = 256;
constexpr int kRecordPerThread = 4;
constexpr int kRecordMaxV = 262144;

__global__ void __launch_bounds__(kRecordThreads)
record_row_kernel(const float* __restrict__ row, int V, const vl2_score_record_params* __restrict__ P, int which,
                  const int64_t* __restrict__ step_dev, int64_t add) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t slot = *step_dev + add;
  float* base = which == VL2_RECORD_SCORES ? P->scores : P->logits;
  if (base == nullptr || P->V != V || slot < 0 || slot >= P->capacity) return;
  float* dst = base + slot * (int64_t)V;
  const int i0 = blockIdx.x * (kRecordThreads * kRecordPerThread) + threadIdx.x;
  float v[kRecordPerThread];
#pragma unroll
  for (int u = 0; u < kRecordPerThread; ++u) {
    const int i = i0 + u * kRecordThreads;
    v[u] = i < V ? __ldg(row + i) : 0.f;
  }
#pragma unroll
  for (int u = 0; u < kRecordPerThread; ++u) {
    const int i = i0 + u * kRecordThreads;
    if (i < V) dst[i] = v[u];
  }
}

}  // namespace vl2

using namespace vl2;

extern "C" int vl2_record_row(const float* row, int V, const vl2_score_record_params* params, int which,
                              const int64_t* step_dev, int64_t add, void* stream) {
  VL2_REQUIRE(V > 0 && V <= kRecordMaxV, VL2_E_BADSHAPE, "vl2_record_row: V = %d outside [1, %d]", V, kRecordMaxV);
  VL2_REQUIRE(which == VL2_RECORD_LOGITS || which == VL2_RECORD_SCORES, VL2_E_BADSHAPE,
              "vl2_record_row: which = %d is neither VL2_RECORD_LOGITS nor VL2_RECORD_SCORES", which);
  VL2_REQUIRE(row && params && step_dev, VL2_E_BADALIGN, "vl2_record_row: null pointer");
  VL2_REQUIRE((reinterpret_cast<uintptr_t>(row) & 3) == 0 && (reinterpret_cast<uintptr_t>(params) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(step_dev) & 7) == 0,
              VL2_E_BADALIGN, "vl2_record_row: row needs 4-byte, params / step 8-byte alignment");
  const int blocks = (V + kRecordThreads * kRecordPerThread - 1) / (kRecordThreads * kRecordPerThread);
  launch_kernel(record_row_kernel, dim3(blocks), dim3(kRecordThreads), 0, (cudaStream_t)stream, 1, row, V, params, which,
                step_dev, add);
  VL2_CHECK_LAUNCH("record_row_kernel");
  return VL2_OK;
}
