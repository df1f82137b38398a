// Host-side helpers shared by the C-ABI translation units: error reporting, launch counting, TMA tensor maps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/vl2.h"

namespace vl2 {

int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);
int sm_count();        // of the CURRENT device (cached per device)
int device_slot();     // cudaGetDevice(), clamped to [0, kMaxDevices): index of per-device host caches
static constexpr int kMaxDevices = 64;

// Encode a tiled bf16 tensor map with 128-byte swizzle (swizzle_bytes = 64 / 32: 64- / 32-byte swizzle, for boxes whose
// rows are 64 / 32 bytes) and zero OOB fill.  dims/strides are innermost-first; strides (bytes) are given for dims 1..rank-1.
int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes = 128);

#define VL2_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return ::vl2::set_error(VL2_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                              __FILE__, __LINE__);                                                \
  } while (0)

#define VL2_CHECK_LAUNCH(name)                                                                              \
  do {                                                                                                      \
    cudaError_t _e = cudaGetLastError();                                                                    \
    if (_e != cudaSuccess)                                                                                  \
      return ::vl2::set_error(VL2_E_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e));         \
    ::vl2::count_launch();                                                                                  \
  } while (0)

#define VL2_REQUIRE(cond, code, ...)                           \
  do {                                                         \
    if (!(cond)) return ::vl2::set_error(code, __VA_ARGS__);   \
  } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device (context): opt in once per (kernel, device), so a
// process that drives several GPUs (torch.cuda.device(i) around the calls) gets the attribute on each of them.
#define VL2_SMEM_OPT_IN(kernel, bytes)                                                                              \
  do {                                                                                                              \
    static bool _vl2_done[::vl2::kMaxDevices] = {};                                                                 \
    const int _vl2_dev = ::vl2::device_slot();                                                                      \
    if (!_vl2_done[_vl2_dev]) {                                                                                     \
      VL2_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));      \
      _vl2_done[_vl2_dev] = true;                                                                                   \
    }                                                                                                               \
  } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

void set_pdl_override(int v);  // -1: follow VL2_PDL, 0: off, 1: on (vl2_set_pdl)
bool pdl_enabled();  // VL2_PDL=1 enables programmatic dependent launch (default off: profiles/r01_bench_v10_*.json)

// One launch path for every kernel: optional thread-block cluster, programmatic dependent launch attribute.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                        int cluster_x, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace vl2
