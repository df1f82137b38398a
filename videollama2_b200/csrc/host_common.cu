// Error state, launch counter and the cuTensorMapEncodeTiled trampoline (resolved through the runtime so that
// libvl2.so does not link libcuda directly and still loads on a CPU-only box for the symbol-export test).
#include "host_common.h"

#include <stdlib.h>

#include <atomic>
#include <mutex>

namespace vl2 {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static std::atomic<int> g_pdl_override{-1};
void set_pdl_override(int v) { g_pdl_override.store(v); }

bool pdl_enabled() {
  const int ov = g_pdl_override.load(std::memory_order_relaxed);
  if (ov >= 0) return ov == 1;
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VL2_PDL");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;   // measured neutral-to-slightly-negative on this path: opt-in
  }
  return v == 1;
}

int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) return 0;
  return dev < kMaxDevices ? dev : kMaxDevices - 1;
}

int sm_count() {
  static int cached[kMaxDevices] = {};
  const int slot = device_slot();
  if (cached[slot] <= 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;   // no device: plan for an H100 SXM
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cached[slot] = n;
  }
  return cached[slot];
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_tiled_fn>(p);
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes) {
  encode_tiled_fn enc = get_encode();
  if (!enc) return set_error(VL2_E_CUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
#ifdef VL2_HALF
  const CUtensorMapDataType elem_type = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
#else
  const CUtensorMapDataType elem_type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
#endif
  const CUtensorMapSwizzle swz = swizzle_bytes == 32   ? CU_TENSOR_MAP_SWIZZLE_32B
                                 : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                       : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(map, elem_type, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(VL2_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dim0 %llu, box0 %u)", (int)r,
                     rank, (unsigned long long)dims[0], box[0]);
  return VL2_OK;
}

}  // namespace vl2

extern "C" {
int vl2_version(void) { return VL2_VERSION; }
#ifdef VL2_HALF
int vl2_storage_dtype(void) { return 1; }
#else
int vl2_storage_dtype(void) { return 0; }
#endif
const char* vl2_last_error(void) { return vl2::g_err; }
int64_t vl2_launch_count(void) { return vl2::g_launches.load(); }
int vl2_set_pdl(int mode) {
  if (mode < -1 || mode > 1) return vl2::set_error(VL2_E_BADSHAPE, "vl2_set_pdl: mode must be -1, 0 or 1");
  vl2::set_pdl_override(mode);
  return VL2_OK;
}
}
