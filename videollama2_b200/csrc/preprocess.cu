// Frame preprocessing in front of the vision tower, on the device (SURVEY.md §8f row 3):
//   uint8 RGB frames [T,H,W,3] -> (virtual) expand2square canvas -> Pillow-exact antialiased bicubic resize
//   (two integer passes, horizontal first, each rounded and clipped to uint8) -> centre crop -> rescale + normalise
//   through a [3,256] table -> bf16 [T,3,S,S] (what CLIPVisionTower / SiglipVisionTower consume).
// Reference: videollama2/mm_utils.py:27-38,91-103,132-202 + transformers 4.40 CLIPImageProcessor + Pillow
// libImaging/Resample.c (ImagingResampleHorizontal_8bpc / Vertical_8bpc).  Integer work: bit-exact with Pillow.
// The 22-bit fixed-point coefficient tables are computed on the host exactly as Pillow does (double arithmetic) and
// passed in; HBM-bound byte work: reads T*H*W*3 bytes once, one uint8 intermediate of T*canvas_h*out_w*3 bytes.
#include "host_common.h"
#include "ptx.cuh"

namespace vl2 {

constexpr int kPrecisionBits = 32 - 8 - 2;

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kPrecisionBits;   // arithmetic shift: floor, as Pillow's clip8 lookup index
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One canvas row per CTA: the row (image pixels or the pad colour) is staged in shared memory with coalesced loads,
// then every thread produces output pixels of that row.
__global__ void __launch_bounds__(256)
resample_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ tmp, int H, int W, int canvas_h, int canvas_w,
                  int off_y, int off_x, uint32_t pad_rgb, int out_w, const int* __restrict__ bounds,
                  const int* __restrict__ kk, int ksize) {
  extern __shared__ uint8_t row[];   // [canvas_w * 3]
  pdl_wait();   // under PDL the producer of the frames may still be running, or still reading what tmp overwrites
  const int cy = blockIdx.x, t = blockIdx.y;
  const int iy = cy - off_y;
  const uint8_t pr = pad_rgb & 0xff, pg = (pad_rgb >> 8) & 0xff, pb = (pad_rgb >> 16) & 0xff;
  const bool in_rows = iy >= 0 && iy < H;
  const uint8_t* srow = src + ((int64_t)t * H + (in_rows ? iy : 0)) * W * 3;
  for (int i = threadIdx.x; i < canvas_w * 3; i += blockDim.x) {
    const int cx = i / 3, c = i - cx * 3;
    const int ix = cx - off_x;
    uint8_t v = c == 0 ? pr : (c == 1 ? pg : pb);
    if (in_rows && ix >= 0 && ix < W) v = srow[ix * 3 + c];
    row[i] = v;
  }
  __syncthreads();
  uint8_t* orow = tmp + ((int64_t)t * canvas_h + cy) * out_w * 3;
  for (int ox = threadIdx.x; ox < out_w; ox += blockDim.x) {
    const int x0 = bounds[2 * ox], n = bounds[2 * ox + 1];
    const int* k = kk + (int64_t)ox * ksize;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int j = 0; j < n; ++j) {
      const int w = __ldg(k + j);
      const uint8_t* p = row + (x0 + j) * 3;
      a0 += p[0] * w;
      a1 += p[1] * w;
      a2 += p[2] * w;
    }
    orow[ox * 3 + 0] = clip8(a0);
    orow[ox * 3 + 1] = clip8(a1);
    orow[ox * 3 + 2] = clip8(a2);
  }
}

// Vertical pass over the cropped window only + rescale/normalise table + planar bf16 store.
__global__ void __launch_bounds__(128)
resample_v_kernel(const uint8_t* __restrict__ tmp, __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ out_u8,
                  int canvas_h, int out_w, int crop_top, int crop_left, int crop, const int* __restrict__ bounds,
                  const int* __restrict__ kk, int ksize, const float* __restrict__ lut) {
  pdl_wait();   // tmp is resample_h's output, and the kernels after this one wait only for this grid
  const int x = blockIdx.x * blockDim.x + threadIdx.x;   // column inside the crop window
  const int y = blockIdx.y, t = blockIdx.z;
  if (x >= crop) return;
  const int oy = crop_top + y, ox = crop_left + x;
  const int y0 = bounds[2 * oy], n = bounds[2 * oy + 1];
  const int* k = kk + (int64_t)oy * ksize;
  const uint8_t* col = tmp + (((int64_t)t * canvas_h + y0) * out_w + ox) * 3;
  int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
  for (int j = 0; j < n; ++j) {
    const int w = __ldg(k + j);
    const uint8_t* p = col + (int64_t)j * out_w * 3;
    a0 += p[0] * w;
    a1 += p[1] * w;
    a2 += p[2] * w;
  }
  const uint8_t r = clip8(a0), g = clip8(a1), b = clip8(a2);
  const int64_t plane = (int64_t)crop * crop;
  __nv_bfloat16* o = out + (int64_t)t * 3 * plane + (int64_t)y * crop + x;
  o[0] = __float2bfloat16_rn(lut[r]);
  o[plane] = __float2bfloat16_rn(lut[256 + g]);
  o[2 * plane] = __float2bfloat16_rn(lut[512 + b]);
  if (out_u8 != nullptr) {
    uint8_t* u = out_u8 + (((int64_t)t * crop + y) * crop + x) * 3;
    u[0] = r;
    u[1] = g;
    u[2] = b;
  }
}

}  // namespace vl2

using namespace vl2;

extern "C" size_t vl2_preprocess_workspace(const vl2_preprocess_args* a) {
  if (a == nullptr || a->T <= 0 || a->canvas_h <= 0 || a->out_w <= 0) return 0;
  return (size_t)a->T * a->canvas_h * a->out_w * 3;
}

extern "C" int vl2_preprocess_frames(const vl2_preprocess_args* a, void* stream) {
  VL2_REQUIRE(a != nullptr, VL2_E_BADSHAPE, "vl2_preprocess_frames: null args");
  VL2_REQUIRE(a->T > 0 && a->H > 0 && a->W > 0 && a->canvas_h >= a->H && a->canvas_w >= a->W && a->off_y >= 0 &&
                  a->off_x >= 0 && a->off_y + a->H <= a->canvas_h && a->off_x + a->W <= a->canvas_w,
              VL2_E_BADSHAPE, "vl2_preprocess_frames: bad frame / canvas geometry (T=%d H=%d W=%d canvas %dx%d off %d,%d)",
              a->T, a->H, a->W, a->canvas_h, a->canvas_w, a->off_y, a->off_x);
  VL2_REQUIRE(a->out_h > 0 && a->out_w > 0 && a->crop > 0 && a->crop_top >= 0 && a->crop_left >= 0 &&
                  a->crop_top + a->crop <= a->out_h && a->crop_left + a->crop <= a->out_w,
              VL2_E_BADSHAPE, "vl2_preprocess_frames: bad resize / crop geometry (%dx%d, crop %d at %d,%d)", a->out_h,
              a->out_w, a->crop, a->crop_top, a->crop_left);
  VL2_REQUIRE(a->canvas_w <= 16384 && a->ksize_h > 0 && a->ksize_v > 0, VL2_E_UNSUPPORTED,
              "vl2_preprocess_frames: canvas wider than 16384 pixels or empty coefficient tables");
  VL2_REQUIRE(a->frames && a->bounds_h && a->kk_h && a->bounds_v && a->kk_v && a->lut && a->tmp && a->out_bf16,
              VL2_E_BADSHAPE, "vl2_preprocess_frames: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)a->canvas_w * 3;
  if (smem > 48 * 1024) {
    VL2_SMEM_OPT_IN(resample_h_kernel, 64 * 1024);
  }
  const uint32_t pad = (uint32_t)a->pad_rgb[0] | ((uint32_t)a->pad_rgb[1] << 8) | ((uint32_t)a->pad_rgb[2] << 16);
  launch_kernel(resample_h_kernel, dim3(a->canvas_h, a->T), dim3(256), smem, st, 1, a->frames, a->tmp, a->H, a->W, a->canvas_h,
                a->canvas_w, a->off_y, a->off_x, pad, a->out_w, a->bounds_h, a->kk_h, a->ksize_h);
  VL2_CHECK_LAUNCH("resample_h_kernel");
  launch_kernel(resample_v_kernel, dim3((a->crop + 127) / 128, a->crop, a->T), dim3(128), 0, st, 1, (const uint8_t*)a->tmp,
                (__nv_bfloat16*)a->out_bf16, a->out_u8, a->canvas_h, a->out_w, a->crop_top, a->crop_left, a->crop, a->bounds_v,
                a->kk_v, a->ksize_v, a->lut);
  VL2_CHECK_LAUNCH("resample_v_kernel");
  return VL2_OK;
}
