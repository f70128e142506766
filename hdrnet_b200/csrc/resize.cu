// resize.cu -- bilinear resize with align_corners=True (+ optional fused add), NHWC float32.
// Replaces tf.image.resize_images(..., BILINEAR, align_corners=True) as used by
// HDRNetGaussianPyrNN._multiscale_input and ._output (hdrnet/models.py:249-289), TF1 legacy
// semantics: src = dst * (in - 1) / (out - 1), lo = floor(src), hi = min(lo + 1, in - 1),
// value = top + (bottom - top) * fy with top = tl + (tr - tl) * fx.
#include <cuda_runtime.h>

#include "hdrnet_b200.h"

namespace hdrnet_b200 {

__global__ void __launch_bounds__(256)
resize_bilinear_ac_kernel(const float* __restrict__ in, const float* __restrict__ add,
                          float* __restrict__ out, int B, int H, int W, int C, int OH, int OW,
                          float sy, float sx, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % C);
    const int ox = static_cast<int>((e / C) % OW);
    const int oy = static_cast<int>((e / (static_cast<long long>(C) * OW)) % OH);
    const int b = static_cast<int>(e / (static_cast<long long>(C) * OW * OH));
    const float fy_src = oy * sy, fx_src = ox * sx;
    const int y0 = static_cast<int>(floorf(fy_src)), x0 = static_cast<int>(floorf(fx_src));
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float fy = fy_src - y0, fx = fx_src - x0;
    const float* img = in + static_cast<size_t>(b) * H * W * C;
    const float tl = __ldg(img + (static_cast<size_t>(y0) * W + x0) * C + c);
    const float tr = __ldg(img + (static_cast<size_t>(y0) * W + x1) * C + c);
    const float bl = __ldg(img + (static_cast<size_t>(y1) * W + x0) * C + c);
    const float br = __ldg(img + (static_cast<size_t>(y1) * W + x1) * C + c);
    const float top = tl + (tr - tl) * fx;
    const float bot = bl + (br - bl) * fx;
    float v = top + (bot - top) * fy;
    if (add) v += __ldg(add + e);
    out[e] = v;
  }
}

}  // namespace hdrnet_b200

extern "C" int hdrnet_resize_bilinear_f32(const float* in, const float* add, float* out, int B,
                                          int H, int W, int C, int OH, int OW, void* stream) {
  if (B < 0 || H < 1 || W < 1 || C < 1 || OH < 1 || OW < 1) return HDRNET_E_BAD_SHAPE;
  const long long total = static_cast<long long>(B) * OH * OW * C;
  if (total == 0) return HDRNET_OK;
  if (!in || !out) return HDRNET_E_NULL_POINTER;
  const float sy = (OH > 1) ? static_cast<float>(H - 1) / static_cast<float>(OH - 1) : 0.0f;
  const float sx = (OW > 1) ? static_cast<float>(W - 1) / static_cast<float>(OW - 1) : 0.0f;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  hdrnet_b200::resize_bilinear_ac_kernel<<<static_cast<unsigned>(blocks), 256, 0,
                                           static_cast<cudaStream_t>(stream)>>>(
      in, add, out, B, H, W, C, OH, OW, sy, sx, total);
  return static_cast<int>(cudaGetLastError());
}

// ---- nearest-neighbour low-resolution input from the decoded image (row f-3) -----------------
namespace hdrnet_b200 {

// img_as_float of one code value: bit-exact with float32(float64(v) / D) for every v (one
// Newton step on v * (1/D); exhaustive check in tests/test_px_gpu.py).
template <int kFmt>
__device__ __forceinline__ float code_to_float(const void* image, long long idx) {
  if constexpr (kFmt == HDRNET_PX_F32) {
    return __ldg(static_cast<const float*>(image) + idx);
  } else {
    constexpr float D = (kFmt == HDRNET_PX_U8) ? 255.0f : 65535.0f;
    constexpr float R = 1.0f / D;
    const float f = (kFmt == HDRNET_PX_U8)
                        ? static_cast<float>(__ldg(static_cast<const unsigned char*>(image) + idx))
                        : static_cast<float>(__ldg(static_cast<const unsigned short*>(image) + idx));
    const float q0 = f * R;
    return fmaf(fmaf(-q0, D, f), R, q0);
  }
}

template <int kFmt>
__global__ void __launch_bounds__(256)
lowres_nearest_kernel(const void* __restrict__ image, float* __restrict__ lowres, int B, int H,
                      int W, int SH, int SW, long long total) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += stride) {
    const int c = static_cast<int>(e % 3);
    const long long px = e / 3;
    const int ox = static_cast<int>(px % SW);
    const int oy = static_cast<int>((px / SW) % SH);
    const long long b = px / (static_cast<long long>(SW) * SH);
    // floor((o + 0.5) * H / S) in exact integer arithmetic
    const int iy = min(static_cast<int>((2LL * oy + 1) * H / (2LL * SH)), H - 1);
    const int ix = min(static_cast<int>((2LL * ox + 1) * W / (2LL * SW)), W - 1);
    lowres[e] = code_to_float<kFmt>(image, ((b * H + iy) * W + ix) * 3 + c);
  }
}

}  // namespace hdrnet_b200

extern "C" int hdrnet_lowres_nearest_f32(const void* image, int fmt, float* lowres, int B, int H,
                                         int W, int SH, int SW, void* stream) {
  if (B < 0 || H < 1 || W < 1 || SH < 1 || SW < 1) return HDRNET_E_BAD_SHAPE;
  const long long total = static_cast<long long>(B) * SH * SW * 3;
  if (total == 0) return HDRNET_OK;
  if (!image || !lowres) return HDRNET_E_NULL_POINTER;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned nb = static_cast<unsigned>(blocks);
  switch (fmt) {
    case HDRNET_PX_F32:
      hdrnet_b200::lowres_nearest_kernel<HDRNET_PX_F32><<<nb, 256, 0, st>>>(image, lowres, B, H, W, SH, SW, total);
      break;
    case HDRNET_PX_U8:
      hdrnet_b200::lowres_nearest_kernel<HDRNET_PX_U8><<<nb, 256, 0, st>>>(image, lowres, B, H, W, SH, SW, total);
      break;
    case HDRNET_PX_U16:
      hdrnet_b200::lowres_nearest_kernel<HDRNET_PX_U16><<<nb, 256, 0, st>>>(image, lowres, B, H, W, SH, SW, total);
      break;
    default:
      return HDRNET_E_UNSUPPORTED;
  }
  return static_cast<int>(cudaGetLastError());
}
