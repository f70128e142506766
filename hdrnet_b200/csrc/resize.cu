// resize.cu -- bilinear resize with align_corners=True (+ optional fused add), NHWC float32.
// Replaces tf.image.resize_images(..., BILINEAR, align_corners=True) as used by
// HDRNetGaussianPyrNN._multiscale_input and ._output (hdrnet/models.py:249-289), TF1 legacy
// semantics: src = dst * (in - 1) / (out - 1), lo = floor(src), hi = min(lo + 1, in - 1),
// value = top + (bottom - top) * fy with top = tl + (tr - tl) * fx.  Its VJP
// (hdrnet_resize_bilinear_grad_f32) gathers the transpose of that map; the fused add's VJP is the
// identity and needs no kernel.
#include <cuda_runtime.h>

#include <algorithm>

#include "hdrnet_b200.h"
#include "slice_rows.cuh"

namespace hdrnet_b200 {

// One output coordinate's source taps: src = o * s rounded to float32, lo = floor(src),
// hi = min(lo + 1, n - 1), frac = src - lo.  The forward and its VJP both take their taps from
// here, so the VJP sends each gradient back to exactly the pixels and weights the forward read.
struct AcTaps {
  int lo, hi;
  float frac;
};

__device__ __forceinline__ AcTaps ac_taps(int o, float s, int n) {
  // __fmul_rn: the product is rounded before frac = src - lo, in every caller.  A plain `o * s`
  // may be contracted into fma(o, s, -lo) where the compiler rematerialises it, which gives a frac
  // the forward never used.
  const float src = __fmul_rn(static_cast<float>(o), s);
  const int lo = static_cast<int>(floorf(src));
  return {lo, min(lo + 1, n - 1), src - lo};
}

// Output element e of the resize (+ add): the one arithmetic of the float forward and of its
// quantising form below, so both compute the same float.
__device__ __forceinline__ float resize_ac_value(const float* __restrict__ in, const float* __restrict__ add,
                                                 int H, int W, int C, int OH, int OW, float sy,
                                                 float sx, long long e) {
  const int c = static_cast<int>(e % C);
  const int ox = static_cast<int>((e / C) % OW);
  const int oy = static_cast<int>((e / (static_cast<long long>(C) * OW)) % OH);
  const int b = static_cast<int>(e / (static_cast<long long>(C) * OW * OH));
  const AcTaps ty = ac_taps(oy, sy, H), tx = ac_taps(ox, sx, W);
  const int y0 = ty.lo, y1 = ty.hi, x0 = tx.lo, x1 = tx.hi;
  const float fy = ty.frac, fx = tx.frac;
  const float* img = in + static_cast<size_t>(b) * H * W * C;
  const float tl = __ldg(img + (static_cast<size_t>(y0) * W + x0) * C + c);
  const float tr = __ldg(img + (static_cast<size_t>(y0) * W + x1) * C + c);
  const float bl = __ldg(img + (static_cast<size_t>(y1) * W + x0) * C + c);
  const float br = __ldg(img + (static_cast<size_t>(y1) * W + x1) * C + c);
  const float top = tl + (tr - tl) * fx;
  const float bot = bl + (br - bl) * fx;
  float v = top + (bot - top) * fy;
  if (add) v += __ldg(add + e);
  return v;
}

__global__ void __launch_bounds__(256)
resize_bilinear_ac_kernel(const float* __restrict__ in, const float* __restrict__ add,
                          float* __restrict__ out, int B, int H, int W, int C, int OH, int OW,
                          float sy, float sx, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x)
    out[e] = resize_ac_value(in, add, H, W, C, OH, OW, sy, sx, e);
}

// The same resize (+ add) with the model path's quantising epilogue: the uint8 cast of
// tf.cast(255 * clip(v, 0, 1)) or the uint16 rint(65535 * clip(v, 0, 1)) of the fused slice-apply
// kernels (slice_rows.cuh).  The pyramid's last upsample-and-add writes its result with it.
template <int kOut>
__global__ void __launch_bounds__(256)
resize_bilinear_ac_quantize_kernel(const float* __restrict__ in, const float* __restrict__ add,
                                   void* __restrict__ out, int H, int W, int C, int OH, int OW,
                                   float sy, float sx, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = resize_ac_value(in, add, H, W, C, OH, OW, sy, sx, e);
    if constexpr (kOut == kPxU8)
      static_cast<unsigned char*>(out)[e] = static_cast<unsigned char>(float_to_u8(v));
    else
      static_cast<unsigned short*>(out)[e] = static_cast<unsigned short>(float_to_u16(v));
  }
}

// [first, last] output coordinates whose taps may reach input coordinate i: the inverse map of
// src in [i - 1, i + 1), widened by one on each side for the rounding of src = o * s.  With s = 0
// (n = 1, or one output) every output is a candidate.
__device__ __forceinline__ int2 ac_candidates(int i, float s, int on) {
  if (s == 0.0f) return make_int2(0, on - 1);
  const float lo = floorf(static_cast<float>(i - 1) / s) - 1.0f;
  const float hi = ceilf(static_cast<float>(i + 1) / s) + 1.0f;
  return make_int2(static_cast<int>(fmaxf(lo, 0.0f)),
                   static_cast<int>(fminf(hi, static_cast<float>(on - 1))));
}

// The weight output coordinate o's taps give input coordinate i, and whether they reach it at all:
// (1 - frac) on lo, frac on hi, both where lo == hi on the last row or column.
__device__ __forceinline__ bool ac_weight(int o, float s, int n, int i, float* w) {
  const AcTaps t = ac_taps(o, s, n);
  if (t.lo != i && t.hi != i) return false;
  *w = (t.lo == i ? 1.0f - t.frac : 0.0f) + (t.hi == i ? t.frac : 0.0f);
  return true;
}

// din[b, y, x, c] = sum over the output pixels whose taps reach (y, x) of wy * wx * dout, gathered
// in a fixed order (output rows ascending, and within a row the columns ascending): no atomics, so
// the result is the same bits on every run.
__global__ void __launch_bounds__(256)
resize_bilinear_ac_grad_kernel(const float* __restrict__ dout, float* __restrict__ din, int H,
                               int W, int C, int OH, int OW, float sy, float sx,
                               long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % C);
    const int x = static_cast<int>((e / C) % W);
    const int y = static_cast<int>((e / (static_cast<long long>(C) * W)) % H);
    const long long b = e / (static_cast<long long>(C) * W * H);
    const int2 ry = ac_candidates(y, sy, OH), rx = ac_candidates(x, sx, OW);
    const float* img = dout + b * OH * OW * C + c;
    float acc = 0.0f;
    for (int oy = ry.x; oy <= ry.y; ++oy) {
      float wy;
      if (!ac_weight(oy, sy, H, y, &wy)) continue;
      const float* row = img + static_cast<long long>(oy) * OW * C;
      float racc = 0.0f;
      for (int ox = rx.x; ox <= rx.y; ++ox) {
        float wx;
        if (ac_weight(ox, sx, W, x, &wx)) racc = fmaf(wx, __ldg(row + static_cast<long long>(ox) * C), racc);
      }
      acc = fmaf(wy, racc, acc);
    }
    din[e] = acc;
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

extern "C" int hdrnet_resize_bilinear_grad_f32(const float* dout, float* din, int B, int H, int W,
                                               int C, int OH, int OW, void* stream) {
  if (B < 0 || H < 1 || W < 1 || C < 1 || OH < 1 || OW < 1) return HDRNET_E_BAD_SHAPE;
  const long long total = static_cast<long long>(B) * H * W * C;
  if (total == 0) return HDRNET_OK;
  if (!dout || !din) return HDRNET_E_NULL_POINTER;
  const float sy = (OH > 1) ? static_cast<float>(H - 1) / static_cast<float>(OH - 1) : 0.0f;
  const float sx = (OW > 1) ? static_cast<float>(W - 1) / static_cast<float>(OW - 1) : 0.0f;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  hdrnet_b200::resize_bilinear_ac_grad_kernel<<<static_cast<unsigned>(blocks), 256, 0,
                                                static_cast<cudaStream_t>(stream)>>>(
      dout, din, H, W, C, OH, OW, sy, sx, total);
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

// ---- the network input of a ragged batch (hdrnet_lowres_nearest_ragged_f32) -------------------
namespace hdrnet_b200 {

struct RaggedLowres {
  int n;
  struct { const void* image; int H, W; } img[HDRNET_RAGGED_MAX_IMAGES];
};

// lowres_nearest_kernel with each image's own pointer and extent: the same source index and
// conversion per output element, so image b's rows equal that kernel's on image b alone.
template <int kFmt>
__global__ void __launch_bounds__(256)
lowres_nearest_ragged_kernel(const __grid_constant__ RaggedLowres a, float* __restrict__ lowres, int SH,
                             int SW, long long total) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += stride) {
    const int c = static_cast<int>(e % 3);
    const long long px = e / 3;
    const int ox = static_cast<int>(px % SW);
    const int oy = static_cast<int>((px / SW) % SH);
    const int b = static_cast<int>(px / (static_cast<long long>(SW) * SH));
    const int H = a.img[b].H, W = a.img[b].W;
    const int iy = min(static_cast<int>((2LL * oy + 1) * H / (2LL * SH)), H - 1);
    const int ix = min(static_cast<int>((2LL * ox + 1) * W / (2LL * SW)), W - 1);
    lowres[e] = code_to_float<kFmt>(a.img[b].image, (static_cast<long long>(iy) * W + ix) * 3 + c);
  }
}

int validate_ragged(const hdrnet_image_desc* images, int B, int in_fmt, int out_fmt, bool need_out, int min_hw);

}  // namespace hdrnet_b200

extern "C" int hdrnet_lowres_nearest_ragged_f32(const hdrnet_image_desc* images, int B, int fmt, float* lowres,
                                                int SH, int SW, void* stream) {
  using namespace hdrnet_b200;
  if (SH < 1 || SW < 1) return HDRNET_E_BAD_SHAPE;
  int rc = validate_ragged(images, B, fmt, HDRNET_PX_F32, false, 1);
  if (rc != HDRNET_OK || B == 0) return rc;
  if (!lowres) return HDRNET_E_NULL_POINTER;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int c0 = 0; c0 < B; c0 += HDRNET_RAGGED_MAX_IMAGES) {
    RaggedLowres a;
    a.n = std::min(HDRNET_RAGGED_MAX_IMAGES, B - c0);
    for (int i = 0; i < a.n; ++i) a.img[i] = {images[c0 + i].image, images[c0 + i].H, images[c0 + i].W};
    const long long total = static_cast<long long>(a.n) * SH * SW * 3;
    const unsigned nb = static_cast<unsigned>(std::min<long long>((total + 255) / 256, 132LL * 32));
    float* dst = lowres + static_cast<size_t>(c0) * SH * SW * 3;
    if (fmt == HDRNET_PX_F32) lowres_nearest_ragged_kernel<HDRNET_PX_F32><<<nb, 256, 0, st>>>(a, dst, SH, SW, total);
    else if (fmt == HDRNET_PX_U8) lowres_nearest_ragged_kernel<HDRNET_PX_U8><<<nb, 256, 0, st>>>(a, dst, SH, SW, total);
    else lowres_nearest_ragged_kernel<HDRNET_PX_U16><<<nb, 256, 0, st>>>(a, dst, SH, SW, total);
    rc = static_cast<int>(cudaGetLastError());
    if (rc != HDRNET_OK) return rc;
  }
  return HDRNET_OK;
}

// ---- pieces of the whole-model C path (model.cu) ---------------------------------------------
namespace hdrnet_b200 {

// img_as_float of a whole image (code_to_float per element): the float full-resolution image the
// pyramid's levels are resized from, bit-exact where models.image_to_float is not (row f-11).
template <int kFmt>
__global__ void __launch_bounds__(256)
image_to_float_kernel(const void* __restrict__ image, float* __restrict__ out, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x)
    out[e] = code_to_float<kFmt>(image, e);
}

static unsigned elementwise_blocks(long long total) {
  const long long blocks = (total + 255) / 256;
  return static_cast<unsigned>(blocks > 132LL * 32 ? 132LL * 32 : blocks);
}

// `total` uint8 / uint16 code values -> float32.
int launch_image_to_float(const void* image, int fmt, float* out, long long total, cudaStream_t st) {
  if (total == 0) return HDRNET_OK;
  if (fmt == HDRNET_PX_U8)
    image_to_float_kernel<HDRNET_PX_U8><<<elementwise_blocks(total), 256, 0, st>>>(image, out, total);
  else if (fmt == HDRNET_PX_U16)
    image_to_float_kernel<HDRNET_PX_U16><<<elementwise_blocks(total), 256, 0, st>>>(image, out, total);
  else
    return HDRNET_E_UNSUPPORTED;
  return static_cast<int>(cudaGetLastError());
}

// hdrnet_resize_bilinear_f32(in, add, ...) written through the uint8 or uint16 epilogue.
int launch_resize_quantize(const float* in, const float* add, void* out, int out_fmt, int B, int H,
                           int W, int C, int OH, int OW, cudaStream_t st) {
  if (B < 0 || H < 1 || W < 1 || C < 1 || OH < 1 || OW < 1) return HDRNET_E_BAD_SHAPE;
  const long long total = static_cast<long long>(B) * OH * OW * C;
  if (total == 0) return HDRNET_OK;
  if (!in || !out) return HDRNET_E_NULL_POINTER;
  const float sy = (OH > 1) ? static_cast<float>(H - 1) / static_cast<float>(OH - 1) : 0.0f;
  const float sx = (OW > 1) ? static_cast<float>(W - 1) / static_cast<float>(OW - 1) : 0.0f;
  const unsigned nb = elementwise_blocks(total);
  if (out_fmt == HDRNET_PX_U8)
    resize_bilinear_ac_quantize_kernel<HDRNET_PX_U8><<<nb, 256, 0, st>>>(in, add, out, H, W, C, OH, OW, sy, sx, total);
  else if (out_fmt == HDRNET_PX_U16)
    resize_bilinear_ac_quantize_kernel<HDRNET_PX_U16><<<nb, 256, 0, st>>>(in, add, out, H, W, C, OH, OW, sy, sx, total);
  else
    return HDRNET_E_UNSUPPORTED;
  return static_cast<int>(cudaGetLastError());
}

}  // namespace hdrnet_b200
