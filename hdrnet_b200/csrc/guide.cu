// guide.cu -- standalone full-resolution guidance-map kernels (SURVEY.md rows a8, a9).
//
// The reference builds the guide from a chain of TF elementwise ops that materialise a
// [B,H,W,3,16] temporary (16x the image) in HBM (hdrnet/models.py:168-175).  Here one pass
// reads 12 B/px and writes 4 B/px; a thread owns 4 consecutive pixels (3 x LDG.128 in,
// 1 x STG.128 out), and all coefficients are constant-bank operands.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "guide.cuh"
#include "hdrnet_b200.h"

namespace hdrnet_b200 {

struct CurvesFn {
  CurvesGuideParams p;
  __device__ __forceinline__ float operator()(float r, float g, float b) const {
    return curves_guide(p, r, g, b);
  }
};
template <int kFeats>
struct NNFn {
  NNGuideParams p;
  __device__ __forceinline__ float operator()(float r, float g, float b) const {
    return nn_guide<kFeats>(p, r, g, b);
  }
};

template <class Fn>
__global__ void __launch_bounds__(256)
guide_kernel(const float* __restrict__ rgb, float* __restrict__ guide, long long npix,
             bool vec_ok, const __grid_constant__ Fn fn) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long tid0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nquads = vec_ok ? npix / 4 : 0;
  for (long long q = tid0; q < nquads; q += stride) {
    const float4* in4 = reinterpret_cast<const float4*>(rgb) + 3 * q;
    const float4 c0 = __ldg(in4), c1 = __ldg(in4 + 1), c2 = __ldg(in4 + 2);
    float4 o;
    o.x = fn(c0.x, c0.y, c0.z);
    o.y = fn(c0.w, c1.x, c1.y);
    o.z = fn(c1.z, c1.w, c2.x);
    o.w = fn(c2.y, c2.z, c2.w);
    reinterpret_cast<float4*>(guide)[q] = o;
  }
  // tail (npix % 4) or the whole image when the buffers are not 16-byte aligned
  for (long long p = nquads * 4 + tid0; p < npix; p += stride)
    guide[p] = fn(__ldg(rgb + 3 * p), __ldg(rgb + 3 * p + 1), __ldg(rgb + 3 * p + 2));
}

template <class Fn>
static int launch_guide(const float* rgb, float* guide, long long npix, const Fn& fn,
                        cudaStream_t stream) {
  if (npix < 0) return HDRNET_E_BAD_SHAPE;
  if (npix == 0) return HDRNET_OK;
  if (!rgb || !guide) return HDRNET_E_NULL_POINTER;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(rgb) | reinterpret_cast<uintptr_t>(guide)) & 15u) == 0;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long work = vec_ok ? (npix + 3) / 4 : npix;
  long long blocks = (work + 255) / 256;
  if (blocks > static_cast<long long>(sms) * 8) blocks = static_cast<long long>(sms) * 8;
  guide_kernel<Fn><<<static_cast<int>(blocks), 256, 0, stream>>>(rgb, guide, npix, vec_ok, fn);
  return static_cast<int>(cudaGetLastError());
}

// Host-side parameter packing, shared with slice_apply.cu's guide-fused entry points.
int pack_curves_params(CurvesGuideParams* p, const float* ccm, const float* ccm_bias,
                       const float* shifts, const float* slopes, const float* mix,
                       float mix_bias) {
  if (!ccm || !ccm_bias || !shifts || !slopes || !mix) return HDRNET_E_NULL_POINTER;
  std::memcpy(p->ccm, ccm, sizeof(p->ccm));
  std::memcpy(p->ccm_bias, ccm_bias, sizeof(p->ccm_bias));
  std::memcpy(p->shifts, shifts, sizeof(p->shifts));
  std::memcpy(p->slopes, slopes, sizeof(p->slopes));
  std::memcpy(p->mix, mix, sizeof(p->mix));
  p->mix_bias = mix_bias;
  double folded = mix_bias;
  for (int c = 0; c < 3; ++c) {
    double cs = 0.0;
    for (int k = 0; k < kCurvePts; ++k)
      cs += static_cast<double>(slopes[c * kCurvePts + k]) * static_cast<double>(shifts[c * kCurvePts + k]);
    folded -= static_cast<double>(mix[c]) * cs;
  }
  p->folded_bias = static_cast<float>(folded);
  return HDRNET_OK;
}

int pack_nn_params(NNGuideParams* p, const float* w1, const float* b1, const float* w2, float b2,
                   int feats) {
  if (!w1 || !b1 || !w2) return HDRNET_E_NULL_POINTER;
  if (feats < 1 || feats > kMaxGuideFeats) return HDRNET_E_UNSUPPORTED;
  std::memset(p, 0, sizeof(*p));
  p->feats = (feats + 1) & ~1;  // processed in pairs; the pad feature has zero weights
  for (int c = 0; c < 3; ++c)
    for (int f = 0; f < feats; ++f) p->w1[c][f] = w1[c * feats + f];
  std::memcpy(p->b1, b1, sizeof(float) * feats);
  std::memcpy(p->w2, w2, sizeof(float) * feats);
  p->b2 = b2;
  return HDRNET_OK;
}

}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

int hdrnet_guide_curves_f32(const float* input, float* guide, long long npix, const float* ccm,
                            const float* ccm_bias, const float* shifts, const float* slopes,
                            const float* mix, float mix_bias, void* stream) {
  CurvesFn fn;
  const int rc = pack_curves_params(&fn.p, ccm, ccm_bias, shifts, slopes, mix, mix_bias);
  if (rc != HDRNET_OK) return rc;
  return launch_guide(input, guide, npix, fn, static_cast<cudaStream_t>(stream));
}

int hdrnet_guide_nn_f32(const float* input, float* guide, long long npix, const float* w1,
                        const float* b1, const float* w2, float b2, int feats, void* stream) {
  NNGuideParams np;
  const int rc = pack_nn_params(&np, w1, b1, w2, b2, feats);
  if (rc != HDRNET_OK) return rc;
  if (np.feats <= 16) {
    NNFn<16> fn; fn.p = np;
    return launch_guide(input, guide, npix, fn, static_cast<cudaStream_t>(stream));
  }
  NNFn<kMaxGuideFeats> fn; fn.p = np;
  return launch_guide(input, guide, npix, fn, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
