// guide.cuh -- per-pixel guidance-map functions, shared by the standalone guide kernels
// (guide.cu) and the guide-fused slice-apply kernel (slice_apply.cu).
//
// Parameters travel BY VALUE in the kernel argument block (constant bank), so every
// coefficient is a free constant operand of the FMA that uses it: no loads, no shared memory.
#pragma once

#include <cuda_runtime.h>

#include "common.cuh"

namespace hdrnet_b200 {

constexpr int kCurvePts = 16;     // hdrnet/models.py:147 (npts, hard-coded in the reference)
constexpr int kMaxGuideFeats = 32;

// HDRNetCurves._guide (hdrnet/models.py:145-190):
//   t = rgb . ccm + ccm_bias; u_c = sum_k slopes[c][k] * relu(t_c - shifts[c][k]);
//   guide = clip(sum_c mix[c] * u_c + mix_bias, 0, 1)
struct CurvesGuideParams {
  float ccm[3][3];   // [in][out]: t_out = sum_in x_in * ccm[in][out]  (tf.matmul(x, ccm))
  float ccm_bias[3];
  float shifts[3][kCurvePts];
  float slopes[3][kCurvePts];
  float mix[3];
  float mix_bias;
  // Folded by pack_curves_params():  slope * relu(t - s) = slope * max(t, s) - slope * s, so
  //   sum_c mix_c * u_c + mix_bias = sum_c mix_c * sum_k slope_ck * max(t_c, s_ck) + folded_bias
  // with folded_bias = mix_bias - sum_c mix_c * sum_k slope_ck * s_ck (computed in double).
  float folded_bias;
};

// HDRNetPointwiseNNGuide._guide (hdrnet/models.py:199-210) with the batch norm of conv1
// folded into w1/b1 on the host (inference form, hdrnet/bin/freeze_graph.py:141-142):
//   h_f = relu(sum_c x_c * w1[c][f] + b1[f]); guide = sigmoid(sum_f h_f * w2[f] + b2)
struct NNGuideParams {
  int feats;
  float w1[3][kMaxGuideFeats];
  float b1[kMaxGuideFeats];
  float w2[kMaxGuideFeats];
  float b2;
};

// The curves guide before its clip: returns a = sum_c mix_c * u_c + mix_bias and stores the
// colour-corrected t_c.  The guide VJP (guide_grad.cu) decides its masks [0 <= a <= 1] and
// [t_c > shift] from these very floats, so they agree with the forward pixel by pixel.
__device__ __forceinline__ float curves_guide_preclip(const CurvesGuideParams& p, float r, float g,
                                                      float b, float t[3]) {
  // One FMNMX and one FFMA per knot (vs FADD + FMNMX + FFMA each).
  float acc = p.folded_bias;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    t[c] = fmaf(b, p.ccm[2][c], fmaf(g, p.ccm[1][c], fmaf(r, p.ccm[0][c], p.ccm_bias[c])));
    unsigned long long u2 = 0ull;  // (0.0f, 0.0f)
#pragma unroll
    for (int k = 0; k < kCurvePts; k += 2) {
      const unsigned long long m2 = pack2(fmaxf(t[c], p.shifts[c][k]), fmaxf(t[c], p.shifts[c][k + 1]));
      u2 = fma2(pack2(p.slopes[c][k], p.slopes[c][k + 1]), m2, u2);
    }
    float u0, u1;
    unpack2(u2, u0, u1);
    acc = fmaf(p.mix[c], u0 + u1, acc);
  }
  return acc;
}

__device__ __forceinline__ float curves_guide(const CurvesGuideParams& p, float r, float g,
                                              float b) {
  float t[3];
  return fminf(fmaxf(curves_guide_preclip(p, r, g, b, t), 0.0f), 1.0f);
}

// The pointwise-NN guide in pieces, so that its VJP (guide_nn_grad.cu) recomputes the forward's
// own floats: nn_guide_preact2 is the pre-activation of features f and f + 1 (its relu masks),
// nn_guide_sigmoid the output from the two lanes of sum_f relu(h_f) w2_f.
__device__ __forceinline__ unsigned long long nn_guide_preact2(const NNGuideParams& p, unsigned long long r2,
                                                               unsigned long long g2, unsigned long long b2v,
                                                               int f) {
  unsigned long long h2 = fma2(r2, pack2(p.w1[0][f], p.w1[0][f + 1]), pack2(p.b1[f], p.b1[f + 1]));
  h2 = fma2(g2, pack2(p.w1[1][f], p.w1[1][f + 1]), h2);
  return fma2(b2v, pack2(p.w1[2][f], p.w1[2][f + 1]), h2);
}

__device__ __forceinline__ float nn_guide_sigmoid(const NNGuideParams& p, unsigned long long y2) {
  float y0, y1;
  unpack2(y2, y0, y1);
  const float y = (y0 + y1) + p.b2;
  return __fdividef(1.0f, 1.0f + __expf(-y));
}

// kFeats is a compile-time bound (16 or 32): the loop unrolls fully and every weight is a
// constant-bank operand with a static offset (a runtime feature count costs an indexed LDC per
// weight).  Weights beyond p.feats are zero (pack_nn_params), so the extra features add 0.
template <int kFeats>
__device__ __forceinline__ float nn_guide(const NNGuideParams& p, float r, float g, float b) {
  // Features in pairs (fma2); sigmoid through ex2.approx / rcp.approx: ~3e-7 absolute.
  const unsigned long long r2 = pack2(r, r), g2 = pack2(g, g), b2v = pack2(b, b);
  unsigned long long y2 = 0ull;
#pragma unroll
  for (int f = 0; f < kFeats; f += 2) {
    float h0, h1;
    unpack2(nn_guide_preact2(p, r2, g2, b2v, f), h0, h1);
    y2 = fma2(pack2(fmaxf(h0, 0.0f), fmaxf(h1, 0.0f)), pack2(p.w2[f], p.w2[f + 1]), y2);
  }
  return nn_guide_sigmoid(p, y2);
}

}  // namespace hdrnet_b200
