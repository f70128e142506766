// guide_grad.cu -- vector-Jacobian product of the curves guide (HDRNetCurves._guide,
// hdrnet/models.py:145-190; forward in guide.cuh): the gradients of its 112 variables and of the
// full-resolution RGB input, for training the guide with the rest of the model.
//
// Per pixel, with x the RGB input and g the upstream gradient of the guide:
//   t_c = sum_i x_i ccm[i][c] + ccm_bias[c],  u_c = sum_k slope_ck relu(t_c - s_ck),
//   a = sum_c mix_c u_c + mix_bias,  guide = clip(a, 0, 1)
//   g^ = g [0 <= a <= 1]                (clip_by_value / torch.clamp pass the gradient at equality)
//   u'_c = sum_k slope_ck [t_c > s_ck]  (TF's ReluGrad: 0 at t = s)
//   d mix_bias = g^,  d mix_c = g^ u_c,  d slope_ck = g^ mix_c relu(t_c - s_ck),
//   d s_ck = -g^ mix_c slope_ck [t_c > s_ck],  d ccm_bias_c = g^ mix_c u'_c,
//   d ccm[i][c] = x_i g^ mix_c u'_c,  dx_i = sum_c ccm[i][c] g^ mix_c u'_c
// t_c and a come from curves_guide_preclip, the forward's own arithmetic, so every mask is the
// one the forward's floats decide.
//
//   guide_grad_partial_kernel  one pass: reads x (12 B/px) and g (4 B/px), writes dx (12 B/px)
//                              when asked.  Each CTA sums the 112 parameter gradients over one
//                              fixed chunk of pixels (per thread in registers, then a fixed
//                              shuffle / shared-memory tree) into the caller's workspace.
//   guide_grad_reduce_kernel   adds the chunks in a fixed order (as wgrad_reduce_kernel does) and
//                              scales the shift sums by -slope.
// The chunk size depends on npix alone and there are no atomics, so a call gives the same bits on
// every run and every device.
#include <cuda_runtime.h>

#include <cstdint>

#include "guide.cuh"
#include "hdrnet_b200.h"

namespace hdrnet_b200 {

int pack_curves_params(CurvesGuideParams* p, const float* ccm, const float* ccm_bias,
                       const float* shifts, const float* slopes, const float* mix,
                       float mix_bias);

namespace {

// dparams layout (include/hdrnet_b200.h): ccm 9 ([in][out]), ccm_bias 3, shifts 48, slopes 48,
// mix 3, mix_bias 1.
constexpr int kOffCcm = 0, kOffCcmBias = 9, kOffShifts = 12, kOffSlopes = 60, kOffMix = 108,
              kOffMixBias = 111, kNumParams = 112;
constexpr int kThreads = 128;
constexpr int kMaxChunks = 1024;   // chunks grow with npix beyond kMaxChunks * 512 pixels

// Pixels per chunk: a multiple of 4 * kThreads (whole quads per thread), from npix alone.
long long chunk_pixels(long long npix) {
  const long long base = 4LL * kThreads;
  long long q = (npix + base * kMaxChunks - 1) / (base * kMaxChunks);
  if (q < 1) q = 1;
  return base * q;
}

long long num_chunks(long long npix) {
  const long long cp = chunk_pixels(npix);
  return (npix + cp - 1) / cp;
}

// Accumulators of the CTAs of channel C (blockIdx.y): ccm[0..2][C], ccm_bias[C], the 16 shift
// sums (sum g^ mix_C [t_C > s_Ck]; the reduce kernel scales them by -slope_Ck), the 16 slopes,
// mix[C], and for C == 0 mix_bias.  37 or 38 registers instead of 112: no spills.
constexpr int kAccCcm = 0, kAccCcmBias = 3, kAccShifts = 4, kAccSlopes = 20, kAccMix = 36,
              kAccMixBias = 37, kNumAcc = 38;

__device__ __forceinline__ int acc_offset(int C, int j) {
  if (j < kAccCcmBias) return kOffCcm + j * 3 + C;
  if (j == kAccCcmBias) return kOffCcmBias + C;
  if (j < kAccSlopes) return kOffShifts + C * kCurvePts + (j - kAccShifts);
  if (j < kAccMix) return kOffSlopes + C * kCurvePts + (j - kAccSlopes);
  if (j == kAccMix) return kOffMix + C;
  return kOffMixBias;
}

// u'_c = sum_k slope_ck [t_c > s_ck]
__device__ __forceinline__ float curve_slope(const CurvesGuideParams& p, int c, float t) {
  float up = 0.0f;
#pragma unroll
  for (int k = 0; k < kCurvePts; ++k) up += t > p.shifts[c][k] ? p.slopes[c][k] : 0.0f;
  return up;
}

// One pixel: channel C's parameter gradients into acc (kParams); dx over all channels (kDx).
template <int C, bool kDx, bool kParams>
__device__ __forceinline__ void pixel_vjp(const CurvesGuideParams& p, float x0, float x1, float x2,
                                          float g, float (&acc)[kNumAcc], float& dx0,
                                          float& dx1, float& dx2) {
  float t[3];
  const float a = curves_guide_preclip(p, x0, x1, x2, t);
  const float gh = (a >= 0.0f && a <= 1.0f) ? g : 0.0f;
  if (kParams) {
    const float gc = gh * p.mix[C];
    float u = 0.0f, up = 0.0f;
#pragma unroll
    for (int k = 0; k < kCurvePts; ++k) {
      const bool on = t[C] > p.shifts[C][k];
      const float r = fmaxf(t[C] - p.shifts[C][k], 0.0f);
      up += on ? p.slopes[C][k] : 0.0f;
      u = fmaf(p.slopes[C][k], r, u);
      acc[kAccSlopes + k] = fmaf(gc, r, acc[kAccSlopes + k]);
      acc[kAccShifts + k] += on ? gc : 0.0f;
    }
    const float w = gc * up;
    acc[kAccMix] = fmaf(gh, u, acc[kAccMix]);
    acc[kAccCcmBias] += w;
    acc[kAccCcm + 0] = fmaf(x0, w, acc[kAccCcm + 0]);
    acc[kAccCcm + 1] = fmaf(x1, w, acc[kAccCcm + 1]);
    acc[kAccCcm + 2] = fmaf(x2, w, acc[kAccCcm + 2]);
    if (C == 0) acc[kAccMixBias] += gh;
  }
  if (kDx) {
    dx0 = dx1 = dx2 = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float w = gh * p.mix[c] * curve_slope(p, c, t[c]);
      dx0 = fmaf(p.ccm[0][c], w, dx0);
      dx1 = fmaf(p.ccm[1][c], w, dx1);
      dx2 = fmaf(p.ccm[2][c], w, dx2);
    }
  }
}

template <int C, bool kDx, bool kParams>
__device__ __forceinline__ void chunk_vjp(const float* __restrict__ x, const float* __restrict__ dguide,
                                          float* __restrict__ dx, float* __restrict__ ws,
                                          long long npix, long long chunk_px, bool vec_ok,
                                          const CurvesGuideParams& p) {
  float acc[kNumAcc];
#pragma unroll
  for (int i = 0; i < kNumAcc; ++i) acc[i] = 0.0f;
  const long long p0 = static_cast<long long>(blockIdx.x) * chunk_px;
  const long long p1 = p0 + chunk_px < npix ? p0 + chunk_px : npix;
  long long scalar0 = p0;
  if (vec_ok) {
    // whole quads of this chunk: chunk_px is a multiple of 4, so only the last chunk has a tail
    const long long q0 = p0 / 4, q1 = p1 / 4;
    for (long long q = q0 + threadIdx.x; q < q1; q += kThreads) {
      const float4* in4 = reinterpret_cast<const float4*>(x) + 3 * q;
      const float4 c0 = __ldg(in4), c1 = __ldg(in4 + 1), c2 = __ldg(in4 + 2);
      const float4 g = __ldg(reinterpret_cast<const float4*>(dguide) + q);
      float4 o0, o1, o2;
      pixel_vjp<C, kDx, kParams>(p, c0.x, c0.y, c0.z, g.x, acc, o0.x, o0.y, o0.z);
      pixel_vjp<C, kDx, kParams>(p, c0.w, c1.x, c1.y, g.y, acc, o0.w, o1.x, o1.y);
      pixel_vjp<C, kDx, kParams>(p, c1.z, c1.w, c2.x, g.z, acc, o1.z, o1.w, o2.x);
      pixel_vjp<C, kDx, kParams>(p, c2.y, c2.z, c2.w, g.w, acc, o2.y, o2.z, o2.w);
      if (kDx) {
        float4* out4 = reinterpret_cast<float4*>(dx) + 3 * q;
        out4[0] = o0;
        out4[1] = o1;
        out4[2] = o2;
      }
    }
    scalar0 = q1 * 4;
  }
  // the tail (npix % 4), or the whole chunk when a buffer is not 16-byte aligned
  for (long long i = scalar0 + threadIdx.x; i < p1; i += kThreads) {
    float d0, d1, d2;
    pixel_vjp<C, kDx, kParams>(p, __ldg(x + 3 * i), __ldg(x + 3 * i + 1), __ldg(x + 3 * i + 2),
                               __ldg(dguide + i), acc, d0, d1, d2);
    if (kDx) {
      dx[3 * i] = d0;
      dx[3 * i + 1] = d1;
      dx[3 * i + 2] = d2;
    }
  }
  if (!kParams) return;
  // CTA sum in a fixed order: xor tree within each warp, then the warps in order.
  constexpr int kN = C == 0 ? kNumAcc : kNumAcc - 1;
  __shared__ float warp_sums[kThreads / 32][kNumAcc];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kN; ++i) {
    float s = acc[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) warp_sums[warp][i] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kN; i += kThreads) {
    float s = warp_sums[0][i];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) s += warp_sums[w][i];
    ws[static_cast<size_t>(blockIdx.x) * kNumParams + acc_offset(C, i)] = s;
  }
}

// blockIdx.y = the channel whose parameter gradients the CTA sums; the channel-0 CTAs also write
// dx.  Every CTA recomputes the whole forward of its pixels (a needs all three channels).
template <bool kDx, bool kParams>
__global__ void __launch_bounds__(kThreads)
guide_grad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dguide,
                          float* __restrict__ dx, float* __restrict__ ws, long long npix,
                          long long chunk_px, bool vec_ok, const __grid_constant__ CurvesGuideParams p) {
  if (blockIdx.y == 0) chunk_vjp<0, kDx, kParams>(x, dguide, dx, ws, npix, chunk_px, vec_ok, p);
  else if (blockIdx.y == 1) chunk_vjp<1, false, kParams>(x, dguide, dx, ws, npix, chunk_px, vec_ok, p);
  else chunk_vjp<2, false, kParams>(x, dguide, dx, ws, npix, chunk_px, vec_ok, p);
}

// One warp per parameter: lane l sums chunks l, l + 32, ... in order, then a fixed xor tree.
__global__ void __launch_bounds__(256)
guide_grad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dparams, int chunks,
                         const __grid_constant__ CurvesGuideParams p) {
  const int e = static_cast<int>((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (e >= kNumParams) return;
  float s = 0.0f;
  for (int c = lane; c < chunks; c += 32) s += ws[static_cast<size_t>(c) * kNumParams + e];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) {
    if (e >= kOffShifts && e < kOffSlopes) {
      const int c = (e - kOffShifts) / kCurvePts, k = (e - kOffShifts) % kCurvePts;
      s *= -p.slopes[c][k];
    }
    dparams[e] = s;
  }
}

template <bool kDx, bool kParams>
void launch_partial(const float* x, const float* dguide, float* dx, float* ws, long long npix,
                    bool vec_ok, const CurvesGuideParams& p, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>(num_chunks(npix)), kParams ? 3 : 1);
  guide_grad_partial_kernel<kDx, kParams><<<grid, kThreads, 0, st>>>(
      x, dguide, dx, ws, npix, chunk_pixels(npix), vec_ok, p);
}

}  // namespace
}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_guide_curves_grad_workspace_bytes(long long npix) {
  if (npix <= 0) return 0;
  return static_cast<size_t>(num_chunks(npix)) * kNumParams * sizeof(float);
}

int hdrnet_guide_curves_grad_f32(const float* input, const float* dguide, float* dinput,
                                 long long npix, const float* ccm, const float* ccm_bias,
                                 const float* shifts, const float* slopes, const float* mix,
                                 float mix_bias, float* dparams, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  CurvesGuideParams p;
  const int rc = pack_curves_params(&p, ccm, ccm_bias, shifts, slopes, mix, mix_bias);
  if (rc != HDRNET_OK) return rc;
  if (npix < 0) return HDRNET_E_BAD_SHAPE;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (npix == 0) {   // nothing to sum: the parameter gradients are zero
    if (dparams) return static_cast<int>(cudaMemsetAsync(dparams, 0, kNumParams * sizeof(float), st));
    return HDRNET_OK;
  }
  if (!dinput && !dparams) return HDRNET_OK;
  if (!input || !dguide) return HDRNET_E_NULL_POINTER;
  if (dparams) {
    if (!workspace) return HDRNET_E_NULL_POINTER;
    if (workspace_bytes < hdrnet_guide_curves_grad_workspace_bytes(npix)) return HDRNET_E_BAD_SHAPE;
  }
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(input) | reinterpret_cast<uintptr_t>(dguide) |
                        reinterpret_cast<uintptr_t>(dinput)) & 15u) == 0;
  float* ws = static_cast<float*>(workspace);
  if (dinput && dparams) launch_partial<true, true>(input, dguide, dinput, ws, npix, vec_ok, p, st);
  else if (dinput) launch_partial<true, false>(input, dguide, dinput, ws, npix, vec_ok, p, st);
  else launch_partial<false, true>(input, dguide, dinput, ws, npix, vec_ok, p, st);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || !dparams) return static_cast<int>(e);
  guide_grad_reduce_kernel<<<(kNumParams * 32 + 255) / 256, 256, 0, st>>>(
      ws, dparams, static_cast<int>(num_chunks(npix)), p);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
