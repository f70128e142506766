// slice_grad.cu -- vector-Jacobian products of bilateral_slice / bilateral_slice_apply
// (SURVEY.md section 8f rank 1).  Replaces the six backward kernels of the reference:
//   hdrnet/ops/bilateral_slice_apply.cu.cc:128-364 (grid / guide / input VJP), launchers :384-417
//   hdrnet/ops/bilateral_slice.cu.cc:93-227       (grid / guide VJP),        launchers :246-272
// with two kernels, each serving both ops (slice == slice-apply with in' = 1 and c = i*J+j):
//
//   slice_grad_pixel_kernel  one thread per pixel: ONE 8-corner gather yields both the sliced
//                            coefficients (-> input VJP) and their depth derivative (-> guide
//                            VJP); the reference runs two kernels that each redo the gather.
//   slice_grad_grid_kernel   one CTA per grid (b, gy, gx) column.  The reference gathers per
//                            OUTPUT ELEMENT (gd*gc threads re-walk the same ~2W/gw x 2H/gh
//                            pixel footprint, 8x of them hitting zero depth weights); here the
//                            footprint is walked once per column, every thread keeps the whole
//                            [gd][gc] column in registers (static indices, predicated depth
//                            weights), and one deterministic block reduction writes it out.
//                            No atomics: results are bitwise reproducible.
//
// Semantics follow the reference's CPU loops exactly (hdrnet/ops/bilateral_slice_apply.cc:
// 84-259, bilateral_slice.cc:72-168): mirror boundary for the footprint, wz forced to 1 at the
// depth borders, dwz = gd * SmoothedLerpWeightGrad.  Checked against the compiled reference.
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"

namespace hdrnet_b200 {

// numerics.h:83-91, :108-126 with dx = (gz + 0.5) - gzf.  The guide VJP sums derivatives of
// opposite sign (two depth corners), so these follow the reference operation for operation --
// x*x + eps WITHOUT fusing, IEEE sqrt and division -- instead of the forward's fast forms:
// a 1-ulp difference here survives the cancellation as a 1e-4-relative error.
__device__ __forceinline__ float smoothed_abs(float dx) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), 1.0e-8f));
}
__device__ __forceinline__ float smoothed_lerp_weight_grad(float dx) {
  const float a = smoothed_abs(dx);
  return (a > 1.0f) ? 0.0f : __fdiv_rn(dx, a);
}
__device__ __forceinline__ float smoothed_lerp_weight(float dx) {
  return fmaxf(__fsub_rn(1.0f, smoothed_abs(dx)), 0.0f);
}
__device__ __forceinline__ int mirror_boundary(int x, int extent) {  // numerics.h:72-80
  return x < 0 ? -x - 1 : (x >= extent ? 2 * extent - 1 - x : x);
}

struct GradGeom {
  int B, H, W, gh, gw, gd;
  int n_in, n_out, J;   // slice mode: n_in = 0, n_out = gc, J = 1
  int apply;            // 1 = slice-apply, 0 = slice
};

// ---- per-pixel VJPs: guide (and input) -----------------------------------------------------
__global__ void __launch_bounds__(256)
slice_grad_pixel_kernel(const float* __restrict__ grid, const float* __restrict__ guide,
                        const float* __restrict__ input, const float* __restrict__ ct,
                        float* __restrict__ guide_vjp, float* __restrict__ input_vjp, GradGeom g,
                        long long npix) {
  const int gc = g.n_out * g.J;
  const float scale_x = static_cast<float>(g.gw) / g.W;
  const float scale_y = static_cast<float>(g.gh) / g.H;
  const long long grid_image = static_cast<long long>(g.gh) * g.gw * g.gd * gc;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < npix;
       p += stride) {
    const int x = static_cast<int>(p % g.W);
    const int y = static_cast<int>((p / g.W) % g.H);
    const int b = static_cast<int>(p / (static_cast<long long>(g.W) * g.H));
    const Axis ax = spatial_axis(x, scale_x);
    const Axis ay = spatial_axis(y, scale_y);
    const float gzf = __fmul_rn(__ldg(guide + p), static_cast<float>(g.gd));
    const int gz0 = static_cast<int>(floorf(__fsub_rn(gzf, 0.5f)));
    int off[8];
    float w[8], dw[8];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int gyc = clampi(ay.i0 + dy, 0, g.gh - 1);
      const float wy = dy ? ay.f : 1.0f - ay.f;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int gxc = clampi(ax.i0 + dx, 0, g.gw - 1);
        const float wxy = (dx ? ax.f : 1.0f - ax.f) * wy;
#pragma unroll
        for (int dz = 0; dz < 2; ++dz) {
          const int gz = gz0 + dz;
          const float d = (gz + 0.5f) - gzf;
          const int k = dy * 4 + dx * 2 + dz;
          off[k] = ((gyc * g.gw + gxc) * g.gd + clampi(gz, 0, g.gd - 1)) * gc;
          w[k] = wxy * smoothed_lerp_weight(d);
          dw[k] = wxy * (g.gd * smoothed_lerp_weight_grad(d));
        }
      }
    }
    const float* grid_b = grid + b * grid_image;
    const float* ctp = ct + p * g.n_out;
    float gvjp = 0.0f;
    if (g.apply) {
      const float* inp = input + p * g.n_in;
      for (int j = 0; j < g.n_in; ++j) input_vjp[p * g.n_in + j] = 0.0f;
      for (int i = 0; i < g.n_out; ++i) {
        const float cti = __ldg(ctp + i);
        float dsum = 0.0f;
        for (int j = 0; j < g.J; ++j) {
          float s = 0.0f, ds = 0.0f;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float v = __ldg(grid_b + off[k] + i * g.J + j);
            s = fmaf(w[k], v, s);
            ds = __fadd_rn(ds, __fmul_rn(dw[k], v));  // as the reference: no fusing (cancellation)
          }
          const float iv = (j < g.n_in) ? __ldg(inp + j) : 1.0f;
          dsum = fmaf(ds, iv, dsum);
          if (j < g.n_in) input_vjp[p * g.n_in + j] += s * cti;
        }
        gvjp = fmaf(dsum, cti, gvjp);
      }
    } else {
      for (int c = 0; c < gc; ++c) {
        float ds = 0.0f;
#pragma unroll
        for (int k = 0; k < 8; ++k) ds = __fadd_rn(ds, __fmul_rn(dw[k], __ldg(grid_b + off[k] + c)));
        gvjp = fmaf(ds, __ldg(ctp + c), gvjp);
      }
    }
    guide_vjp[p] = gvjp;
  }
}

// ---- grid VJP ----------------------------------------------------------------------------------
constexpr int kGgThreads = 256;
constexpr int kGgMaxGd = 8;
constexpr int kGgMaxGc = 12;

// Accumulates a pixel's contribution into the per-thread [gd][gc] column.
template <int GC>
__device__ __forceinline__ void accumulate_column(float (&acc)[kGgMaxGd][GC], const float (&v)[GC],
                                                  float wxy, float gzf, int gd) {
#pragma unroll
  for (int gz = 0; gz < kGgMaxGd; ++gz) {
    if (gz < gd) {
      float wz = smoothed_lerp_weight((gz + 0.5f) - gzf);
      // border override (bilateral_slice_apply.cc:115-118): both depth corners clamp here
      if ((gz == 0 && gzf < 0.5f) || (gz == gd - 1 && gzf > gd - 0.5f)) wz = 1.0f;
      const float wgt = wxy * wz;
#pragma unroll
      for (int c = 0; c < GC; ++c) acc[gz][c] = fmaf(wgt, v[c], acc[gz][c]);
    }
  }
}

template <int GC>
__global__ void __launch_bounds__(kGgThreads)
slice_grad_grid_kernel(const float* __restrict__ guide, const float* __restrict__ input,
                       const float* __restrict__ ct, float* __restrict__ grid_vjp, GradGeom g) {
  __shared__ float red[kGgThreads / 32][kGgMaxGd * GC];
  const int gc = g.n_out * g.J;  // == GC or smaller (padded channels stay zero)
  const int col = blockIdx.x;    // (b, gy, gx)
  const int gx = col % g.gw;
  const int gy = (col / g.gw) % g.gh;
  const int b = col / (g.gw * g.gh);
  const float scale_x = static_cast<float>(g.W) / g.gw;   // note: pixels per cell here
  const float scale_y = static_cast<float>(g.H) / g.gh;
  const int x0 = static_cast<int>(floorf(scale_x * (gx + 0.5f - 1.0f)));
  const int x1e = static_cast<int>(ceilf(scale_x * (gx + 0.5f + 1.0f)));
  const int y0 = static_cast<int>(floorf(scale_y * (gy + 0.5f - 1.0f)));
  const int y1e = static_cast<int>(ceilf(scale_y * (gy + 0.5f + 1.0f)));
  const int fw = x1e - x0, fh = y1e - y0;

  float acc[kGgMaxGd][GC];
#pragma unroll
  for (int z = 0; z < kGgMaxGd; ++z)
#pragma unroll
    for (int c = 0; c < GC; ++c) acc[z][c] = 0.0f;

  const long long img = static_cast<long long>(b) * g.H * g.W;
  for (int e = threadIdx.x; e < fw * fh; e += kGgThreads) {
    const int yy = y0 + e / fw, xx = x0 + e % fw;
    const float gyf = (yy + 0.5f) / scale_y;
    const float gxf = (xx + 0.5f) / scale_x;
    const float wy = fmaxf(1.0f - fabsf((gy + 0.5f) - gyf), 0.0f);
    const float wx = fmaxf(1.0f - fabsf((gx + 0.5f) - gxf), 0.0f);
    const float wxy = wx * wy;
    if (wxy == 0.0f) continue;
    const long long p = img + static_cast<long long>(mirror_boundary(yy, g.H)) * g.W +
                        mirror_boundary(xx, g.W);
    const float gzf = __ldg(guide + p) * g.gd;
    float v[GC];
    if (g.apply) {
#pragma unroll
      for (int c = 0; c < GC; ++c) {
        const int i = c / g.J, j = c - i * g.J;
        v[c] = (c < gc) ? ((j < g.n_in ? __ldg(input + p * g.n_in + j) : 1.0f) * __ldg(ct + p * g.n_out + i))
                        : 0.0f;
      }
    } else {
#pragma unroll
      for (int c = 0; c < GC; ++c) v[c] = (c < gc) ? __ldg(ct + p * gc + c) : 0.0f;
    }
    accumulate_column<GC>(acc, v, wxy, gzf, g.gd);
  }

  // Deterministic block reduction: warp shuffle tree, then a fixed-order sum over warps.
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int z = 0; z < kGgMaxGd; ++z)
#pragma unroll
    for (int c = 0; c < GC; ++c) {
      float s = acc[z][c];
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
      if (lane == 0) red[warp][z * GC + c] = s;
    }
  __syncthreads();
  for (int e = threadIdx.x; e < g.gd * gc; e += kGgThreads) {
    const int z = e / gc, c = e - z * gc;
    float s = 0.0f;
#pragma unroll
    for (int w = 0; w < kGgThreads / 32; ++w) s += red[w][z * GC + c];
    grid_vjp[(static_cast<size_t>(col) * g.gd + z) * gc + c] = s;
  }
}

// Any gd / gc: one thread per output element, the reference's own formulation
// (bilateral_slice_apply.cu.cc:128-206).
__global__ void __launch_bounds__(128)
slice_grad_grid_generic_kernel(const float* __restrict__ guide, const float* __restrict__ input,
                               const float* __restrict__ ct, float* __restrict__ grid_vjp,
                               GradGeom g, long long nelem) {
  const int gc = g.n_out * g.J;
  const float scale_x = static_cast<float>(g.W) / g.gw;
  const float scale_y = static_cast<float>(g.H) / g.gh;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < nelem;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(e % gc);
    const int gz = static_cast<int>((e / gc) % g.gd);
    const int gx = static_cast<int>((e / (static_cast<long long>(gc) * g.gd)) % g.gw);
    const int gy = static_cast<int>((e / (static_cast<long long>(gc) * g.gd * g.gw)) % g.gh);
    const int b = static_cast<int>(e / (static_cast<long long>(gc) * g.gd * g.gw * g.gh));
    const int i = c / g.J, j = c - i * g.J;
    const int x0 = static_cast<int>(floorf(scale_x * (gx + 0.5f - 1.0f)));
    const int x1e = static_cast<int>(ceilf(scale_x * (gx + 0.5f + 1.0f)));
    const int y0 = static_cast<int>(floorf(scale_y * (gy + 0.5f - 1.0f)));
    const int y1e = static_cast<int>(ceilf(scale_y * (gy + 0.5f + 1.0f)));
    float s = 0.0f;
    for (int yy = y0; yy < y1e; ++yy) {
      const int ym = mirror_boundary(yy, g.H);
      const float wy = fmaxf(1.0f - fabsf((gy + 0.5f) - (yy + 0.5f) / scale_y), 0.0f);
      for (int xx = x0; xx < x1e; ++xx) {
        const int xm = mirror_boundary(xx, g.W);
        const float wx = fmaxf(1.0f - fabsf((gx + 0.5f) - (xx + 0.5f) / scale_x), 0.0f);
        const long long p = (static_cast<long long>(b) * g.H + ym) * g.W + xm;
        const float gzf = __ldg(guide + p) * g.gd;
        float wz = smoothed_lerp_weight((gz + 0.5f) - gzf);
        if ((gz == 0 && gzf < 0.5f) || (gz == g.gd - 1 && gzf > g.gd - 0.5f)) wz = 1.0f;
        float v;
        if (g.apply)
          v = (j < g.n_in ? __ldg(input + p * g.n_in + j) : 1.0f) * __ldg(ct + p * g.n_out + i);
        else
          v = __ldg(ct + p * gc + c);
        s = fmaf(wx * wy * wz, v, s);
      }
    }
    grid_vjp[e] = s;
  }
}

static int launch_grads(const float* grid, const float* guide, const float* input, const float* ct,
                        float* grid_vjp, float* guide_vjp, float* input_vjp, const GradGeom& g,
                        cudaStream_t stream) {
  const long long npix = static_cast<long long>(g.B) * g.H * g.W;
  if (npix == 0) return HDRNET_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int gc = g.n_out * g.J;
  long long blocks = (npix + 255) / 256;
  if (blocks > static_cast<long long>(sms) * 16) blocks = static_cast<long long>(sms) * 16;
  slice_grad_pixel_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      grid, guide, input, ct, guide_vjp, input_vjp, g, npix);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long cols = static_cast<long long>(g.B) * g.gh * g.gw;
  if (g.gd <= kGgMaxGd && gc <= kGgMaxGc) {
    slice_grad_grid_kernel<kGgMaxGc><<<static_cast<unsigned>(cols), kGgThreads, 0, stream>>>(
        guide, input, ct, grid_vjp, g);
  } else {
    const long long nelem = cols * g.gd * gc;
    long long gb = (nelem + 127) / 128;
    if (gb > static_cast<long long>(sms) * 32) gb = static_cast<long long>(sms) * 32;
    slice_grad_grid_generic_kernel<<<static_cast<unsigned>(gb), 128, 0, stream>>>(
        guide, input, ct, grid_vjp, g, nelem);
  }
  return static_cast<int>(cudaGetLastError());
}

}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

int hdrnet_slice_apply_grad_f32(const float* grid, const float* guide, const float* input,
                                const float* codomain_tangent, float* grid_vjp, float* guide_vjp,
                                float* input_vjp, int B, int H, int W, int gh, int gw, int gd,
                                int n_in, int n_out, int has_offset, void* stream) {
  if (B < 0 || H < 0 || W < 0 || gh < 1 || gw < 1 || gd < 1 || n_in < 1 || n_out < 1)
    return HDRNET_E_BAD_SHAPE;
  if (static_cast<long long>(B) * H * W == 0) {
    // no pixels: the pixel-shaped VJPs are empty, but the grid VJP is a full tensor of zeros when
    // B > 0 (the reference's kernels write 0 for a cell without a footprint)
    const size_t n = static_cast<size_t>(B) * gh * gw * gd * n_out * (n_in + (has_offset ? 1 : 0));
    if (n == 0) return HDRNET_OK;
    if (!grid_vjp) return HDRNET_E_NULL_POINTER;
    return static_cast<int>(cudaMemsetAsync(grid_vjp, 0, n * sizeof(float), static_cast<cudaStream_t>(stream)));
  }
  if (!grid || !guide || !input || !codomain_tangent || !grid_vjp || !guide_vjp || !input_vjp)
    return HDRNET_E_NULL_POINTER;
  GradGeom g{B, H, W, gh, gw, gd, n_in, n_out, n_in + (has_offset ? 1 : 0), 1};
  return launch_grads(grid, guide, input, codomain_tangent, grid_vjp, guide_vjp, input_vjp, g,
                      static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_grad_f32(const float* grid, const float* guide, const float* codomain_tangent,
                          float* grid_vjp, float* guide_vjp, int B, int H, int W, int gh, int gw,
                          int gd, int gc, void* stream) {
  if (B < 0 || H < 0 || W < 0 || gh < 1 || gw < 1 || gd < 1 || gc < 1) return HDRNET_E_BAD_SHAPE;
  if (static_cast<long long>(B) * H * W == 0) {
    const size_t n = static_cast<size_t>(B) * gh * gw * gd * gc;
    if (n == 0) return HDRNET_OK;
    if (!grid_vjp) return HDRNET_E_NULL_POINTER;
    return static_cast<int>(cudaMemsetAsync(grid_vjp, 0, n * sizeof(float), static_cast<cudaStream_t>(stream)));
  }
  if (!grid || !guide || !codomain_tangent || !grid_vjp || !guide_vjp) return HDRNET_E_NULL_POINTER;
  GradGeom g{B, H, W, gh, gw, gd, 0, gc, 1, 0};
  return launch_grads(grid, guide, nullptr, codomain_tangent, grid_vjp, guide_vjp, nullptr, g,
                      static_cast<cudaStream_t>(stream));
}

}  // extern "C"
