// slice_apply.cu -- fused BilateralSliceApply for H100 (sm_90a), plus the generic
// any-shape slice / slice-apply kernel and the cell-index debug kernel.
//
// Replaces hdrnet/ops/bilateral_slice_apply.cu.cc:36-126 (BilateralSliceApplyKernel, one
// thread per OUTPUT ELEMENT, 32 scalar grid loads each, no shared memory) with a design
// built around what bounds the op: 28 B of HBM traffic per pixel against ~250 fp32 lane
// operations per pixel at the HBM roofline (132 SMs x 128 lanes x ~1.8 GHz over 3.35 TB/s / 28 B;
// DESIGN.md section 3).
//
// slice_apply_rows_tma_kernel -- persistent, one CTA per resident slot:
//   * every HBM byte moves through the TMA engine: 1-D bulk copies (cp.async.bulk ->
//     UBLKCP) bring a row segment's RGB (12 B/px) and guide (4 B/px) into a multi-stage
//     shared-memory ring, completion on mbarriers; results are written IN PLACE over the
//     RGB tile and leave with one bulk store per segment.  No LDG/STG address arithmetic
//     in the math warps, perfectly coalesced traffic whatever the per-thread access shape.
//   * the grid rows a pixel row touches (gy0, gy0+1: gw*gd*12 floats each) are staged once
//     by TMA and stay resident while consecutive rows share them; per image row they are
//     pre-blended along y (wy is constant on a row) into a slab Gy[gx][gz][12], so a pixel
//     blends 4 corners instead of 8: 48 FMAs instead of 96, + 9 for
//     the affine apply.
//   * one thread owns 4 consecutive pixels: 3 LDS.128 of RGB + 1 LDS.128 of guide, 12
//     16-byte slab chunks per pixel (conflict-free within an x cell: its 8 depth cells map to
//     disjoint 4-bank groups), 3 STS.128 of output.
//   * the kernel is bound by the shared-memory data pipe (ncu), so its texture-assisted form
//     (template parameter kTexChunks, HDRNET_VARIANT_TEX) reads the y-pre-blended slab rows
//     from a pre-pass workspace and serves 4 of the 12 chunks through the texture pipe -- the
//     only on-chip gather path that does not share the LSU crossbar (DESIGN.md section 3).
//   * template parameter GuideFn fuses the curves / pointwise-NN guide (model path, 24 B/px).
// slice_rows_tma_kernel is the un-fused bilateral_slice on the same plan (write-bound).
//
// Files: slice_rows.cuh (device code shared by the row kernels: tile accessors, 4-corner blend,
// guide sources, plan / argument structs), this file (generic kernels, the block-synchronous row
// kernel, the un-fused slice kernel, the y pre-pass, planning, kernel selection, C-ABI),
// slice_apply_async.cu (issuer-warp form: what AUTO runs for large images with a workspace).
// Forms that measured slower (z-bucketed, texture-fed input, producer-warp, tensor-core gather
// forms) are not part of the library.
#include <cuda_runtime.h>

#include <atomic>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <mutex>
#include <new>
#include <vector>

#include "slice_rows.cuh"

namespace hdrnet_b200 {

// =========================================================================================
// Generic kernels: one thread per pixel, any n_in / n_out / alignment / width.
// =========================================================================================

// Corners / make_corners / sample: slice_rows.cuh.
// kApply = true : out[p, i] = sum_j sample(i*J + j) * (j < n_in ? input[p, j] : 1)
// kApply = false: out[p, c] = sample(c), c < gc
template <bool kApply>
__global__ void __launch_bounds__(256)
slice_generic_kernel(const float* __restrict__ grid, const float* __restrict__ guide,
                     const float* __restrict__ input, float* __restrict__ out, SliceGeom g,
                     int n_in, int n_out, int J, long long npix) {
  const int gc = kApply ? n_out * J : J;
  const long long grid_image = static_cast<long long>(g.gh) * g.gw * g.gd * gc;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < npix;
       p += stride) {
    const int x = static_cast<int>(p % g.W);
    const long long row = p / g.W;
    const int r = static_cast<int>(row % g.rows);
    const int b = static_cast<int>(row / g.rows);
    const Corners c = make_corners(g, x, g.y_off + r, __ldg(guide + p), gc);
    const float* grid_b = grid + b * grid_image;
    if (kApply) {
      for (int i = 0; i < n_out; ++i) {
        float value = 0.0f;
        for (int j = 0; j < J; ++j) {
          const float s = sample(grid_b, c, i * J + j);
          value = (j < n_in) ? fmaf(s, __ldg(input + p * n_in + j), value) : value + s;
        }
        out[p * n_out + i] = value;
      }
    } else {
      for (int ch = 0; ch < gc; ++ch) out[p * gc + ch] = sample(grid_b, c, ch);
    }
  }
}

// =========================================================================================
// Any-shape ROW kernel: the row kernels' organisation without their alignment contract.
// =========================================================================================
// The TMA row kernels take the 3 -> 3 affine op with offset on 16-byte aligned rows (W % 4 == 0);
// everything else -- has_offset = False (ops_test.py:345-365), other n_in / n_out
// (HDRNetGaussianPyrNN's 9 x 4 grids sliced directly, hdrnet_ops_test.py:91-100), odd widths,
// unaligned views, and the un-fused slice with gc != 12 -- used to fall to slice_generic_kernel:
// 8 corners x gc scalar L2 loads per pixel.
// This kernel keeps what makes the row kernels fast and drops only the bulk copies: a persistent
// CTA owns contiguous rows; the two grid rows a pixel row touches are staged in shared memory
// (plain loads, reloaded only when the row pair changes) and pre-blended along y into a slab
// [gw][gd][gc], so a pixel gathers 4 corners from shared memory instead of 8 from L2; pixels are
// one per thread with plain (coalesced, any alignment) global loads / stores.
constexpr int kAnyThreads = 256;

struct AnyArgs {
  const float* grid;
  const float* guide;
  const float* input;   // kApply only
  float* out;
  SliceGeom g;
  int n_in, n_out, J, gc;   // kApply: gc = n_out * J;  slice: gc channels, n_out = gc
  int row_floats;           // gw * gd * gc
};

// kGc > 0: the channel counts are compile-time (kGc grid channels; kApply: kIn inputs, kOut
// outputs, offset when kGc == kOut * (kIn + 1)).  The slab then pads each cell to a multiple of 4
// floats, a corner is kGc / 4 128-bit shared loads instead of kGc scalar ones, and the affine
// apply runs out of registers.  kGc == 0: any counts at run time (scalar loads).  Same order of
// floating-point operations in both.
template <bool kApply, int kGc, int kIn, int kOut>
__global__ void __launch_bounds__(kAnyThreads, 4)
slice_rows_any_kernel(const AnyArgs a) {
  extern __shared__ __align__(16) float sm_any[];
  const SliceGeom& g = a.g;
  constexpr int kGcp = (kGc + 3) / 4 * 4;            // padded cell stride of the slab (kGc > 0)
  const int gc = kGc > 0 ? kGc : a.gc;
  const int cell_stride = kGc > 0 ? kGcp : a.gc;
  const int cells = g.gw * g.gd;
  float* raw0 = sm_any;
  float* raw1 = raw0 + ((a.row_floats + 3) & ~3);
  float* slab = raw1 + ((a.row_floats + 3) & ~3);
  const int tid = threadIdx.x;
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  const long long r_begin = total_rows * blockIdx.x / gridDim.x;
  const long long r_end = total_rows * (blockIdx.x + 1) / gridDim.x;
  const float gd_f = static_cast<float>(g.gd);
  const int x_stride = g.gd * cell_stride;
  const bool out_vec = (reinterpret_cast<uintptr_t>(a.out) & 15u) == 0;
  int cur_b = -1, cur_gy0 = INT_MIN;
  for (long long row = r_begin; row < r_end; ++row) {
    const int b = static_cast<int>(row / g.rows);
    const int y = g.y_off + static_cast<int>(row - static_cast<long long>(b) * g.rows);
    const Axis ay = spatial_axis(y, g.scale_y);
    __syncthreads();   // the previous row's pixels are done with the slab
    if (b != cur_b || ay.i0 != cur_gy0) {
      const float* gb = a.grid + static_cast<size_t>(b) * g.gh * a.row_floats;
      const float* r0 = gb + static_cast<size_t>(clampi(ay.i0, 0, g.gh - 1)) * a.row_floats;
      const float* r1 = gb + static_cast<size_t>(clampi(ay.i0 + 1, 0, g.gh - 1)) * a.row_floats;
      for (int e = tid; e < a.row_floats; e += kAnyThreads) { raw0[e] = __ldg(r0 + e); raw1[e] = __ldg(r1 + e); }
      cur_b = b;
      cur_gy0 = ay.i0;
      __syncthreads();
    }
    const float wy1 = ay.f, wy0 = 1.0f - ay.f;
    if constexpr (kGc > 0 && kGcp != kGc) {
      for (int e = tid; e < cells * kGcp; e += kAnyThreads) {
        const int cell = e / kGcp, ch = e - cell * kGcp;
        slab[e] = ch < kGc ? fmaf(wy1, raw1[cell * kGc + ch], wy0 * raw0[cell * kGc + ch]) : 0.0f;
      }
    } else {
      for (int e = tid; e < a.row_floats; e += kAnyThreads) slab[e] = fmaf(wy1, raw1[e], wy0 * raw0[e]);   // lerp4's order
    }
    __syncthreads();
    const size_t pix0 = static_cast<size_t>(row) * g.W;
    for (int x = tid; x < g.W; x += kAnyThreads) {
      const size_t p = pix0 + x;
      const Axis ax = spatial_axis(x, g.scale_x);
      const Axis az = range_axis(__ldg(a.guide + p), gd_f);
      const int xo0 = clampi(ax.i0, 0, g.gw - 1) * x_stride, xo1 = clampi(ax.i0 + 1, 0, g.gw - 1) * x_stride;
      const int zo0 = clampi(az.i0, 0, g.gd - 1) * cell_stride, zo1 = clampi(az.i0 + 1, 0, g.gd - 1) * cell_stride;
      float wz0, wz1;
      smoothed_weights(az.f, wz0, wz1);
      const float wx1 = ax.f, wx0 = 1.0f - ax.f;
      const float w00 = wx0 * wz0, w01 = wx0 * wz1, w10 = wx1 * wz0, w11 = wx1 * wz1;
      const float* c00 = slab + xo0 + zo0;
      const float* c01 = slab + xo0 + zo1;
      const float* c10 = slab + xo1 + zo0;
      const float* c11 = slab + xo1 + zo1;
      if constexpr (kGc > 0) {
        float cf[kGcp];
#pragma unroll
        for (int q4 = 0; q4 < kGcp / 4; ++q4) {
          const float4 v00 = *reinterpret_cast<const float4*>(c00 + 4 * q4);
          const float4 v01 = *reinterpret_cast<const float4*>(c01 + 4 * q4);
          const float4 v10 = *reinterpret_cast<const float4*>(c10 + 4 * q4);
          const float4 v11 = *reinterpret_cast<const float4*>(c11 + 4 * q4);
          cf[4 * q4 + 0] = fmaf(w11, v11.x, fmaf(w10, v10.x, fmaf(w01, v01.x, w00 * v00.x)));
          cf[4 * q4 + 1] = fmaf(w11, v11.y, fmaf(w10, v10.y, fmaf(w01, v01.y, w00 * v00.y)));
          cf[4 * q4 + 2] = fmaf(w11, v11.z, fmaf(w10, v10.z, fmaf(w01, v01.z, w00 * v00.z)));
          cf[4 * q4 + 3] = fmaf(w11, v11.w, fmaf(w10, v10.w, fmaf(w01, v01.w, w00 * v00.w)));
        }
        if constexpr (kApply) {
          constexpr int kJ = kGc / kOut;
          float in[kIn];
#pragma unroll
          for (int j = 0; j < kIn; ++j) in[j] = __ldg(a.input + p * kIn + j);
#pragma unroll
          for (int i = 0; i < kOut; ++i) {
            float value = 0.0f;
#pragma unroll
            for (int j = 0; j < kJ; ++j)
              value = (j < kIn) ? fmaf(cf[i * kJ + j], in[j], value) : value + cf[i * kJ + j];
            a.out[p * kOut + i] = value;
          }
        } else if ((kGc % 4 == 0) && out_vec) {   // a pixel is kGc * 4 bytes: 16-byte aligned whenever the base is
#pragma unroll
          for (int q4 = 0; q4 < kGc / 4; ++q4)
            *reinterpret_cast<float4*>(a.out + p * kGc + 4 * q4) =
                make_float4(cf[4 * q4], cf[4 * q4 + 1], cf[4 * q4 + 2], cf[4 * q4 + 3]);
        } else {
#pragma unroll
          for (int ch = 0; ch < kGc; ++ch) a.out[p * kGc + ch] = cf[ch];
        }
      } else {
        auto coef = [&](int ch) {   // the row kernels' order of operations
          return fmaf(w11, c11[ch], fmaf(w10, c10[ch], fmaf(w01, c01[ch], w00 * c00[ch])));
        };
        if constexpr (kApply) {
          for (int i = 0; i < a.n_out; ++i) {
            float value = 0.0f;
            for (int j = 0; j < a.J; ++j) {
              const float sv = coef(i * a.J + j);
              value = (j < a.n_in) ? fmaf(sv, __ldg(a.input + p * a.n_in + j), value) : value + sv;
            }
            a.out[p * a.n_out + i] = value;
          }
        } else {
          for (int ch = 0; ch < gc; ++ch) a.out[p * gc + ch] = coef(ch);
        }
      }
    }
  }
}

// Compile-time channel count of the any-shape row kernel for these counts (0: run-time counts).  The
// common shapes get one: the 3 -> 3 affine op with and without offset (what the TMA kernels take, at
// widths / alignments they do not; ops_test.py:345-365), the pyramid grid (hdrnet_ops_test.py:91-100),
// and the un-fused slice of a 12-channel grid.
static int rows_any_gc(const AnyArgs& a, bool apply) {
  if (!apply) return a.gc == 12 ? 12 : 0;
  if (a.n_in == 3 && a.n_out == 3 && (a.J == 4 || a.J == 3)) return 3 * a.J;
  if (a.n_in == 3 && a.n_out == 9 && a.J == 4) return 36;
  return 0;
}

static int rows_any_smem_cap(int max_smem) { return (max_smem + 1024) / 4 - 1024; }   // 4 CTAs per SM

// Dynamic shared memory of the any-shape row kernel, or 0 where the shape does not suit it (slab rows
// larger than a quarter SM's shared memory, images too narrow to fill a CTA): slice_generic_kernel
// runs then.
static size_t rows_any_smem(const AnyArgs& a, bool apply, int max_smem) {
  const int gc = rows_any_gc(a, apply);
  const size_t raw = (static_cast<size_t>(a.row_floats) + 3) & ~static_cast<size_t>(3);
  const size_t slab = gc > 0 ? static_cast<size_t>(a.g.gw) * a.g.gd * ((gc + 3) / 4 * 4) : raw;
  const size_t smem = (2 * raw + slab) * sizeof(float);
  if (a.g.W < 64 || smem > static_cast<size_t>(rows_any_smem_cap(max_smem))) return 0;
  return smem;
}

static int rows_any_ctas(const SliceGeom& g, int sms) {
  return static_cast<int>(std::min<long long>(static_cast<long long>(g.B) * g.rows, static_cast<long long>(sms) * 4));
}

template <bool kApply, int kGc, int kIn, int kOut>
static int launch_rows_any_t(const AnyArgs& a, int ctas, size_t smem, int max_smem, cudaStream_t stream) {
  auto kern = slice_rows_any_kernel<kApply, kGc, kIn, kOut>;
  static std::atomic<int> granted{0};   // sticky per-function attribute: only ever raise it
  if (granted.load(std::memory_order_relaxed) < static_cast<int>(smem)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_any_smem_cap(max_smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    granted.store(rows_any_smem_cap(max_smem), std::memory_order_relaxed);
  }
  kern<<<ctas, kAnyThreads, smem, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

// smem: rows_any_smem, non-zero
template <bool kApply>
static int launch_rows_any(const AnyArgs& a, int ctas, size_t smem, int max_smem, cudaStream_t stream) {
  const int gc = rows_any_gc(a, kApply);
  if constexpr (kApply) {
    if (gc == 12) return launch_rows_any_t<true, 12, 3, 3>(a, ctas, smem, max_smem, stream);
    if (gc == 9) return launch_rows_any_t<true, 9, 3, 3>(a, ctas, smem, max_smem, stream);
    if (gc == 36) return launch_rows_any_t<true, 36, 3, 9>(a, ctas, smem, max_smem, stream);
    return launch_rows_any_t<true, 0, 0, 0>(a, ctas, smem, max_smem, stream);
  } else {
    if (gc == 12) return launch_rows_any_t<false, 12, 0, 0>(a, ctas, smem, max_smem, stream);
    return launch_rows_any_t<false, 0, 0, 0>(a, ctas, smem, max_smem, stream);
  }
}

__global__ void __launch_bounds__(256)
slice_indices_kernel(const float* __restrict__ guide, int32_t* __restrict__ idx, SliceGeom g,
                     long long npix) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < npix;
       p += stride) {
    const int x = static_cast<int>(p % g.W);
    const int r = static_cast<int>((p / g.W) % g.rows);
    idx[3 * p + 0] = spatial_axis(x, g.scale_x).i0;
    idx[3 * p + 1] = spatial_axis(g.y_off + r, g.scale_y).i0;
    idx[3 * p + 2] = range_axis(__ldg(guide + p), static_cast<float>(g.gd)).i0;
  }
}

// Any-shape fallback of the model-path forms with integer pixel I/O: one thread per pixel, guide
// computed in registers, 8-corner gather as slice_generic_kernel<true> (same summation order, so
// its float32 result equals guide kernel + generic kernel bit for bit).
template <class GuideFn, int kIn, int kOut>
__global__ void __launch_bounds__(256)
slice_apply_px_generic_kernel(const float* __restrict__ grid, const unsigned char* __restrict__ input,
                              unsigned char* __restrict__ out, float* __restrict__ guide_out,
                              SliceGeom g, long long npix, const __grid_constant__ GuideFn guide_fn) {
  const long long grid_image = static_cast<long long>(g.gh) * g.gw * g.gd * 12;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < npix;
       p += stride) {
    const int x = static_cast<int>(p % g.W);
    const long long row = p / g.W;
    const int r = static_cast<int>(row % g.rows);
    const int b = static_cast<int>(row / g.rows);
    const float in[3] = {load_channel<kIn>(input, 3 * p), load_channel<kIn>(input, 3 * p + 1),
                         load_channel<kIn>(input, 3 * p + 2)};
    const float gv = guide_fn(in[0], in[1], in[2]);
    if (guide_out != nullptr) guide_out[p] = gv;
    const Corners c = make_corners(g, x, g.y_off + r, gv, 12);
    const float* grid_b = grid + b * grid_image;
    float o[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      float value = 0.0f;
#pragma unroll
      for (int j = 0; j < 3; ++j) value = fmaf(sample(grid_b, c, i * 4 + j), in[j], value);
      o[i] = value + sample(grid_b, c, i * 4 + 3);
    }
    if constexpr (kOut == kPxF32) {
      float* op = reinterpret_cast<float*>(out) + 3 * p;
      op[0] = o[0]; op[1] = o[1]; op[2] = o[2];
    } else if constexpr (kOut == kPxU16) {
      unsigned short* op = reinterpret_cast<unsigned short*>(out) + 3 * p;
      op[0] = static_cast<unsigned short>(float_to_u16(o[0]));
      op[1] = static_cast<unsigned short>(float_to_u16(o[1]));
      op[2] = static_cast<unsigned short>(float_to_u16(o[2]));
    } else {
      out[3 * p] = static_cast<unsigned char>(float_to_u8(o[0]));
      out[3 * p + 1] = static_cast<unsigned char>(float_to_u8(o[1]));
      out[3 * p + 2] = static_cast<unsigned char>(float_to_u8(o[2]));
    }
  }
}

template <class GuideFn, int kTexChunks, int kMinBlocks = 2, int kThreads = kTmaThreads,
          int kIn = kPxF32, int kOut = kPxF32>
__global__ void __launch_bounds__(kThreads, kMinBlocks)
slice_apply_rows_tma_kernel(const TmaArgs args, const __grid_constant__ GuideFn guide_fn) {
  constexpr bool kGuideIn = GuideFn::kFromInput;
  constexpr uint32_t kInBpp = 3u * px_bytes_per_channel(kIn), kOutBpp = 3u * px_bytes_per_channel(kOut);
  extern __shared__ __align__(128) unsigned char smem[];
  const SliceGeom& g = args.g;
  const TmaPlan& pl = args.p;
  const int tid = threadIdx.x;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);        // [kMaxStages]
  uint64_t* gridbar = full + kMaxStages;                      // [2]
  float* raw0 = reinterpret_cast<float*>(smem + pl.off_raw);
  float* raw1 = raw0 + pl.row_floats;
  float* slab = reinterpret_cast<float*>(smem + pl.off_slab);
  int tex_row = 0;
  unsigned char* stage_base = smem + pl.off_stage;

  // Contiguous block of buffer rows per CTA (neighbouring rows share grid rows).
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  const long long r_begin = total_rows * blockIdx.x / gridDim.x;
  const long long r_end = total_rows * (blockIdx.x + 1) / gridDim.x;
  const int nitems = static_cast<int>(r_end - r_begin) * pl.nseg;
  if (nitems <= 0) return;

  if (tid == 0) {
    for (int s = 0; s < pl.stages; ++s) mbar_init(&full[s], 1);
    mbar_init(&gridbar[0], 1);
    mbar_init(&gridbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int NS = pl.stages;

  auto stage_rgb = [&](int s) { return stage_base + static_cast<size_t>(s) * pl.stage_bytes; };
  auto stage_guide = [&](int s) { return stage_rgb(s) + pl.off_guide; };
  // same pixel size in and out: the result overwrites the input tile (plan.off_out == 0)
  auto stage_out = [&](int s) { return stage_rgb(s) + (kInBpp == kOutBpp ? 0 : pl.off_out); };
  // Work item -> (buffer row, first pixel of the segment, pixels in the segment).
  auto item_span = [&](int item, long long& row, int& x0, int& npx) {
    const int rr = item / pl.nseg;
    const int seg = item - rr * pl.nseg;
    row = r_begin + rr;
    x0 = seg * pl.seg_px;
    npx = min(pl.seg_px, g.W - x0);
  };
  auto issue_load = [&](int item) {  // thread 0 only
    long long row; int x0, npx;
    item_span(item, row, x0, npx);
    const int s = item % NS;
    const size_t pix = static_cast<size_t>(row) * g.W + x0;
    mbar_expect_tx(&full[s], static_cast<uint32_t>(npx) * (kInBpp + (kGuideIn ? 4u : 0u)));
    tma_load_1d(stage_rgb(s), args.input + pix * kInBpp, static_cast<uint32_t>(npx) * kInBpp, &full[s]);
    if (kGuideIn)
      tma_load_1d(stage_guide(s), args.guide + pix, static_cast<uint32_t>(npx) * 4u, &full[s]);
  };

  if (tid == 0) {
    if constexpr (kTexChunks > 0) {  // slab of the first row
      const uint32_t bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
      mbar_expect_tx(&gridbar[0], bytes);
      tma_load_1d(raw0, args.yslab + static_cast<size_t>(r_begin) * pl.row_floats, bytes, &gridbar[0]);
    }
    const int pre = min(NS - 1, nitems);
    for (int it = 0; it < pre; ++it) issue_load(it);
  }

  int cur_b = -1, cur_gy0 = INT_MIN;
  uint32_t grid_phase = 0;

  for (int item = 0; item < nitems; ++item) {
    long long row; int x0, npx;
    item_span(item, row, x0, npx);

    if (x0 == 0) {
      if constexpr (kTexChunks > 0) {
        // Texture-assisted form: the y-pre-blended slab rows were produced by a pre-pass
        // (yblend_rows_kernel) into a global workspace, so that the texture pipe may read
        // them (texture reads of data written by the SAME kernel are not coherent).  The
        // row's slab arrives by one TMA copy, double-buffered one row ahead in raw0 / raw1.
        const int rowk = item / pl.nseg;
        const int cur = rowk & 1;
        slab = raw0 + cur * pl.row_floats;
        mbar_wait(&gridbar[cur], static_cast<uint32_t>(rowk >> 1) & 1u);
        if (tid == 0 && row + 1 < r_end) {
          const uint32_t bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
          mbar_expect_tx(&gridbar[cur ^ 1], bytes);
          tma_load_1d(raw0 + (cur ^ 1) * pl.row_floats,
                      args.yslab + static_cast<size_t>(row + 1) * pl.row_floats, bytes,
                      &gridbar[cur ^ 1]);
        }
        tex_row = static_cast<int>(row) * (pl.row_floats / 4);
      } else {
      // New image row: (re)stage its two grid rows if they changed, then pre-blend in y.
      // Every thread is past the previous item's post-compute barrier, so raw/slab are idle.
      const int b = static_cast<int>(row / g.rows);
      const int y = g.y_off + static_cast<int>(row - static_cast<long long>(b) * g.rows);
      const Axis ay = spatial_axis(y, g.scale_y);
      if (b != cur_b || ay.i0 != cur_gy0) {
        if (tid == 0) {
          const int gy0c = clampi(ay.i0, 0, g.gh - 1);
          const int gy1c = clampi(ay.i0 + 1, 0, g.gh - 1);
          const float* gb = args.grid + static_cast<size_t>(b) * g.gh * pl.row_floats;
          const uint32_t bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
          mbar_expect_tx(gridbar, 2u * bytes);
          tma_load_1d(raw0, gb + static_cast<size_t>(gy0c) * pl.row_floats, bytes, gridbar);
          tma_load_1d(raw1, gb + static_cast<size_t>(gy1c) * pl.row_floats, bytes, gridbar);
        }
        mbar_wait(gridbar, grid_phase);
        grid_phase ^= 1u;
        cur_b = b;
        cur_gy0 = ay.i0;
      }
      const float wy1 = ay.f, wy0 = 1.0f - ay.f;
      const float4* a4 = reinterpret_cast<const float4*>(raw0);
      const float4* b4 = reinterpret_cast<const float4*>(raw1);
      float4* s4 = reinterpret_cast<float4*>(slab);
      for (int e = tid; e < pl.row_floats / 4; e += kThreads) s4[e] = lerp4(wy0, a4[e], wy1, b4[e]);
      __syncthreads();
      }
    }

    const int s = item % NS;
    mbar_wait(&full[s], static_cast<uint32_t>(item / NS) & 1u);

    if (tid * 4 < npx)
      process_quad<GuideFn, kTexChunks, kIn, kOut>(args, guide_fn, stage_rgb(s), stage_out(s),
                                                   stage_guide(s), slab, tex_row, row, x0, tid);
    __syncthreads();

    if (tid == 0) {
      const size_t pix = static_cast<size_t>(row) * g.W + x0;
      tma_store_1d(args.out + pix * kOutBpp, stage_out(s), static_cast<uint32_t>(npx) * kOutBpp);
      tma_store_commit();
      const int nxt = item + NS - 1;
      if (nxt < nitems) {
        tma_store_wait_read<1>();  // the store of item-1 has drained its stage
        issue_load(nxt);
      }
    }
  }
  if (tid == 0) tma_store_wait_all<0>();
}



// =========================================================================================
// Un-fused slice, persistent TMA row kernel (gc = 12, W % 4 == 0): out[b,y,x,0..11].
// =========================================================================================
// Same organisation as the fused kernel, but the op is WRITE-bound (4 B in, 48 B out per pixel):
// the guide arrives through a deep ring of small TMA copies, each thread blends the 4 slab
// corners of its pixels (48 FFMA per pixel, no apply) and writes the 12 coefficients into one of
// kSliceOutBufs shared-memory output tiles that leave by TMA bulk stores; an mbarrier per
// output tile (armed by the store-issuing thread after cp.async.bulk.wait_group.read) gates
// its reuse.  Thread t owns pixels t and t + 256 of a 512-pixel segment: 48-byte stride between
// lanes keeps the 3 x STS.128 per pixel conflict-free.
constexpr int kSliceThreads = 256;
constexpr int kSliceSegPx = 512;
constexpr int kSliceOutBufs = 3;
constexpr int kSliceGuideStages = 8;

struct SlicePlan {
  int ctas, nseg, seg_px, row_floats, smem_bytes;
  int off_raw, off_slab, off_guide, off_out, out_bytes;
};

struct SliceArgs {
  const float* grid;
  const float* guide;
  float* out;
  SliceGeom g;
  SlicePlan p;
};

__global__ void __launch_bounds__(kSliceThreads, 2)
slice_rows_tma_kernel(const SliceArgs args) {
  extern __shared__ __align__(128) unsigned char smem[];
  const SliceGeom& g = args.g;
  const SlicePlan& pl = args.p;
  const int tid = threadIdx.x;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);   // [kSliceGuideStages]
  uint64_t* out_free = full + kSliceGuideStages;         // [kSliceOutBufs]
  uint64_t* gridbar = out_free + kSliceOutBufs;          // [1]
  float* raw0 = reinterpret_cast<float*>(smem + pl.off_raw);
  float* raw1 = raw0 + pl.row_floats;
  float* slab = reinterpret_cast<float*>(smem + pl.off_slab);
  float* guide_ring = reinterpret_cast<float*>(smem + pl.off_guide);  // [stages][seg_px]
  unsigned char* out_base = smem + pl.off_out;

  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  const long long r_begin = total_rows * blockIdx.x / gridDim.x;
  const long long r_end = total_rows * (blockIdx.x + 1) / gridDim.x;
  const int nitems = static_cast<int>(r_end - r_begin) * pl.nseg;
  if (nitems <= 0) return;

  if (tid == 0) {
    for (int s = 0; s < kSliceGuideStages; ++s) mbar_init(&full[s], 1);
    for (int s = 0; s < kSliceOutBufs; ++s) mbar_init(&out_free[s], 1);
    mbar_init(gridbar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto item_span = [&](int item, long long& row, int& x0, int& npx) {
    const int rr = item / pl.nseg;
    const int seg = item - rr * pl.nseg;
    row = r_begin + rr;
    x0 = seg * pl.seg_px;
    npx = min(pl.seg_px, g.W - x0);
  };
  auto issue_load = [&](int item) {  // thread 0 only
    long long row; int x0, npx;
    item_span(item, row, x0, npx);
    const int s = item % kSliceGuideStages;
    mbar_expect_tx(&full[s], static_cast<uint32_t>(npx) * 4u);
    tma_load_1d(guide_ring + static_cast<size_t>(s) * pl.seg_px,
                args.guide + static_cast<size_t>(row) * g.W + x0, static_cast<uint32_t>(npx) * 4u,
                &full[s]);
  };
  if (tid == 0) {
    // every output tile starts free: one arrival completes phase 0 of its barrier
    for (int s = 0; s < kSliceOutBufs; ++s)
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&out_free[s])) : "memory");
    const int pre = min(kSliceGuideStages - 1, nitems);
    for (int it = 0; it < pre; ++it) issue_load(it);
  }

  const float gd_f = static_cast<float>(g.gd);
  const int x_stride = g.gd * kGc;
  int cur_b = -1, cur_gy0 = INT_MIN;
  uint32_t grid_phase = 0;

  for (int item = 0; item < nitems; ++item) {
    long long row; int x0, npx;
    item_span(item, row, x0, npx);

    if (x0 == 0) {  // new image row: grid rows + y pre-blend, as in the fused kernel
      const int b = static_cast<int>(row / g.rows);
      const int y = g.y_off + static_cast<int>(row - static_cast<long long>(b) * g.rows);
      const Axis ay = spatial_axis(y, g.scale_y);
      if (b != cur_b || ay.i0 != cur_gy0) {
        if (tid == 0) {
          const int gy0c = clampi(ay.i0, 0, g.gh - 1);
          const int gy1c = clampi(ay.i0 + 1, 0, g.gh - 1);
          const float* gb = args.grid + static_cast<size_t>(b) * g.gh * pl.row_floats;
          const uint32_t bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
          mbar_expect_tx(gridbar, 2u * bytes);
          tma_load_1d(raw0, gb + static_cast<size_t>(gy0c) * pl.row_floats, bytes, gridbar);
          tma_load_1d(raw1, gb + static_cast<size_t>(gy1c) * pl.row_floats, bytes, gridbar);
        }
        mbar_wait(gridbar, grid_phase);
        grid_phase ^= 1u;
        cur_b = b;
        cur_gy0 = ay.i0;
      }
      const float wy1 = ay.f, wy0 = 1.0f - ay.f;
      const float4* a4 = reinterpret_cast<const float4*>(raw0);
      const float4* b4 = reinterpret_cast<const float4*>(raw1);
      float4* s4 = reinterpret_cast<float4*>(slab);
      for (int e = tid; e < pl.row_floats / 4; e += kSliceThreads) s4[e] = lerp4(wy0, a4[e], wy1, b4[e]);
      __syncthreads();
    }

    const int s = item % kSliceGuideStages;
    const int ob = item % kSliceOutBufs;
    mbar_wait(&full[s], static_cast<uint32_t>(item / kSliceGuideStages) & 1u);
    mbar_wait(&out_free[ob], static_cast<uint32_t>(item / kSliceOutBufs) & 1u);
    const float* gseg = guide_ring + static_cast<size_t>(s) * pl.seg_px;
    float* otile = reinterpret_cast<float*>(out_base + static_cast<size_t>(ob) * pl.out_bytes);
#pragma unroll
    for (int h = 0; h < kSliceSegPx / kSliceThreads; ++h) {
      const int px = tid + h * kSliceThreads;
      if (px < npx) {
        const Axis ax = spatial_axis(x0 + px, g.scale_x);
        const Axis az = range_axis(gseg[px], gd_f);
        const int xo0 = clampi(ax.i0, 0, g.gw - 1) * x_stride;
        const int xo1 = clampi(ax.i0 + 1, 0, g.gw - 1) * x_stride;
        const int zo0 = clampi(az.i0, 0, g.gd - 1) * kGc;
        const int zo1 = clampi(az.i0 + 1, 0, g.gd - 1) * kGc;
        float wz0, wz1;
        smoothed_weights(az.f, wz0, wz1);
        const float wx1 = ax.f, wx0 = 1.0f - ax.f;
        const unsigned long long W00 = pack2(wx0 * wz0, wx0 * wz0), W01 = pack2(wx0 * wz1, wx0 * wz1);
        const unsigned long long W10 = pack2(wx1 * wz0, wx1 * wz0), W11 = pack2(wx1 * wz1, wx1 * wz1);
        const ulonglong2* v00 = reinterpret_cast<const ulonglong2*>(slab + xo0 + zo0);
        const ulonglong2* v01 = reinterpret_cast<const ulonglong2*>(slab + xo0 + zo1);
        const ulonglong2* v10 = reinterpret_cast<const ulonglong2*>(slab + xo1 + zo0);
        const ulonglong2* v11 = reinterpret_cast<const ulonglong2*>(slab + xo1 + zo1);
        ulonglong2* dst = reinterpret_cast<ulonglong2*>(otile + static_cast<size_t>(px) * kGc);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const ulonglong2 a = v00[k], bq = v01[k], c = v10[k], d = v11[k];
          ulonglong2 r;
          r.x = fma2(W11, d.x, fma2(W10, c.x, fma2(W01, bq.x, mul2(W00, a.x))));
          r.y = fma2(W11, d.y, fma2(W10, c.y, fma2(W01, bq.y, mul2(W00, a.y))));
          dst[k] = r;
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();

    if (tid == 0) {
      const size_t pix = static_cast<size_t>(row) * g.W + x0;
      tma_store_1d(args.out + pix * kGc, otile, static_cast<uint32_t>(npx) * (kGc * 4u));
      tma_store_commit();
      // the tile the NEXT item writes is free once all but the newest (kSliceOutBufs-1) stores
      // have finished reading shared memory
      tma_store_wait_read<kSliceOutBufs - 1>();
      if (item + 1 >= kSliceOutBufs)  // first uses were released by the initial arrivals
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(
                         smem_u32(&out_free[(item + 1) % kSliceOutBufs]))
                     : "memory");
      const int nxt = item + kSliceGuideStages - 1;
      if (nxt < nitems) issue_load(nxt);
    }
  }
  if (tid == 0) tma_store_wait_all<0>();
}

static bool make_slice_plan(const SliceGeom& g, int max_smem, int sms, SlicePlan* out) {
  if (g.W < 4 || (g.W % 4) != 0) return false;
  SlicePlan p;
  p.row_floats = g.gw * g.gd * kGc;
  const int quads = g.W / 4;
  const int max_quads = kSliceSegPx / 4;
  p.nseg = (quads + max_quads - 1) / max_quads;
  p.seg_px = 4 * ((quads + p.nseg - 1) / p.nseg);
  p.out_bytes = round_up(p.seg_px * kGc * 4, 128);
  p.off_raw = 128;  // (8 + 3 + 1) barriers = 96 bytes
  p.off_slab = p.off_raw + round_up(2 * p.row_floats * 4, 128);
  p.off_guide = p.off_slab + round_up(p.row_floats * 4, 128);
  p.off_out = p.off_guide + round_up(kSliceGuideStages * p.seg_px * 4, 128);
  p.smem_bytes = p.off_out + kSliceOutBufs * p.out_bytes;
  if (p.smem_bytes > max_smem) return false;
  const int resident = (p.smem_bytes <= (max_smem + 1024) / 2 - 1024) ? 2 : 1;
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  p.ctas = static_cast<int>(std::min<long long>(total_rows, static_cast<long long>(sms) * resident));
  *out = p;
  return true;
}

// Pre-pass of the texture-assisted forms: yslab[r] = (1 - fy) * G[b][gy0] + fy * G[b][gy1] for
// every buffer row r = (b, y) -- the same y pre-blend the row kernel does in shared memory,
// materialised once (gw*gd*48 B per image row: +11 % HBM bytes at 4K / 16x16x8).
// One CTA owns kYblendRows consecutive rows and a thread one output float4 column of them: the two
// grid rows it blends change every H / gh image rows, so they live in registers and the kernel
// is a stream of coalesced stores (one CTA per row, with two dependent L2 loads per thread, is
// latency-bound).
constexpr int kYblendRows = 16;
__global__ void __launch_bounds__(256)
yblend_rows_kernel(const float* __restrict__ grid, float4* __restrict__ ws, SliceGeom g,
                   int row_floats) {
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  const long long r0 = static_cast<long long>(blockIdx.x) * kYblendRows;
  const long long r1 = min(r0 + kYblendRows, total_rows);
  const int n_out = row_floats / 4;   // float4 per output row
  for (int e = threadIdx.x; e < n_out; e += blockDim.x) {
    int cur_b = -1, cur_i0 = INT_MIN;
    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
    int b = static_cast<int>(r0 / g.rows);                                   // one division per CTA column
    int yl = static_cast<int>(r0 - static_cast<long long>(b) * g.rows);      // row inside the image's band
    for (long long row = r0; row < r1; ++row, ++yl) {
      if (yl == g.rows) { yl = 0; ++b; }
      const Axis ay = spatial_axis(g.y_off + yl, g.scale_y);
      if (b != cur_b || ay.i0 != cur_i0) {
        const float* gb = grid + static_cast<size_t>(b) * g.gh * row_floats;
        va = __ldg(reinterpret_cast<const float4*>(gb + static_cast<size_t>(clampi(ay.i0, 0, g.gh - 1)) * row_floats) + e);
        vb = __ldg(reinterpret_cast<const float4*>(gb + static_cast<size_t>(clampi(ay.i0 + 1, 0, g.gh - 1)) * row_floats) + e);
        cur_b = b;
        cur_i0 = ay.i0;
      }
      ws[static_cast<size_t>(row) * n_out + e] = lerp4(1.0f - ay.f, va, ay.f, vb);
    }
  }
}

static int launch_yblend(const float* grid, float* ws, const SliceGeom& g, int row_floats, cudaStream_t stream) {
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  const unsigned blocks = static_cast<unsigned>((total_rows + kYblendRows - 1) / kYblendRows);
  yblend_rows_kernel<<<blocks, 256, 0, stream>>>(grid, reinterpret_cast<float4*>(ws), g, row_floats);
  return static_cast<int>(cudaGetLastError());
}

// =========================================================================================
// Host side: planning, validation, launch.
// =========================================================================================

static int device_sm_count() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
  return sms > 0 ? sms : 132;
}

static int device_max_smem_optin() {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 227 * 1024;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return 227 * 1024;
  return v;
}

// Base alignment a texture object over linear memory needs (512 bytes on H100): the texture-assisted
// forms fetch the slab workspace through one, and cudaCreateTextureObject refuses other bases.
static int device_texture_alignment() {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 512;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrTextureAlignment, dev) != cudaSuccess) return 512;
  return v > 0 ? v : 512;
}


// Returns false when the TMA kernel cannot run these shapes.  threads: the threads that process
// pixels (a quad each per segment).
// tex_mode: the texture-assisted form double-buffers whole slab rows in raw0 / raw1 and needs no
// separate slab region (lets 32x32x16 grids keep two CTAs per SM).
// grid_rows: grid rows staged next to the slab rows (the slab warp of the issuer-warp form).
static bool make_tma_plan(const SliceGeom& g, int max_smem, int sms, TmaPlan* out, bool tex_mode,
                          int threads, int in_fmt = kPxF32, int out_fmt = kPxF32, int grid_rows = 0) {
  // Bulk copies move 16-byte units: a row and every segment must start on one.  float32 pixels
  // need W % 4 == 0, uint16 W % 8 == 0, uint8 W % 16 == 0 (12 / 6 / 3 bytes per pixel).
  const int in_bpp = 3 * px_bytes_per_channel(in_fmt), out_bpp = 3 * px_bytes_per_channel(out_fmt);
  const int gran = std::max(4, std::max(16 / std::__gcd(16, in_bpp), 16 / std::__gcd(16, out_bpp)));
  if (g.W < gran || (g.W % gran) != 0) return false;
  TmaPlan p;
  p.threads = threads;
  p.row_floats = g.gw * g.gd * kGc;
  p.in_bpp = in_bpp;
  p.out_bpp = out_bpp;
  const int quads = g.W / 4;
  p.nseg = (quads + threads - 1) / threads;
  p.seg_px = round_up(4 * ((quads + p.nseg - 1) / p.nseg), gran);  // <= 4 * threads (a multiple of 16)
  // stage = input tile | guide tile (always reserved) | output tile unless it fits in place
  p.off_guide = round_up(p.seg_px * in_bpp, 16);
  p.off_out = (out_bpp == in_bpp) ? 0 : p.off_guide + p.seg_px * 4;
  p.stage_bytes = round_up((p.off_out ? p.off_out + p.seg_px * out_bpp : p.off_guide + p.seg_px * 4), 128);
  p.off_raw = 256;  // barriers: up to 2 * kMaxStages + 4 (warp-specialised form) = 160 bytes
  p.off_slab = p.off_raw + round_up(2 * p.row_floats * 4, 128);
  p.off_grid = p.off_slab;
  p.off_stage = p.off_slab + (tex_mode ? grid_rows * round_up(p.row_floats * 4, 128) : round_up(p.row_floats * 4, 128));
  // Residency: two CTAs per SM with a 4-stage ring; shrink the ring before giving up residency.
  const int per_cta_2 = (max_smem + 1024) / 2 - 1024;  // ~113 KB when 227 KB opt-in
  int stages = 0, resident = 0;
  for (int ns = 4; ns >= 2 && stages == 0; --ns)
    if (p.off_stage + ns * p.stage_bytes <= per_cta_2) { stages = ns; resident = 2; }
  for (int ns = 4; ns >= 2 && stages == 0; --ns)
    if (p.off_stage + ns * p.stage_bytes <= max_smem) { stages = ns; resident = 1; }
  if (stages == 0) return false;
  p.stages = stages;
  p.resident = resident;
  p.smem_bytes = p.off_stage + stages * p.stage_bytes;
  const long long total_rows = static_cast<long long>(g.B) * g.rows;
  p.ctas = static_cast<int>(std::min<long long>(total_rows, static_cast<long long>(sms) * resident));
  *out = p;
  return true;
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int validate_common(int B, int H, int W, int gh, int gw, int gd) {
  if (B < 0 || H < 0 || W < 0) return HDRNET_E_BAD_SHAPE;
  if (gh < 1 || gw < 1 || gd < 1) return HDRNET_E_BAD_SHAPE;
  return HDRNET_OK;
}

static int generic_grid(long long npix, int sms) {
  const long long blocks = (npix + 255) / 256;
  return static_cast<int>(std::min<long long>(blocks, static_cast<long long>(sms) * 16));
}

template <class GuideFn, int kTexChunks = 0, int kMinBlocks = 2, int kThreads = kTmaThreads,
          int kIn = kPxF32, int kOut = kPxF32>
static int launch_tma_occ(const TmaArgs& a, const GuideFn& fn, cudaStream_t stream) {
  auto kern = slice_apply_rows_tma_kernel<GuideFn, kTexChunks, kMinBlocks, kThreads, kIn, kOut>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       a.p.smem_bytes);
  if (e != cudaSuccess) return static_cast<int>(e);
  kern<<<a.p.ctas, kThreads, a.p.smem_bytes, stream>>>(a, fn);
  return static_cast<int>(cudaGetLastError());
}

template <class GuideFn, int kTexChunks = 0>
static int launch_tma(const TmaArgs& a, const GuideFn& fn, cudaStream_t stream, int in_fmt = kPxF32,
                      int out_fmt = kPxF32) {
  if constexpr (GuideFn::kFromInput) {
    // the texture-assisted form of the op API: 512 threads, 64 registers per thread (no spills), 32
    // warps per SM (plan_slice_apply gives it no other plan)
    if constexpr (kTexChunks > 0) return launch_tma_occ<GuideFn, kTexChunks, 2, kTexThreads>(a, fn, stream);
    else return launch_tma_occ<GuideFn, 0, 2>(a, fn, stream);
  } else {
    // The fused-guide forms are issue-bound and need their registers: 256 threads x 2 CTAs.
    // (chosen against 256 x 3 and 512 x 2 on the previous target; not re-tuned on H100).  Integer
    // pixel formats exist for them only.
    if (in_fmt == kPxU8 && out_fmt == kPxU8)
      return launch_tma_occ<GuideFn, kTexChunks, 2, kTmaThreads, kPxU8, kPxU8>(a, fn, stream);
    if (in_fmt == kPxU16 && out_fmt == kPxU8)
      return launch_tma_occ<GuideFn, kTexChunks, 2, kTmaThreads, kPxU16, kPxU8>(a, fn, stream);
    if (in_fmt == kPxU8 && out_fmt == kPxU16)
      return launch_tma_occ<GuideFn, kTexChunks, 2, kTmaThreads, kPxU8, kPxU16>(a, fn, stream);
    if (in_fmt == kPxU16 && out_fmt == kPxU16)
      return launch_tma_occ<GuideFn, kTexChunks, 2, kTmaThreads, kPxU16, kPxU16>(a, fn, stream);
    if (in_fmt != kPxF32 || out_fmt != kPxF32) return HDRNET_E_UNSUPPORTED;
    return launch_tma_occ<GuideFn, kTexChunks, 2>(a, fn, stream);
  }
}

// Texture objects over caller workspaces.  Creating one is a host-side driver call that should
// not sit inside a timed loop, so they are cached, keyed by (device, pointer, lent bytes) -- the
// whole workspace, not the part a call uses, so one entry serves every shape.  An entry remembers
// an event recorded after the last launch that uses it; an evicted texture is destroyed only once
// that event has completed (else it waits in a graveyard that later calls drain): a texture object
// is never destroyed under a kernel that may still fetch through it.  A call that a CUDA graph is
// capturing takes no cached texture (a graph replays long after any event recorded at capture, and
// the cache may have evicted the entry by then): it creates a texture of its own that the graph owns
// (graph_slab_texture).  This cache and the list of textures released by graphs are the library's
// only process-wide state.
struct TexCacheEntry { const void* ptr; size_t bytes; int dev; cudaTextureObject_t tex; cudaEvent_t last_use; };
constexpr int kTexCacheEntries = 16;
static std::mutex g_tex_mutex;
static TexCacheEntry g_tex_cache[kTexCacheEntries];
static int g_tex_next = 0;
static std::vector<TexCacheEntry> g_tex_graveyard;
// Textures whose graphs are gone.  Filled by user-object destructors, which may not call CUDA and
// may run on a driver thread, so this list has a lock of its own that is never held across a CUDA
// call; the next texture request destroys them.
static std::mutex g_graph_tex_mutex;
static std::vector<cudaTextureObject_t> g_graph_tex_released;

static void drain_tex_graveyard_locked() {
  for (size_t i = 0; i < g_tex_graveyard.size();) {
    TexCacheEntry& e = g_tex_graveyard[i];
    if (cudaEventQuery(e.last_use) == cudaSuccess) {
      cudaDestroyTextureObject(e.tex);
      cudaEventDestroy(e.last_use);
      g_tex_graveyard[i] = g_tex_graveyard.back();
      g_tex_graveyard.pop_back();
    } else {
      ++i;
    }
  }
  (void)cudaGetLastError();   // cudaErrorNotReady of a pending event is not an error of this call
}

static void destroy_released_graph_textures() {
  std::vector<cudaTextureObject_t> released;
  {
    std::lock_guard<std::mutex> lock(g_graph_tex_mutex);
    released.swap(g_graph_tex_released);
  }
  for (cudaTextureObject_t t : released) cudaDestroyTextureObject(t);
}

static int create_slab_texture(const float* ws, size_t bytes, cudaTextureObject_t* tex) {
  cudaResourceDesc rd = {};
  rd.resType = cudaResourceTypeLinear;
  rd.res.linear.devPtr = const_cast<float*>(ws);
  rd.res.linear.desc = cudaCreateChannelDesc<float4>();
  rd.res.linear.sizeInBytes = bytes;
  cudaTextureDesc td = {};
  td.readMode = cudaReadModeElementType;
  *tex = 0;
  cudaError_t err = cudaCreateTextureObject(tex, &rd, &td, nullptr);
  if (err != cudaSuccess) (void)cudaGetLastError();   // report it from this call only: the next launch's check must not see it
  return static_cast<int>(err);
}

// The texture over [ws, ws + bytes); `*use` must be recorded on the launch stream after the last
// kernel of this call that fetches through it.
static int get_slab_texture(const float* ws, size_t bytes, cudaTextureObject_t* out, cudaEvent_t* use) {
  destroy_released_graph_textures();
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_tex_mutex);
  if (!g_tex_graveyard.empty()) drain_tex_graveyard_locked();
  for (auto& e : g_tex_cache)
    if (e.tex && e.ptr == ws && e.bytes == bytes && e.dev == dev) { *out = e.tex; *use = e.last_use; return 0; }
  cudaTextureObject_t tex = 0;
  const int rc = create_slab_texture(ws, bytes, &tex);
  if (rc != 0) return rc;
  cudaEvent_t ev = nullptr;
  cudaError_t err = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (err != cudaSuccess) { cudaDestroyTextureObject(tex); return static_cast<int>(err); }
  TexCacheEntry& slot = g_tex_cache[g_tex_next];
  g_tex_next = (g_tex_next + 1) % kTexCacheEntries;
  if (slot.tex) { g_tex_graveyard.push_back(slot); drain_tex_graveyard_locked(); }
  slot = TexCacheEntry{ws, bytes, dev, tex, ev};
  *out = tex;
  *use = ev;
  return 0;
}

// User-object destructor of a graph-owned texture: runs once the graph and every executable graph
// made from it are destroyed and their launches have completed.
static void release_graph_texture(void* p) {
  cudaTextureObject_t* t = static_cast<cudaTextureObject_t*>(p);
  {
    std::lock_guard<std::mutex> lock(g_graph_tex_mutex);
    g_graph_tex_released.push_back(*t);
  }
  delete t;
}

// The texture over [ws, ws + bytes) for a call that `graph` is capturing: created for this call and
// owned by the graph through a user object, so it lives exactly as long as the graph can be replayed.
static int graph_slab_texture_relaxed(const float* ws, size_t bytes, cudaGraph_t graph, cudaTextureObject_t* out) {
  destroy_released_graph_textures();
  cudaTextureObject_t tex = 0;
  int rc = create_slab_texture(ws, bytes, &tex);
  if (rc != 0) return rc;
  cudaTextureObject_t* owned = new (std::nothrow) cudaTextureObject_t(tex);
  if (!owned) { cudaDestroyTextureObject(tex); return static_cast<int>(cudaErrorMemoryAllocation); }
  cudaUserObject_t obj = nullptr;
  cudaError_t err = cudaUserObjectCreate(&obj, owned, release_graph_texture, 1, cudaUserObjectNoDestructorSync);
  if (err != cudaSuccess) {
    (void)cudaGetLastError();
    delete owned;
    cudaDestroyTextureObject(tex);
    return static_cast<int>(err);
  }
  err = cudaGraphRetainUserObject(graph, obj, 1, cudaGraphUserObjectMove);
  if (err != cudaSuccess) {
    (void)cudaGetLastError();
    cudaUserObjectRelease(obj, 1);   // the destructor queues the texture for destruction
    return static_cast<int>(err);
  }
  *out = tex;
  return 0;
}

// Texture creation counts as an unsafe call while a capture in the global mode is in progress (the
// mode torch.cuda.graph uses), which would invalidate the capture; it does not touch any stream, so
// this thread makes it in the relaxed mode and restores its mode after.
static int graph_slab_texture(const float* ws, size_t bytes, cudaGraph_t graph, cudaTextureObject_t* out) {
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaError_t err = cudaThreadExchangeStreamCaptureMode(&mode);
  if (err != cudaSuccess) { (void)cudaGetLastError(); return static_cast<int>(err); }
  const int rc = graph_slab_texture_relaxed(ws, bytes, graph, out);
  cudaThreadExchangeStreamCaptureMode(&mode);
  return rc;
}

// Guide source of a launch: an input tensor, or one of the fused per-pixel guide networks.
struct GuideSpec {
  int mode;  // 0 = input tensor, 1 = curves, 2 = pointwise NN
  const float* guide;
  float* guide_out;
  const CurvesGuideParams* curves;
  const NNGuideParams* nn;
  float* workspace = nullptr;  // HDRNET_VARIANT_TEX: slab rows, B * rows * gw * gd * 48 bytes
  size_t workspace_bytes = 0;
  int in_fmt = kPxF32;         // pixel storage of `input` / `out` (fused-guide modes only)
  int out_fmt = kPxF32;
};


template <class GuideFn>
static int launch_px_generic(const float* grid, const void* input, void* out, float* guide_out,
                             const SliceGeom& g, long long npix, int blocks, int in_fmt, int out_fmt,
                             const GuideFn& fn, cudaStream_t stream) {
  const unsigned char* in = static_cast<const unsigned char*>(input);
  unsigned char* o = static_cast<unsigned char*>(out);
#define HDRNET_PX_CASE(I, O)                                                                    \
  if (in_fmt == I && out_fmt == O) {                                                            \
    slice_apply_px_generic_kernel<GuideFn, I, O><<<blocks, 256, 0, stream>>>(grid, in, o,       \
                                                                           guide_out, g, npix, fn); \
    return static_cast<int>(cudaGetLastError());                                                \
  }
  HDRNET_PX_CASE(kPxU8, kPxU8)
  HDRNET_PX_CASE(kPxU16, kPxU8)
  HDRNET_PX_CASE(kPxF32, kPxU8)
  HDRNET_PX_CASE(kPxU8, kPxF32)
  HDRNET_PX_CASE(kPxU16, kPxF32)
  HDRNET_PX_CASE(kPxU8, kPxU16)
  HDRNET_PX_CASE(kPxU16, kPxU16)
  HDRNET_PX_CASE(kPxF32, kPxU16)
#undef HDRNET_PX_CASE
  return HDRNET_E_UNSUPPORTED;
}

// Which kernels one slice-apply call runs.  plan_slice_apply is the only place that decides it: the
// launcher runs what it returns, and hdrnet_slice_apply_plan_ws reports it.
struct ApplyForm {
  int variant;        // HDRNET_VARIANT_GENERIC, _TMA, _TEX or _TEX_ASYNC
  TmaPlan p;          // the row kernels' plan
  bool pre_pass;      // texture-assisted forms: yblend_rows_kernel writes the slab rows first ...
  bool slab_warp;     // ... or (issuer-warp form) a slab warp inside the kernel blends them
  bool lean;          // issuer-warp form: index arithmetic per quad (x cells at least 4 pixels wide)
  bool fused_async;   // texture-assisted, fused curves guide: the issuer-warp form
  bool rows_any;      // GENERIC: the any-shape row kernel, else one thread per pixel
  int ctas, threads;  // launch of the main kernel
  size_t smem_bytes;
};

// g, n_in / n_out / has_offset, the guide mode and pixel formats of GuideSpec; aligned: every buffer
// the call passes is 16-byte aligned; ws_base / ws_bytes: address and size of the lent workspace (0
// without one).  HDRNET_E_UNSUPPORTED when a forced variant cannot run the call, or a float32
// fused-guide call has no row-kernel form (the caller then runs the guide kernel first).
static int plan_slice_apply(const SliceGeom& g, int n_in, int n_out, int has_offset, int mode, int in_fmt,
                            int out_fmt, bool aligned, uintptr_t ws_base, size_t ws_bytes, int variant,
                            ApplyForm* f) {
  const int sms = device_sm_count();
  const int max_smem = device_max_smem_optin();
  const bool px = in_fmt != kPxF32 || out_fmt != kPxF32;
  const long long npix = static_cast<long long>(g.B) * g.rows * g.W;
  *f = ApplyForm{};

  // The persistent row kernels take the 3 -> 3 affine op with offset on 16-byte aligned, bulk-copy
  // sized rows, with (u8 | u16) -> (u8 | u16) or f32 -> f32 pixels; everything else runs a generic
  // kernel.
  TmaPlan plan;
  const bool row_shape = n_in == 3 && n_out == 3 && has_offset && aligned &&
                         (!px || (in_fmt != kPxF32 && (out_fmt == kPxU8 || out_fmt == kPxU16))) &&
                         make_tma_plan(g, max_smem, sms, &plan, false, kTmaThreads, in_fmt, out_fmt);
  // Texture-assisted forms: possible when the caller lent a workspace for the slab rows, at the
  // texture alignment.
  const bool tex_ok = row_shape && ws_base != 0 && ws_base % device_texture_alignment() == 0 &&
                      ws_bytes >= static_cast<size_t>(g.B) * g.rows * plan.row_floats * sizeof(float) &&
                      ws_bytes / 16 <= (1u << 27);
  // Issuer-warp form: float32 pixels, guide as an input, two CTAs per SM.
  TmaPlan aplan, splan;
  const bool async_ok = tex_ok && mode == 0 && !px &&
                        make_tma_plan(g, max_smem, sms, &aplan, true, kAsyncThreads - 32) &&
                        aplan.resident == 2 && aplan.seg_px <= aplan.threads * 4;
  // ... with a SLAB WARP that blends each row's slab inside the kernel (no pre-pass launch): needs
  // two more grid rows of shared memory next to the two slab rows, and still a ring of >= 3 stages,
  // and workspace rows that are whole 128-byte cache lines (row bytes and base): a CTA fetches a
  // workspace row through the texture path only after its own slab warp wrote it in THIS launch, and
  // the caches start a launch invalid -- but a line shared by rows r and r + 1 would be cached,
  // with row r + 1's bytes of the previous call, when row r is fetched (seen: 252-float rows)
  const bool slab_lines = (static_cast<size_t>(plan.row_floats) * sizeof(float)) % 128 == 0 && ws_base % 128 == 0;
  const bool slab_warp = async_ok && slab_lines &&
                         make_tma_plan(g, max_smem, sms, &splan, true, kAsyncThreads - 32, kPxF32, kPxF32, 2) &&
                         splan.resident == 2 && splan.seg_px <= splan.threads * 4 &&
                         splan.stages >= kAsyncAutoMinStages;

  const bool auto_req = variant == HDRNET_VARIANT_AUTO;
  if (auto_req) {
    // the texture-assisted forms pay a pre-pass launch or a slab warp: large images only
    if (tex_ok && g.W >= 128 && npix >= (1LL << 21))
      variant = (async_ok && aplan.stages >= kAsyncAutoMinStages) ? HDRNET_VARIANT_TEX_ASYNC : HDRNET_VARIANT_TEX;
    else
      variant = (row_shape && g.W >= 128) ? HDRNET_VARIANT_TMA : HDRNET_VARIANT_GENERIC;
  }
  f->variant = variant;

  if (variant == HDRNET_VARIANT_GENERIC) {
    // The float32 fused-guide forms exist only in the row kernels (the caller runs the standalone
    // guide kernel first: see hdrnet_slice_apply_{curves,nn}_f32); integer pixels have a per-pixel
    // fused kernel.  GENERIC on request is the one-thread-per-pixel L2 gather; AUTO takes the
    // any-shape row kernel where it fits.
    if (mode != 0 && !px) return HDRNET_E_UNSUPPORTED;
    const int J = n_in + (has_offset ? 1 : 0);
    const AnyArgs aa{nullptr, nullptr, nullptr, nullptr, g, n_in, n_out, J, n_out * J, g.gw * g.gd * n_out * J};
    const size_t smem = (auto_req && mode == 0) ? rows_any_smem(aa, true, max_smem) : 0;
    f->rows_any = smem != 0;
    f->ctas = f->rows_any ? rows_any_ctas(g, sms) : generic_grid(npix, sms);
    f->threads = f->rows_any ? kAnyThreads : 256;
    f->smem_bytes = smem;
    return HDRNET_OK;
  }
  if (variant == HDRNET_VARIANT_TMA) {
    if (!row_shape) return HDRNET_E_UNSUPPORTED;
    f->p = plan;
  } else if (variant == HDRNET_VARIANT_TEX_ASYNC) {
    if (!async_ok) return HDRNET_E_UNSUPPORTED;
    f->slab_warp = slab_warp;
    f->pre_pass = !slab_warp;
    f->lean = static_cast<long long>(g.W) >= 4LL * g.gw;
    f->p = slab_warp ? splan : aplan;
  } else {   // HDRNET_VARIANT_TEX
    if (!tex_ok) return HDRNET_E_UNSUPPORTED;
    f->pre_pass = true;
    // the fused-guide issuer-warp form (8 math warps + the issuer), for the curves guide only: for
    // the pointwise-NN guide the block-synchronous form was as fast
    TmaPlan fplan;
    f->fused_async = mode == 1 &&
                     make_tma_plan(g, max_smem, sms, &fplan, true, kFusedAsyncMathThreads, in_fmt, out_fmt) &&
                     fplan.resident == kFusedAsyncResident && fplan.stages >= 3;
    // the block-synchronous texture form: 512 threads for the op API, 256 for fused guides.  It holds
    // no slab region, so it fits wherever the row plan does (at twice the row plan's threads too)
    if (f->fused_async) {
      f->p = fplan;
    } else if (!make_tma_plan(g, max_smem, sms, &f->p, true, mode != 0 ? kTmaThreads : kTexThreads, in_fmt, out_fmt)) {
      return HDRNET_E_UNSUPPORTED;
    }
  }
  // launch threads: the issuer-warp forms add the issuer warp, and the slab warp where there is one
  const bool issuer = variant == HDRNET_VARIANT_TEX_ASYNC || f->fused_async;
  f->ctas = f->p.ctas;
  f->threads = f->p.threads + (issuer ? 32 : 0) + (f->slab_warp ? 32 : 0);
  f->smem_bytes = f->p.smem_bytes;
  return HDRNET_OK;
}

// The block-synchronous row kernel for the call's guide source (kTexChunks > 0: texture-assisted).
template <int kTexChunks>
static int launch_block_sync(const TmaArgs& a, const GuideSpec& gs, cudaStream_t stream) {
  if (gs.mode == 1) { GuideCurves fn; fn.p = *gs.curves; return launch_tma<GuideCurves, kTexChunks>(a, fn, stream, gs.in_fmt, gs.out_fmt); }
  if (gs.mode == 2 && gs.nn->feats <= 16) {
    GuideNN<16> fn; fn.p = *gs.nn;
    return launch_tma<GuideNN<16>, kTexChunks>(a, fn, stream, gs.in_fmt, gs.out_fmt);
  }
  if (gs.mode == 2) {
    GuideNN<kMaxGuideFeats> fn; fn.p = *gs.nn;
    return launch_tma<GuideNN<kMaxGuideFeats>, kTexChunks>(a, fn, stream, gs.in_fmt, gs.out_fmt);
  }
  return launch_tma<GuideFromInput, kTexChunks>(a, GuideFromInput{}, stream);
}

static int launch_slice_apply_impl(const float* grid, const GuideSpec& gs, const void* input_v,
                                   void* out_v, int B, int H, int W, int rows, int y_off, int gh,
                                   int gw, int gd, int n_in, int n_out, int has_offset,
                                   int variant, cudaStream_t stream) {
  const float* input = static_cast<const float*>(input_v);   // float32 forms
  float* out = static_cast<float*>(out_v);
  const bool px = gs.in_fmt != kPxF32 || gs.out_fmt != kPxF32;
  if (px) {  // integer pixel I/O: model-path (fused-guide) forms of the 3 -> 3 affine op only
    if (gs.mode == 0 || n_in != 3 || n_out != 3 || !has_offset) return HDRNET_E_UNSUPPORTED;
    if (gs.in_fmt < kPxF32 || gs.in_fmt > kPxU16 || gs.out_fmt < kPxF32 || gs.out_fmt > kPxU16)
      return HDRNET_E_UNSUPPORTED;
  }
  int rc = validate_common(B, H, W, gh, gw, gd);
  if (rc != HDRNET_OK) return rc;
  if (n_in < 1 || n_out < 1 || rows < 0 || y_off < 0 || y_off + rows > H) return HDRNET_E_BAD_SHAPE;
  const long long npix = static_cast<long long>(B) * rows * W;
  if (npix == 0) return HDRNET_OK;
  if (!grid || !input || !out || (gs.mode == 0 && !gs.guide)) return HDRNET_E_NULL_POINTER;
  if (gs.out_fmt == kPxU16) {
    // A uint16 result has its own width (6 bytes per pixel against 3 / 6 / 12 in): written over its
    // input or grid, a segment's store would overwrite pixels or coefficients other threads have not
    // read yet.  These forms do not run in place.
    const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_v), o1 = o0 + static_cast<uintptr_t>(npix) * 6u;
    const uintptr_t i0 = reinterpret_cast<uintptr_t>(input_v),
                    i1 = i0 + static_cast<uintptr_t>(npix) * 3u * px_bytes_per_channel(gs.in_fmt);
    const uintptr_t g0 = reinterpret_cast<uintptr_t>(grid),
                    g1 = g0 + static_cast<uintptr_t>(B) * gh * gw * gd * kGc * sizeof(float);
    if ((o0 < i1 && i0 < o1) || (o0 < g1 && g0 < o1)) return HDRNET_E_UNSUPPORTED;
  }
  const int J = n_in + (has_offset ? 1 : 0);
  const long long grid_floats = static_cast<long long>(gh) * gw * gd * n_out * J;
  if (grid_floats > INT_MAX || static_cast<long long>(rows) * B > INT_MAX / 4) return HDRNET_E_TOO_LARGE;
  if (variant != HDRNET_VARIANT_AUTO && variant != HDRNET_VARIANT_GENERIC && variant != HDRNET_VARIANT_TMA &&
      variant != HDRNET_VARIANT_TEX && variant != HDRNET_VARIANT_TEX_ASYNC)
    return HDRNET_E_UNSUPPORTED;

  const SliceGeom g = make_geom(B, H, W, rows, y_off, gh, gw, gd);
  const bool aligned = aligned16(grid) && aligned16(input) && aligned16(out) &&
                       (gs.mode != 0 || aligned16(gs.guide)) && (gs.guide_out == nullptr || aligned16(gs.guide_out));
  ApplyForm f;
  rc = plan_slice_apply(g, n_in, n_out, has_offset, gs.mode, gs.in_fmt, gs.out_fmt, aligned,
                        reinterpret_cast<uintptr_t>(gs.workspace), gs.workspace_bytes, variant, &f);
  if (rc != HDRNET_OK) return rc;

  if (f.variant == HDRNET_VARIANT_GENERIC) {
    if (px) {   // integer pixel I/O on shapes the row kernel cannot take: the per-pixel fused kernel
      if (gs.mode == 1) { GuideCurves fn; fn.p = *gs.curves;
                          return launch_px_generic(grid, input_v, out_v, gs.guide_out, g, npix, f.ctas, gs.in_fmt, gs.out_fmt, fn, stream); }
      if (gs.nn->feats <= 16) { GuideNN<16> fn; fn.p = *gs.nn;
                                return launch_px_generic(grid, input_v, out_v, gs.guide_out, g, npix, f.ctas, gs.in_fmt, gs.out_fmt, fn, stream); }
      GuideNN<kMaxGuideFeats> fn; fn.p = *gs.nn;
      return launch_px_generic(grid, input_v, out_v, gs.guide_out, g, npix, f.ctas, gs.in_fmt, gs.out_fmt, fn, stream);
    }
    if (f.rows_any) {
      const AnyArgs aa{grid, gs.guide, input, out, g, n_in, n_out, J, n_out * J, gw * gd * n_out * J};
      return launch_rows_any<true>(aa, f.ctas, f.smem_bytes, device_max_smem_optin(), stream);
    }
    slice_generic_kernel<true><<<f.ctas, 256, 0, stream>>>(grid, gs.guide, input, out, g, n_in, n_out, J, npix);
    return static_cast<int>(cudaGetLastError());
  }

  TmaArgs a;
  a.grid = grid; a.guide = gs.guide; a.guide_out = gs.guide_out;
  a.input = static_cast<const unsigned char*>(input_v); a.out = static_cast<unsigned char*>(out_v);
  a.g = g; a.p = f.p; a.slab_tex = 0; a.yslab = nullptr;
  if (f.variant == HDRNET_VARIANT_TMA) return launch_block_sync<0>(a, gs, stream);

  // texture-assisted forms
  a.yslab = gs.workspace;
  cudaEvent_t tex_use = nullptr;
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  cudaGraph_t graph = nullptr;
  if (cudaStreamGetCaptureInfo(stream, &capture, nullptr, &graph) != cudaSuccess) {
    (void)cudaGetLastError();   // the launch below reports what is wrong with the stream
    capture = cudaStreamCaptureStatusNone;
  }
  rc = capture == cudaStreamCaptureStatusActive
           ? graph_slab_texture(gs.workspace, gs.workspace_bytes, graph, &a.slab_tex)
           : get_slab_texture(gs.workspace, gs.workspace_bytes, &a.slab_tex, &tex_use);
  if (rc != 0) return rc;
  if (f.pre_pass) {   // every row's y-pre-blended slab into the workspace
    rc = launch_yblend(grid, gs.workspace, g, f.p.row_floats, stream);
    if (rc != 0) return rc;
  }
  if (f.variant == HDRNET_VARIANT_TEX_ASYNC) {
    a.guide_out = nullptr;
    rc = launch_async_form(a, f.lean, f.slab_warp, stream);
  } else if (f.fused_async) {
    rc = launch_async_fused(a, *gs.curves, gs.in_fmt, gs.out_fmt, stream);
  } else {
    rc = launch_block_sync<kSyncTexChunks>(a, gs, stream);
  }
  // the texture must outlive every kernel that fetches through it (get_slab_texture; a captured
  // call's texture belongs to its graph)
  if (rc == 0 && tex_use && cudaEventRecord(tex_use, stream) != cudaSuccess) rc = static_cast<int>(cudaGetLastError());
  return rc;
}

// Internal launcher shared with the host path (host_path.cu): pixel buffers hold `rows`
// rows per image starting at image row y_off.
int launch_slice_apply(const float* grid, const float* guide, const float* input, float* out,
                       int B, int H, int W, int rows, int y_off, int gh, int gw, int gd,
                       int n_in, int n_out, int has_offset, int variant, cudaStream_t stream) {
  GuideSpec gs{0, guide, nullptr, nullptr, nullptr};
  return launch_slice_apply_impl(grid, gs, input, out, B, H, W, rows, y_off, gh, gw, gd, n_in,
                                 n_out, has_offset, variant, stream);
}

int pack_curves_params(CurvesGuideParams* p, const float* ccm, const float* ccm_bias,
                       const float* shifts, const float* slopes, const float* mix,
                       float mix_bias);
int pack_nn_params(NNGuideParams* p, const float* w1, const float* b1, const float* w2, float b2,
                   int feats);

int launch_slice(const float* grid, const float* guide, float* out, int B, int H, int W, int rows,
                 int y_off, int gh, int gw, int gd, int gc, int variant, cudaStream_t stream) {
  int rc = validate_common(B, H, W, gh, gw, gd);
  if (rc != HDRNET_OK) return rc;
  if (gc < 1 || rows < 0 || y_off < 0 || y_off + rows > H) return HDRNET_E_BAD_SHAPE;
  const long long npix = static_cast<long long>(B) * rows * W;
  if (npix == 0) return HDRNET_OK;
  if (!grid || !guide || !out) return HDRNET_E_NULL_POINTER;
  if (static_cast<long long>(gh) * gw * gd * gc > INT_MAX) return HDRNET_E_TOO_LARGE;
  if (variant != HDRNET_VARIANT_AUTO && variant != HDRNET_VARIANT_GENERIC &&
      variant != HDRNET_VARIANT_TMA)
    return HDRNET_E_UNSUPPORTED;
  const SliceGeom g = make_geom(B, H, W, rows, y_off, gh, gw, gd);
  const int sms = device_sm_count();
  SlicePlan plan;
  const bool tma_shape = gc == kGc && make_slice_plan(g, device_max_smem_optin(), sms, &plan) &&
                         aligned16(grid) && aligned16(guide) && aligned16(out);
  if (variant == HDRNET_VARIANT_TMA && !tma_shape) return HDRNET_E_UNSUPPORTED;
  const bool use_tma = tma_shape && (variant == HDRNET_VARIANT_TMA ||
                                     (variant == HDRNET_VARIANT_AUTO && W >= 128));
  if (use_tma) {
    cudaError_t e = cudaFuncSetAttribute(slice_rows_tma_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         plan.smem_bytes);
    if (e != cudaSuccess) return static_cast<int>(e);
    SliceArgs a;
    a.grid = grid; a.guide = guide; a.out = out; a.g = g; a.p = plan;
    slice_rows_tma_kernel<<<plan.ctas, kSliceThreads, plan.smem_bytes, stream>>>(a);
  } else {
    if (variant == HDRNET_VARIANT_AUTO) {
      const int max_smem = device_max_smem_optin();
      AnyArgs aa{grid, guide, nullptr, out, g, 0, gc, 1, gc, gw * gd * gc};
      const size_t smem = rows_any_smem(aa, false, max_smem);
      if (smem) return launch_rows_any<false>(aa, rows_any_ctas(g, sms), smem, max_smem, stream);
    }
    slice_generic_kernel<false><<<generic_grid(npix, sms), 256, 0, stream>>>(
        grid, guide, nullptr, out, g, 0, 0, gc, npix);
  }
  return static_cast<int>(cudaGetLastError());
}

// Whether a single-image fused-guide call (hdrnet_slice_apply_{curves,nn}_px_ws, B = 1) on these
// shapes and buffers runs a row-kernel form (TMA or texture-assisted: the 4-corner blend of the
// y-pre-blended slab) rather than a per-pixel one: the ragged kernel (slice_apply_ragged.cu) runs
// the same arithmetic per image.  mode: 1 = curves, 2 = pointwise NN.
bool fused_call_runs_row_form(int H, int W, int gh, int gw, int gd, int mode, int in_fmt, int out_fmt,
                              bool aligned) {
  ApplyForm f;
  return plan_slice_apply(make_geom(1, H, W, H, 0, gh, gw, gd), 3, 3, 1, mode, in_fmt, out_fmt, aligned, 0, 0,
                          HDRNET_VARIANT_AUTO, &f) == HDRNET_OK &&
         f.variant != HDRNET_VARIANT_GENERIC;
}

}  // namespace hdrnet_b200

// =========================================================================================
// C-ABI (include/hdrnet_b200.h)
// =========================================================================================
using namespace hdrnet_b200;

extern "C" {

int hdrnet_b200_abi_version(void) { return HDRNET_B200_ABI_VERSION; }

const char* hdrnet_b200_error_string(int code) {
  switch (code) {
    case HDRNET_OK: return "ok";
    case HDRNET_E_NULL_POINTER: return "a required pointer is NULL";
    case HDRNET_E_BAD_SHAPE: return "invalid dimension";
    case HDRNET_E_BAD_CHANNELS: return "grid channels do not match n_out * (n_in + has_offset)";
    case HDRNET_E_TOO_LARGE: return "extent exceeds the kernels' 32-bit index range";
    case HDRNET_E_UNSUPPORTED: return "requested kernel variant cannot run these shapes";
    case HDRNET_E_BAD_CONTEXT: return "invalid or destroyed context or model object, or not its device";
    case HDRNET_E_BAD_MODEL: return "malformed frozen model (magic, version, lengths, shapes or CRC-32C)";
    default: break;
  }
  if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
  return "unknown hdrnet_b200 error";
}

int hdrnet_slice_apply_f32_variant(const float* grid, const float* guide, const float* input,
                                   float* out, int B, int H, int W, int gh, int gw, int gd,
                                   int n_in, int n_out, int has_offset, int variant,
                                   void* stream) {
  return launch_slice_apply(grid, guide, input, out, B, H, W, H, 0, gh, gw, gd, n_in, n_out,
                            has_offset, variant, static_cast<cudaStream_t>(stream));
}

size_t hdrnet_slice_apply_workspace_bytes(int B, int H, int gw, int gd) {
  if (B < 0 || H < 0 || gw < 1 || gd < 1) return 0;
  return static_cast<size_t>(B) * H * gw * gd * kGc * sizeof(float);
}

int hdrnet_slice_apply_f32_ws(const float* grid, const float* guide, const float* input,
                              float* out, int B, int H, int W, int gh, int gw, int gd, int n_in,
                              int n_out, int has_offset, int variant, void* workspace,
                              size_t workspace_bytes, void* stream) {
  GuideSpec gs{0, guide, nullptr, nullptr, nullptr};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  return launch_slice_apply_impl(grid, gs, input, out, B, H, W, H, 0, gh, gw, gd, n_in, n_out,
                                 has_offset, variant, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_rows_f32_ws(const float* grid, const float* guide, const float* input,
                                   float* out, int B, int H, int W, int rows, int y_off, int gh,
                                   int gw, int gd, int n_in, int n_out, int has_offset, int variant,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  GuideSpec gs{0, guide, nullptr, nullptr, nullptr};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  return launch_slice_apply_impl(grid, gs, input, out, B, H, W, rows, y_off, gh, gw, gd, n_in, n_out,
                                 has_offset, variant, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_f32(const float* grid, const float* guide, const float* input,
                           float* out, int B, int H, int W, int gh, int gw, int gd, int n_in,
                           int n_out, int has_offset, void* stream) {
  return launch_slice_apply(grid, guide, input, out, B, H, W, H, 0, gh, gw, gd, n_in, n_out,
                            has_offset, HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
}

// Model-path forms: guide computed per pixel inside the slice-apply kernel (24 B/px).
// Shapes the TMA kernel cannot take fall back to: standalone guide kernel into `guide_out`
// (required in that case) followed by the generic slice-apply.
extern "C" int hdrnet_guide_curves_f32(const float*, float*, long long, const float*, const float*,
                                       const float*, const float*, const float*, float, void*);
extern "C" int hdrnet_guide_nn_f32(const float*, float*, long long, const float*, const float*,
                                   const float*, float, int, void*);

int hdrnet_slice_apply_curves_f32_ws(const float* grid, const float* input, float* out,
                                     float* guide_out, int B, int H, int W, int gh, int gw, int gd,
                                     const float* ccm, const float* ccm_bias, const float* shifts,
                                     const float* slopes, const float* mix, float mix_bias,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  CurvesGuideParams cp;
  int rc = pack_curves_params(&cp, ccm, ccm_bias, shifts, slopes, mix, mix_bias);
  if (rc != HDRNET_OK) return rc;
  GuideSpec gs{1, nullptr, guide_out, &cp, nullptr};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  rc = launch_slice_apply_impl(grid, gs, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                               HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
  if (rc != HDRNET_E_UNSUPPORTED) return rc;
  if (!guide_out) return HDRNET_E_NULL_POINTER;
  rc = hdrnet_guide_curves_f32(input, guide_out, static_cast<long long>(B) * H * W, ccm, ccm_bias,
                               shifts, slopes, mix, mix_bias, stream);
  if (rc != HDRNET_OK) return rc;
  return launch_slice_apply(grid, guide_out, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                            HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_curves_f32(const float* grid, const float* input, float* out,
                                  float* guide_out, int B, int H, int W, int gh, int gw, int gd,
                                  const float* ccm, const float* ccm_bias, const float* shifts,
                                  const float* slopes, const float* mix, float mix_bias,
                                  void* stream) {
  return hdrnet_slice_apply_curves_f32_ws(grid, input, out, guide_out, B, H, W, gh, gw, gd, ccm,
                                          ccm_bias, shifts, slopes, mix, mix_bias, nullptr, 0,
                                          stream);
}

int hdrnet_slice_apply_nn_f32_ws(const float* grid, const float* input, float* out,
                                 float* guide_out, int B, int H, int W, int gh, int gw, int gd,
                                 const float* w1, const float* b1, const float* w2, float b2,
                                 int feats, void* workspace, size_t workspace_bytes, void* stream) {
  NNGuideParams np;
  int rc = pack_nn_params(&np, w1, b1, w2, b2, feats);
  if (rc != HDRNET_OK) return rc;
  GuideSpec gs{2, nullptr, guide_out, nullptr, &np};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  rc = launch_slice_apply_impl(grid, gs, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                               HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
  if (rc != HDRNET_E_UNSUPPORTED) return rc;
  if (!guide_out) return HDRNET_E_NULL_POINTER;
  rc = hdrnet_guide_nn_f32(input, guide_out, static_cast<long long>(B) * H * W, w1, b1, w2, b2,
                           feats, stream);
  if (rc != HDRNET_OK) return rc;
  return launch_slice_apply(grid, guide_out, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                            HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_nn_f32(const float* grid, const float* input, float* out, float* guide_out,
                              int B, int H, int W, int gh, int gw, int gd, const float* w1,
                              const float* b1, const float* w2, float b2, int feats,
                              void* stream) {
  return hdrnet_slice_apply_nn_f32_ws(grid, input, out, guide_out, B, H, W, gh, gw, gd, w1, b1, w2,
                                      b2, feats, nullptr, 0, stream);
}

int hdrnet_slice_apply_curves_px_ws(const float* grid, const void* input, int in_fmt, void* out,
                                    int out_fmt, float* guide_out, int B, int H, int W, int gh,
                                    int gw, int gd, const float* ccm, const float* ccm_bias,
                                    const float* shifts, const float* slopes, const float* mix,
                                    float mix_bias, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  if (in_fmt == HDRNET_PX_F32 && out_fmt == HDRNET_PX_F32)
    return hdrnet_slice_apply_curves_f32_ws(grid, static_cast<const float*>(input),
                                            static_cast<float*>(out), guide_out, B, H, W, gh, gw,
                                            gd, ccm, ccm_bias, shifts, slopes, mix, mix_bias,
                                            workspace, workspace_bytes, stream);
  CurvesGuideParams cp;
  const int rc = pack_curves_params(&cp, ccm, ccm_bias, shifts, slopes, mix, mix_bias);
  if (rc != HDRNET_OK) return rc;
  GuideSpec gs{1, nullptr, guide_out, &cp, nullptr};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  gs.in_fmt = in_fmt;
  gs.out_fmt = out_fmt;
  return launch_slice_apply_impl(grid, gs, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                                 HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_nn_px_ws(const float* grid, const void* input, int in_fmt, void* out,
                                int out_fmt, float* guide_out, int B, int H, int W, int gh, int gw,
                                int gd, const float* w1, const float* b1, const float* w2, float b2,
                                int feats, void* workspace, size_t workspace_bytes, void* stream) {
  if (in_fmt == HDRNET_PX_F32 && out_fmt == HDRNET_PX_F32)
    return hdrnet_slice_apply_nn_f32_ws(grid, static_cast<const float*>(input),
                                        static_cast<float*>(out), guide_out, B, H, W, gh, gw, gd,
                                        w1, b1, w2, b2, feats, workspace, workspace_bytes, stream);
  NNGuideParams np;
  const int rc = pack_nn_params(&np, w1, b1, w2, b2, feats);
  if (rc != HDRNET_OK) return rc;
  GuideSpec gs{2, nullptr, guide_out, nullptr, &np};
  gs.workspace = static_cast<float*>(workspace);
  gs.workspace_bytes = workspace_bytes;
  gs.in_fmt = in_fmt;
  gs.out_fmt = out_fmt;
  return launch_slice_apply_impl(grid, gs, input, out, B, H, W, H, 0, gh, gw, gd, 3, 3, 1,
                                 HDRNET_VARIANT_AUTO, static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_f32_variant(const float* grid, const float* guide, float* out, int B, int H,
                             int W, int gh, int gw, int gd, int gc, int variant, void* stream) {
  return launch_slice(grid, guide, out, B, H, W, H, 0, gh, gw, gd, gc, variant,
                      static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_f32(const float* grid, const float* guide, float* out, int B, int H, int W,
                     int gh, int gw, int gd, int gc, void* stream) {
  return launch_slice(grid, guide, out, B, H, W, H, 0, gh, gw, gd, gc, HDRNET_VARIANT_AUTO,
                      static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_indices_i32(const float* guide, int32_t* idx, int B, int H, int W, int gh,
                             int gw, int gd, void* stream) {
  int rc = validate_common(B, H, W, gh, gw, gd);
  if (rc != HDRNET_OK) return rc;
  const long long npix = static_cast<long long>(B) * H * W;
  if (npix == 0) return HDRNET_OK;
  if (!guide || !idx) return HDRNET_E_NULL_POINTER;
  const SliceGeom g = make_geom(B, H, W, H, 0, gh, gw, gd);
  slice_indices_kernel<<<generic_grid(npix, device_sm_count()), 256, 0,
                         static_cast<cudaStream_t>(stream)>>>(guide, idx, g, npix);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_slice_apply_plan_ws(int B, int H, int W, int gh, int gw, int gd, int n_in, int n_out,
                               int has_offset, int with_workspace, int* variant, int* ctas,
                               int* threads, int* smem_bytes) {
  int rc = validate_common(B, H, W, gh, gw, gd);
  if (rc != HDRNET_OK) return rc;
  // the call described: AUTO, 16-byte aligned buffers and, with_workspace, a workspace of
  // hdrnet_slice_apply_workspace_bytes at the device's texture alignment
  ApplyForm f;
  rc = plan_slice_apply(make_geom(B, H, W, H, 0, gh, gw, gd), n_in, n_out, has_offset, 0, kPxF32, kPxF32, true,
                        with_workspace ? static_cast<uintptr_t>(device_texture_alignment()) : 0,
                        with_workspace ? hdrnet_slice_apply_workspace_bytes(B, H, gw, gd) : 0,
                        HDRNET_VARIANT_AUTO, &f);
  if (rc != HDRNET_OK) return rc;
  if (variant) *variant = f.variant;
  if (ctas) *ctas = f.ctas;
  if (threads) *threads = f.threads;
  if (smem_bytes) *smem_bytes = static_cast<int>(f.smem_bytes);
  return HDRNET_OK;
}

int hdrnet_slice_apply_plan(int B, int H, int W, int gh, int gw, int gd, int n_in, int n_out,
                            int has_offset, int* variant, int* ctas, int* threads,
                            int* smem_bytes) {
  return hdrnet_slice_apply_plan_ws(B, H, W, gh, gw, gd, n_in, n_out, has_offset, 0, variant, ctas,
                                    threads, smem_bytes);
}

}  // extern "C"
