// slice_rows.cuh -- device code and plan / argument structs shared by the persistent row kernels
// of the fused slice-apply (slice_apply.cu: block-synchronous form and host side;
// slice_apply_async.cu: issuer-warp form; slice_apply_variants.cu: the opt-in negative-result
// forms): pixel storage formats, the staged-tile accessors, the 4-corner blend + affine apply,
// the guide sources, one thread's quad of pixels.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "guide.cuh"

namespace hdrnet_b200 {

// =========================================================================================
// Pixel storage formats of the model-path forms (row f-3): the full-resolution image may stay
// in the integer format it was decoded to, and the result may leave as the uint8 the reference
// writes (hdrnet/bin/run.py:145-169 img_as_float; :95 uint8(255 * clip(out, 0, 1))).
// =========================================================================================
constexpr int kPxF32 = HDRNET_PX_F32, kPxU8 = HDRNET_PX_U8, kPxU16 = HDRNET_PX_U16;

__host__ __device__ constexpr int px_bytes_per_channel(int fmt) {
  return fmt == kPxU8 ? 1 : (fmt == kPxU16 ? 2 : 4);
}

// skimage.img_as_float: v / 255 (uint8) or v / 65535 (uint16), evaluated in float64 and handed
// to a float32 placeholder.  q0 = v * (1/D) with one Newton correction reproduces that float32
// for EVERY code value (exhaustive check: tests/test_px_gpu.py) at 3 FMA-pipe instructions.
template <int kFmt>
__device__ __forceinline__ float px_to_float(unsigned v) {
  constexpr float D = (kFmt == kPxU8) ? 255.0f : 65535.0f;
  constexpr float R = 1.0f / D;
  const float f = static_cast<float>(v);
  const float q0 = f * R;
  return fmaf(fmaf(-q0, D, f), R, q0);
}

// tf.cast(255.0 * tf.clip_by_value(x, 0, 1), tf.uint8): truncating conversion.
__device__ __forceinline__ unsigned float_to_u8(float x) {
  return __float2uint_rz(255.0f * fminf(fmaxf(x, 0.0f), 1.0f));
}

// One thread's 4 consecutive pixels, from / to a staged tile (shared memory) or global memory.
template <int kFmt>
__device__ __forceinline__ void load_quad(const unsigned char* tile, int q, float (&pr)[4],
                                          float (&pg)[4], float (&pb)[4]) {
  if constexpr (kFmt == kPxF32) {
    const float4* rgb4 = reinterpret_cast<const float4*>(tile) + 3 * q;
    const float4 c0 = rgb4[0], c1 = rgb4[1], c2 = rgb4[2];
    pr[0] = c0.x; pg[0] = c0.y; pb[0] = c0.z; pr[1] = c0.w;
    pg[1] = c1.x; pb[1] = c1.y; pr[2] = c1.z; pg[2] = c1.w;
    pb[2] = c2.x; pr[3] = c2.y; pg[3] = c2.z; pb[3] = c2.w;
  } else if constexpr (kFmt == kPxU8) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(tile) + 3 * q;  // 12 bytes
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    pr[0] = px_to_float<kPxU8>(w0 & 0xffu);         pg[0] = px_to_float<kPxU8>((w0 >> 8) & 0xffu);
    pb[0] = px_to_float<kPxU8>((w0 >> 16) & 0xffu); pr[1] = px_to_float<kPxU8>(w0 >> 24);
    pg[1] = px_to_float<kPxU8>(w1 & 0xffu);         pb[1] = px_to_float<kPxU8>((w1 >> 8) & 0xffu);
    pr[2] = px_to_float<kPxU8>((w1 >> 16) & 0xffu); pg[2] = px_to_float<kPxU8>(w1 >> 24);
    pb[2] = px_to_float<kPxU8>(w2 & 0xffu);         pr[3] = px_to_float<kPxU8>((w2 >> 8) & 0xffu);
    pg[3] = px_to_float<kPxU8>((w2 >> 16) & 0xffu); pb[3] = px_to_float<kPxU8>(w2 >> 24);
  } else {
    const uint2* w = reinterpret_cast<const uint2*>(tile) + 3 * q;        // 24 bytes
    const uint2 w0 = w[0], w1 = w[1], w2 = w[2];
    pr[0] = px_to_float<kPxU16>(w0.x & 0xffffu); pg[0] = px_to_float<kPxU16>(w0.x >> 16);
    pb[0] = px_to_float<kPxU16>(w0.y & 0xffffu); pr[1] = px_to_float<kPxU16>(w0.y >> 16);
    pg[1] = px_to_float<kPxU16>(w1.x & 0xffffu); pb[1] = px_to_float<kPxU16>(w1.x >> 16);
    pr[2] = px_to_float<kPxU16>(w1.y & 0xffffu); pg[2] = px_to_float<kPxU16>(w1.y >> 16);
    pb[2] = px_to_float<kPxU16>(w2.x & 0xffffu); pr[3] = px_to_float<kPxU16>(w2.x >> 16);
    pg[3] = px_to_float<kPxU16>(w2.y & 0xffffu); pb[3] = px_to_float<kPxU16>(w2.y >> 16);
  }
}

template <int kFmt>
__device__ __forceinline__ void store_quad(unsigned char* tile, int q, const float (&o_r)[4],
                                           const float (&o_g)[4], const float (&o_b)[4]) {
  if constexpr (kFmt == kPxF32) {
    float4* rgb4 = reinterpret_cast<float4*>(tile) + 3 * q;
    rgb4[0] = make_float4(o_r[0], o_g[0], o_b[0], o_r[1]);
    rgb4[1] = make_float4(o_g[1], o_b[1], o_r[2], o_g[2]);
    rgb4[2] = make_float4(o_b[2], o_r[3], o_g[3], o_b[3]);
  } else {
    static_assert(kFmt == kPxU8, "results leave as float32 or uint8");
    uint32_t* w = reinterpret_cast<uint32_t*>(tile) + 3 * q;
    w[0] = float_to_u8(o_r[0]) | (float_to_u8(o_g[0]) << 8) | (float_to_u8(o_b[0]) << 16) | (float_to_u8(o_r[1]) << 24);
    w[1] = float_to_u8(o_g[1]) | (float_to_u8(o_b[1]) << 8) | (float_to_u8(o_r[2]) << 16) | (float_to_u8(o_g[2]) << 24);
    w[2] = float_to_u8(o_b[2]) | (float_to_u8(o_r[3]) << 8) | (float_to_u8(o_g[3]) << 16) | (float_to_u8(o_b[3]) << 24);
  }
}

template <int kFmt>
__device__ __forceinline__ float load_channel(const unsigned char* base, long long idx) {
  if constexpr (kFmt == kPxF32) return __ldg(reinterpret_cast<const float*>(base) + idx);
  else if constexpr (kFmt == kPxU8) return px_to_float<kPxU8>(__ldg(base + idx));
  else return px_to_float<kPxU16>(__ldg(reinterpret_cast<const unsigned short*>(base) + idx));
}

// =========================================================================================
// Persistent TMA row kernel: n_in = 3, n_out = 3, has_offset (gc = 12), W % 4 == 0.
// =========================================================================================

constexpr int kTmaThreads = 256;    // all-LSU form, and every form of the block-synchronous kernel with a fused guide
constexpr int kTexThreads = 512;    // block-synchronous texture-assisted form of the op API (64 registers)
constexpr int kAsyncThreads = 352;  // issuer-warp form: 10 math warps + the issuer, two CTAs per SM, 88 registers
// AUTO takes the issuer-warp form only with a ring of >= 3 stages at two CTAs per SM: with the two
// stages that 32x32 grids leave (24 / 48 KB of slab rows) the block-synchronous form was faster.
// Checked on an H100 (tools/ab_lib.py, 4K x 8, medians of interleaved bursts, 400 W card): at
// 16x16x8 the kept form (352 + slab warp, 5 texture chunks) 0.805 ms against 0.827 without the slab
// warp, 0.838 with 4 texture chunks, 0.841 at 512 threads, 0.931 block-synchronous texture form,
// 0.949 all-LSU; at 32x32x16 1.258 against 1.255 (4 chunks), 1.388 (512), 1.370 (block-synchronous).
// The 4-chunk and 512-thread shapes of the issuer-warp form were removed on these numbers.
constexpr int kAsyncAutoMinStages = 3;
constexpr int kAsyncTexChunks = 5;  // corner chunks per pixel through the texture pipe in the issuer-warp form
constexpr int kMaxStages = 8;
constexpr int kSyncTexChunks = 4;   // texture chunks of the block-synchronous forms (and of the fused-guide
                                    // issuer-warp form, which runs their per-pixel code)
constexpr int kGc = 12;

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

struct TmaPlan {
  int ctas;
  int threads;     // threads that process pixels (issuer-warp forms: the math warps)
  int resident;    // CTAs per SM the plan was sized for (1 or 2)
  int stages;
  int nseg;        // segments per row
  int seg_px;      // pixels per segment (multiple of 4, <= 4 * kTmaThreads)
  int row_floats;  // gw * gd * 12
  int smem_bytes;
  // byte offsets into dynamic shared memory
  int off_raw, off_slab, off_stage, stage_bytes;
  int off_grid;    // issuer-warp form with a slab warp: two staged grid rows (else unused)
  // pixel formats: bytes per pixel of the staged input / output tiles, and where the guide and
  // output tiles sit inside a stage (off_out == 0: the result overwrites the input tile)
  int in_bpp, out_bpp, off_guide, off_out;
};

struct TmaArgs {
  const float* grid;
  const float* guide;   // guide input (GuideFromInput), else unused
  float* guide_out;     // optional guide dump for the fused forms, else nullptr
  const unsigned char* input;   // [B * rows][W][3] in the kernel's input pixel format
  unsigned char* out;           // [B * rows][W][3] in the kernel's output pixel format
  cudaTextureObject_t slab_tex;  // kTexChunks > 0: float4 view of the y-pre-blended slab rows
  const float* yslab;            // kTexChunks > 0: [B * rows][gw * gd * 12] slab rows (workspace)
  SliceGeom g;
  TmaPlan p;
};

__device__ __forceinline__ float4 lerp4(float w0, float4 a, float w1, float4 b) {
  return make_float4(fmaf(w1, b.x, w0 * a.x), fmaf(w1, b.y, w0 * a.y), fmaf(w1, b.z, w0 * a.z),
                     fmaf(w1, b.w, w0 * a.w));
}

// One 16-byte chunk (4 coefficients) of a corner vector: from the shared-memory slab through
// the LSU, or -- for the last kTexChunks of the 12 chunks a pixel needs -- from the same slab
// row in global memory through the TEXTURE pipe, the one on-chip gather path that does not
// share the LSU crossbar (tools/ubench/gather_paths.cu: LDS.128 + tex float4 overlap fully).
// kBytes: `off` is a BYTE offset into the slab row (the lean index path) instead of a float one.
template <int kTexChunks, int kChunkId, bool kBytes = false>
__device__ __forceinline__ ulonglong2 corner_chunk(const float* __restrict__ slab,
                                                   cudaTextureObject_t tex, int tex_row, int off) {
  if constexpr (kChunkId >= 12 - kTexChunks) {
    const float4 v = tex1Dfetch<float4>(tex, tex_row + (off >> (kBytes ? 4 : 2)) + (kChunkId % 3));
    ulonglong2 r;
    r.x = pack2(v.x, v.y);
    r.y = pack2(v.z, v.w);
    return r;
  } else if constexpr (kBytes) {
    return reinterpret_cast<const ulonglong2*>(reinterpret_cast<const unsigned char*>(slab) + off)[kChunkId % 3];
  } else {
    return reinterpret_cast<const ulonglong2*>(slab + off)[kChunkId % 3];
  }
}

// Blend the four (x, z) corners of the y-pre-blended slab for one pixel and apply the
// 3x4 affine transform to (r, g, b, 1).
template <int kTexChunks, bool kBytes = false>
__device__ __forceinline__ void blend_apply(const float* __restrict__ slab,
                                            cudaTextureObject_t tex, int tex_row, int o00,
                                            int o01, int o10, int o11, float w00, float w01,
                                            float w10, float w11, float r, float g, float b,
                                            float& out_r, float& out_g, float& out_b) {
  const unsigned long long W00 = pack2(w00, w00), W01 = pack2(w01, w01);
  const unsigned long long W10 = pack2(w10, w10), W11 = pack2(w11, w11);
  // chunk ids: v00 -> 0..2, v01 -> 3..5, v10 -> 6..8, v11 -> 9..11
  const ulonglong2 a0 = corner_chunk<kTexChunks, 0, kBytes>(slab, tex, tex_row, o00);
  const ulonglong2 a1 = corner_chunk<kTexChunks, 1, kBytes>(slab, tex, tex_row, o00);
  const ulonglong2 a2 = corner_chunk<kTexChunks, 2, kBytes>(slab, tex, tex_row, o00);
  const ulonglong2 b0 = corner_chunk<kTexChunks, 3, kBytes>(slab, tex, tex_row, o01);
  const ulonglong2 b1 = corner_chunk<kTexChunks, 4, kBytes>(slab, tex, tex_row, o01);
  const ulonglong2 b2 = corner_chunk<kTexChunks, 5, kBytes>(slab, tex, tex_row, o01);
  const ulonglong2 c0 = corner_chunk<kTexChunks, 6, kBytes>(slab, tex, tex_row, o10);
  const ulonglong2 c1 = corner_chunk<kTexChunks, 7, kBytes>(slab, tex, tex_row, o10);
  const ulonglong2 c2 = corner_chunk<kTexChunks, 8, kBytes>(slab, tex, tex_row, o10);
  const ulonglong2 d0 = corner_chunk<kTexChunks, 9, kBytes>(slab, tex, tex_row, o11);
  const ulonglong2 d1 = corner_chunk<kTexChunks, 10, kBytes>(slab, tex, tex_row, o11);
  const ulonglong2 d2 = corner_chunk<kTexChunks, 11, kBytes>(slab, tex, tex_row, o11);
  unsigned long long acc[6];
  acc[0] = fma2(W11, d0.x, fma2(W10, c0.x, fma2(W01, b0.x, mul2(W00, a0.x))));
  acc[1] = fma2(W11, d0.y, fma2(W10, c0.y, fma2(W01, b0.y, mul2(W00, a0.y))));
  acc[2] = fma2(W11, d1.x, fma2(W10, c1.x, fma2(W01, b1.x, mul2(W00, a1.x))));
  acc[3] = fma2(W11, d1.y, fma2(W10, c1.y, fma2(W01, b1.y, mul2(W00, a1.y))));
  acc[4] = fma2(W11, d2.x, fma2(W10, c2.x, fma2(W01, b2.x, mul2(W00, a2.x))));
  acc[5] = fma2(W11, d2.y, fma2(W10, c2.y, fma2(W01, b2.y, mul2(W00, a2.y))));
  float a0f, a1f, a2f, a3f;
  unpack2(acc[0], a0f, a1f);
  unpack2(acc[1], a2f, a3f);
  out_r = fmaf(a2f, b, fmaf(a1f, g, fmaf(a0f, r, a3f)));
  unpack2(acc[2], a0f, a1f);
  unpack2(acc[3], a2f, a3f);
  out_g = fmaf(a2f, b, fmaf(a1f, g, fmaf(a0f, r, a3f)));
  unpack2(acc[4], a0f, a1f);
  unpack2(acc[5], a2f, a3f);
  out_b = fmaf(a2f, b, fmaf(a1f, g, fmaf(a0f, r, a3f)));
}

// Guide sources.  kFromInput: the op-API form, guide is an input tensor staged by TMA
// (28 B/px).  The fused forms compute the guide from the pixel's RGB in registers
// (24 B/px; the guide map never touches HBM) -- the model path of HDRNetCurves /
// HDRNetPointwiseNNGuide (hdrnet/models.py:43-59).
struct GuideFromInput {
  static constexpr bool kFromInput = true;
  __device__ __forceinline__ float operator()(float, float, float) const { return 0.0f; }
};
struct GuideCurves {
  static constexpr bool kFromInput = false;
  CurvesGuideParams p;
  __device__ __forceinline__ float operator()(float r, float g, float b) const {
    return curves_guide(p, r, g, b);
  }
};
template <int kFeats>
struct GuideNN {
  static constexpr bool kFromInput = false;
  NNGuideParams p;
  __device__ __forceinline__ float operator()(float r, float g, float b) const {
    return nn_guide<kFeats>(p, r, g, b);
  }
};


// One thread's 4 consecutive pixels (quad `q` of a staged segment): guide (staged, or computed
// from RGB), bit-exact cell indices, 4-corner blend + affine apply, result written IN PLACE over
// the RGB tile.  Shared by the block-synchronous and the warp-specialised row kernels.
template <class GuideFn, int kTexChunks, int kIn = kPxF32, int kOut = kPxF32>
__device__ __forceinline__ void process_quad(const TmaArgs& args, const GuideFn& guide_fn,
                                             const unsigned char* in_tile, unsigned char* out_tile,
                                             const unsigned char* guide_tile, const float* slab,
                                             int tex_row, long long row, int x0, int q) {
  constexpr bool kGuideIn = GuideFn::kFromInput;
  const SliceGeom& g = args.g;
  const float gd_f = static_cast<float>(g.gd);
  const int x_stride = g.gd * kGc;
  float pr[4], pg[4], pb[4];
  load_quad<kIn>(in_tile, q, pr, pg, pb);
  float gv[4];
  if (kGuideIn) {
    const float4 gq = lds128(reinterpret_cast<const float4*>(guide_tile) + q);
    gv[0] = gq.x; gv[1] = gq.y; gv[2] = gq.z; gv[3] = gq.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) gv[i] = guide_fn(pr[i], pg[i], pb[i]);
    if (args.guide_out != nullptr) {  // optional dump (hdrnet/bin/run.py --debug)
      const size_t pix = static_cast<size_t>(row) * g.W + x0 + 4 * q;
      *reinterpret_cast<float4*>(args.guide_out + pix) = make_float4(gv[0], gv[1], gv[2], gv[3]);
    }
  }
  float o_r[4], o_g[4], o_b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const Axis ax = spatial_axis(x0 + 4 * q + i, g.scale_x);
    const Axis az = range_axis(gv[i], gd_f);
    const int xo0 = clampi(ax.i0, 0, g.gw - 1) * x_stride;
    const int xo1 = clampi(ax.i0 + 1, 0, g.gw - 1) * x_stride;
    const int zo0 = clampi(az.i0, 0, g.gd - 1) * kGc;
    const int zo1 = clampi(az.i0 + 1, 0, g.gd - 1) * kGc;
    float wz0, wz1;
    smoothed_weights(az.f, wz0, wz1);
    const float wx1 = ax.f, wx0 = 1.0f - ax.f;
    blend_apply<kTexChunks>(slab, args.slab_tex, tex_row, xo0 + zo0, xo0 + zo1, xo1 + zo0,
                            xo1 + zo1, wx0 * wz0, wx0 * wz1, wx1 * wz0, wx1 * wz1, pr[i], pg[i],
                            pb[i], o_r[i], o_g[i], o_b[i]);
  }
  store_quad<kOut>(out_tile, q, o_r, o_g, o_b);
  fence_proxy_async_smem();
}

// Entry points of slice_apply_async.cu (non-template: the arguments select the instantiation).
int launch_async_form(const TmaArgs& a, bool lean, bool slab_warp, cudaStream_t stream);
int launch_async_fused(const TmaArgs& a, const CurvesGuideParams& curves, int in_fmt, int out_fmt,
                       cudaStream_t stream);
// fused-guide issuer-warp form (curves guide only: for the pointwise-NN guide the block-synchronous
// form was as fast, and its issuer-warp form was removed): 8 math warps + the issuer warp, 2 CTAs per
// SM (96 registers); preferred to 6 math warps x 3 CTAs and 10 x 2 (both 80 registers).
constexpr int kFusedAsyncMathThreads = 256;
constexpr int kFusedAsyncResident = 2;

}  // namespace hdrnet_b200
