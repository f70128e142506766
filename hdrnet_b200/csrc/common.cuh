// common.cuh -- shared device helpers for the bilateral-slice kernels (sm_90a).
//
// Numerics contract (SURVEY.md section 7.3, BASELINE.json north_star):
//   * cell-index arithmetic is BIT-EXACT with the reference:
//       gxf = (x + 0.5f) * scale_x,  gx0 = floor(gxf - 0.5f),  scale_x = float(gw) / W
//     (hdrnet/ops/bilateral_slice_apply.cu.cc:51-52, :73-80; jax/bilateral_slice.py:317-327).
//     Every step is an explicitly rounded intrinsic so nvcc cannot contract mul+sub into FMA.
//   * interpolation weights only need <= 1e-5 relative agreement; x/y use the plain tent
//     (numerics.h:53-57), z the smoothed tent max(1 - sqrt(d*d + 1e-8), 0)
//     (numerics.h:83-85, :108-113).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "hdrnet_b200.h"

namespace hdrnet_b200 {

// Geometry shared by every slice kernel.  Pixel buffers (guide / input / out) hold `rows`
// image rows per image starting at image row `y_off` of an image that is `H` rows tall:
// the whole-batch entry points use y_off = 0, rows = H; the host path streams row bands.
struct SliceGeom {
  int B;      // images in the pixel buffers
  int H;      // full image height (defines scale_y)
  int W;      // image width
  int rows;   // rows per image present in the buffers
  int y_off;  // image row of buffer row 0
  int gh, gw, gd;
  float scale_x;  // float(gw) / W   (host float division, as the reference)
  float scale_y;  // float(gh) / H
};

__host__ inline SliceGeom make_geom(int B, int H, int W, int rows, int y_off, int gh, int gw,
                                    int gd) {
  SliceGeom g;
  g.B = B; g.H = H; g.W = W; g.rows = rows; g.y_off = y_off;
  g.gh = gh; g.gw = gw; g.gd = gd;
  g.scale_x = static_cast<float>(gw) / static_cast<float>(W > 0 ? W : 1);
  g.scale_y = static_cast<float>(gh) / static_cast<float>(H > 0 ? H : 1);
  return g;
}

// One axis of the trilinear lookup: lower cell index (unclamped) and fractional position.
struct Axis {
  int i0;    // floor(gf - 0.5f), bit-exact with the reference
  float f;   // (gf - 0.5f) - i0 in [0, 1): the reference's weights are w0 = 1 - f, w1 = f
};

// Spatial axis: integer pixel coordinate -> grid coordinate.
__device__ __forceinline__ Axis spatial_axis(int p, float scale) {
  const float gf = __fmul_rn(__fadd_rn(static_cast<float>(p), 0.5f), scale);
  const float t = __fsub_rn(gf, 0.5f);
  const float fl = floorf(t);
  Axis a;
  a.i0 = static_cast<int>(fl);
  a.f = t - fl;
  return a;
}

// Range axis: guide value -> grid depth coordinate (no 0.5 offset on the guide itself,
// bilateral_slice_apply.cu.cc:75-76).
__device__ __forceinline__ Axis range_axis(float guide, float gd_f) {
  const float gf = __fmul_rn(guide, gd_f);
  const float t = __fsub_rn(gf, 0.5f);
  const float fl = floorf(t);
  Axis a;
  // CUDA's float->int conversion saturates (and maps NaN to 0), so pathological guides --
  // undefined behaviour in the reference's cast -- stay harmless: indices are clamped
  // before use and the weights of far-away cells evaluate to 0.
  a.i0 = static_cast<int>(fl);
  a.f = t - fl;
  return a;
}

// Smoothed tent weights of the two depth corners (numerics.h:108-113): d0 = -f, d1 = 1 - f.
// sqrt.approx (one MUFU op, max relative error 2^-23) instead of the IEEE sqrtf sequence
// (MUFU.RSQ + Newton + slow-path call): the argument is >= 1e-8, always normal.
__device__ __forceinline__ float sqrt_fast(float v) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
}
__device__ __forceinline__ void smoothed_weights(float f, float& w0, float& w1) {
  const float u = 1.0f - f;
  w0 = fmaxf(1.0f - sqrt_fast(fmaf(f, f, 1.0e-8f)), 0.0f);
  w1 = fmaxf(1.0f - sqrt_fast(fmaf(u, u, 1.0e-8f)), 0.0f);
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// One 128-bit shared-memory load that the compiler may not split or rematerialise: under
// register pressure nvcc turned `float4 g = guide4[tid]` into four LDS.32 issued right before
// each use -- 4-way bank conflicted (lanes 16 B apart).
__device__ __forceinline__ float4 lds128(const void* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))));
  return v;
}

// ---- fp32 pairs: two lanes of a 64-bit register pair, each rounded on its own ---------------
// Hopper has no packed fp32 FMA, so a pair op is two scalar FFMA / FMUL.  Both halves use the
// explicitly rounded intrinsics: nvcc may not contract a mul2 into a following fma2, which keeps
// every blend bit-identical to the order written at the call site.
__device__ __forceinline__ unsigned long long pack2(float lo, float hi) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(unsigned long long v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ unsigned long long fma2(unsigned long long a, unsigned long long b,
                                                   unsigned long long c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ unsigned long long mul2(unsigned long long a, unsigned long long b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// ---- programmatic dependent launch (sm_90+); both are no-ops in a grid launched without the
// programmatic-stream-serialization attribute
__device__ __forceinline__ void grid_dependency_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void grid_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ---- mbarrier / TMA bulk-copy PTX wrappers (cp.async.bulk -> SASS UBLKCP) ---------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_wait_addr(uint32_t bar_smem_addr, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar_smem_addr),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes % 16 == 0).
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global bulk copy, tracked by the bulk async-group of the issuing thread.
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src,
                                             uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// Ask the L2 to fetch a span of global memory (no destination): warms it for later loads.
__device__ __forceinline__ void l2_prefetch_bulk(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
// Make this thread's generic-proxy shared-memory writes visible to the async proxy (TMA).
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- L2 eviction priorities (cache-policy operands of the .L2::cache_hint forms) -------------
// evict_first: data touched once (streamed pixels) goes first, so it does not push out lines that
// will be read again soon; evict_last: data written now and read back later in the same launch.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// tma_load_1d / tma_store_1d with an L2 cache policy.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes,
                                             uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
               ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy)
               : "memory");
}
// One 16-byte global store with an L2 cache policy.
__device__ __forceinline__ void st_global_hint(float4* p, const float4& v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
               ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(policy)
               : "memory");
}
// Drop the 128-byte L2 line at p (128-byte aligned) without writing it back: the line's memory
// holds undefined bytes afterwards.  For scratch data no one reads again.
__device__ __forceinline__ void l2_discard_line(const void* p) {
  asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory");
}

}  // namespace hdrnet_b200
