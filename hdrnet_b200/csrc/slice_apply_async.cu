// slice_apply_async.cu -- the issuer-warp form of the texture-assisted row kernel
// (HDRNET_VARIANT_TEX_ASYNC; what AUTO runs for large images when a workspace is lent).
// Shared device code: slice_rows.cuh.  Host dispatch: launch_slice_apply_impl in slice_apply.cu.
#include <cuda_runtime.h>

#include <climits>
#include <cstdint>
#include <cstdlib>

#include "slice_rows.cuh"

namespace hdrnet_b200 {

// =========================================================================================
// Issuer-warp form of the texture-assisted row kernel (HDRNET_VARIANT_TEX_ASYNC).
// =========================================================================================
// What the block-synchronous kernel loses: barrier stalls, and warp instructions per item spent
// outside the pixel body.  After
// every segment's __syncthreads thread 0 runs a SERIAL section (bulk store, wait for the previous
// store, an integer division for the next item, expect_tx, two bulk loads) while its own warp's
// pixels wait -- so warp 0 reaches the next barrier late by that section and the other fifteen
// warps wait for it, every item.  The first warp-specialised form (above) moved the loads to a
// producer warp but left a serial store / wait / arrive section in lane 0 of EVERY math warp.
//
// Here the serial work has a warp of its own and nothing else is synchronous:
//   * warps 0..N-2 are MATH warps.  Per item a warp waits for the stage's TMA barrier (full[s]),
//     processes its 128 pixels in place, and one lane ARRIVES on done[s] -- an mbarrier arrive
//     does not block, the warp goes straight on to the next stage.  No __syncthreads, no bulk
//     copies, no divisions (row / segment are nested loop counters) in a math warp.
//   * warp N-1 (one lane) is the ISSUER: it waits on done[s], issues the segment's ONE bulk store,
//     refills the stage freed one item earlier, and after a row's last segment prefetches the slab
//     row two rows ahead into the buffer that row just released.
// 352 threads = 10 math warps (320 quads = one 1280-pixel segment, a third of a 4K row) + the issuer.
//
// kLean: index arithmetic per QUAD instead of per pixel where the x cells are at least 4 pixels
// wide (W >= 4 gw).  floor(t_i) of the quad's pixels is floor(t_0) or floor(t_0) + 1 (t grows by
// scale_x <= 1/4 per pixel), so one float->int conversion serves four pixels and the cell offsets
// are one of three precomputed values; the depth cell uses F2I.FLOOR + I2FP (one XU-pipe op)
// instead of FRND + F2I (two).  t_i, the fractions and every weight are computed by the same
// rounded operations as spatial_axis / range_axis: results are bitwise those of the other forms.
//
// Tried on this form and removed because they were slower or no faster: results stored by STG.128
// from registers, slab rows blended by the issuer warp from L2, texture fetches software-pipelined
// one pixel ahead, programmatic dependent launch of the pre-pass.

// Which of a pixel's 12 corner chunks -- corner c = 0..3 (v00, v01, v10, v11), part p = 0..2 --
// travel through the texture pipe: the last kTexChunks of the ids 3 c + p.
template <int kTexChunks>
__host__ __device__ constexpr bool chunk_on_tex(int c, int p) { return c * 3 + p >= 12 - kTexChunks; }

template <int kTexChunks, int kC, int kP>
__device__ __forceinline__ ulonglong2 fetch_chunk(const unsigned char* __restrict__ slab_b,
                                                  cudaTextureObject_t tex, int off_b, int tex_idx) {
  if constexpr (chunk_on_tex<kTexChunks>(kC, kP)) {
    const float4 v = tex1Dfetch<float4>(tex, tex_idx + kP);   // tex_idx: texel of the cell's part 0
    ulonglong2 r;
    r.x = pack2(v.x, v.y);
    r.y = pack2(v.z, v.w);
    return r;
  } else {
    return *reinterpret_cast<const ulonglong2*>(slab_b + off_b + 16 * kP);
  }
}

// blend_apply with byte offsets and per-corner texel indices (unused ones are dead code).
template <int kTexChunks>
__device__ __forceinline__ void blend_apply_q(const unsigned char* __restrict__ slab_b,
                                              cudaTextureObject_t tex, const int (&off)[4],
                                              const int (&tix)[4], const float (&w)[4], float r,
                                              float g, float b, float& out_r, float& out_g,
                                              float& out_b) {
  const unsigned long long W00 = pack2(w[0], w[0]), W01 = pack2(w[1], w[1]);
  const unsigned long long W10 = pack2(w[2], w[2]), W11 = pack2(w[3], w[3]);
  const ulonglong2 a0 = fetch_chunk<kTexChunks, 0, 0>(slab_b, tex, off[0], tix[0]);
  const ulonglong2 a1 = fetch_chunk<kTexChunks, 0, 1>(slab_b, tex, off[0], tix[0]);
  const ulonglong2 a2 = fetch_chunk<kTexChunks, 0, 2>(slab_b, tex, off[0], tix[0]);
  const ulonglong2 b0 = fetch_chunk<kTexChunks, 1, 0>(slab_b, tex, off[1], tix[1]);
  const ulonglong2 b1 = fetch_chunk<kTexChunks, 1, 1>(slab_b, tex, off[1], tix[1]);
  const ulonglong2 b2 = fetch_chunk<kTexChunks, 1, 2>(slab_b, tex, off[1], tix[1]);
  const ulonglong2 c0 = fetch_chunk<kTexChunks, 2, 0>(slab_b, tex, off[2], tix[2]);
  const ulonglong2 c1 = fetch_chunk<kTexChunks, 2, 1>(slab_b, tex, off[2], tix[2]);
  const ulonglong2 c2 = fetch_chunk<kTexChunks, 2, 2>(slab_b, tex, off[2], tix[2]);
  const ulonglong2 d0 = fetch_chunk<kTexChunks, 3, 0>(slab_b, tex, off[3], tix[3]);
  const ulonglong2 d1 = fetch_chunk<kTexChunks, 3, 1>(slab_b, tex, off[3], tix[3]);
  const ulonglong2 d2 = fetch_chunk<kTexChunks, 3, 2>(slab_b, tex, off[3], tix[3]);
  unsigned long long acc[6];  // same order of operations as blend_apply: identical bits
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

// tex_base: texel of the row's first cell in the slab workspace (row * gw * gd * 3).
template <int kTexChunks>
__device__ __forceinline__ void process_quad_lean(const TmaArgs& args, const unsigned char* tile,
                                                  unsigned char* out_tile,
                                                  const unsigned char* guide_tile,
                                                  const unsigned char* slab_b, int tex_base, int x0, int q) {
  const SliceGeom& g = args.g;
  const float gd_f = static_cast<float>(g.gd);
  float pr[4], pg[4], pb[4];
  load_quad<kPxF32>(tile, q, pr, pg, pb);
  const float4 gq = lds128(reinterpret_cast<const float4*>(guide_tile) + q);
  const float gv[4] = {gq.x, gq.y, gq.z, gq.w};

  // x axis, once per quad: t_i = (x_i + 0.5f) * scale - 0.5f with the reference's roundings
  // (float(X + i) + 0.5f == float(X) + (i + 0.5f): both exact below 2^22).
  const float xf = static_cast<float>(x0 + 4 * q);
  float tx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    tx[i] = __fsub_rn(__fmul_rn(__fadd_rn(xf, static_cast<float>(i) + 0.5f), g.scale_x), 0.5f);
  const int ix0 = __float2int_rd(tx[0]);
  const float fl0 = static_cast<float>(ix0), fl1 = fl0 + 1.0f;
  // the three x cells a quad can touch, as byte offsets into the slab row (x-major, gd depth cells each)
  const int b0 = clampi(ix0, 0, g.gw - 1) * g.gd * 48;
  const int b1 = clampi(ix0 + 1, 0, g.gw - 1) * g.gd * 48;
  const int b2 = clampi(ix0 + 2, 0, g.gw - 1) * g.gd * 48;

  float o_r[4], o_g[4], o_b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool step = (i > 0) && (tx[i] >= fl1);     // this pixel sits in the next x cell
    const float fx = tx[i] - (step ? fl1 : fl0);
    const int xo0 = step ? b1 : b0;
    const int xo1 = step ? b2 : b1;
    // depth axis (range_axis with one conversion)
    const float tz = __fsub_rn(__fmul_rn(gv[i], gd_f), 0.5f);
    const int iz = __float2int_rd(tz);
    const float fz = tz - static_cast<float>(iz);
    const int zc0 = clampi(iz, 0, g.gd - 1);
    const int zc1 = clampi(iz + 1, 0, g.gd - 1);
    float wz0, wz1;
    smoothed_weights(fz, wz0, wz1);
    const float wx1 = fx, wx0 = 1.0f - fx;
    const int off[4] = {zc0 * 48 + xo0, zc1 * 48 + xo0, zc0 * 48 + xo1, zc1 * 48 + xo1};
    int tix[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) tix[c] = tex_base + (off[c] >> 4);
    const float w[4] = {wx0 * wz0, wx0 * wz1, wx1 * wz0, wx1 * wz1};
    blend_apply_q<kTexChunks>(slab_b, args.slab_tex, off, tix, w, pr[i], pg[i], pb[i], o_r[i], o_g[i], o_b[i]);
  }
  store_quad<kPxF32>(out_tile, q, o_r, o_g, o_b);
  fence_proxy_async_smem();
}

// process_quad_lean for the model-path forms: the guide is COMPUTED from the pixel (curves / pointwise
// NN, guide.cuh) instead of read, pixels arrive and leave in their storage format (f32 / u8 / u16).
// Same per-quad x arithmetic, same rounded operations: bitwise the results of process_quad.
template <class GuideFn, int kTexChunks, int kIn, int kOut>
__device__ __forceinline__ void process_quad_lean_fused(const TmaArgs& args, const GuideFn& guide_fn,
                                                        const unsigned char* in_tile, unsigned char* out_tile,
                                                        const unsigned char* slab_b, int tex_base,
                                                        long long row, int x0, int q) {
  const SliceGeom& g = args.g;
  const float gd_f = static_cast<float>(g.gd);
  float pr[4], pg[4], pb[4];
  load_quad<kIn>(in_tile, q, pr, pg, pb);
  float gv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) gv[i] = guide_fn(pr[i], pg[i], pb[i]);
  if (args.guide_out != nullptr) {  // optional dump (hdrnet/bin/run.py --debug)
    const size_t pix = static_cast<size_t>(row) * g.W + x0 + 4 * q;
    *reinterpret_cast<float4*>(args.guide_out + pix) = make_float4(gv[0], gv[1], gv[2], gv[3]);
  }
  const float xf = static_cast<float>(x0 + 4 * q);
  float tx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    tx[i] = __fsub_rn(__fmul_rn(__fadd_rn(xf, static_cast<float>(i) + 0.5f), g.scale_x), 0.5f);
  const int ix0 = __float2int_rd(tx[0]);
  const float fl0 = static_cast<float>(ix0), fl1 = fl0 + 1.0f;
  const int b0 = clampi(ix0, 0, g.gw - 1) * g.gd * 48;
  const int b1 = clampi(ix0 + 1, 0, g.gw - 1) * g.gd * 48;
  const int b2 = clampi(ix0 + 2, 0, g.gw - 1) * g.gd * 48;
  float o_r[4], o_g[4], o_b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool step = (i > 0) && (tx[i] >= fl1);
    const float fx = tx[i] - (step ? fl1 : fl0);
    const int xo0 = step ? b1 : b0;
    const int xo1 = step ? b2 : b1;
    const float tz = __fsub_rn(__fmul_rn(gv[i], gd_f), 0.5f);
    const int iz = __float2int_rd(tz);
    const float fz = tz - static_cast<float>(iz);
    const int zc0 = clampi(iz, 0, g.gd - 1);
    const int zc1 = clampi(iz + 1, 0, g.gd - 1);
    float wz0, wz1;
    smoothed_weights(fz, wz0, wz1);
    const float wx1 = fx, wx0 = 1.0f - fx;
    const int off[4] = {zc0 * 48 + xo0, zc1 * 48 + xo0, zc0 * 48 + xo1, zc1 * 48 + xo1};
    int tix[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) tix[c] = tex_base + (off[c] >> 4);
    const float w[4] = {wx0 * wz0, wx0 * wz1, wx1 * wz0, wx1 * wz1};
    blend_apply_q<kTexChunks>(slab_b, args.slab_tex, off, tix, w, pr[i], pg[i], pb[i], o_r[i], o_g[i], o_b[i]);
  }
  store_quad<kOut>(out_tile, q, o_r, o_g, o_b);
  fence_proxy_async_smem();
}

// kSlabWarp: one more warp blends each image row's slab INSIDE the kernel, two rows ahead of the math
// warps -- from the two grid rows it keeps staged in shared memory (TMA, reloaded only when the pair
// changes) into (i) the shared-memory slab buffer the LSU chunks are read from and (ii) the row's
// place in the caller's workspace, from where the texture chunks are fetched a row later.  The
// separate pre-pass launch and the slab-row bulk loads
// disappear.  A CTA only ever fetches workspace rows its own slab warp wrote earlier in this launch
// (a row split between two CTAs is written by both, with identical bytes), after a device-scope
// fence and the slab barrier; L1 / texture caches start a launch invalid, so no stale line of an
// earlier call can be hit.
template <int kTexChunks, bool kLean, int kThreads, int kMinBlocks, bool kSlabWarp>
__global__ void __launch_bounds__(kThreads, kMinBlocks)
slice_apply_rows_async_kernel(const TmaArgs args) {
  static_assert(kTexChunks > 0, "the issuer-warp kernel serves part of the gather by texture");
  constexpr int kMathWarps = kThreads / 32 - 1 - (kSlabWarp ? 1 : 0);
  extern __shared__ __align__(128) unsigned char smem[];
  const SliceGeom& g = args.g;
  const TmaPlan& pl = args.p;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);   // [kMaxStages]  TMA landed
  uint64_t* done = full + kMaxStages;                    // [kMaxStages]  every math warp is through
  uint64_t* slab_full = done + kMaxStages;               // [2]
  uint64_t* row_free = slab_full + 2;                    // [2]  kSlabWarp: the row's slab buffer may be rewritten
  uint64_t* grid_full = row_free + 2;                    // [2]  kSlabWarp: a staged grid row landed
  unsigned char* raw0 = smem + pl.off_raw;               // two slab rows
  unsigned char* stage_base = smem + pl.off_stage;

  // Work split in ITEMS (row segments), not rows: 17280 rows (4K x 8) over 264 CTAs give 120 CTAs
  // 66 rows and 144 CTAs 65, a tail of one whole row; in half-row items the tail is half a row.
  // A CTA covers items [i_begin, i_end): rows r_begin .. r_end-1, the first row from pixel
  // x_first, the last row up to pixel x_last (a row split between two CTAs has its slab row
  // loaded by both).
  const long long total_items = static_cast<long long>(g.B) * g.rows * pl.nseg;
  const long long i_begin = total_items * blockIdx.x / gridDim.x;
  const long long i_end = total_items * (blockIdx.x + 1) / gridDim.x;
  if (i_end <= i_begin) return;
  const long long r_begin = i_begin / pl.nseg, r_end = (i_end - 1) / pl.nseg + 1;
  const int x_first = static_cast<int>(i_begin - r_begin * pl.nseg) * pl.seg_px;
  const int x_last = min(g.W, (static_cast<int>((i_end - 1) - (r_end - 1) * pl.nseg) + 1) * pl.seg_px);
  auto row_x0 = [&](long long row) { return row == r_begin ? x_first : 0; };
  auto row_x1 = [&](long long row) { return row == r_end - 1 ? x_last : g.W; };

  if (tid == 0) {
    for (int s = 0; s < pl.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], kMathWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&slab_full[i], 1); mbar_init(&row_free[i], 1); mbar_init(&grid_full[i], 1); }
    fence_mbar_init();
  }
  __syncthreads();  // the only block-wide barrier

  const int NS = pl.stages;
  const uint32_t slab_bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
  auto arrive = [&](uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
  };

  if (kSlabWarp && warp == kMathWarps + 1) {
    // -------------------------------- slab warp ---------------------------------------------
    float* graw = reinterpret_cast<float*>(smem + pl.off_grid);   // two staged grid rows
    const int gstride = (static_cast<int>(slab_bytes) + 127) / 128 * 32;   // floats between the two slots
    int key0 = -1, key1 = -1;          // grid row (b * gh + gy) held by slot 0 / 1
    uint32_t gpar0 = 0u, gpar1 = 0u;
    const int n4 = pl.row_floats / 4;
    float4* ws4 = reinterpret_cast<float4*>(const_cast<float*>(args.yslab));
    const uint64_t ws_pol = l2_policy_evict_last();
    // Once the issuer has released a row every texture fetch of it has returned: a row this CTA
    // owns whole (no other CTA fetches it) is dropped from L2 without a write-back to HBM.  Rows
    // are whole 128-byte lines (slab_lines in launch_slice_apply_impl); the workspace's contents
    // are undefined after the call.
    auto discard_row = [&](long long r) {
      if (row_x0(r) != 0 || row_x1(r) != g.W) return;
      const unsigned char* base = reinterpret_cast<const unsigned char*>(ws4 + static_cast<size_t>(r) * n4);
      for (int l = lane; l < static_cast<int>(slab_bytes / 128u); l += 32) l2_discard_line(base + 128 * l);
    };
    for (long long row = r_begin; row < r_end; ++row) {
      const int rowk = static_cast<int>(row - r_begin), rb = rowk & 1;
      const int b = static_cast<int>(row / g.rows);
      const int y = g.y_off + static_cast<int>(row - static_cast<long long>(b) * g.rows);
      const Axis ay = spatial_axis(y, g.scale_y);
      const int k0 = b * g.gh + clampi(ay.i0, 0, g.gh - 1);
      const int k1 = b * g.gh + clampi(ay.i0 + 1, 0, g.gh - 1);
      int s0 = (key0 == k0) ? 0 : ((key1 == k0) ? 1 : -1);
      int s1 = (key0 == k1) ? 0 : ((key1 == k1) ? 1 : -1);
      auto fetch = [&](int slot, int k) {   // grid row k -> slot (warp-uniform); the warp itself is the only reader
        if (lane == 0) {
          mbar_expect_tx(&grid_full[slot], slab_bytes);
          tma_load_1d(graw + slot * gstride, args.grid + static_cast<size_t>(k) * pl.row_floats, slab_bytes,
                      &grid_full[slot]);
        }
        if (slot == 0) { key0 = k; mbar_wait(&grid_full[0], gpar0); gpar0 ^= 1u; }
        else { key1 = k; mbar_wait(&grid_full[1], gpar1); gpar1 ^= 1u; }
      };
      __syncwarp();   // every lane is done reading the slot a load may overwrite
      if (s0 < 0) { s0 = (s1 == 0) ? 1 : 0; fetch(s0, k0); if (k1 == k0) s1 = s0; }
      if (s1 < 0) { s1 = s0 ^ 1; fetch(s1, k1); }
      // the slab buffer of row - 2 is free once the issuer has seen that row's last item done
      if (rowk >= 2) mbar_wait(&row_free[rb], static_cast<uint32_t>((rowk >> 1) - 1) & 1u);
      const float wy1 = ay.f, wy0 = 1.0f - ay.f;
      const float4* a4 = reinterpret_cast<const float4*>(graw + s0 * gstride);
      const float4* b4 = reinterpret_cast<const float4*>(graw + s1 * gstride);
      float4* slab4 = reinterpret_cast<float4*>(raw0 + static_cast<size_t>(rb) * slab_bytes);
      float4* wrow = ws4 + static_cast<size_t>(row) * n4;
      for (int e = lane; e < n4; e += 32) {   // exactly yblend_rows_kernel's arithmetic
        const float4 v = lerp4(wy0, a4[e], wy1, b4[e]);
        slab4[e] = v;
        st_global_hint(wrow + e, v, ws_pol);   // kept in L2 until the texture chunks have read it
      }
      __threadfence();   // the workspace row is visible device-wide before anyone is told it exists
      __syncwarp();
      if (lane == 0) arrive(&slab_full[rb]);
      if (rowk >= 2) discard_row(row - 2);   // released: waited on row_free above
    }
    for (long long row = max(r_begin, r_end - 2); row < r_end; ++row) {   // the last two rows
      const int rowk = static_cast<int>(row - r_begin);
      mbar_wait(&row_free[rowk & 1], static_cast<uint32_t>(rowk >> 1) & 1u);
      discard_row(row);
    }
    return;
  }

  if (warp == kMathWarps) {
    // ------------------------------- issuer warp --------------------------------------------
    // Lane 0 issues every bulk copy.  Pixels are touched once: evict_first keeps them from pushing
    // the slab rows out of L2 between their write and their texture fetches.
    if (lane != 0) return;
    const uint64_t px_pol = l2_policy_evict_first();
    auto make_slab = [&](long long row) {   // the row's y-pre-blended slab, from the pre-pass workspace
      if constexpr (kSlabWarp) return;
      const int rb = static_cast<int>(row - r_begin) & 1;
      mbar_expect_tx(&slab_full[rb], slab_bytes);
      tma_load_1d(raw0 + static_cast<size_t>(rb) * slab_bytes,
                  args.yslab + static_cast<size_t>(row) * pl.row_floats, slab_bytes, &slab_full[rb]);
    };
    // load cursor: runs NS - 1 items ahead of the math warps
    long long l_row = r_begin;
    int l_x0 = x_first, l_s = 0;
    auto issue_next_load = [&]() {
      if (l_row >= r_end) return;
      const int npx = min(pl.seg_px, g.W - l_x0);
      unsigned char* st = stage_base + static_cast<size_t>(l_s) * pl.stage_bytes;
      const size_t pix = static_cast<size_t>(l_row) * g.W + l_x0;
      mbar_expect_tx(&full[l_s], static_cast<uint32_t>(npx) * 16u);
      tma_load_1d(st, args.input + pix * 12, static_cast<uint32_t>(npx) * 12u, &full[l_s], px_pol);
      tma_load_1d(st + pl.off_guide, args.guide + pix, static_cast<uint32_t>(npx) * 4u, &full[l_s], px_pol);
      if (++l_s == NS) l_s = 0;
      l_x0 += pl.seg_px;
      if (l_x0 >= row_x1(l_row)) { l_x0 = 0; ++l_row; }
    };
    // the stage refilled after item i is item i-1's (its bulk store must have drained)
    for (int i = 0; i < NS - 1; ++i) issue_next_load();
    make_slab(r_begin);
    if (r_begin + 1 < r_end) make_slab(r_begin + 1);

    int s = 0;
    uint32_t ph = 0;
    for (long long row = r_begin; row < r_end; ++row) {
      const int x_end = row_x1(row);
      for (int x0 = row_x0(row); x0 < x_end; x0 += pl.seg_px) {
        mbar_wait(&done[s], ph);  // every math warp is through with this stage (results written in place, proxy-fenced)
        const int npx = min(pl.seg_px, g.W - x0);
        unsigned char* st = stage_base + static_cast<size_t>(s) * pl.stage_bytes;
        const size_t pix = static_cast<size_t>(row) * g.W + x0;
        tma_store_1d(args.out + pix * 12, st, static_cast<uint32_t>(npx) * 12u, px_pol);
        tma_store_commit();
        if (l_row < r_end) {
          tma_store_wait_read<1>();  // the previous item's store has drained the stage refilled now
          issue_next_load();
        }
        if (++s == NS) { s = 0; ph ^= 1u; }
      }
      // the row's slab buffer is free: every math warp arrived after its last read of it
      if constexpr (kSlabWarp) arrive(&row_free[static_cast<int>(row - r_begin) & 1]);
      else if (row + 2 < r_end) make_slab(row + 2);
    }
    tma_store_wait_all<0>();
    return;
  }

  // --------------------------------- math warps ---------------------------------------------
  const int q = warp * 32 + lane;  // this thread's quad inside a segment
  const int cells = g.gw * g.gd;
  int s = 0;
  uint32_t ph = 0;
  for (long long row = r_begin; row < r_end; ++row) {
    const int rowk = static_cast<int>(row - r_begin), rb = rowk & 1;
    mbar_wait(&slab_full[rb], static_cast<uint32_t>(rowk >> 1) & 1u);
    const unsigned char* slab_b = raw0 + static_cast<size_t>(rb) * slab_bytes;
    const int tex_base = static_cast<int>(row) * cells * 3;
    const int x_end = row_x1(row);
    for (int x0 = row_x0(row); x0 < x_end; x0 += pl.seg_px) {
      const int npx = min(pl.seg_px, g.W - x0);
      unsigned char* st = stage_base + static_cast<size_t>(s) * pl.stage_bytes;
      mbar_wait(&full[s], ph);
      if (q * 4 < npx) {
        if constexpr (kLean)
          process_quad_lean<kTexChunks>(args, st, st, st + pl.off_guide, slab_b, tex_base, x0, q);
        else
          process_quad<GuideFromInput, kTexChunks>(args, GuideFromInput{}, st, st, st + pl.off_guide,
                                                   reinterpret_cast<const float*>(slab_b), tex_base,
                                                   row, x0, q);
      }
      __syncwarp();
      if (lane == 0) arrive(&done[s]);
      if (++s == NS) { s = 0; ph ^= 1u; }
    }
  }
}

template <bool kLean, bool kSlabWarp>
static int launch_async(const TmaArgs& a, cudaStream_t stream) {
  constexpr int kLaunchThreads = kAsyncThreads + (kSlabWarp ? 32 : 0);   // + the slab warp
  auto kern = slice_apply_rows_async_kernel<kAsyncTexChunks, kLean, kLaunchThreads, 2, kSlabWarp>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, a.p.smem_bytes);
  if (e != cudaSuccess) return static_cast<int>(e);
  kern<<<a.p.ctas, kLaunchThreads, a.p.smem_bytes, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

int launch_async_form(const TmaArgs& a, bool lean, bool slab_warp, cudaStream_t stream) {
  if (slab_warp) return lean ? launch_async<true, true>(a, stream) : launch_async<false, true>(a, stream);
  return lean ? launch_async<true, false>(a, stream) : launch_async<false, false>(a, stream);
}

// =========================================================================================
// Issuer-warp control flow for the FUSED-GUIDE (model path) forms.
// =========================================================================================
// HDRNetCurves computes the guide from the pixel's RGB in registers (24 B/px, models.py:43-59) and
// may read / write integer pixels.  This is the block-synchronous
// kernel's per-pixel code (slice_apply.cu, process_quad:
// identical bits) under the issuer-warp control flow above: math warps that only wait for their
// stage and ARRIVE on done[s], one warp that issues every bulk copy.  8 math warps + the issuer
// (288 threads, 112 registers at two CTAs per SM: the fused forms are issue-bound and want their
// registers), texture chunks as the block-synchronous fused form (4).
constexpr int kFusedAsyncThreads = kFusedAsyncMathThreads + 32;

template <class GuideFn, int kTexChunks, int kIn, int kOut>
__global__ void __launch_bounds__(kFusedAsyncThreads, kFusedAsyncResident)
slice_apply_rows_async_fused_kernel(const TmaArgs args, const __grid_constant__ GuideFn guide_fn) {
  static_assert(!GuideFn::kFromInput, "fused-guide forms only");
  constexpr int kMathWarps = kFusedAsyncThreads / 32 - 1;
  constexpr uint32_t kInBpp = 3u * px_bytes_per_channel(kIn), kOutBpp = 3u * px_bytes_per_channel(kOut);
  extern __shared__ __align__(128) unsigned char smem[];
  const SliceGeom& g = args.g;
  const TmaPlan& pl = args.p;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* done = full + kMaxStages;
  uint64_t* slab_full = done + kMaxStages;
  unsigned char* raw0 = smem + pl.off_raw;
  unsigned char* stage_base = smem + pl.off_stage;

  const long long total_items = static_cast<long long>(g.B) * g.rows * pl.nseg;
  const long long i_begin = total_items * blockIdx.x / gridDim.x;
  const long long i_end = total_items * (blockIdx.x + 1) / gridDim.x;
  if (i_end <= i_begin) return;
  const long long r_begin = i_begin / pl.nseg, r_end = (i_end - 1) / pl.nseg + 1;
  const int x_first = static_cast<int>(i_begin - r_begin * pl.nseg) * pl.seg_px;
  const int x_last = min(g.W, (static_cast<int>((i_end - 1) - (r_end - 1) * pl.nseg) + 1) * pl.seg_px);
  auto row_x0 = [&](long long row) { return row == r_begin ? x_first : 0; };
  auto row_x1 = [&](long long row) { return row == r_end - 1 ? x_last : g.W; };

  if (tid == 0) {
    for (int s = 0; s < pl.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], kMathWarps); }
    mbar_init(&slab_full[0], 1);
    mbar_init(&slab_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int NS = pl.stages;
  const uint32_t slab_bytes = static_cast<uint32_t>(pl.row_floats) * 4u;
  // same pixel size in and out: the result overwrites the input tile (plan.off_out == 0)
  auto stage_out = [&](unsigned char* st) { return st + (kInBpp == kOutBpp ? 0 : pl.off_out); };

  if (warp == kMathWarps) {
    // ------------------------------- issuer (lane 0) ----------------------------------------
    if (lane != 0) return;
    auto load_slab = [&](long long row) {
      const int rb = static_cast<int>(row - r_begin) & 1;
      mbar_expect_tx(&slab_full[rb], slab_bytes);
      tma_load_1d(raw0 + static_cast<size_t>(rb) * slab_bytes,
                  args.yslab + static_cast<size_t>(row) * pl.row_floats, slab_bytes, &slab_full[rb]);
    };
    long long l_row = r_begin;
    int l_x0 = x_first, l_s = 0;
    auto issue_next_load = [&]() {
      if (l_row >= r_end) return;
      const int npx = min(pl.seg_px, g.W - l_x0);
      unsigned char* st = stage_base + static_cast<size_t>(l_s) * pl.stage_bytes;
      const size_t pix = static_cast<size_t>(l_row) * g.W + l_x0;
      mbar_expect_tx(&full[l_s], static_cast<uint32_t>(npx) * kInBpp);
      tma_load_1d(st, args.input + pix * kInBpp, static_cast<uint32_t>(npx) * kInBpp, &full[l_s]);
      if (++l_s == NS) l_s = 0;
      l_x0 += pl.seg_px;
      if (l_x0 >= row_x1(l_row)) { l_x0 = 0; ++l_row; }
    };
    for (int i = 0; i < NS - 1; ++i) issue_next_load();
    load_slab(r_begin);
    if (r_begin + 1 < r_end) load_slab(r_begin + 1);
    int s = 0;
    uint32_t ph = 0;
    for (long long row = r_begin; row < r_end; ++row) {
      const int x_end = row_x1(row);
      for (int x0 = row_x0(row); x0 < x_end; x0 += pl.seg_px) {
        mbar_wait(&done[s], ph);
        const int npx = min(pl.seg_px, g.W - x0);
        unsigned char* st = stage_base + static_cast<size_t>(s) * pl.stage_bytes;
        const size_t pix = static_cast<size_t>(row) * g.W + x0;
        tma_store_1d(args.out + pix * kOutBpp, stage_out(st), static_cast<uint32_t>(npx) * kOutBpp);
        tma_store_commit();
        if (l_row < r_end) {
          tma_store_wait_read<1>();
          issue_next_load();
        }
        if (++s == NS) { s = 0; ph ^= 1u; }
      }
      if (row + 2 < r_end) load_slab(row + 2);
    }
    tma_store_wait_all<0>();
    return;
  }

  // --------------------------------- math warps ---------------------------------------------
  const int q = warp * 32 + lane;
  int s = 0;
  uint32_t ph = 0;
  for (long long row = r_begin; row < r_end; ++row) {
    const int rowk = static_cast<int>(row - r_begin), rb = rowk & 1;
    mbar_wait(&slab_full[rb], static_cast<uint32_t>(rowk >> 1) & 1u);
    const float* slab = reinterpret_cast<const float*>(raw0 + static_cast<size_t>(rb) * slab_bytes);
    const int tex_row = static_cast<int>(row) * (pl.row_floats / 4);
    const int x_end = row_x1(row);
    for (int x0 = row_x0(row); x0 < x_end; x0 += pl.seg_px) {
      const int npx = min(pl.seg_px, g.W - x0);
      unsigned char* st = stage_base + static_cast<size_t>(s) * pl.stage_bytes;
      mbar_wait(&full[s], ph);
      if (q * 4 < npx)   // per-quad x arithmetic: -2.6 % for the curves guide against process_quad, same bits
        process_quad_lean_fused<GuideFn, kTexChunks, kIn, kOut>(args, guide_fn, st, stage_out(st),
                                                                reinterpret_cast<const unsigned char*>(slab),
                                                                tex_row, row, x0, q);
      __syncwarp();
      if (lane == 0)
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&done[s])) : "memory");
      if (++s == NS) { s = 0; ph ^= 1u; }
    }
  }
}

template <int kIn, int kOut>
static int launch_async_fused_fmt(const TmaArgs& a, const GuideCurves& fn, cudaStream_t stream) {
  auto kern = slice_apply_rows_async_fused_kernel<GuideCurves, kSyncTexChunks, kIn, kOut>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, a.p.smem_bytes);
  if (e != cudaSuccess) return static_cast<int>(e);
  kern<<<a.p.ctas, kFusedAsyncThreads, a.p.smem_bytes, stream>>>(a, fn);
  return static_cast<int>(cudaGetLastError());
}

// plan: (kFusedAsyncThreads - 32) quads per segment
int launch_async_fused(const TmaArgs& a, const CurvesGuideParams& curves, int in_fmt, int out_fmt,
                       cudaStream_t stream) {
  GuideCurves fn;
  fn.p = curves;
  if (in_fmt == kPxF32 && out_fmt == kPxF32) return launch_async_fused_fmt<kPxF32, kPxF32>(a, fn, stream);
  if (in_fmt == kPxU8 && out_fmt == kPxU8) return launch_async_fused_fmt<kPxU8, kPxU8>(a, fn, stream);
  if (in_fmt == kPxU16 && out_fmt == kPxU8) return launch_async_fused_fmt<kPxU16, kPxU8>(a, fn, stream);
  return HDRNET_E_UNSUPPORTED;
}

}  // namespace hdrnet_b200
