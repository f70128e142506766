// cnn.cu -- the low-resolution coefficient network (SURVEY.md row a7): replaces the TF
// conv / fully_connected layers of HDRNetCurves._coefficients (hdrnet/models.py:62-142,
// hdrnet/layers.py:25-93) with three hand-written fp32 kernels:
//
//   conv2d_nhwc_kernel   k x k (1 or 3), stride 1/2, TF 'SAME' padding (asymmetric for
//                        stride 2 on even extents), HWIO weights, bias + ReLU epilogue.
//                        Batch norm is folded into weights/bias on the host (inference form).
//   fc_kernel            x[B,I] @ W[I,O] + b (+ReLU), weights streamed once for 8 images.
//   fuse_predict_kernel  fusion relu(local + global) (models.py:122-125), the 1x1 prediction
//                        conv (:129-132) and the unroll_grid permutation (:134-139) in one
//                        pass, writing the [B,gh,gw,gd,n_out*n_in] grid slice-apply reads.
//
// The whole network is ~83 MFLOP per image: launch-latency bound, not tensor bound.  fp32 CUDA-core math keeps the coefficients within float32 round-off of the
// float64-accumulated oracle, which bf16 / tf32 tensor-core math could not.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdint>

#include "hdrnet_b200.h"

namespace hdrnet_b200 {

constexpr int kConvThreads = 128;  // 32 pixel groups x 4 channel groups

struct ConvArgs {
  const float* in;
  const float* w;     // [k][k][Cin][Cout]
  const float* bias;  // [Cout] or nullptr
  float* out;
  int B, H, W, Cin, OH, OW, Cout, k, stride, pad_t, pad_l, relu, ci_chunk;
  int w_vec;  // Cout % 4 == 0 and 16-byte aligned weights: cp.async staging
};

// Register tile per thread: kConvPx output pixels x kConvCo output channels.  <2, 8> is the
// throughput shape (64 px x 32 channels per CTA); <1, 4> quadruples the CTA count for the
// tiny late layers at batch 1, which are otherwise a handful of CTAs on 132 SMs.
template <int kConvPx, int kConvCo>
__global__ void __launch_bounds__(kConvThreads)
conv2d_nhwc_kernel(const ConvArgs a) {
  constexpr int kConvTilePx = 32 * kConvPx;
  constexpr int kConvTileCo = 4 * kConvCo;
  static_assert(kConvCo == 4 || kConvCo == 8, "channel tile is one or two float4");
  extern __shared__ __align__(16) float wsm[];  // [k*k][ci_chunk][kConvTileCo]
  const int tid = threadIdx.x;
  const int pg = tid & 31, cg = tid >> 5;
  const int co0 = blockIdx.y * kConvTileCo;
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  const long long tile_px0 = static_cast<long long>(blockIdx.x) * kConvTilePx;

  // This thread's output pixels.
  int pb[kConvPx], py[kConvPx], px[kConvPx];
  bool pv[kConvPx];
#pragma unroll
  for (int p = 0; p < kConvPx; ++p) {
    const long long q = tile_px0 + pg * kConvPx + p;
    pv[p] = q < total_px;
    const long long qq = pv[p] ? q : 0;
    px[p] = static_cast<int>(qq % a.OW);
    py[p] = static_cast<int>((qq / a.OW) % a.OH);
    pb[p] = static_cast<int>(qq / (static_cast<long long>(a.OW) * a.OH));
  }
  float acc[kConvPx][kConvCo];
#pragma unroll
  for (int p = 0; p < kConvPx; ++p)
#pragma unroll
    for (int c = 0; c < kConvCo; ++c) acc[p][c] = 0.0f;

  const int kk = a.k * a.k;
  const bool vec_in = (a.Cin % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.in) & 15u) == 0);
  for (int ci0 = 0; ci0 < a.Cin; ci0 += a.ci_chunk) {
    const int cn = min(a.ci_chunk, a.Cin - ci0);
    __syncthreads();
    // Stage weights [kk][cn][32 co] (zero-fill channels beyond Cout).  16-byte cp.async
    // (LDGSTS) keeps every copy of the tile in flight at once: the tile is up to 72 KB and a
    // register-staged loop would serialise on global-load latency.
    if (a.w_vec) {
      for (int e4 = tid; e4 < kk * cn * (kConvTileCo / 4); e4 += kConvThreads) {
        const int co = (e4 % (kConvTileCo / 4)) * 4;
        const int ci = (e4 / (kConvTileCo / 4)) % cn;
        const int t = e4 / ((kConvTileCo / 4) * cn);
        float* dst = wsm + static_cast<size_t>(e4) * 4;
        if (co0 + co < a.Cout) {
          const float* src = a.w + (static_cast<size_t>(t) * a.Cin + ci0 + ci) * a.Cout + co0 + co;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                           static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
                       "l"(src)
                       : "memory");
        } else {
          *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    } else {
      for (int e = tid; e < kk * cn * kConvTileCo; e += kConvThreads) {
        const int co = e % kConvTileCo;
        const int ci = (e / kConvTileCo) % cn;
        const int t = e / (kConvTileCo * cn);
        const int gco = co0 + co;
        wsm[e] = (gco < a.Cout)
                     ? __ldg(a.w + (static_cast<size_t>(t) * a.Cin + ci0 + ci) * a.Cout + gco)
                     : 0.0f;
      }
    }
    __syncthreads();
    for (int t = 0; t < kk; ++t) {
      const int ky = t / a.k, kx = t - ky * a.k;
      const float* src[kConvPx];
      bool ok[kConvPx];
#pragma unroll
      for (int p = 0; p < kConvPx; ++p) {
        const int iy = py[p] * a.stride - a.pad_t + ky;
        const int ix = px[p] * a.stride - a.pad_l + kx;
        ok[p] = pv[p] && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
        src[p] = a.in + ((static_cast<size_t>(pb[p]) * a.H + (ok[p] ? iy : 0)) * a.W +
                         (ok[p] ? ix : 0)) * a.Cin + ci0;
      }
      const float* wt = wsm + static_cast<size_t>(t) * cn * kConvTileCo + cg * kConvCo;
      if (vec_in && (cn % 4 == 0)) {
        // unrolled so that several iterations' input loads are in flight at once: a late layer at
        // batch 1 is a few dozen CTAs of 4 warps, and every new (tap, 4 channels) is an L2 round trip
        // that nothing else on the SM hides (tools/time_cnn.py times the layers)
#pragma unroll(kConvPx == 1 ? 8 : 4)
        for (int ci = 0; ci < cn; ci += 4) {
          float xin[kConvPx][4];
#pragma unroll
          for (int p = 0; p < kConvPx; ++p) {
            const float4 v = ok[p] ? __ldg(reinterpret_cast<const float4*>(src[p] + ci))
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
            xin[p][0] = v.x; xin[p][1] = v.y; xin[p][2] = v.z; xin[p][3] = v.w;
          }
#pragma unroll
          for (int d = 0; d < 4; ++d) {
            const float4 w0 = *reinterpret_cast<const float4*>(wt + (ci + d) * kConvTileCo);
            const float4 w1 = (kConvCo == 8)
                                  ? *reinterpret_cast<const float4*>(wt + (ci + d) * kConvTileCo + 4)
                                  : w0;
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int p = 0; p < kConvPx; ++p)
#pragma unroll
              for (int c = 0; c < kConvCo; ++c) acc[p][c] = fmaf(xin[p][d], wv[c], acc[p][c]);
          }
        }
      } else {
        for (int ci = 0; ci < cn; ++ci) {
          const float4 w0 = *reinterpret_cast<const float4*>(wt + ci * kConvTileCo);
          const float4 w1 = (kConvCo == 8)
                                ? *reinterpret_cast<const float4*>(wt + ci * kConvTileCo + 4)
                                : w0;
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int p = 0; p < kConvPx; ++p) {
            const float x = ok[p] ? __ldg(src[p] + ci) : 0.0f;
#pragma unroll
            for (int c = 0; c < kConvCo; ++c) acc[p][c] = fmaf(x, wv[c], acc[p][c]);
          }
        }
      }
    }
  }

  // Epilogue: bias, ReLU, store.
#pragma unroll
  for (int p = 0; p < kConvPx; ++p) {
    if (!pv[p]) continue;
    float* dst = a.out + ((static_cast<size_t>(pb[p]) * a.OH + py[p]) * a.OW + px[p]) * a.Cout;
#pragma unroll
    for (int c = 0; c < kConvCo; ++c) {
      const int gco = co0 + cg * kConvCo + c;
      if (gco < a.Cout) {
        float v = acc[p][c] + (a.bias ? __ldg(a.bias + gco) : 0.0f);
        if (a.relu) v = fmaxf(v, 0.0f);
        dst[gco] = v;
      }
    }
  }
}

// ---- fully connected --------------------------------------------------------------------
constexpr int kFcThreads = 256;   // 64 outputs x 4 k-slices
constexpr int kFcOut = 64;
constexpr int kFcSlices = 4;
constexpr int kFcBatch = 8;       // images per pass (weights streamed once for all of them)
constexpr int kFcChunk = 512;     // inputs staged per step: 8 x 512 x 4 B = 16 KB

__global__ void __launch_bounds__(kFcThreads)
fc_kernel(const float* __restrict__ in, const float* __restrict__ w,
          const float* __restrict__ bias, float* __restrict__ out, int B, int I, int O,
          int relu) {
  __shared__ float xs[kFcBatch][kFcChunk];
  __shared__ float red[kFcSlices][kFcBatch][kFcOut];
  const int tid = threadIdx.x;
  const int o = tid % kFcOut, ks = tid / kFcOut;
  const int go = blockIdx.x * kFcOut + o;
  const int b0 = blockIdx.y * kFcBatch;
  const int nb = min(kFcBatch, B - b0);
  float acc[kFcBatch];
#pragma unroll
  for (int b = 0; b < kFcBatch; ++b) acc[b] = 0.0f;

  for (int i0 = 0; i0 < I; i0 += kFcChunk) {
    const int n = min(kFcChunk, I - i0);
    __syncthreads();
    for (int e = tid; e < kFcBatch * kFcChunk; e += kFcThreads) {
      const int b = e / kFcChunk, i = e % kFcChunk;
      xs[b][i] = (b < nb && i < n) ? __ldg(in + static_cast<size_t>(b0 + b) * I + i0 + i) : 0.0f;
    }
    __syncthreads();
    if (go < O) {
      // k-slices interleave so consecutive rows of W stream from consecutive threads' loops
#pragma unroll 8
      for (int i = ks; i < n; i += kFcSlices) {
        const float wv = __ldg(w + static_cast<size_t>(i0 + i) * O + go);
#pragma unroll
        for (int b = 0; b < kFcBatch; ++b) acc[b] = fmaf(xs[b][i], wv, acc[b]);
      }
    }
  }
#pragma unroll
  for (int b = 0; b < kFcBatch; ++b) red[ks][b][o] = acc[b];
  __syncthreads();
  for (int e = tid; e < kFcBatch * kFcOut; e += kFcThreads) {
    const int b = e / kFcOut, oo = e % kFcOut;
    const int goo = blockIdx.x * kFcOut + oo;
    if (b < nb && goo < O) {
      float v = ((red[0][b][oo] + red[1][b][oo]) + (red[2][b][oo] + red[3][b][oo])) +
                (bias ? __ldg(bias + goo) : 0.0f);
      if (relu) v = fmaxf(v, 0.0f);
      out[static_cast<size_t>(b0 + b) * O + goo] = v;
    }
  }
}


// ---- fully connected, split-K over a thread-block cluster ----------------------------------------
// At batch <= 8 a fully connected layer is a weight stream (fc1: 1 MB) that a handful of CTAs
// cannot pull fast enough.  Here the K dimension is split over the
// CTAs of a cluster (up to 8): every CTA streams its slice of W with 128-bit loads (16 rows x 16
// float4 columns in flight per pass), reduces its 16 row-lanes in shared memory, and the
// cluster's rank 0 sums the per-CTA partials through DISTRIBUTED SHARED MEMORY in a fixed order
// (deterministic; no atomics), then applies bias / ReLU.
constexpr int kFcCThreads = 256;
constexpr int kFcCOut = 64;       // outputs per cluster (16 float4 columns)
constexpr int kFcCRows = 16;      // k rows streamed in parallel
constexpr int kFcCMaxSlice = 256; // inputs per CTA staged in shared memory (static smem <= 48 KB)

__global__ void __launch_bounds__(kFcCThreads)
fc_cluster_kernel(const float* __restrict__ in, const float* __restrict__ w,
                  const float* __restrict__ bias, float* __restrict__ out, int B, int I, int O,
                  int relu, int slice) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ float xs[kFcBatch][kFcCMaxSlice];
  __shared__ float red[kFcCRows][kFcBatch][kFcCOut];   // 32 KB
  __shared__ float partial[kFcBatch][kFcCOut];
  const int tid = threadIdx.x;
  const int col = tid % 16, krow = tid / 16;
  const int o0 = blockIdx.x * kFcCOut + col * 4;
  const int b0 = blockIdx.z * kFcBatch;
  const int nb = min(kFcBatch, B - b0);
  const unsigned rank = cluster.block_rank();
  const int k0 = static_cast<int>(rank) * slice;
  const int kn = max(0, min(slice, I - k0));

  for (int e = tid; e < kFcBatch * slice; e += kFcCThreads) {
    const int b = e / slice, i = e % slice;
    xs[b][i] = (b < nb && i < kn) ? __ldg(in + static_cast<size_t>(b0 + b) * I + k0 + i) : 0.0f;
  }
  __syncthreads();

  float acc[kFcBatch][4];
#pragma unroll
  for (int b = 0; b < kFcBatch; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.0f;
  if (o0 < O) {
#pragma unroll 4
    for (int i = krow; i < kn; i += kFcCRows) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + static_cast<size_t>(k0 + i) * O + o0));
#pragma unroll
      for (int b = 0; b < kFcBatch; ++b) {
        const float x = xs[b][i];
        acc[b][0] = fmaf(x, wv.x, acc[b][0]);
        acc[b][1] = fmaf(x, wv.y, acc[b][1]);
        acc[b][2] = fmaf(x, wv.z, acc[b][2]);
        acc[b][3] = fmaf(x, wv.w, acc[b][3]);
      }
    }
  }
#pragma unroll
  for (int b = 0; b < kFcBatch; ++b)
    *reinterpret_cast<float4*>(&red[krow][b][col * 4]) = make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
  __syncthreads();
  for (int e = tid; e < kFcBatch * kFcCOut; e += kFcCThreads) {
    const int b = e / kFcCOut, o = e % kFcCOut;
    float s = 0.0f;
#pragma unroll
    for (int r = 0; r < kFcCRows; ++r) s += red[r][b][o];
    partial[b][o] = s;
  }
  cluster.sync();  // every CTA's partial is complete and visible cluster-wide
  if (rank == 0) {
    const unsigned nranks = cluster.num_blocks();
    for (int e = tid; e < kFcBatch * kFcCOut; e += kFcCThreads) {
      const int b = e / kFcCOut, o = e % kFcCOut;
      const int go = blockIdx.x * kFcCOut + o;
      if (b < nb && go < O) {
        float s = 0.0f;
        for (unsigned r = 0; r < nranks; ++r)
          s += cluster.map_shared_rank(&partial[0][0], r)[b * kFcCOut + o];
        s += bias ? __ldg(bias + go) : 0.0f;
        out[static_cast<size_t>(b0 + b) * O + go] = relu ? fmaxf(s, 0.0f) : s;
      }
    }
  }
  cluster.sync();  // keep the remote shared memory alive until rank 0 has read it
}

// ---- fusion + prediction + unroll_grid ----------------------------------------------------
constexpr int kFpThreads = 256;
constexpr int kFpCells = 8;  // grid cells per CTA (one warp each)

__global__ void __launch_bounds__(kFpThreads)
fuse_predict_kernel(const float* __restrict__ local, const float* __restrict__ global_feat,
                    const float* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ grid, int B, int cells_per_image, int C, int gd,
                    int n_out, int n_in, int stage_w, int pdl) {
  extern __shared__ __align__(16) float sm[];  // [w[C][O] when stage_w] then f[kFpCells][C]
  const int O = gd * n_out * n_in;
  // stage_w == 0: the prediction weights do not fit shared memory next to the features (e.g.
  // HDRNetGaussianPyrNN with channel_multiplier 4: C = 256, O = 288, 295 KB): read them through L1
  float* fsm = sm + (stage_w ? static_cast<size_t>(C) * O : 0);
  const float* wsm = stage_w ? sm : w;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (stage_w) {
    if ((C * O) % 4 == 0 && (reinterpret_cast<uintptr_t>(w) & 15u) == 0) {
      for (int e = tid; e < C * O / 4; e += kFpThreads)
        reinterpret_cast<float4*>(sm)[e] = __ldg(reinterpret_cast<const float4*>(w) + e);
    } else {
      for (int e = tid; e < C * O; e += kFpThreads) sm[e] = __ldg(w + e);
    }
  }
  // launched with programmatic stream serialisation (hdrnet_coefficients_f32): the weights above do
  // not depend on the previous kernels, the features below do
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long total = static_cast<long long>(B) * cells_per_image;
  const long long cell = static_cast<long long>(blockIdx.x) * kFpCells + warp;
  const bool valid = cell < total;
  if (valid) {
    const int b = static_cast<int>(cell / cells_per_image);
    for (int c = lane; c < C; c += 32)
      fsm[warp * C + c] = fmaxf(__ldg(local + cell * C + c) + __ldg(global_feat + static_cast<size_t>(b) * C + c), 0.0f);
  }
  __syncthreads();
  if (!valid) return;
  const float* f = fsm + warp * C;
  for (int o = lane; o < O; o += 32) {
    float acc = 0.0f;
    for (int c = 0; c < C; ++c) acc = fmaf(f[c], wsm[c * O + o], acc);
    acc += bias ? __ldg(bias + o) : 0.0f;
    // unroll_grid (models.py:134-139): prediction channel o = (j*n_out + i)*gd + z
    const int z = o % gd;
    const int i = (o / gd) % n_out;
    const int j = o / (gd * n_out);
    grid[((cell * gd + z) * n_out + i) * n_in + j] = acc;
  }
}

// conv_wgmma.cu: tensor-core (wgmma, 3xTF32) implicit-GEMM form of the same layer.
int launch_conv_wgmma(const float* in, const float* w, const float* bias, float* out, int B,
                      int H, int W, int Cin, int Cout, int k, int stride, int relu, int OH,
                      int OW, int pad_t, int pad_l, cudaStream_t stream);

static void same_pad(int size, int k, int s, int* out, int* before) {
  *out = (size + s - 1) / s;
  int total = (*out - 1) * s + k - size;
  if (total < 0) total = 0;
  *before = total / 2;
}

// ---------------------------------------------------------------------------------------------
// Latency form for the small late layers (batch 1-2: a few thousand output pixels at most).
// conv2d_nhwc_kernel walks its k*k*Cin reduction with one dependent L2 round trip per 4 input
// channels and 4 warps per SM, mostly waiting on those round trips.
// Here a CTA owns 32 output pixels (lane = pixel) x 4*kCoGroups output channels and
//   1. copies every lane's k x k x Cin input patch and the CTA's weight columns into shared
//      memory with 16-byte cp.async -- ALL of them in flight at once, one memory round trip;
//   2. splits the reduction four ways across warps (kPatchSlices), each warp doing
//      LDS.128 (its pixel's 4 inputs, conflict-free row stride) + 4 broadcast LDS.128 (weights)
//      + 16 FFMA per step, no global access;
//   3. adds the four partial sums through shared memory, bias + ReLU, 16-byte stores.
// The patches overlap (9x redundant for stride 1), which is why this form is for SMALL layers
// only: the redundancy is L2 -> shared traffic of tens of KB per CTA.
// Input channels that are not a multiple of 4 (the first layer: 3) are staged with 4-byte copies and
// the reduction is zero-padded to a multiple of 4; reductions of <= 64 terms are not split across
// warps (kSlices = 1: the first layer is 27 terms).
constexpr int kPatchPx = 32;

__host__ __device__ inline int patch_k4(int K) { return (K + 3) / 4 * 4; }
__host__ __device__ inline int patch_row_floats(int K) {
  const int q = patch_k4(K) / 4;
  return ((q & 1) ? q : q + 1) * 4;  // odd number of 16-byte chunks: lanes hit distinct banks
}

//
// The kernel takes TWO layers: x-tiles [0, tiles0) belong to a0, the rest to a1 (a1.B == 0: none).
// That is how the global and the local branch of the network (models.py:86-118: both read the
// splat features, neither reads the other) share one launch.  kPdl: launched with programmatic
// stream serialisation -- the weight copies (independent of the previous layer) are issued
// BEFORE griddepcontrol.wait, the input patch after it, so the previous layer's tail and this
// layer's launch + weight fetch overlap.
template <int kCoGroups, int kPatchSlices>
__global__ void __launch_bounds__(32 * kPatchSlices * kCoGroups)
conv2d_patch_kernel(const ConvArgs a0, const ConvArgs a1, const int tiles0, const int pdl) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // let the next layer's prologue start
  const bool second = static_cast<int>(blockIdx.x) >= tiles0;
  ConvArgs a;   // scalar selects: the structs are kernel parameters (constant bank)
  a.in = second ? a1.in : a0.in;       a.w = second ? a1.w : a0.w;
  a.bias = second ? a1.bias : a0.bias; a.out = second ? a1.out : a0.out;
  a.B = second ? a1.B : a0.B;          a.H = second ? a1.H : a0.H;
  a.W = second ? a1.W : a0.W;          a.Cin = second ? a1.Cin : a0.Cin;
  a.OH = second ? a1.OH : a0.OH;       a.OW = second ? a1.OW : a0.OW;
  a.Cout = second ? a1.Cout : a0.Cout; a.k = second ? a1.k : a0.k;
  a.stride = second ? a1.stride : a0.stride;
  a.pad_t = second ? a1.pad_t : a0.pad_t; a.pad_l = second ? a1.pad_l : a0.pad_l;
  a.relu = second ? a1.relu : a0.relu;
  const int tile_x = static_cast<int>(blockIdx.x) - (second ? tiles0 : 0);
  constexpr int kTileCo = 4 * kCoGroups;
  constexpr int kWarps = kPatchSlices * kCoGroups;
  constexpr int kThreads = 32 * kWarps;
  extern __shared__ __align__(16) float psm[];
  const int kk = a.k * a.k;
  const int K = kk * a.Cin;
  const int K4 = patch_k4(K);
  const int Kp = patch_row_floats(K);
  float* in_s = psm;                                  // [32][Kp]
  float* w_s = in_s + kPatchPx * Kp;                  // [K4][kTileCo]
  float* red = w_s + static_cast<size_t>(K4) * kTileCo;  // [kPatchSlices-1][kCoGroups][32][4]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int co0 = blockIdx.y * kTileCo;
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  const long long q = static_cast<long long>(tile_x) * kPatchPx + lane;
  const bool pv = q < total_px;
  const long long qq = pv ? q : 0;
  const int px = static_cast<int>(qq % a.OW);
  const int py = static_cast<int>((qq / a.OW) % a.OH);
  const int pb = static_cast<int>(qq / (static_cast<long long>(a.OW) * a.OH));

  // 1a. weights: row k of the CTA's column block = kCoGroups 16-byte chunks
  for (int e = tid; e < K4 * kCoGroups; e += kThreads) {
    const int krow = e / kCoGroups, g = e - krow * kCoGroups;
    float* dst = w_s + static_cast<size_t>(krow) * kTileCo + g * 4;
    if (krow < K && co0 + g * 4 < a.Cout) {  // Cout % 4 == 0 (launch precondition): whole chunk or nothing
      const float* src = a.w + static_cast<size_t>(krow) * a.Cout + co0 + g * 4;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                       static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
                   "l"(src)
                   : "memory");
    } else {
      *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // 1b. this lane's input patch: tap t -> Cin / 4 chunks, the warps interleave over the chunks
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");   // the previous layer's output is complete
  {
    const bool vec = (a.Cin & 3) == 0;
    const int cpr = vec ? a.Cin / 4 : a.Cin;   // copies per tap: 16-byte chunks, or single floats
    float* row = in_s + static_cast<size_t>(lane) * Kp;
    if (warp == 0)
      for (int c = K; c < K4; ++c) row[c] = 0.0f;
    for (int t = 0; t < kk; ++t) {
      const int ky = t / a.k, kx = t - ky * a.k;
      const int iy = py * a.stride - a.pad_t + ky;
      const int ix = px * a.stride - a.pad_l + kx;
      const bool ok = pv && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
      const float* src = a.in + ((static_cast<size_t>(pb) * a.H + (ok ? iy : 0)) * a.W +
                                 (ok ? ix : 0)) * a.Cin;
      float* dst = row + t * a.Cin;
      for (int c4 = warp; c4 < cpr; c4 += kWarps) {
        if (!vec) {
          if (ok) {
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(
                             static_cast<uint32_t>(__cvta_generic_to_shared(dst + c4))),
                         "l"(src + c4)
                         : "memory");
          } else {
            dst[c4] = 0.0f;
          }
        } else if (ok) {
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                           static_cast<uint32_t>(__cvta_generic_to_shared(dst + c4 * 4))),
                       "l"(src + c4 * 4)
                       : "memory");
        } else {
          *reinterpret_cast<float4*>(dst + c4 * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  // 2. this warp's quarter of the reduction
  const int ks = warp % kPatchSlices, cg = warp / kPatchSlices;
  const int nq = K4 / 4;
  const int q0 = (nq * ks) / kPatchSlices, q1 = (nq * (ks + 1)) / kPatchSlices;
  const float* xs = in_s + static_cast<size_t>(lane) * Kp;
  const float* ws = w_s + cg * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int i = q0; i < q1; ++i) {
    const float4 x = *reinterpret_cast<const float4*>(xs + 4 * i);
    const float4 w0 = *reinterpret_cast<const float4*>(ws + static_cast<size_t>(4 * i + 0) * kTileCo);
    const float4 w1 = *reinterpret_cast<const float4*>(ws + static_cast<size_t>(4 * i + 1) * kTileCo);
    const float4 w2 = *reinterpret_cast<const float4*>(ws + static_cast<size_t>(4 * i + 2) * kTileCo);
    const float4 w3 = *reinterpret_cast<const float4*>(ws + static_cast<size_t>(4 * i + 3) * kTileCo);
    acc.x = fmaf(x.x, w0.x, acc.x); acc.y = fmaf(x.x, w0.y, acc.y);
    acc.z = fmaf(x.x, w0.z, acc.z); acc.w = fmaf(x.x, w0.w, acc.w);
    acc.x = fmaf(x.y, w1.x, acc.x); acc.y = fmaf(x.y, w1.y, acc.y);
    acc.z = fmaf(x.y, w1.z, acc.z); acc.w = fmaf(x.y, w1.w, acc.w);
    acc.x = fmaf(x.z, w2.x, acc.x); acc.y = fmaf(x.z, w2.y, acc.y);
    acc.z = fmaf(x.z, w2.z, acc.z); acc.w = fmaf(x.z, w2.w, acc.w);
    acc.x = fmaf(x.w, w3.x, acc.x); acc.y = fmaf(x.w, w3.y, acc.y);
    acc.z = fmaf(x.w, w3.z, acc.z); acc.w = fmaf(x.w, w3.w, acc.w);
  }

  // 3. partial sums -> slice 0, epilogue
  if (kPatchSlices > 1) {
    if (ks > 0)
      *reinterpret_cast<float4*>(red + ((static_cast<size_t>(ks - 1) * kCoGroups + cg) * 32 + lane) * 4) = acc;
    __syncthreads();
  }
  if (ks == 0 && pv) {
#pragma unroll
    for (int s = 0; s < kPatchSlices - 1; ++s) {
      const float4 r = *reinterpret_cast<const float4*>(
          red + ((static_cast<size_t>(s) * kCoGroups + cg) * 32 + lane) * 4);
      acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
    }
    const int gco = co0 + cg * 4;
    if (gco < a.Cout) {
      if (a.bias) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(a.bias + gco));
        acc.x += bv.x; acc.y += bv.y; acc.z += bv.z; acc.w += bv.w;
      }
      if (a.relu) {
        acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f);
        acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
      }
      float* dst = a.out + ((static_cast<size_t>(pb) * a.OH + py) * a.OW + px) * a.Cout + gco;
      *reinterpret_cast<float4*>(dst) = acc;
    }
  }
}

inline int patch_slices(int K) { return patch_k4(K) <= 64 ? 1 : 4; }

inline size_t patch_smem_bytes(int K, int co_groups) {
  return (static_cast<size_t>(kPatchPx) * patch_row_floats(K) + static_cast<size_t>(patch_k4(K)) * 4 * co_groups +
          static_cast<size_t>(patch_slices(K) - 1) * co_groups * 32 * 4) * sizeof(float);
}

// Preconditions for the patch form: float4 weights / outputs (Cout % 4, 16-byte bases); input
// channels % 4 with a 16-byte base, or any count with 4-byte copies.
inline bool patch_ok(const ConvArgs& a) {
  const auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  return (a.Cin % 4 != 0 || al(a.in)) && a.Cout % 4 == 0 && al(a.w) && al(a.out) &&
         (!a.bias || al(a.bias)) && patch_smem_bytes(a.k * a.k * a.Cin, 1) <= 200 * 1024;
}

// One launch for one layer (b == nullptr) or two independent layers of equal Cout and equal
// reduction split.
template <int kCoGroups, int kSlices>
static int launch_conv_patch_t(const ConvArgs& a, const ConvArgs* b, bool pdl, cudaStream_t stream) {
  size_t smem = patch_smem_bytes(a.k * a.k * a.Cin, kCoGroups);
  if (b) smem = std::max(smem, patch_smem_bytes(b->k * b->k * b->Cin, kCoGroups));
  // the attribute is per function and sticky: raise it once, never lower it (threads may race
  // here; every value written is a valid upper bound for every launch that follows)
  static std::atomic<int> raised{0};
  if (!raised.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(conv2d_patch_kernel<kCoGroups, kSlices>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    raised.store(1, std::memory_order_relaxed);
  }
  const auto tiles = [](const ConvArgs& c) {
    return static_cast<int>((static_cast<long long>(c.B) * c.OH * c.OW + kPatchPx - 1) / kPatchPx);
  };
  const int tiles0 = tiles(a), tiles1 = b ? tiles(*b) : 0;
  ConvArgs none = a;
  none.B = 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(tiles0 + tiles1),
                     static_cast<unsigned>((a.Cout + 4 * kCoGroups - 1) / (4 * kCoGroups)));
  cfg.blockDim = dim3(32 * kSlices * kCoGroups);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, conv2d_patch_kernel<kCoGroups, kSlices>, a, b ? *b : none, tiles0,
                                     static_cast<int>(pdl));
  return static_cast<int>(e != cudaSuccess ? e : cudaGetLastError());
}

template <int kCoGroups>
static int launch_conv_patch(const ConvArgs& a, const ConvArgs* b, bool pdl, cudaStream_t stream) {
  return patch_slices(a.k * a.k * a.Cin) == 1 ? launch_conv_patch_t<kCoGroups, 1>(a, b, pdl, stream)
                                              : launch_conv_patch_t<kCoGroups, 4>(a, b, pdl, stream);
}

template <int kPx, int kCo>
static int launch_conv(ConvArgs a, cudaStream_t stream) {
  constexpr int kTilePx = 32 * kPx, kTileCo = 4 * kCo;
  // weights staged per input-channel chunk: k*k*chunk*kTileCo floats <= 72 KB
  int chunk = a.Cin;
  const int max_chunk = (72 * 1024 / 4) / (a.k * a.k * kTileCo);
  if (chunk > max_chunk) chunk = max_chunk / 4 * 4;
  a.ci_chunk = chunk;
  const size_t smem = static_cast<size_t>(a.k) * a.k * chunk * kTileCo * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(conv2d_nhwc_kernel<kPx, kCo>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  dim3 grid(static_cast<unsigned>((total_px + kTilePx - 1) / kTilePx),
            static_cast<unsigned>((a.Cout + kTileCo - 1) / kTileCo));
  conv2d_nhwc_kernel<kPx, kCo><<<grid, kConvThreads, smem, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

// ---- fc1 -> fc2 -> fc3 in ONE cluster (models.py:94-104) ------------------------------------
// Three launches of 0.6 MFLOP cost 3 x 4 us.  Here one cluster of 8 CTAs runs all three: every
// layer is split over K by cluster rank (rank r multiplies inputs [r*I/8, (r+1)*I/8) into ALL the
// outputs: its 1/8 of the weight matrix, streamed once), the per-rank partial sums meet through
// distributed shared memory, and rank r reduces outputs [r*O/8, (r+1)*O/8) -- which are exactly
// the inputs of ITS K-slice of the next layer, so activations never leave shared memory.
constexpr int kFcChainRanks = 8;
constexpr int kFcChainThreads = 256;
constexpr int kFcChainBatch = 4;

struct FcChainArgs {
  const float* x;      // [B][n[0]]
  const float* w[3];   // [n[l]][n[l+1]]
  const float* b[3];
  float* out;          // [B][n[3]]
  int B, n[4], max_slice, max_o, pdl;
  int stage_w;   // this rank's three weight slices fit shared memory: copied there before the dependency wait
};

__global__ void __launch_bounds__(kFcChainThreads)
fc_chain_kernel(const FcChainArgs a) {
  namespace cg = cooperative_groups;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) float fsm[];
  float* xs = fsm;                                                  // [kFcChainBatch][max_slice]
  float* partial = xs + kFcChainBatch * a.max_slice;                // [2][kFcChainBatch][max_o]
  float* red = partial + 2 * kFcChainBatch * a.max_o;               // [krows][kFcChainBatch][O]: 256 float4 x batch
  float* wsm = red + kFcChainThreads * 4 * kFcChainBatch;            // [3 layers][slice][O] when stage_w
  const int tid = threadIdx.x;
  const int rank = static_cast<int>(cluster.block_rank());
  if (a.stage_w) {
    // the weights do not depend on the previous kernel: every 16-byte copy of all three layers is
    // in flight before the wait (one memory round trip, hidden behind the previous layer's tail)
    float* dst = wsm;
    for (int l = 0; l < 3; ++l) {
      const int slice = a.n[l] / kFcChainRanks, O = a.n[l + 1];
      const float* src = a.w[l] + static_cast<size_t>(rank) * slice * O;
      for (int e = tid; e < slice * O / 4; e += kFcChainThreads)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                         static_cast<uint32_t>(__cvta_generic_to_shared(dst + e * 4))),
                     "l"(src + e * 4)
                     : "memory");
      dst += slice * O;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  if (a.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  {
    const int slice = a.n[0] / kFcChainRanks;
    for (int e = tid; e < kFcChainBatch * slice; e += kFcChainThreads) {
      const int b = e / slice, i = e - b * slice;
      xs[b * a.max_slice + i] = (b < a.B) ? __ldg(a.x + static_cast<size_t>(b) * a.n[0] + rank * slice + i) : 0.0f;
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  const float* wstaged = wsm;
#pragma unroll 1
  for (int l = 0; l < 3; ++l) {
    const int I = a.n[l], O = a.n[l + 1];
    const int slice = I / kFcChainRanks, ncol = O / 4, krows = kFcChainThreads / ncol;
    const int col = tid % ncol, kr = tid / ncol;
    float acc[kFcChainBatch][4];
#pragma unroll
    for (int b = 0; b < kFcChainBatch; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.0f;
    const float* wp = a.stage_w ? wstaged + col * 4 : a.w[l] + (static_cast<size_t>(rank) * slice) * O + col * 4;
    wstaged += slice * O;
#pragma unroll 8
    for (int i = kr; i < slice; i += krows) {
      const float4 wv = a.stage_w ? *reinterpret_cast<const float4*>(wp + static_cast<size_t>(i) * O)
                                  : __ldg(reinterpret_cast<const float4*>(wp + static_cast<size_t>(i) * O));
#pragma unroll
      for (int b = 0; b < kFcChainBatch; ++b) {
        const float x = xs[b * a.max_slice + i];
        acc[b][0] = fmaf(x, wv.x, acc[b][0]);
        acc[b][1] = fmaf(x, wv.y, acc[b][1]);
        acc[b][2] = fmaf(x, wv.z, acc[b][2]);
        acc[b][3] = fmaf(x, wv.w, acc[b][3]);
      }
    }
#pragma unroll
    for (int b = 0; b < kFcChainBatch; ++b)
      *reinterpret_cast<float4*>(red + (static_cast<size_t>(kr) * kFcChainBatch + b) * O + col * 4) =
          make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
    __syncthreads();
    float* mine = partial + static_cast<size_t>(l & 1) * kFcChainBatch * a.max_o;
    for (int e = tid; e < kFcChainBatch * O; e += kFcChainThreads) {
      const int b = e / O, o = e - b * O;
      float sum = 0.0f;
      for (int r = 0; r < krows; ++r) sum += red[(static_cast<size_t>(r) * kFcChainBatch + b) * O + o];
      mine[b * a.max_o + o] = sum;
    }
    cluster.sync();   // every rank's partial of layer l is complete and visible cluster-wide
    // (the buffer of layer l is rewritten by layer l + 2, behind the sync of layer l + 1: no rank
    // can still be reading it then)
    const int oslice = O / kFcChainRanks;
    for (int e = tid; e < kFcChainBatch * oslice; e += kFcChainThreads) {
      const int b = e / oslice, oo = e - b * oslice, o = rank * oslice + oo;
      float sum = 0.0f;
#pragma unroll
      for (int r = 0; r < kFcChainRanks; ++r) sum += cluster.map_shared_rank(mine, r)[b * a.max_o + o];
      sum += a.b[l] ? __ldg(a.b[l] + o) : 0.0f;
      if (l < 2) {
        xs[b * a.max_slice + oo] = fmaxf(sum, 0.0f);   // my K-slice of the next layer's input
      } else if (b < a.B) {
        a.out[static_cast<size_t>(b) * O + o] = sum;    // fc3: no activation (models.py:103)
      }
    }
    __syncthreads();
  }
  cluster.sync();   // keep this CTA's shared memory alive until every rank has read it
}

// Shapes the cluster chain takes: each width a power of two in [32, 1024] (so that 256 threads
// tile the float4 columns and every rank's slice is a multiple of 4), batch <= kFcChainBatch.
static bool fc_chain_ok(int B, const int n[4], const float* const w[3]) {
  if (B < 1 || B > kFcChainBatch) return false;
  for (int l = 0; l < 4; ++l)
    if (n[l] < 32 || (n[l] & (n[l] - 1))) return false;
  for (int l = 1; l < 4; ++l)
    if (n[l] > 1024) return false;
  if (n[0] / kFcChainRanks > 1024) return false;
  for (int l = 0; l < 3; ++l)
    if (reinterpret_cast<uintptr_t>(w[l]) & 15u) return false;
  return true;
}

static int launch_fc_chain(const float* x, const float* const w[3], const float* const b[3], float* out,
                           int B, const int n[4], bool pdl, cudaStream_t stream) {
  FcChainArgs a;
  a.x = x; a.out = out; a.B = B; a.pdl = pdl;
  a.max_slice = 0; a.max_o = 0;
  for (int l = 0; l < 3; ++l) {
    a.w[l] = w[l]; a.b[l] = b[l];
    a.max_slice = std::max(a.max_slice, n[l] / kFcChainRanks);
    a.max_o = std::max(a.max_o, n[l + 1]);
  }
  for (int l = 0; l < 4; ++l) a.n[l] = n[l];
  const size_t red_floats = static_cast<size_t>(kFcChainThreads) * 4 * kFcChainBatch;   // krows * (O / 4) = 256 float4 per image
  size_t smem = (static_cast<size_t>(kFcChainBatch) * a.max_slice +
                 2 * static_cast<size_t>(kFcChainBatch) * a.max_o + red_floats) * sizeof(float);
  if (smem > 200 * 1024) return HDRNET_E_UNSUPPORTED;
  size_t w_bytes = 0;
  for (int l = 0; l < 3; ++l) w_bytes += static_cast<size_t>(n[l] / kFcChainRanks) * n[l + 1] * sizeof(float);
  a.stage_w = smem + w_bytes <= 200 * 1024;
  if (a.stage_w) smem += w_bytes;
  static std::atomic<int> raised{0};
  if (!raised.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(fc_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    raised.store(1, std::memory_order_relaxed);
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kFcChainRanks);
  cfg.blockDim = dim3(kFcChainThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kFcChainRanks;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 2 : 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, fc_chain_kernel, a);
  return static_cast<int>(e != cudaSuccess ? e : cudaGetLastError());
}







// Layer dispatch shared by hdrnet_conv2d_nhwc_f32 and the network chain (hdrnet_coefficients_f32).
// pdl: the launch may overlap the tail of the previous kernel on the stream (patch form only; the
// other forms are launched in plain stream order, which is always correct).
static int conv_fill(ConvArgs* a, const float* in, const float* w, const float* bias, float* out, int B,
                     int H, int W, int Cin, int Cout, int k, int stride, int relu) {
  if (B < 0 || H < 1 || W < 1 || Cin < 1 || Cout < 1) return HDRNET_E_BAD_SHAPE;
  if ((k != 1 && k != 3) || (stride != 1 && stride != 2)) return HDRNET_E_UNSUPPORTED;
  if (B > 0 && (!in || !w || !out)) return HDRNET_E_NULL_POINTER;
  a->in = in; a->w = w; a->bias = bias; a->out = out;
  a->B = B; a->H = H; a->W = W; a->Cin = Cin; a->Cout = Cout; a->k = k; a->stride = stride; a->relu = relu;
  same_pad(H, k, stride, &a->OH, &a->pad_t);
  same_pad(W, k, stride, &a->OW, &a->pad_l);
  a->w_vec = (Cout % 4 == 0) && ((reinterpret_cast<uintptr_t>(w) & 15u) == 0);
  a->ci_chunk = Cin;
  return HDRNET_OK;
}

static int device_sms() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// 4 or 8 output channels per CTA for `ctas1` CTAs of the 4-channel form (tools/time_conv_layers.py):
// a second CTA on an SM doubles its staging time
static bool patch_two_groups(long long ctas1, int Cout, int K, int sms) {
  return ctas1 > sms && Cout % 8 == 0 && patch_smem_bytes(K, 2) <= 200 * 1024;
}

static int conv_dispatch_cuda_cores(const ConvArgs& a, bool pdl, cudaStream_t stream);

static int conv_dispatch(const ConvArgs& a, bool pdl, cudaStream_t stream) {
  if (a.B == 0) return HDRNET_OK;
  {  // Tensor-core path (conv_wgmma.cu).  Each 128-pixel tile runs a fixed-latency chunk loop,
     // so it pays off once there are about as many tiles as SMs (H100, tools/conv_bench.py: about
     // even with the CUDA-core kernels at 64 tiles, 1.8-3.7x faster at 128).
    const long long tiles = (static_cast<long long>(a.B) * a.OH * a.OW + 127) / 128;
    if (tiles >= 96) {
      const int rc = launch_conv_wgmma(a.in, a.w, a.bias, a.out, a.B, a.H, a.W, a.Cin, a.Cout, a.k, a.stride,
                                       a.relu, a.OH, a.OW, a.pad_t, a.pad_l, stream);
      if (rc != HDRNET_E_UNSUPPORTED) return rc;
    }
  }
  return conv_dispatch_cuda_cores(a, pdl, stream);
}

// The CUDA-core forms alone (float32 FMAs, round to nearest), for every shape.
static int conv_dispatch_cuda_cores(const ConvArgs& a, bool pdl, cudaStream_t stream) {
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  const int sms = device_sms();
  const long long big_ctas = ((total_px + 63) / 64) * ((a.Cout + 31) / 32);
  // The shared-memory patch form: one memory round trip instead of one per 4 input channels, for
  // batch 1-8 of every layer of the network (tools/time_conv_layers.py compares the forms); the
  // bound below caps its 9x-redundant staging traffic, it is not a measured crossover.
  if (patch_ok(a)) {
    const long long tiles = (total_px + kPatchPx - 1) / kPatchPx;
    const long long ctas1 = tiles * (a.Cout / 4);
    const bool two = patch_two_groups(ctas1, a.Cout, a.k * a.k * a.Cin, sms);
    if ((two ? ctas1 / 2 : ctas1) <= 32LL * sms)
      return two ? launch_conv_patch<2>(a, nullptr, pdl, stream) : launch_conv_patch<1>(a, nullptr, pdl, stream);
  }
  return (big_ctas >= 2LL * sms) ? launch_conv<2, 8>(a, stream) : launch_conv<1, 4>(a, stream);
}

// Two independent layers of equal Cout (the global and the local branch): one launch when both
// take the patch form, else two.
static int conv_dispatch_pair(const ConvArgs& a, const ConvArgs& b, bool pdl, cudaStream_t stream) {
  const int sms = device_sms();
  const auto small = [&](const ConvArgs& c) {   // not a tensor-core-sized layer, and the patch form takes it
    const long long px = static_cast<long long>(c.B) * c.OH * c.OW;
    return ((px + 127) / 128) < 96 && patch_ok(c);
  };
  if (a.Cout == b.Cout && a.B > 0 && b.B > 0 && small(a) && small(b) &&
      patch_slices(a.k * a.k * a.Cin) == patch_slices(b.k * b.k * b.Cin)) {
    const auto tiles = [](const ConvArgs& c) {
      return (static_cast<long long>(c.B) * c.OH * c.OW + kPatchPx - 1) / kPatchPx;
    };
    const long long ctas1 = (tiles(a) + tiles(b)) * (a.Cout / 4);
    const int K = std::max(a.k * a.k * a.Cin, b.k * b.k * b.Cin);
    if (patch_two_groups(ctas1, a.Cout, K, sms)) return launch_conv_patch<2>(a, &b, pdl, stream);
    return launch_conv_patch<1>(a, &b, pdl, stream);
  }
  const int rc = conv_dispatch(a, pdl, stream);
  return rc ? rc : conv_dispatch(b, false, stream);
}

}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

int hdrnet_conv2d_nhwc_f32(const float* in, const float* w, const float* bias, float* out, int B,
                           int H, int W, int Cin, int Cout, int k, int stride, int relu,
                           void* stream) {
  ConvArgs a;
  const int rc = conv_fill(&a, in, w, bias, out, B, H, W, Cin, Cout, k, stride, relu);
  return rc ? rc : conv_dispatch(a, false, static_cast<cudaStream_t>(stream));
}

int hdrnet_conv2d_nhwc_fp32_f32(const float* in, const float* w, const float* bias, float* out, int B,
                                int H, int W, int Cin, int Cout, int k, int stride, int relu,
                                void* stream) {
  ConvArgs a;
  const int rc = conv_fill(&a, in, w, bias, out, B, H, W, Cin, Cout, k, stride, relu);
  if (rc || a.B == 0) return rc;
  return conv_dispatch_cuda_cores(a, false, static_cast<cudaStream_t>(stream));
}

int hdrnet_fc_f32(const float* in, const float* w, const float* bias, float* out, int B, int I,
                  int O, int relu, void* stream) {
  if (B < 0 || I < 1 || O < 1) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!in || !w || !out) return HDRNET_E_NULL_POINTER;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // Cluster split-K form: needs float4 rows of W (O % 4 == 0, aligned) and a K worth splitting.
  int ksplit = 1;
  while (ksplit < 8 && I / (ksplit * 2) >= 64) ksplit *= 2;
  const int slice = (I + ksplit - 1) / ksplit;
  if (O % 4 == 0 && (reinterpret_cast<uintptr_t>(w) & 15u) == 0 && ksplit >= 2 &&
      slice <= kFcCMaxSlice) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((O + kFcCOut - 1) / kFcCOut, ksplit, (B + kFcBatch - 1) / kFcBatch);
    cfg.blockDim = dim3(kFcCThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = ksplit;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, fc_cluster_kernel, in, w, bias, out, B, I, O, relu, slice);
    return static_cast<int>(e != cudaSuccess ? e : cudaGetLastError());
  }
  dim3 grid((O + kFcOut - 1) / kFcOut, (B + kFcBatch - 1) / kFcBatch);
  fc_kernel<<<grid, kFcThreads, 0, st>>>(in, w, bias, out, B, I, O, relu);
  return static_cast<int>(cudaGetLastError());
}

static int fuse_predict_launch(const float* local, const float* global_feat, const float* w,
                               const float* bias, float* grid, int B, int gh, int gw, int C, int gd,
                               int n_out, int n_in, bool pdl, cudaStream_t stream) {
  if (B < 0 || gh < 1 || gw < 1 || C < 1 || gd < 1 || n_out < 1 || n_in < 1) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!local || !global_feat || !w || !grid) return HDRNET_E_NULL_POINTER;
  const int O = gd * n_out * n_in;
  size_t smem = (static_cast<size_t>(C) * O + static_cast<size_t>(kFpCells) * C) * sizeof(float);
  const int stage_w = smem <= 200 * 1024;
  if (!stage_w) smem = static_cast<size_t>(kFpCells) * C * sizeof(float);
  if (smem > 200 * 1024) return HDRNET_E_UNSUPPORTED;
  static std::atomic<int> raised{0};   // sticky per-function attribute: raise once, never lower
  if (!raised.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(fuse_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    raised.store(1, std::memory_order_relaxed);
  }
  const long long cells = static_cast<long long>(B) * gh * gw;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>((cells + kFpCells - 1) / kFpCells));
  cfg.blockDim = dim3(kFpThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, fuse_predict_kernel, local, global_feat, w, bias, grid, B, gh * gw, C,
                                     gd, n_out, n_in, stage_w, static_cast<int>(pdl));
  return static_cast<int>(e != cudaSuccess ? e : cudaGetLastError());
}

int hdrnet_fuse_predict_f32(const float* local, const float* global_feat, const float* w,
                            const float* bias, float* grid, int B, int gh, int gw, int C, int gd,
                            int n_out, int n_in, void* stream) {
  return fuse_predict_launch(local, global_feat, w, bias, grid, B, gh, gw, C, gd, n_out, n_in, false,
                             static_cast<cudaStream_t>(stream));
}

// ---- the whole coefficient network behind one call ------------------------------------------
// HDRNetCurves._coefficients (hdrnet/models.py:62-142): splat convs, global convs + 3 fc, local
// convs, fusion + prediction + unroll_grid.  One FFI crossing and 8 launches at small batch
// (n_ds splat + [global conv1 || local conv1] + [global conv2 || local conv2] + fc cluster chain
// + fuse/predict), each launched with programmatic stream serialisation so that a layer's launch
// latency and weight fetch hide behind the previous layer.  Layer i of the network writes buffer i
// of the caller's scratch: nothing is written twice inside a call.
namespace {

struct CoefPlan {
  int n_ds, c_splat[8], c8, f1, f2, g1, g2;   // g1, g2: spatial extent after global conv1 / conv2
  size_t act_floats;
};

bool coef_plan(int S, int sb, int gd, int cm, int B, CoefPlan* d) {
  if (S < 1 || sb < 1 || gd < 1 || cm < 1 || B < 1 || S % sb) return false;
  int n_ds = 0;
  for (int s = S; s > sb; s >>= 1) {
    if (s & 1) return false;
    ++n_ds;
  }
  if (n_ds < 1 || n_ds > 8 || (sb << n_ds) != S) return false;   // models.py:69: int(log2(S / sb)) halvings
  d->n_ds = n_ds;
  size_t fl = 0;
  const auto take = [&](size_t n) { fl += (n + 3) & ~static_cast<size_t>(3); };
  for (int i = 0; i < n_ds; ++i) {
    d->c_splat[i] = cm * (1 << i) * gd;
    const size_t sp = static_cast<size_t>(S >> (i + 1));
    take(static_cast<size_t>(B) * sp * sp * d->c_splat[i]);
  }
  d->c8 = 8 * cm * gd; d->f1 = 32 * cm * gd; d->f2 = 16 * cm * gd;
  d->g1 = (sb + 1) / 2; d->g2 = (d->g1 + 1) / 2;
  take(static_cast<size_t>(B) * d->g1 * d->g1 * d->c8);
  take(static_cast<size_t>(B) * d->g2 * d->g2 * d->c8);
  take(static_cast<size_t>(B) * sb * sb * d->c8);
  take(static_cast<size_t>(B) * sb * sb * d->c8);
  take(static_cast<size_t>(B) * d->f1);
  take(static_cast<size_t>(B) * d->f2);
  take(static_cast<size_t>(B) * d->c8);
  d->act_floats = fl;
  return true;
}

}  // namespace

size_t hdrnet_coefficients_scratch_bytes(int B, int net_input_size, int spatial_bin, int luma_bins,
                                         int channel_multiplier, int n_out, int n_in) {
  CoefPlan d;
  if (n_out < 1 || n_in < 1 || !coef_plan(net_input_size, spatial_bin, luma_bins, channel_multiplier, B, &d))
    return 0;
  return d.act_floats * sizeof(float);
}

int hdrnet_coefficients_f32(const float* lowres, float* grid, const float* const* weights,
                            const float* const* biases, int n_layers, void* scratch, size_t scratch_bytes,
                            int B, int net_input_size, int spatial_bin, int luma_bins,
                            int channel_multiplier, int n_out, int n_in, void* stream) {
  if (B < 0 || n_out < 1 || n_in < 1) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!lowres || !grid || !weights || !biases || !scratch) return HDRNET_E_NULL_POINTER;
  CoefPlan d;
  if (!coef_plan(net_input_size, spatial_bin, luma_bins, channel_multiplier, B, &d)) return HDRNET_E_UNSUPPORTED;
  if (n_layers != d.n_ds + 8) return HDRNET_E_BAD_SHAPE;
  if (scratch_bytes < d.act_floats * sizeof(float)) return HDRNET_E_BAD_SHAPE;
  for (int i = 0; i < n_layers; ++i)
    if (!weights[i]) return HDRNET_E_NULL_POINTER;
  if (reinterpret_cast<uintptr_t>(scratch) & 15u) return HDRNET_E_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* cur = static_cast<float*>(scratch);
  const auto take = [&](size_t n) { float* p = cur; cur += (n + 3) & ~static_cast<size_t>(3); return p; };
  int rc = HDRNET_OK;
  // layer order of `weights` / `biases`: splat conv1..n_ds, global conv1, conv2, fc1, fc2, fc3,
  // local conv1, conv2, prediction conv1
  const float* in = lowres;
  int H = net_input_size, C = 3, li = 0;
  for (int i = 0; i < d.n_ds; ++i, ++li) {
    const int OH = H / 2;
    float* out = take(static_cast<size_t>(B) * OH * OH * d.c_splat[i]);
    ConvArgs a;
    rc = conv_fill(&a, in, weights[li], biases[li], out, B, H, H, C, d.c_splat[i], 3, 2, 1);
    if (!rc) rc = conv_dispatch(a, /*pdl=*/i > 0, st);
    if (rc) return rc;
    in = out; H = OH; C = d.c_splat[i];
  }
  const float* splat = in;   // [B, sb, sb, C]
  const int sb = spatial_bin, c8 = d.c8;
  float* g1 = take(static_cast<size_t>(B) * d.g1 * d.g1 * c8);
  float* g2 = take(static_cast<size_t>(B) * d.g2 * d.g2 * c8);
  float* l1 = take(static_cast<size_t>(B) * sb * sb * c8);
  float* l2 = take(static_cast<size_t>(B) * sb * sb * c8);
  float* f1 = take(static_cast<size_t>(B) * d.f1);
  float* f2 = take(static_cast<size_t>(B) * d.f2);
  float* f3 = take(static_cast<size_t>(B) * c8);
  const int gi = li, fi = li + 2, lci = li + 5, pi = li + 7;
  ConvArgs ga, la;
  rc = conv_fill(&ga, splat, weights[gi], biases[gi], g1, B, sb, sb, C, c8, 3, 2, 1);
  if (!rc) rc = conv_fill(&la, splat, weights[lci], biases[lci], l1, B, sb, sb, C, c8, 3, 1, 1);
  if (!rc) rc = conv_dispatch_pair(la, ga, true, st);
  if (rc) return rc;
  rc = conv_fill(&ga, g1, weights[gi + 1], biases[gi + 1], g2, B, d.g1, d.g1, c8, c8, 3, 2, 1);
  if (!rc) rc = conv_fill(&la, l1, weights[lci + 1], biases[lci + 1], l2, B, sb, sb, c8, c8, 3, 1, 0);
  if (!rc) rc = conv_dispatch_pair(la, ga, true, st);
  if (rc) return rc;
  const int n[4] = {d.g2 * d.g2 * c8, d.f1, d.f2, c8};   // NHWC flatten = the buffer as it lies (models.py:94-95)
  const float* fw[3] = {weights[fi], weights[fi + 1], weights[fi + 2]};
  const float* fb[3] = {biases[fi], biases[fi + 1], biases[fi + 2]};
  if (fc_chain_ok(B, n, fw)) {
    rc = launch_fc_chain(g2, fw, fb, f3, B, n, true, st);
  } else {
    rc = hdrnet_fc_f32(g2, fw[0], fb[0], f1, B, n[0], n[1], 1, stream);
    if (!rc) rc = hdrnet_fc_f32(f1, fw[1], fb[1], f2, B, n[1], n[2], 1, stream);
    if (!rc) rc = hdrnet_fc_f32(f2, fw[2], fb[2], f3, B, n[2], n[3], 0, stream);
  }
  if (rc) return rc;
  return fuse_predict_launch(l2, f3, weights[pi], biases[pi], grid, B, sb, sb, c8, luma_bins, n_out, n_in, true, st);
}

}  // extern "C"
