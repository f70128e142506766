// cnn_grad.cu -- vector-Jacobian products of the coefficient network's layers (cnn.cu): the
// backward of HDRNetCurves._coefficients (hdrnet/models.py:62-142) for fine-tuning the network
// through the slice-apply VJP (slice_grad.cu).
//
//   conv_dgrad_kernel    input VJP of conv2d: dx[b,iy,ix,ci] = sum over (ky,kx,co) with
//                        iy = oy*s + ky - pad_t (same for x) of W[ky,kx,ci,co] * dy'[b,oy,ox,co],
//                        dy' = dy * (out > 0) for a ReLU layer (TF's ReluGrad masks on the output).
//                        One thread per input element; taps and channels in a fixed order.
//   wgrad_partial_kernel weight + bias VJP as a GEMM over output pixels:
//                        dW[kk*Cin + ci, co] = sum_p x_im2col[p, kk*Cin + ci] * dy'[p, co], with one
//                        extra row of ones whose result is db.  Each CTA reduces one chunk of
//                        kWgChunk pixels for a 64 x 64 tile of (row, co) into the caller's
//                        workspace; wgrad_reduce_kernel then sums the chunks in a fixed order.
//   fuse_*_kernel        the transpose of fuse_predict_kernel: dpred is read from dgrid through the
//                        unroll_grid map, fused = relu(local + global) is recomputed, not stored.
//
// fully_connected is the same computation as a 1 x 1 conv on a 1 x 1 image (I input channels), so
// the fc VJP runs the conv kernels.  No floating-point atomics anywhere: every sum has one fixed
// order, so two identical calls give bitwise-identical gradients (the policy of slice_grad.cu).
#include <cuda_runtime.h>

#include <cstdint>

#include "hdrnet_b200.h"

namespace hdrnet_b200 {
namespace {

constexpr int kDgThreads = 256;
constexpr int kWgThreads = 256;   // 16 x 16 threads, 4 x 4 outputs each
constexpr int kWgTileK = 64;      // im2col rows per CTA
constexpr int kWgTileC = 64;      // output channels per CTA
constexpr int kWgSub = 32;        // pixels staged in shared memory per step
constexpr int kWgChunk = 128;     // pixels per CTA (per workspace partial)

struct Geom {
  int B, H, W, Cin, OH, OW, Cout, k, stride, pad_t, pad_l, relu;
};

void same_pad(int size, int k, int s, int* out, int* before) {
  *out = (size + s - 1) / s;
  int total = (*out - 1) * s + k - size;
  if (total < 0) total = 0;
  *before = total / 2;
}

Geom make_geom(int B, int H, int W, int Cin, int Cout, int k, int stride, int relu) {
  Geom g;
  g.B = B; g.H = H; g.W = W; g.Cin = Cin; g.Cout = Cout; g.k = k; g.stride = stride; g.relu = relu;
  same_pad(H, k, stride, &g.OH, &g.pad_t);
  same_pad(W, k, stride, &g.OW, &g.pad_l);
  return g;
}

__device__ __forceinline__ float masked(const float* dy, const float* out, long long i, int relu) {
  const float d = __ldg(dy + i);
  return (relu && !(__ldg(out + i) > 0.0f)) ? 0.0f : d;
}

// ---- conv2d input VJP -------------------------------------------------------------------------
__global__ void __launch_bounds__(kDgThreads)
conv_dgrad_kernel(const float* __restrict__ w, const float* __restrict__ out,
                  const float* __restrict__ dy, float* __restrict__ dx, const Geom g) {
  const long long total = static_cast<long long>(g.B) * g.H * g.W * g.Cin;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(e % g.Cin);
    const long long pix = e / g.Cin;
    const int ix = static_cast<int>(pix % g.W);
    const int iy = static_cast<int>((pix / g.W) % g.H);
    const int b = static_cast<int>(pix / (static_cast<long long>(g.W) * g.H));
    float acc = 0.0f;
    for (int ky = 0; ky < g.k; ++ky) {
      const int ny = iy + g.pad_t - ky;            // = oy * stride
      if (ny < 0 || ny % g.stride) continue;
      const int oy = ny / g.stride;
      if (oy >= g.OH) continue;
      for (int kx = 0; kx < g.k; ++kx) {
        const int nx = ix + g.pad_l - kx;
        if (nx < 0 || nx % g.stride) continue;
        const int ox = nx / g.stride;
        if (ox >= g.OW) continue;
        const long long o0 = ((static_cast<long long>(b) * g.OH + oy) * g.OW + ox) * g.Cout;
        const float* wr = w + (static_cast<size_t>(ky * g.k + kx) * g.Cin + ci) * g.Cout;
        for (int co = 0; co < g.Cout; ++co)
          acc = fmaf(__ldg(wr + co), masked(dy, out, o0 + co, g.relu), acc);
      }
    }
    dx[e] = acc;
  }
}

// ---- weight + bias VJP: per-chunk partial sums ------------------------------------------------
// Mode kConv: rows are the im2col columns of a conv input (x NHWC, HWIO row order), the bias row
// is K = k*k*Cin.  Mode kFuse: rows are the channels of fused = relu(local + global[b]) (C rows),
// and dy is the prediction gradient gathered from dgrid (o = (j*n_out + i)*gd + z, models.py:134-139).
enum WgMode { kConv = 0, kFuse = 1 };

struct WgArgs {
  Geom g;
  const float* x;        // conv: layer input; fuse: local [P][C]
  const float* glob;     // fuse: global [B][C]
  const float* dy;       // conv: dy [P][Cout]; fuse: dgrid [P][gd][n_out][n_in]
  const float* out;      // conv: layer output (ReLU mask) or nullptr
  float* ws;             // [chunks][K + 1][Cout]
  int K, cells, gd, n_out, n_in;   // cells: fuse, pixels per image
  long long P;
};

template <int kMode>
__device__ __forceinline__ float wg_x(const WgArgs& a, long long p, int r) {
  if (r == a.K) return 1.0f;        // the bias row
  if (r > a.K) return 0.0f;
  if (kMode == kFuse) {
    const long long b = p / a.cells;
    return fmaxf(__ldg(a.x + p * a.K + r) + __ldg(a.glob + b * a.K + r), 0.0f);
  }
  const Geom& g = a.g;
  const int ci = r % g.Cin, t = r / g.Cin;
  const int ky = t / g.k, kx = t - ky * g.k;
  const int ox = static_cast<int>(p % g.OW);
  const int oy = static_cast<int>((p / g.OW) % g.OH);
  const long long b = p / (static_cast<long long>(g.OW) * g.OH);
  const int iy = oy * g.stride - g.pad_t + ky, ix = ox * g.stride - g.pad_l + kx;
  if (iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) return 0.0f;
  return __ldg(a.x + ((b * g.H + iy) * g.W + ix) * g.Cin + ci);
}

template <int kMode>
__device__ __forceinline__ float wg_dy(const WgArgs& a, long long p, int co) {
  if (co >= a.g.Cout) return 0.0f;
  if (kMode == kFuse) {
    const int z = co % a.gd, i = (co / a.gd) % a.n_out, j = co / (a.gd * a.n_out);
    return __ldg(a.dy + ((p * a.gd + z) * a.n_out + i) * a.n_in + j);
  }
  return masked(a.dy, a.out, p * a.g.Cout + co, a.g.relu);
}

template <int kMode>
__global__ void __launch_bounds__(kWgThreads)
wgrad_partial_kernel(const WgArgs a) {
  __shared__ __align__(16) float xs[kWgSub][kWgTileK];
  __shared__ __align__(16) float ds[kWgSub][kWgTileC];
  const int tid = threadIdx.x;
  const int tr = tid / 16, tc = tid % 16;   // 4 rows x 4 channels per thread
  const int r0 = blockIdx.x * kWgTileK, c0 = blockIdx.y * kWgTileC;
  const long long p0 = static_cast<long long>(blockIdx.z) * kWgChunk;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  for (int s = 0; s < kWgChunk; s += kWgSub) {
    __syncthreads();
    for (int e = tid; e < kWgSub * kWgTileK; e += kWgThreads) {
      const int pp = e / kWgTileK, r = e % kWgTileK;
      const long long p = p0 + s + pp;
      xs[pp][r] = (p < a.P) ? wg_x<kMode>(a, p, r0 + r) : 0.0f;
    }
    for (int e = tid; e < kWgSub * kWgTileC; e += kWgThreads) {
      const int pp = e / kWgTileC, c = e % kWgTileC;
      const long long p = p0 + s + pp;
      ds[pp][c] = (p < a.P) ? wg_dy<kMode>(a, p, c0 + c) : 0.0f;
    }
    __syncthreads();
#pragma unroll 4
    for (int pp = 0; pp < kWgSub; ++pp) {
      const float4 xv = *reinterpret_cast<const float4*>(&xs[pp][tr * 4]);
      const float4 dv = *reinterpret_cast<const float4*>(&ds[pp][tc * 4]);
      const float xr[4] = {xv.x, xv.y, xv.z, xv.w};
      const float dr[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xr[i], dr[j], acc[i][j]);
    }
  }
  const int rows = a.K + 1;
  float* dst = a.ws + static_cast<size_t>(blockIdx.z) * rows * a.g.Cout;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + tr * 4 + i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = c0 + tc * 4 + j;
      if (co < a.g.Cout) dst[static_cast<size_t>(r) * a.g.Cout + co] = acc[i][j];
    }
  }
}

// One warp per (row, co): lane l sums chunks l, l + 32, ... in order, then a fixed xor tree.
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, float* __restrict__ db,
                    int K, int Cout, int chunks) {
  const long long warp = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long n = static_cast<long long>(K + 1) * Cout;
  if (warp >= n) return;
  float s = 0.0f;
  for (int c = lane; c < chunks; c += 32) s += ws[static_cast<size_t>(c) * n + warp];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) {
    const int r = static_cast<int>(warp / Cout), co = static_cast<int>(warp % Cout);
    if (r < K) {
      if (dw) dw[warp] = s;
    } else if (db) {
      db[co] = s;
    }
  }
}

long long wg_chunks(long long P) { return (P + kWgChunk - 1) / kWgChunk; }

size_t wg_bytes(long long P, int K, int Cout) {
  return static_cast<size_t>(wg_chunks(P)) * (K + 1) * Cout * sizeof(float);
}

template <int kMode>
int launch_wgrad(const WgArgs& a, float* dw, float* db, size_t ws_bytes, cudaStream_t st) {
  if (!dw && !db) return HDRNET_OK;
  if (!a.ws) return HDRNET_E_NULL_POINTER;
  if (ws_bytes < wg_bytes(a.P, a.K, a.g.Cout)) return HDRNET_E_BAD_SHAPE;
  const long long chunks = wg_chunks(a.P);
  if (chunks > 65535) return HDRNET_E_TOO_LARGE;
  dim3 grid((a.K + 1 + kWgTileK - 1) / kWgTileK, (a.g.Cout + kWgTileC - 1) / kWgTileC,
            static_cast<unsigned>(chunks));
  wgrad_partial_kernel<kMode><<<grid, kWgThreads, 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long warps = static_cast<long long>(a.K + 1) * a.g.Cout;
  wgrad_reduce_kernel<<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, st>>>(
      a.ws, dw, db, a.K, a.g.Cout, static_cast<int>(chunks));
  return static_cast<int>(cudaGetLastError());
}

unsigned grid_for(long long n, int threads) {
  const long long b = (n + threads - 1) / threads;
  return static_cast<unsigned>(b < (1LL << 20) ? (b > 0 ? b : 1) : (1LL << 20));
}

// ---- fusion + prediction VJP --------------------------------------------------------------------
struct FuseArgs {
  const float* local;   // [P][C]
  const float* glob;    // [B][C]
  const float* w;       // [C][O]
  const float* dgrid;   // [P][gd][n_out][n_in]
  int B, cells, C, gd, n_out, n_in, O;
};

// dfused[p][c] = (sum_o dpred[p][o] * Wp[c][o]) * (fused[p][c] > 0)
__device__ __forceinline__ float fuse_dfused(const FuseArgs& a, long long p, int c) {
  const long long b = p / a.cells;
  const float f = __ldg(a.local + p * a.C + c) + __ldg(a.glob + b * a.C + c);
  if (!(f > 0.0f)) return 0.0f;
  const float* wr = a.w + static_cast<size_t>(c) * a.O;
  const float* dg = a.dgrid + p * a.O;
  float acc = 0.0f;
  for (int z = 0; z < a.gd; ++z)
    for (int i = 0; i < a.n_out; ++i)
      for (int j = 0; j < a.n_in; ++j)
        acc = fmaf(__ldg(dg + (z * a.n_out + i) * a.n_in + j), __ldg(wr + (j * a.n_out + i) * a.gd + z), acc);
  return acc;
}

__global__ void __launch_bounds__(kDgThreads)
fuse_dlocal_kernel(const FuseArgs a, float* __restrict__ dlocal) {
  const long long total = static_cast<long long>(a.B) * a.cells * a.C;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x)
    dlocal[e] = fuse_dfused(a, e / a.C, static_cast<int>(e % a.C));
}

// dglobal[b][c] = sum over the image's cells of dfused: one warp per (b, c), lane l takes cells
// l, l + 32, ... in order, then a fixed xor tree.
__global__ void __launch_bounds__(256)
fuse_dglobal_kernel(const FuseArgs a, float* __restrict__ dglobal) {
  const long long warp = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= static_cast<long long>(a.B) * a.C) return;
  const long long b = warp / a.C;
  const int c = static_cast<int>(warp % a.C);
  float s = 0.0f;
  for (int q = lane; q < a.cells; q += 32) s += fuse_dfused(a, b * a.cells + q, c);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) dglobal[warp] = s;
}

int conv_grad(const float* in, const float* w, const float* out, const float* dout, float* din,
              float* dw, float* db, int B, int H, int W, int Cin, int Cout, int k, int stride,
              int relu, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (B < 0 || H < 1 || W < 1 || Cin < 1 || Cout < 1) return HDRNET_E_BAD_SHAPE;
  if ((k != 1 && k != 3) || (stride != 1 && stride != 2)) return HDRNET_E_UNSUPPORTED;
  if (B == 0 || (!din && !dw && !db)) return HDRNET_OK;
  if (!dout || (relu && !out)) return HDRNET_E_NULL_POINTER;
  if (din && !w) return HDRNET_E_NULL_POINTER;
  if ((dw || db) && !in) return HDRNET_E_NULL_POINTER;
  const Geom g = make_geom(B, H, W, Cin, Cout, k, stride, relu);
  if (din) {
    const long long n = static_cast<long long>(B) * H * W * Cin;
    conv_dgrad_kernel<<<grid_for(n, kDgThreads), kDgThreads, 0, st>>>(w, out, dout, din, g);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  WgArgs a = {};
  a.g = g; a.x = in; a.dy = dout; a.out = out; a.ws = static_cast<float*>(workspace);
  a.K = k * k * Cin;
  a.P = static_cast<long long>(B) * g.OH * g.OW;
  return launch_wgrad<kConv>(a, dw, db, workspace_bytes, st);
}

}  // namespace
}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_conv2d_grad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k, int stride) {
  if (B < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || k < 1 || stride < 1) return 0;
  const long long P = static_cast<long long>(B) * ((H + stride - 1) / stride) * ((W + stride - 1) / stride);
  return wg_bytes(P, k * k * Cin, Cout);
}

int hdrnet_conv2d_grad_f32(const float* in, const float* w, const float* out, const float* dout,
                           float* din, float* dw, float* db, int B, int H, int W, int Cin, int Cout,
                           int k, int stride, int relu, void* workspace, size_t workspace_bytes,
                           void* stream) {
  return conv_grad(in, w, out, dout, din, dw, db, B, H, W, Cin, Cout, k, stride, relu, workspace,
                   workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t hdrnet_fc_grad_workspace_bytes(int B, int I, int O) {
  return hdrnet_conv2d_grad_workspace_bytes(B, 1, 1, I, O, 1, 1);
}

int hdrnet_fc_grad_f32(const float* in, const float* w, const float* out, const float* dout,
                       float* din, float* dw, float* db, int B, int I, int O, int relu,
                       void* workspace, size_t workspace_bytes, void* stream) {
  if (B < 0 || I < 1 || O < 1) return HDRNET_E_BAD_SHAPE;
  // in[B, I] @ w[I, O] is a 1 x 1 conv on a 1 x 1 image with I input channels
  return conv_grad(in, w, out, dout, din, dw, db, B, 1, 1, I, O, 1, 1, relu, workspace,
                   workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t hdrnet_fuse_predict_grad_workspace_bytes(int B, int gh, int gw, int C, int gd, int n_out,
                                                int n_in) {
  if (B < 1 || gh < 1 || gw < 1 || C < 1 || gd < 1 || n_out < 1 || n_in < 1) return 0;
  return wg_bytes(static_cast<long long>(B) * gh * gw, C, gd * n_out * n_in);
}

int hdrnet_fuse_predict_grad_f32(const float* local, const float* global_feat, const float* w,
                                 const float* dgrid, float* dlocal, float* dglobal, float* dw,
                                 float* db, int B, int gh, int gw, int C, int gd, int n_out,
                                 int n_in, void* workspace, size_t workspace_bytes, void* stream) {
  if (B < 0 || gh < 1 || gw < 1 || C < 1 || gd < 1 || n_out < 1 || n_in < 1) return HDRNET_E_BAD_SHAPE;
  if (B == 0 || (!dlocal && !dglobal && !dw && !db)) return HDRNET_OK;
  if (!local || !global_feat || !dgrid) return HDRNET_E_NULL_POINTER;
  if ((dlocal || dglobal) && !w) return HDRNET_E_NULL_POINTER;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FuseArgs f;
  f.local = local; f.glob = global_feat; f.w = w; f.dgrid = dgrid;
  f.B = B; f.cells = gh * gw; f.C = C; f.gd = gd; f.n_out = n_out; f.n_in = n_in;
  f.O = gd * n_out * n_in;
  if (dlocal) {
    const long long n = static_cast<long long>(B) * f.cells * C;
    fuse_dlocal_kernel<<<grid_for(n, kDgThreads), kDgThreads, 0, st>>>(f, dlocal);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (dglobal) {
    const long long warps = static_cast<long long>(B) * C;
    fuse_dglobal_kernel<<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, st>>>(f, dglobal);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  WgArgs a = {};
  a.g = make_geom(B, gh, gw, C, f.O, 1, 1, 0);
  a.x = local; a.glob = global_feat; a.dy = dgrid; a.out = nullptr;
  a.ws = static_cast<float*>(workspace);
  a.K = C; a.cells = f.cells; a.gd = gd; a.n_out = n_out; a.n_in = n_in;
  a.P = static_cast<long long>(B) * f.cells;
  return launch_wgrad<kFuse>(a, dw, db, workspace_bytes, st);
}

}  // extern "C"
