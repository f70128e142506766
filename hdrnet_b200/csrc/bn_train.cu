// bn_train.cu -- training-mode batch norm of the coefficient network's layers (hdrnet/layers.py:47-54
// with is_training=True; the layers _coefficient_specs marks): batch statistics, the normalised relu
// output with the moving-average update, and the VJP.  z is the layer's conv or fc output without bias
// or relu, an [N, C] row-major float32 view (NHWC flattened; an fc layer has N = B).  Per channel c:
//
//   mu_c, var_c = mean and biased variance of z[:, c],  s_c = 1 / sqrt(var_c + 1e-3)
//   zh = (z - mu_c) s_c,  y = relu(zh + beta_c)                        (center=True, scale=False)
//   moving_mean -= (1 - 0.999) (moving_mean - mu_c)
//   moving_var  -= (1 - 0.999) (moving_var - var_c N / (N - 1))        (N = 1 feeds var_c = 0)
//   dyh = dy [y > 0] (TF's ReluGrad),  A_c = sum dyh (= d beta_c),  B_c = sum dyh zh
//   dz = s_c (dyh - A_c / N - zh B_c / N)
//
//   stats_partial_kernel   each CTA: one fixed chunk of rows x 32 channels; every thread sums its
//                          channel's rows centred on the chunk's first row, in float64, and the CTA
//                          writes the chunk's mean and M2.  A warp reads 32 adjacent channels of a row.
//   stats_reduce_kernel    one warp per channel merges the chunks (Chan et al.) in a fixed order.
//   bn_relu_kernel         y from z; the CTAs of the first row block also move the moving averages.
//   grad_partial_kernel    A and B of one chunk, in float64, the layout of stats_partial_kernel.
//   grad_reduce_kernel     one warp per channel adds the chunks in a fixed order.
//   grad_kernel            dz from z, dy and the (possibly rank-merged) A and B.
// The chunking depends on (N, C) alone and there are no atomics, so every call gives the same bits.
// mu enters the float32 arithmetic as mu_hi + mu_lo (two floats), so a channel whose spread is small
// against its mean (0.9 +- 1e-3) keeps its digits: z - mu_hi is exact there.
#include <cuda_runtime.h>

#include <cstdint>

#include "hdrnet_b200.h"

namespace hdrnet_b200 {
namespace {

constexpr int kTileC = 32;          // channels per CTA (threadIdx.x)
constexpr int kRowLanes = 8;        // rows in flight per CTA (threadIdx.y)
constexpr int kMinChunkRows = 64;
constexpr long long kChunkCtas = 1024;  // target of chunks x channel tiles for the partial passes
constexpr long long kMaxChunks = 512;
constexpr int kReduceWarps = 8;     // channels per CTA of the reduce kernels
constexpr double kBnEps = 1e-3;     // tf.contrib.layers.batch_norm's default epsilon
constexpr double kBnDecay = 0.999;  // ... and its moving-average decay

int channel_tiles(int C) { return (C + kTileC - 1) / kTileC; }

// Rows per chunk, a multiple of kRowLanes, from (N, C) alone.
long long chunk_rows(long long N, int C) {
  long long max_chunks = kChunkCtas / channel_tiles(C);
  if (max_chunks > kMaxChunks) max_chunks = kMaxChunks;
  if (max_chunks < 1) max_chunks = 1;
  long long rows = (N + max_chunks - 1) / max_chunks;
  if (rows < kMinChunkRows) rows = kMinChunkRows;
  return (rows + kRowLanes - 1) / kRowLanes * kRowLanes;
}

long long num_chunks(long long N, int C) {
  const long long r = chunk_rows(N, C);
  return (N + r - 1) / r;
}

// Row blocks of the elementwise kernels: about four rows per thread.
int row_blocks(long long N) {
  long long b = (N + 4 * kRowLanes - 1) / (4 * kRowLanes);
  return static_cast<int>(b > 65535 ? 65535 : b);
}

// One channel's normalisation from its float64 moments [3][C] (count, mean, M2).
struct Norm {
  float mu_hi, mu_lo, s;
};

__device__ __forceinline__ Norm channel_norm(const double* __restrict__ mom, int C, int c, double* var_out) {
  const double n = mom[c], mean = mom[C + c];
  double var = mom[2 * C + c] / n;
  if (var < 0.0) var = 0.0;
  if (var_out) *var_out = var;
  Norm r;
  r.mu_hi = static_cast<float>(mean);
  r.mu_lo = static_cast<float>(mean - static_cast<double>(r.mu_hi));
  r.s = static_cast<float>(1.0 / sqrt(var + kBnEps));
  return r;
}

// z - mu in float32, and the pre-activation (z - mu) s + beta: the forward and both VJP passes
// evaluate the same expression, so the relu mask is the forward's.
__device__ __forceinline__ float centred(float z, const Norm& q) {
  return __fsub_rn(__fsub_rn(z, q.mu_hi), q.mu_lo);
}

__device__ __forceinline__ float preact(float d, const Norm& q, float beta) { return __fmaf_rn(d, q.s, beta); }

// Sums of the kRowLanes lanes of a channel in a fixed order; valid in threadIdx.y == 0.
__device__ __forceinline__ void lane_sums(double a, double b, double* out_a, double* out_b) {
  __shared__ double sh[2][kRowLanes][kTileC];
  sh[0][threadIdx.y][threadIdx.x] = a;
  sh[1][threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y != 0) return;
  double ta = sh[0][0][threadIdx.x], tb = sh[1][0][threadIdx.x];
#pragma unroll
  for (int l = 1; l < kRowLanes; ++l) {
    ta += sh[0][l][threadIdx.x];
    tb += sh[1][l][threadIdx.x];
  }
  *out_a = ta;
  *out_b = tb;
}

// ws[chunk][2][C]: the chunk's mean and its sum of squared deviations M2, per channel.
__global__ void __launch_bounds__(kTileC * kRowLanes)
stats_partial_kernel(const float* __restrict__ z, double* __restrict__ ws, long long N, int C, long long rows) {
  const int c = blockIdx.x * kTileC + threadIdx.x;
  const long long r0 = static_cast<long long>(blockIdx.y) * rows;
  const long long r1 = r0 + rows < N ? r0 + rows : N;
  const bool valid = c < C;
  // Centred on the chunk's first row: a large common offset cancels before anything is squared.
  const double k = valid ? static_cast<double>(__ldg(z + r0 * C + c)) : 0.0;
  double s = 0.0, q = 0.0;
  if (valid) {
    for (long long r = r0 + threadIdx.y; r < r1; r += kRowLanes) {
      const double d = static_cast<double>(__ldg(z + r * C + c)) - k;
      s += d;
      q = fma(d, d, q);
    }
  }
  double ts = 0.0, tq = 0.0;
  lane_sums(s, q, &ts, &tq);
  if (threadIdx.y != 0 || !valid) return;
  const double n = static_cast<double>(r1 - r0);
  double* out = ws + static_cast<size_t>(blockIdx.y) * 2 * C;
  out[c] = k + ts / n;
  out[C + c] = tq - ts * ts / n;
}

// (n, mean, M2) += (nb, mb, M2b): the pairwise update of Chan, Golub and LeVeque.
__device__ __forceinline__ void merge(double& n, double& mean, double& m2, double nb, double mb, double m2b) {
  if (nb == 0.0) return;
  const double nt = n + nb, d = mb - mean;
  mean += d * (nb / nt);
  m2 += m2b + d * d * (n * nb / nt);
  n = nt;
}

// Warp w of CTA b: channel b * kReduceWarps + w.  Lane l merges chunks l, l + 32, ... in order, then a
// fixed tree over the lanes.  moments [3][C]: count, mean, M2.
__global__ void __launch_bounds__(32 * kReduceWarps)
stats_reduce_kernel(const double* __restrict__ ws, double* __restrict__ moments, long long N, int C,
                    long long rows, int chunks) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kReduceWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int k = lane; k < chunks; k += 32) {
    const long long r0 = static_cast<long long>(k) * rows;
    const long long nk = r0 + rows < N ? rows : N - r0;
    const double* w = ws + static_cast<size_t>(k) * 2 * C;
    merge(n, mean, m2, static_cast<double>(nk), w[c], w[C + c]);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, n, off);
    const double mb = __shfl_down_sync(0xffffffffu, mean, off);
    const double m2b = __shfl_down_sync(0xffffffffu, m2, off);
    if (lane < off) merge(n, mean, m2, nb, mb, m2b);
  }
  if (lane != 0) return;
  moments[c] = n;
  moments[C + c] = mean;
  moments[2 * C + c] = m2;
}

__global__ void __launch_bounds__(kTileC * kRowLanes)
bn_relu_kernel(const float* __restrict__ z, const double* __restrict__ moments, const float* __restrict__ beta,
               float* __restrict__ y, float* __restrict__ moving_mean, float* __restrict__ moving_var,
               long long N, int C) {
  const int c = blockIdx.x * kTileC + threadIdx.x;
  if (c >= C) return;
  double var = 0.0;
  const Norm q = channel_norm(moments, C, c, &var);
  const float b = __ldg(beta + c);
  if (moving_mean && blockIdx.y == 0 && threadIdx.y == 0) {
    // TF's assign_moving_average without zero-debias, in float32 as the guide's update runs it
    const double n = moments[c];
    const float f = static_cast<float>(1.0 - kBnDecay);
    const float bm = static_cast<float>(moments[C + c]);
    const float bv = static_cast<float>(var * (n > 1.0 ? n / (n - 1.0) : 1.0));
    moving_mean[c] = __fsub_rn(moving_mean[c], __fmul_rn(__fsub_rn(moving_mean[c], bm), f));
    moving_var[c] = __fsub_rn(moving_var[c], __fmul_rn(__fsub_rn(moving_var[c], bv), f));
  }
  const long long step = static_cast<long long>(gridDim.y) * kRowLanes;
  for (long long r = static_cast<long long>(blockIdx.y) * kRowLanes + threadIdx.y; r < N; r += step) {
    const long long i = r * C + c;
    y[i] = fmaxf(preact(centred(__ldg(z + i), q), q, b), 0.0f);
  }
}

// ws[chunk][2][C]: A and B of the chunk's rows, per channel.
__global__ void __launch_bounds__(kTileC * kRowLanes)
grad_partial_kernel(const float* __restrict__ z, const float* __restrict__ dy, const double* __restrict__ moments,
                    const float* __restrict__ beta, double* __restrict__ ws, long long N, int C, long long rows) {
  const int c = blockIdx.x * kTileC + threadIdx.x;
  const long long r0 = static_cast<long long>(blockIdx.y) * rows;
  const long long r1 = r0 + rows < N ? r0 + rows : N;
  const bool valid = c < C;
  double a = 0.0, bsum = 0.0;
  if (valid) {
    const Norm q = channel_norm(moments, C, c, nullptr);
    const float b = __ldg(beta + c);
    for (long long r = r0 + threadIdx.y; r < r1; r += kRowLanes) {
      const long long i = r * C + c;
      const float d = centred(__ldg(z + i), q);
      if (preact(d, q, b) > 0.0f) {
        const double g = static_cast<double>(__ldg(dy + i));
        a += g;
        bsum = fma(g, static_cast<double>(__fmul_rn(d, q.s)), bsum);
      }
    }
  }
  double ta = 0.0, tb = 0.0;
  lane_sums(a, bsum, &ta, &tb);
  if (threadIdx.y != 0 || !valid) return;
  double* out = ws + static_cast<size_t>(blockIdx.y) * 2 * C;
  out[c] = ta;
  out[C + c] = tb;
}

// sums [2][C]: A and B; dbeta [C] (optional): A as float32.
__global__ void __launch_bounds__(32 * kReduceWarps)
grad_reduce_kernel(const double* __restrict__ ws, double* __restrict__ sums, float* __restrict__ dbeta, int C,
                   int chunks) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kReduceWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int k = lane; k < chunks; k += 32) {
    const double* w = ws + static_cast<size_t>(k) * 2 * C;
    a += w[c];
    b += w[C + c];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
  }
  if (lane != 0) return;
  sums[c] = a;
  sums[C + c] = b;
  if (dbeta) dbeta[c] = static_cast<float>(a);
}

__global__ void __launch_bounds__(kTileC * kRowLanes)
grad_kernel(const float* __restrict__ z, const float* __restrict__ dy, const double* __restrict__ moments,
            const float* __restrict__ beta, const double* __restrict__ sums, float* __restrict__ dz, long long N,
            int C) {
  const int c = blockIdx.x * kTileC + threadIdx.x;
  if (c >= C) return;
  const Norm q = channel_norm(moments, C, c, nullptr);
  const float b = __ldg(beta + c);
  const double n = moments[c];
  const float an = static_cast<float>(sums[c] / n), bn = static_cast<float>(sums[C + c] / n);
  const long long step = static_cast<long long>(gridDim.y) * kRowLanes;
  for (long long r = static_cast<long long>(blockIdx.y) * kRowLanes + threadIdx.y; r < N; r += step) {
    const long long i = r * C + c;
    const float d = centred(__ldg(z + i), q);
    const float g = preact(d, q, b) > 0.0f ? __ldg(dy + i) : 0.0f;
    const float t = __fmaf_rn(-__fmul_rn(d, q.s), bn, __fsub_rn(g, an));
    dz[i] = __fmul_rn(t, q.s);
  }
}

bool misaligned(const void* p, uintptr_t mask) { return (reinterpret_cast<uintptr_t>(p) & mask) != 0; }

int check_shape(long long N, int C) {
  if (N < 1 || C < 1) return HDRNET_E_BAD_SHAPE;
  if (C > HDRNET_BN_MAX_CHANNELS) return HDRNET_E_UNSUPPORTED;
  if (N > (1LL << 40) / C) return HDRNET_E_TOO_LARGE;
  return HDRNET_OK;
}

}  // namespace
}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_bn_stats_workspace_bytes(long long N, int C) {
  if (check_shape(N, C) != HDRNET_OK) return 0;
  return static_cast<size_t>(num_chunks(N, C)) * 2 * static_cast<size_t>(C) * sizeof(double);
}

int hdrnet_bn_stats_f32(const float* z, long long N, int C, double* moments, void* workspace,
                        size_t workspace_bytes, void* stream) {
  int rc = check_shape(N, C);
  if (rc != HDRNET_OK) return rc;
  if (!z || !moments || !workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_bn_stats_workspace_bytes(N, C)) return HDRNET_E_BAD_SHAPE;
  if (misaligned(z, 3) || misaligned(moments, 7) || misaligned(workspace, 7)) return HDRNET_E_BAD_SHAPE;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = chunk_rows(N, C);
  const int chunks = static_cast<int>(num_chunks(N, C));
  double* ws = static_cast<double*>(workspace);
  stats_partial_kernel<<<dim3(channel_tiles(C), chunks), dim3(kTileC, kRowLanes), 0, st>>>(z, ws, N, C, rows);
  stats_reduce_kernel<<<(C + kReduceWarps - 1) / kReduceWarps, 32 * kReduceWarps, 0, st>>>(ws, moments, N, C, rows,
                                                                                           chunks);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_bn_relu_f32(const float* z, long long N, int C, const double* moments, const float* beta, float* y,
                       float* moving_mean, float* moving_var, void* stream) {
  int rc = check_shape(N, C);
  if (rc != HDRNET_OK) return rc;
  if (!z || !moments || !beta || !y) return HDRNET_E_NULL_POINTER;
  if ((moving_mean == nullptr) != (moving_var == nullptr)) return HDRNET_E_NULL_POINTER;
  if (misaligned(z, 3) || misaligned(beta, 3) || misaligned(y, 3) || misaligned(moments, 7) ||
      misaligned(moving_mean, 3) || misaligned(moving_var, 3))
    return HDRNET_E_BAD_SHAPE;
  bn_relu_kernel<<<dim3(channel_tiles(C), row_blocks(N)), dim3(kTileC, kRowLanes), 0,
                   static_cast<cudaStream_t>(stream)>>>(z, moments, beta, y, moving_mean, moving_var, N, C);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_bn_relu_grad_sums_f32(const float* z, const float* dy, long long N, int C, const double* moments,
                                 const float* beta, double* sums, float* dbeta, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  int rc = check_shape(N, C);
  if (rc != HDRNET_OK) return rc;
  if (!z || !dy || !moments || !beta || !sums || !workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_bn_stats_workspace_bytes(N, C)) return HDRNET_E_BAD_SHAPE;
  if (misaligned(z, 3) || misaligned(dy, 3) || misaligned(beta, 3) || misaligned(dbeta, 3) ||
      misaligned(moments, 7) || misaligned(sums, 7) || misaligned(workspace, 7))
    return HDRNET_E_BAD_SHAPE;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = chunk_rows(N, C);
  const int chunks = static_cast<int>(num_chunks(N, C));
  double* ws = static_cast<double*>(workspace);
  grad_partial_kernel<<<dim3(channel_tiles(C), chunks), dim3(kTileC, kRowLanes), 0, st>>>(z, dy, moments, beta, ws,
                                                                                          N, C, rows);
  grad_reduce_kernel<<<(C + kReduceWarps - 1) / kReduceWarps, 32 * kReduceWarps, 0, st>>>(ws, sums, dbeta, C,
                                                                                          chunks);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_bn_relu_grad_f32(const float* z, const float* dy, long long N, int C, const double* moments,
                            const float* beta, const double* sums, float* dz, void* stream) {
  int rc = check_shape(N, C);
  if (rc != HDRNET_OK) return rc;
  if (!z || !dy || !moments || !beta || !sums || !dz) return HDRNET_E_NULL_POINTER;
  if (misaligned(z, 3) || misaligned(dy, 3) || misaligned(beta, 3) || misaligned(dz, 3) ||
      misaligned(moments, 7) || misaligned(sums, 7))
    return HDRNET_E_BAD_SHAPE;
  grad_kernel<<<dim3(channel_tiles(C), row_blocks(N)), dim3(kTileC, kRowLanes), 0,
                static_cast<cudaStream_t>(stream)>>>(z, dy, moments, beta, sums, dz, N, C);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
