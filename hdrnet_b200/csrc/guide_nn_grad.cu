// guide_nn_grad.cu -- the pointwise-NN guide in training mode (HDRNetPointwiseNNGuide._guide with
// is_training=True, hdrnet/models.py:203-210): conv1's batch norm normalises with the batch's
// statistics.  The batch statistics, their fold into the existing forward (guide.cu), and the VJP
// of the whole guide with the gradient through the statistics.
//
// Per pixel p, with x_p the RGB input, F features, N pixels:
//   z_pf = x_p . W1[:, f],  mu_f = m . W1[:, f],  var_f = W1[:, f]' C W1[:, f]   (m, C: the input's
//   mean and biased covariance),  s_f = 1 / sqrt(var_f + 1e-3),  xh_pf = (z_pf - mu_f) s_f,
//   y_pf = xh_pf + beta_f,  o_p = sum_f relu(y_pf) w2_f + b2,  guide_p = sigmoid(o_p)
// The forward is hdrnet_guide_nn_f32 with W1'_if = W1_if s_f and b1'_f = beta_f - mu_f s_f
// (hdrnet_guide_nn_batch_fold).  Given g_p = dL/dguide_p:
//   do_p = g_p guide_p (1 - guide_p),  dy_pf = do_p w2_f [y_pf > 0]   (TF's ReluGrad: 0 at y = 0)
//   A_f = sum_p dy_pf (= d beta_f),  B_f = sum_p dy_pf xh_pf,  D_if = sum_p x_pi dy_pf
//   d w2_f = sum_p do_p relu(y_pf),  d b2 = sum_p do_p
//   dz_pf = s_f (dy_pf - A_f / N - xh_pf B_f / N)
//   d W1_if = sum_p x_pi dz_pf = s_f (D_if - m_i A_f - s_f (C W1)_if B_f),  dx_pi = sum_f W1_if dz_pf
// y and guide are recomputed with nn_guide_preact2 / nn_guide_sigmoid on the folded float32
// weights the forward used, so every relu mask is the one the forward's floats decide.
//
//   stats_partial_kernel   one pass over x (12 B/px): each CTA sums one fixed chunk, centred on the
//                          chunk's first pixel, in float64, and writes the chunk's mean and M2.
//   stats_reduce_kernel    one warp merges the chunks (Chan et al.) in float64, in a fixed order.
//   vjp_partial_kernel     one pass over x and g (16 B/px): the 6 F + 1 sums of one fixed chunk
//                          for one group of kGroup features (blockIdx.x), so nothing spills.
//   vjp_finish_kernel      one CTA per feature adds the chunks in a fixed order and applies the
//                          closed forms above in float64.
//   vjp_dx_kernel          only when dinput is wanted: a second pass (16 B/px in, 12 B/px out).
// The chunking depends on npix alone and there are no atomics, so a call gives the same bits on
// every run and every device.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstring>

#include "guide.cuh"
#include "hdrnet_b200.h"

namespace hdrnet_b200 {

int pack_nn_params(NNGuideParams* p, const float* w1, const float* b1, const float* w2, float b2,
                   int feats);

namespace {

constexpr int kThreads = 128;
constexpr int kMaxChunks = 1024;   // chunks grow with npix beyond kMaxChunks * 512 pixels
constexpr int kMoments = 9;        // m0 m1 m2, c00 c01 c02 c11 c12 c22
constexpr int kGroup = 8;          // features whose sums one VJP CTA keeps (6 * 8 + 1 registers)
constexpr int kKinds = 6;          // per feature: d w2, A, B, D_0, D_1, D_2
constexpr double kBnEps = 1e-3;    // tf.contrib.layers.batch_norm's default epsilon

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

// ---- batch statistics ----------------------------------------------------------------------------

__device__ __forceinline__ void add_moments(const double k[3], float a, float b, float c, double (&v)[kMoments]) {
  const double d0 = static_cast<double>(a) - k[0], d1 = static_cast<double>(b) - k[1],
               d2 = static_cast<double>(c) - k[2];
  v[0] += d0;
  v[1] += d1;
  v[2] += d2;
  v[3] = fma(d0, d0, v[3]);
  v[4] = fma(d0, d1, v[4]);
  v[5] = fma(d0, d2, v[5]);
  v[6] = fma(d1, d1, v[6]);
  v[7] = fma(d1, d2, v[7]);
  v[8] = fma(d2, d2, v[8]);
}

// ws[chunk][9]: the chunk's mean (3) and its sum of centred cross products M2 (6), in float64.
__global__ void __launch_bounds__(kThreads)
stats_partial_kernel(const float* __restrict__ x, double* __restrict__ ws, long long npix,
                     long long chunk_px, bool vec_ok) {
  const long long p0 = static_cast<long long>(blockIdx.x) * chunk_px;
  const long long p1 = p0 + chunk_px < npix ? p0 + chunk_px : npix;
  // Centred on the chunk's first pixel: a large common offset cancels before anything is squared.
  const double k[3] = {__ldg(x + 3 * p0), __ldg(x + 3 * p0 + 1), __ldg(x + 3 * p0 + 2)};
  double v[kMoments];
#pragma unroll
  for (int i = 0; i < kMoments; ++i) v[i] = 0.0;
  long long scalar0 = p0;
  if (vec_ok) {
    const long long q0 = p0 / 4, q1 = p1 / 4;
    for (long long q = q0 + threadIdx.x; q < q1; q += kThreads) {
      const float4* in4 = reinterpret_cast<const float4*>(x) + 3 * q;
      const float4 c0 = __ldg(in4), c1 = __ldg(in4 + 1), c2 = __ldg(in4 + 2);
      add_moments(k, c0.x, c0.y, c0.z, v);
      add_moments(k, c0.w, c1.x, c1.y, v);
      add_moments(k, c1.z, c1.w, c2.x, v);
      add_moments(k, c2.y, c2.z, c2.w, v);
    }
    scalar0 = q1 * 4;
  }
  for (long long i = scalar0 + threadIdx.x; i < p1; i += kThreads)
    add_moments(k, __ldg(x + 3 * i), __ldg(x + 3 * i + 1), __ldg(x + 3 * i + 2), v);
  // CTA sum in a fixed order: xor tree within each warp, then the warps in order.
  __shared__ double warp_sums[kThreads / 32][kMoments];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kMoments; ++i) {
    double s = v[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) warp_sums[warp][i] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double t[kMoments];
#pragma unroll
  for (int i = 0; i < kMoments; ++i) {
    t[i] = warp_sums[0][i];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) t[i] += warp_sums[w][i];
  }
  const double n = static_cast<double>(p1 - p0);
  double* out = ws + static_cast<size_t>(blockIdx.x) * kMoments;
  out[0] = k[0] + t[0] / n;
  out[1] = k[1] + t[1] / n;
  out[2] = k[2] + t[2] / n;
  out[3] = t[3] - t[0] * t[0] / n;
  out[4] = t[4] - t[0] * t[1] / n;
  out[5] = t[5] - t[0] * t[2] / n;
  out[6] = t[6] - t[1] * t[1] / n;
  out[7] = t[7] - t[1] * t[2] / n;
  out[8] = t[8] - t[2] * t[2] / n;
}

// (n, mean, M2) += (nb, mb, M2b): the pairwise update of Chan, Golub and LeVeque.
__device__ __forceinline__ void merge_moments(double& n, double (&a)[kMoments], double nb, const double* b) {
  if (nb == 0.0) return;
  const double nt = n + nb, f = nb / nt, w = n * nb / nt;
  const double d[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]};
  a[0] += d[0] * f;
  a[1] += d[1] * f;
  a[2] += d[2] * f;
  a[3] += b[3] + d[0] * d[0] * w;
  a[4] += b[4] + d[0] * d[1] * w;
  a[5] += b[5] + d[0] * d[2] * w;
  a[6] += b[6] + d[1] * d[1] * w;
  a[7] += b[7] + d[1] * d[2] * w;
  a[8] += b[8] + d[2] * d[2] * w;
  n = nt;
}

// One warp: lane l merges chunks l, l + 32, ... in order, then lane 0 merges the lanes in order.
__global__ void __launch_bounds__(32)
stats_reduce_kernel(const double* __restrict__ ws, double* __restrict__ moments, long long npix,
                    long long chunk_px, int chunks) {
  const int lane = threadIdx.x;
  double n = 0.0, a[kMoments];
#pragma unroll
  for (int i = 0; i < kMoments; ++i) a[i] = 0.0;
  for (int c = lane; c < chunks; c += 32) {
    const long long p0 = static_cast<long long>(c) * chunk_px;
    const long long nc = p0 + chunk_px < npix ? chunk_px : npix - p0;
    merge_moments(n, a, static_cast<double>(nc), ws + static_cast<size_t>(c) * kMoments);
  }
  __shared__ double lanes[32][kMoments + 1];
  lanes[lane][0] = n;
#pragma unroll
  for (int i = 0; i < kMoments; ++i) lanes[lane][i + 1] = a[i];
  __syncwarp();
  if (lane != 0) return;
  for (int l = 1; l < 32; ++l) merge_moments(n, a, lanes[l][0], &lanes[l][1]);
  for (int i = 0; i < 3; ++i) moments[i] = a[i];
  for (int i = 3; i < kMoments; ++i) moments[i] = a[i] / n;    // biased: the one that normalises
}

// ---- the fold (host, float64) ----------------------------------------------------------------------

struct BatchFold {
  double mean[kMaxGuideFeats], var[kMaxGuideFeats], s[kMaxGuideFeats];
  float w1[3 * kMaxGuideFeats], b1[kMaxGuideFeats];
};

void fold_batch_norm(const float* w1, const float* beta, const double* mom, int feats, BatchFold* out) {
  const double C[3][3] = {{mom[3], mom[4], mom[5]}, {mom[4], mom[6], mom[7]}, {mom[5], mom[7], mom[8]}};
  for (int f = 0; f < feats; ++f) {
    double w[3], mu = 0.0, var = 0.0;
    for (int i = 0; i < 3; ++i) {
      w[i] = w1[i * feats + f];
      mu += mom[i] * w[i];
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) var += w[i] * C[i][j] * w[j];
    if (var < 0.0) var = 0.0;          // rounding of a (near-)singular C
    const double s = 1.0 / std::sqrt(var + kBnEps);
    out->mean[f] = mu;
    out->var[f] = var;
    out->s[f] = s;
    for (int i = 0; i < 3; ++i) out->w1[i * feats + f] = static_cast<float>(w[i] * s);
    out->b1[f] = static_cast<float>(static_cast<double>(beta[f]) - mu * s);
  }
}

// ---- VJP -------------------------------------------------------------------------------------------

struct VjpParams {
  NNGuideParams p;                 // the folded forward (pack_nn_params of the fold)
  float beta[kMaxGuideFeats];      // 0 beyond feats
  int feats;                       // the caller's feature count (p.feats is rounded up to even)
};

// One pixel: the 6 kGroup (+ 1 for group 0) sums of features G * kGroup ... into acc.
template <int kFeats, int G>
__device__ __forceinline__ void pixel_sums(const VjpParams& q, float r, float g, float b, float dg,
                                           float (&acc)[kKinds * kGroup + 1]) {
  const unsigned long long r2 = pack2(r, r), g2 = pack2(g, g), b2v = pack2(b, b);
  unsigned long long y2 = 0ull;
  float y[kGroup];
#pragma unroll
  for (int f = 0; f < kFeats; f += 2) {
    float h0, h1;
    unpack2(nn_guide_preact2(q.p, r2, g2, b2v, f), h0, h1);
    y2 = fma2(pack2(fmaxf(h0, 0.0f), fmaxf(h1, 0.0f)), pack2(q.p.w2[f], q.p.w2[f + 1]), y2);
    if (f >= G * kGroup && f < (G + 1) * kGroup) {
      y[f - G * kGroup] = h0;
      y[f + 1 - G * kGroup] = h1;
    }
  }
  const float sg = nn_guide_sigmoid(q.p, y2);
  const float d = dg * sg * (1.0f - sg);
#pragma unroll
  for (int j = 0; j < kGroup; ++j) {
    const int f = G * kGroup + j;
    const float dy = y[j] > 0.0f ? d * q.p.w2[f] : 0.0f;
    const float xh = y[j] - q.beta[f];
    acc[0 * kGroup + j] = fmaf(d, fmaxf(y[j], 0.0f), acc[0 * kGroup + j]);
    acc[1 * kGroup + j] += dy;
    acc[2 * kGroup + j] = fmaf(dy, xh, acc[2 * kGroup + j]);
    acc[3 * kGroup + j] = fmaf(r, dy, acc[3 * kGroup + j]);
    acc[4 * kGroup + j] = fmaf(g, dy, acc[4 * kGroup + j]);
    acc[5 * kGroup + j] = fmaf(b, dy, acc[5 * kGroup + j]);
  }
  if (G == 0) acc[kKinds * kGroup] += d;
}

// ws[chunk][6 feats + 1]: [kind][feature] then d b2.
template <int kFeats, int G>
__device__ __forceinline__ void chunk_sums(const float* __restrict__ x, const float* __restrict__ dguide,
                                           float* __restrict__ ws, long long npix, long long chunk_px,
                                           bool vec_ok, const VjpParams& q) {
  constexpr int kN = kKinds * kGroup + 1;
  float acc[kN];
#pragma unroll
  for (int i = 0; i < kN; ++i) acc[i] = 0.0f;
  const long long p0 = static_cast<long long>(blockIdx.y) * chunk_px;
  const long long p1 = p0 + chunk_px < npix ? p0 + chunk_px : npix;
  long long scalar0 = p0;
  if (vec_ok) {
    const long long q0 = p0 / 4, q1 = p1 / 4;
    for (long long i = q0 + threadIdx.x; i < q1; i += kThreads) {
      const float4* in4 = reinterpret_cast<const float4*>(x) + 3 * i;
      const float4 c0 = __ldg(in4), c1 = __ldg(in4 + 1), c2 = __ldg(in4 + 2);
      const float4 gv = __ldg(reinterpret_cast<const float4*>(dguide) + i);
      pixel_sums<kFeats, G>(q, c0.x, c0.y, c0.z, gv.x, acc);
      pixel_sums<kFeats, G>(q, c0.w, c1.x, c1.y, gv.y, acc);
      pixel_sums<kFeats, G>(q, c1.z, c1.w, c2.x, gv.z, acc);
      pixel_sums<kFeats, G>(q, c2.y, c2.z, c2.w, gv.w, acc);
    }
    scalar0 = q1 * 4;
  }
  for (long long i = scalar0 + threadIdx.x; i < p1; i += kThreads)
    pixel_sums<kFeats, G>(q, __ldg(x + 3 * i), __ldg(x + 3 * i + 1), __ldg(x + 3 * i + 2),
                          __ldg(dguide + i), acc);
  // CTA sum in a fixed order: xor tree within each warp, then the warps in order.
  __shared__ float warp_sums[kThreads / 32][kN];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kN; ++i) {
    float s = acc[i];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) warp_sums[warp][i] = s;
  }
  __syncthreads();
  const int nsum = kKinds * q.feats + 1;
  float* out = ws + static_cast<size_t>(blockIdx.y) * nsum;
  for (int i = threadIdx.x; i < kN; i += kThreads) {
    float s = warp_sums[0][i];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) s += warp_sums[w][i];
    if (i == kKinds * kGroup) {
      if (G == 0) out[kKinds * q.feats] = s;
    } else {
      const int kind = i / kGroup, f = G * kGroup + i % kGroup;
      if (f < q.feats) out[kind * q.feats + f] = s;
    }
  }
}

// blockIdx.x = feature group, blockIdx.y = pixel chunk (the groups of a chunk run side by side and
// share its reads in L2).  Every CTA recomputes the whole forward of its pixels.
template <int kFeats>
__global__ void __launch_bounds__(kThreads)
vjp_partial_kernel(const float* __restrict__ x, const float* __restrict__ dguide, float* __restrict__ ws,
                   long long npix, long long chunk_px, bool vec_ok, const __grid_constant__ VjpParams q) {
  static_assert(kFeats % kGroup == 0 && kFeats <= 4 * kGroup, "feature groups");
  switch (blockIdx.x) {
    case 0: chunk_sums<kFeats, 0>(x, dguide, ws, npix, chunk_px, vec_ok, q); break;
    case 1: chunk_sums<kFeats, 1>(x, dguide, ws, npix, chunk_px, vec_ok, q); break;
    case 2: if (kFeats > 2 * kGroup) chunk_sums<kFeats, 2 % (kFeats / kGroup)>(x, dguide, ws, npix, chunk_px, vec_ok, q); break;
    default: if (kFeats > 3 * kGroup) chunk_sums<kFeats, 3 % (kFeats / kGroup)>(x, dguide, ws, npix, chunk_px, vec_ok, q); break;
  }
}

struct FinishParams {
  double m[3];                      // the input's mean
  double cw1[3][kMaxGuideFeats];    // (C W1)_if
  double s[kMaxGuideFeats];
  int feats;
  double inv_n;
};

// CTA f: warp k sums kind k of feature f over the chunks (lane l: chunks l, l + 32, ... in order,
// then a fixed xor tree), warp 6 of CTA 0 sums d b2.  Thread 0 then applies the closed forms.
// sums [2][32] gets A / N and B / N for the dx pass.
__global__ void __launch_bounds__(32 * (kKinds + 1))
vjp_finish_kernel(const float* __restrict__ ws, int chunks, float* __restrict__ dparams,
                  float* __restrict__ sums, const __grid_constant__ FinishParams fp) {
  const int f = blockIdx.x, F = fp.feats, nsum = kKinds * F + 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ double tot[kKinds + 1];
  if (warp < kKinds || f == 0) {
    const int e = warp < kKinds ? warp * F + f : kKinds * F;
    double s = 0.0;
    for (int c = lane; c < chunks; c += 32) s += ws[static_cast<size_t>(c) * nsum + e];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) tot[warp] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double A = tot[1], B = tot[2], s = fp.s[f];
  sums[f] = static_cast<float>(A * fp.inv_n);
  sums[kMaxGuideFeats + f] = static_cast<float>(B * fp.inv_n);
  if (!dparams) return;
  for (int i = 0; i < 3; ++i)
    dparams[i * F + f] = static_cast<float>(s * (tot[3 + i] - fp.m[i] * A - s * fp.cw1[i][f] * B));
  dparams[3 * F + f] = static_cast<float>(A);
  dparams[4 * F + f] = static_cast<float>(tot[0]);
  if (f == 0) dparams[5 * F] = static_cast<float>(tot[kKinds]);
}

// dx_i = sum_f W1'_if (dy_f - xh_f B_f / N) - sum_f W1'_if A_f / N, with W1' = W1 s the folded
// weights (dz_f = s_f (dy_f - A_f / N - xh_f B_f / N)).
template <int kFeats>
__device__ __forceinline__ void pixel_dx(const VjpParams& q, const float* bn, const float c[3], float r,
                                         float g, float b, float dg, float& d0, float& d1, float& d2) {
  const unsigned long long r2 = pack2(r, r), g2 = pack2(g, g), b2v = pack2(b, b);
  unsigned long long y2 = 0ull;
  float y[kFeats];
#pragma unroll
  for (int f = 0; f < kFeats; f += 2) {
    unpack2(nn_guide_preact2(q.p, r2, g2, b2v, f), y[f], y[f + 1]);
    y2 = fma2(pack2(fmaxf(y[f], 0.0f), fmaxf(y[f + 1], 0.0f)), pack2(q.p.w2[f], q.p.w2[f + 1]), y2);
  }
  const float sg = nn_guide_sigmoid(q.p, y2);
  const float d = dg * sg * (1.0f - sg);
  d0 = -c[0];
  d1 = -c[1];
  d2 = -c[2];
#pragma unroll
  for (int f = 0; f < kFeats; ++f) {
    const float dy = y[f] > 0.0f ? d * q.p.w2[f] : 0.0f;
    const float t = fmaf(-(y[f] - q.beta[f]), bn[f], dy);
    d0 = fmaf(q.p.w1[0][f], t, d0);
    d1 = fmaf(q.p.w1[1][f], t, d1);
    d2 = fmaf(q.p.w1[2][f], t, d2);
  }
}

template <int kFeats>
__global__ void __launch_bounds__(256)
vjp_dx_kernel(const float* __restrict__ x, const float* __restrict__ dguide, float* __restrict__ dx,
              long long npix, bool vec_ok, const float* __restrict__ sums,
              const __grid_constant__ VjpParams q) {
  __shared__ float an[kFeats], bn[kFeats];
  for (int f = threadIdx.x; f < kFeats; f += blockDim.x) {
    an[f] = f < q.feats ? sums[f] : 0.0f;
    bn[f] = f < q.feats ? sums[kMaxGuideFeats + f] : 0.0f;
  }
  __syncthreads();
  float c[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int f = 0; f < kFeats; ++f) {
    c[0] = fmaf(q.p.w1[0][f], an[f], c[0]);
    c[1] = fmaf(q.p.w1[1][f], an[f], c[1]);
    c[2] = fmaf(q.p.w1[2][f], an[f], c[2]);
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long tid0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nquads = vec_ok ? npix / 4 : 0;
  for (long long i = tid0; i < nquads; i += stride) {
    const float4* in4 = reinterpret_cast<const float4*>(x) + 3 * i;
    const float4 c0 = __ldg(in4), c1 = __ldg(in4 + 1), c2 = __ldg(in4 + 2);
    const float4 gv = __ldg(reinterpret_cast<const float4*>(dguide) + i);
    float4 o0, o1, o2;
    pixel_dx<kFeats>(q, bn, c, c0.x, c0.y, c0.z, gv.x, o0.x, o0.y, o0.z);
    pixel_dx<kFeats>(q, bn, c, c0.w, c1.x, c1.y, gv.y, o0.w, o1.x, o1.y);
    pixel_dx<kFeats>(q, bn, c, c1.z, c1.w, c2.x, gv.z, o1.z, o1.w, o2.x);
    pixel_dx<kFeats>(q, bn, c, c2.y, c2.z, c2.w, gv.w, o2.y, o2.z, o2.w);
    float4* out4 = reinterpret_cast<float4*>(dx) + 3 * i;
    out4[0] = o0;
    out4[1] = o1;
    out4[2] = o2;
  }
  // the tail (npix % 4), or every pixel when a buffer is not 16-byte aligned
  for (long long i = nquads * 4 + tid0; i < npix; i += stride) {
    float d0, d1, d2;
    pixel_dx<kFeats>(q, bn, c, __ldg(x + 3 * i), __ldg(x + 3 * i + 1), __ldg(x + 3 * i + 2),
                     __ldg(dguide + i), d0, d1, d2);
    dx[3 * i] = d0;
    dx[3 * i + 1] = d1;
    dx[3 * i + 2] = d2;
  }
}

template <int kFeats>
int launch_vjp(const float* x, const float* dguide, float* dx, long long npix, float* ws,
               float* dparams, const VjpParams& q, const FinishParams& fp, cudaStream_t st) {
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dguide)) & 15u) == 0;
  const int chunks = static_cast<int>(num_chunks(npix));
  const dim3 grid((q.p.feats + kGroup - 1) / kGroup, chunks);
  vjp_partial_kernel<kFeats><<<grid, kThreads, 0, st>>>(x, dguide, ws, npix, chunk_pixels(npix), vec_ok, q);
  float* sums = ws + static_cast<size_t>(chunks) * (kKinds * q.feats + 1);
  vjp_finish_kernel<<<q.feats, 32 * (kKinds + 1), 0, st>>>(ws, chunks, dparams, sums, fp);
  if (!dx) return static_cast<int>(cudaGetLastError());
  const bool dx_vec = vec_ok && (reinterpret_cast<uintptr_t>(dx) & 15u) == 0;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long work = dx_vec ? (npix + 3) / 4 : npix;
  long long blocks = (work + 255) / 256;
  if (blocks > static_cast<long long>(sms) * 8) blocks = static_cast<long long>(sms) * 8;
  vjp_dx_kernel<kFeats><<<static_cast<int>(blocks), 256, 0, st>>>(x, dguide, dx, npix, dx_vec, sums, q);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace
}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_guide_nn_stats_workspace_bytes(long long npix) {
  if (npix <= 0) return 0;
  return static_cast<size_t>(num_chunks(npix)) * kMoments * sizeof(double);
}

int hdrnet_guide_nn_stats_f32(const float* input, long long npix, double* moments, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (npix < 0) return HDRNET_E_BAD_SHAPE;
  if (!moments) return HDRNET_E_NULL_POINTER;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (npix == 0) return static_cast<int>(cudaMemsetAsync(moments, 0, kMoments * sizeof(double), st));
  if (!input || !workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_guide_nn_stats_workspace_bytes(npix)) return HDRNET_E_BAD_SHAPE;
  // float64 partials: the workspace and the moments must be 8-byte aligned
  if ((reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(moments)) & 7u)
    return HDRNET_E_BAD_SHAPE;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(input) & 15u) == 0;
  const long long cp = chunk_pixels(npix);
  const int chunks = static_cast<int>(num_chunks(npix));
  double* ws = static_cast<double*>(workspace);
  stats_partial_kernel<<<chunks, kThreads, 0, st>>>(input, ws, npix, cp, vec_ok);
  stats_reduce_kernel<<<1, 32, 0, st>>>(ws, moments, npix, cp, chunks);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_guide_nn_batch_fold(const float* w1, const float* beta, const double* moments, int feats,
                               float* w1_folded, float* b1_folded, double* batch_mean,
                               double* batch_var) {
  if (!w1 || !beta || !moments || !w1_folded || !b1_folded) return HDRNET_E_NULL_POINTER;
  if (feats < 1 || feats > kMaxGuideFeats) return HDRNET_E_UNSUPPORTED;
  BatchFold bf;
  fold_batch_norm(w1, beta, moments, feats, &bf);
  std::memcpy(w1_folded, bf.w1, sizeof(float) * 3 * feats);
  std::memcpy(b1_folded, bf.b1, sizeof(float) * feats);
  if (batch_mean) std::memcpy(batch_mean, bf.mean, sizeof(double) * feats);
  if (batch_var) std::memcpy(batch_var, bf.var, sizeof(double) * feats);
  return HDRNET_OK;
}

size_t hdrnet_guide_nn_grad_workspace_bytes(long long npix, int feats) {
  if (npix <= 0 || feats < 1 || feats > kMaxGuideFeats) return 0;
  return (static_cast<size_t>(num_chunks(npix)) * (kKinds * feats + 1) + 2 * kMaxGuideFeats) * sizeof(float);
}

int hdrnet_guide_nn_grad_f32(const float* input, const float* dguide, float* dinput, long long npix,
                             const float* w1, const float* beta, const float* w2, float b2, int feats,
                             const double* moments, float* dparams, void* workspace,
                             size_t workspace_bytes, void* stream) {
  if (!w1 || !beta || !w2 || !moments) return HDRNET_E_NULL_POINTER;
  if (feats < 1 || feats > kMaxGuideFeats) return HDRNET_E_UNSUPPORTED;
  if (npix < 0) return HDRNET_E_BAD_SHAPE;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (npix == 0) {   // nothing to sum: the parameter gradients are zero
    if (dparams) return static_cast<int>(cudaMemsetAsync(dparams, 0, (5 * feats + 1) * sizeof(float), st));
    return HDRNET_OK;
  }
  if (!dinput && !dparams) return HDRNET_OK;
  if (!input || !dguide || !workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_guide_nn_grad_workspace_bytes(npix, feats)) return HDRNET_E_BAD_SHAPE;
  BatchFold bf;
  fold_batch_norm(w1, beta, moments, feats, &bf);
  VjpParams q;
  std::memset(&q, 0, sizeof(q));
  const int rc = pack_nn_params(&q.p, bf.w1, bf.b1, w2, b2, feats);
  if (rc != HDRNET_OK) return rc;
  std::memcpy(q.beta, beta, sizeof(float) * feats);
  q.feats = feats;
  FinishParams fp;
  std::memset(&fp, 0, sizeof(fp));
  const double C[3][3] = {{moments[3], moments[4], moments[5]}, {moments[4], moments[6], moments[7]},
                          {moments[5], moments[7], moments[8]}};
  for (int i = 0; i < 3; ++i) fp.m[i] = moments[i];
  for (int f = 0; f < feats; ++f) {
    fp.s[f] = bf.s[f];
    for (int i = 0; i < 3; ++i) {
      double a = 0.0;
      for (int j = 0; j < 3; ++j) a += C[i][j] * static_cast<double>(w1[j * feats + f]);
      fp.cw1[i][f] = a;
    }
  }
  fp.feats = feats;
  fp.inv_n = 1.0 / static_cast<double>(npix);
  float* ws = static_cast<float*>(workspace);
  if (q.p.feats <= 16) return launch_vjp<16>(input, dguide, dinput, npix, ws, dparams, q, fp, st);
  return launch_vjp<kMaxGuideFeats>(input, dguide, dinput, npix, ws, dparams, q, fp, st);
}

}  // extern "C"
