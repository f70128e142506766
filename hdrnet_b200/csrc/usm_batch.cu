// usm_batch.cu -- one training batch of UnsharpMaskDataPipeline (row f-15): the input crop and
// network input of train_batch.cu, and a target computed from the input alone,
//   t = clip(x + sharpen * (x - G_sigma * x), 0, 1),
// with G_sigma the separable Gaussian of scipy.ndimage.gaussian_filter1d (truncate = 4.0, radius
// r = int(4 sigma + 0.5), weights exp(-k^2 / 2 sigma^2) normalised to sum 1) and half-sample
// symmetric reflection at the SOURCE image's edges (scipy's mode "reflect", repeated when r is
// not smaller than the extent).
//
// The blur runs in source coordinates, so a source pixel's target does not depend on the draw:
//   pass 1 (usm_rows_kernel): per sample, each source row of the crop's source window grown by r
//     rows (clipped to the source), over the crop's source columns, blurred along x into float32
//     workspace rows; a block stages one row segment and its 2r reflected halo columns in shared
//     memory (at most (128 + 256) pixels).
//   pass 2 (usm_target_kernel): per output pixel of the augmented crop, the workspace column at its
//     source pixel blurred along y, the unsharp step, the clip and the store at the augmented
//     position; the same launch writes the input crop and the nearest-neighbour network input as
//     train_batch_kernel does (same conversion, same index: the same bits).
// Both passes sum the taps in float64 in one fixed order, w[0] x[0] + sum_{k = 1..r} w[k] (x[-k] +
// x[+k]) with k ascending, and round once to float32; no atomics: bitwise the same from run to run.
// The window a sample's buffer holds may be the whole source (the device tier) or the crop's source
// window grown by r and clipped to the source (the streamed tier): every reflected index of the
// crop's blur lies inside that window, so both give the same bits.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "hdrnet_b200.h"
#include "slice_rows.cuh"

namespace hdrnet_b200 {

constexpr int kUsmSamples = 16;       // descriptors per launch (they travel in the parameter block)
constexpr int kUsmRowTile = 128;      // pass 1: columns per block
constexpr int kUsmX = 32, kUsmY = 8;  // pass 2: 2-D output tiles, as train_batch_kernel
constexpr int kUsmMaxRadius = 128;    // r = int(4 * 32 + 0.5)
constexpr size_t kUsmAlign = 256;     // each sample's workspace rows start 256-byte aligned

struct UsmSample {
  const unsigned char* input;  // the window [h, w, 3], row pitch w pixels
  long long ws;                // first float of the sample's workspace rows
  int fmt;
  int H, W;                    // the full source
  int y0, x0, w;               // the window's origin and row pitch
  int fliplr, flipud, rot90, crop_y, crop_x;
  int cx0, cw;                 // the crop's source columns [cx0, cx0 + cw)
  int gy0, grows;              // workspace rows: source rows [gy0, gy0 + grows)
};

struct UsmArgs {
  UsmSample s[kUsmSamples];
  double wt[kUsmMaxRadius + 1];  // wt[|k|], k = -r..r
  float* ws;
  float* fullres_in;
  float* fullres_out;
  float* lowres_in;
  long long b0;
  double sharpen;
  int radius;
  int ctiles;                    // pass 1: column tiles per row (the launch's widest crop)
  int oh, ow, S;
  int full_tiles_y;
  float sy, sx;
};

// Half-sample symmetric reflection into [0, n), repeated (period 2n): scipy's mode "reflect".
__device__ __forceinline__ int usm_reflect(int i, int n) {
  if (i >= 0 && i < n) return i;
  const int p = 2 * n;
  int m = i % p;
  if (m < 0) m += p;
  return m < n ? m : p - 1 - m;
}

__device__ __forceinline__ float usm_load(const unsigned char* base, int fmt, long long e) {
  if (fmt == kPxU8) return load_channel<kPxU8>(base, e);
  if (fmt == kPxU16) return load_channel<kPxU16>(base, e);
  return load_channel<kPxF32>(base, e);
}

// Element index (pixel * 3) of source pixel (y, x) in the sample's window buffer.
__device__ __forceinline__ long long usm_elem(const UsmSample& s, int y, int x) {
  return (static_cast<long long>(y - s.y0) * s.w + (x - s.x0)) * 3;
}

// Source pixel (y, x) of crop pixel (i, j): train_batch.cu's source_pixel.
__device__ __forceinline__ void usm_source(const UsmSample& s, int i, int j, int& y, int& x) {
  const int r = s.crop_y + i, c = s.crop_x + j;
  switch (s.rot90) {
    case 1: y = c; x = s.W - 1 - r; break;
    case 2: y = s.H - 1 - r; x = s.W - 1 - c; break;
    case 3: y = s.H - 1 - c; x = r; break;
    default: y = r; x = c; break;
  }
  if (s.flipud) y = s.H - 1 - y;
  if (s.fliplr) x = s.W - 1 - x;
}

__global__ void __launch_bounds__(kUsmRowTile) usm_rows_kernel(const __grid_constant__ UsmArgs a) {
  __shared__ float px[(kUsmRowTile + 2 * kUsmMaxRadius) * 3];
  const UsmSample& s = a.s[blockIdx.z];
  const int row = static_cast<int>(blockIdx.x / a.ctiles);
  const int c0 = static_cast<int>(blockIdx.x % a.ctiles) * kUsmRowTile;
  if (row >= s.grows || c0 >= s.cw) return;
  const int r = a.radius;
  const int y = s.gy0 + row;
  const int n = min(kUsmRowTile, s.cw - c0) + 2 * r;
  for (int e = threadIdx.x; e < n; e += kUsmRowTile) {
    const long long p = usm_elem(s, y, usm_reflect(s.cx0 + c0 - r + e, s.W));
    px[3 * e] = usm_load(s.input, s.fmt, p);
    px[3 * e + 1] = usm_load(s.input, s.fmt, p + 1);
    px[3 * e + 2] = usm_load(s.input, s.fmt, p + 2);
  }
  __syncthreads();
  const int j = threadIdx.x;
  if (c0 + j >= s.cw) return;
  const float* q = px + 3 * (j + r);
  double acc[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) acc[c] = a.wt[0] * static_cast<double>(q[c]);
  for (int k = 1; k <= r; ++k) {
    const double wk = a.wt[k];
#pragma unroll
    for (int c = 0; c < 3; ++c)
      acc[c] = fma(wk, static_cast<double>(q[c - 3 * k]) + static_cast<double>(q[c + 3 * k]), acc[c]);
  }
  float* o = a.ws + s.ws + (static_cast<long long>(row) * s.cw + c0 + j) * 3;
  o[0] = static_cast<float>(acc[0]);
  o[1] = static_cast<float>(acc[1]);
  o[2] = static_cast<float>(acc[2]);
}

__global__ void __launch_bounds__(kUsmX * kUsmY) usm_target_kernel(const __grid_constant__ UsmArgs a) {
  const UsmSample& s = a.s[blockIdx.z];
  const long long b = a.b0 + blockIdx.z;
  const int j = blockIdx.x * kUsmX + threadIdx.x;
  int y, x;
  if (static_cast<int>(blockIdx.y) < a.full_tiles_y) {
    const int i = blockIdx.y * kUsmY + threadIdx.y;
    if (i >= a.oh || j >= a.ow) return;
    usm_source(s, i, j, y, x);
    const long long e = usm_elem(s, y, x);
    const long long o = ((b * a.oh + i) * a.ow + j) * 3;
    const float v[3] = {usm_load(s.input, s.fmt, e), usm_load(s.input, s.fmt, e + 1),
                        usm_load(s.input, s.fmt, e + 2)};
    if (a.fullres_in != nullptr) {
      a.fullres_in[o] = v[0];
      a.fullres_in[o + 1] = v[1];
      a.fullres_in[o + 2] = v[2];
    }
    // the workspace column of source column x; row k of it is source row gy0 + k
    const float* col = a.ws + s.ws + static_cast<long long>(x - s.cx0) * 3;
    const long long pitch = static_cast<long long>(s.cw) * 3;
    const int r = a.radius;
    const float* q = col + (y - s.gy0) * pitch;
    double acc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = a.wt[0] * static_cast<double>(q[c]);
    for (int k = 1; k <= r; ++k) {
      const double wk = a.wt[k];
      const float* lo = col + (usm_reflect(y - k, s.H) - s.gy0) * pitch;
      const float* hi = col + (usm_reflect(y + k, s.H) - s.gy0) * pitch;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        acc[c] = fma(wk, static_cast<double>(lo[c]) + static_cast<double>(hi[c]), acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double xv = static_cast<double>(v[c]);
      const float t = static_cast<float>(fma(a.sharpen, xv - acc[c], xv));
      a.fullres_out[o + c] = fminf(fmaxf(t, 0.0f), 1.0f);
    }
  } else {
    const int i = (blockIdx.y - a.full_tiles_y) * kUsmY + threadIdx.y;
    if (i >= a.S || j >= a.S) return;
    const int ci = min(static_cast<int>(floorf(static_cast<float>(i) * a.sy)), a.oh - 1);
    const int cj = min(static_cast<int>(floorf(static_cast<float>(j) * a.sx)), a.ow - 1);
    usm_source(s, ci, cj, y, x);
    const long long e = usm_elem(s, y, x);
    float* o = a.lowres_in + ((b * a.S + i) * a.S + j) * 3;
    o[0] = usm_load(s.input, s.fmt, e);
    o[1] = usm_load(s.input, s.fmt, e + 1);
    o[2] = usm_load(s.input, s.fmt, e + 2);
  }
}

// ---- host side ---------------------------------------------------------------------------------

bool usm_sigma_ok(double sigma) { return sigma > 0.0 && sigma <= 32.0; }   // false for NaN

int usm_radius(double sigma) { return static_cast<int>(4.0 * sigma + 0.5); }

// The crop's rectangle on the un-augmented source: (first row, rows, first column, columns), as
// data_pipeline.source_window.
struct CropRect { int y, h, x, w; };

CropRect usm_crop_rect(const hdrnet_usm_sample& s, int oh, int ow) {
  const int cy = s.crop_y, cx = s.crop_x;
  CropRect c;
  switch (s.rot90) {
    case 1: c = {cx, ow, s.W - cy - oh, oh}; break;
    case 2: c = {s.H - cy - oh, oh, s.W - cx - ow, ow}; break;
    case 3: c = {s.H - cx - ow, ow, cy, oh}; break;
    default: c = {cy, oh, cx, ow}; break;
  }
  if (s.flipud) c.y = s.H - c.y - c.h;
  if (s.fliplr) c.x = s.W - c.x - c.w;
  return c;
}

// Every contract check of one sample but the pointer: HDRNET_OK or the error code.
int usm_check_sample(const hdrnet_usm_sample& s, int oh, int ow, int r) {
  if (s.H <= 0 || s.W <= 0 || s.rot90 < 0 || s.rot90 > 3) return HDRNET_E_BAD_SHAPE;
  const int rh = (s.rot90 & 1) ? s.W : s.H, rw = (s.rot90 & 1) ? s.H : s.W;
  if (s.crop_y < 0 || s.crop_x < 0 || s.crop_y > rh - oh || s.crop_x > rw - ow) return HDRNET_E_BAD_SHAPE;
  if (s.input_fmt != HDRNET_PX_F32 && s.input_fmt != HDRNET_PX_U8 && s.input_fmt != HDRNET_PX_U16)
    return HDRNET_E_UNSUPPORTED;
  if (s.h < 1 || s.w < 1 || s.y0 < 0 || s.x0 < 0 || s.y0 > s.H - s.h || s.x0 > s.W - s.w)
    return HDRNET_E_BAD_SHAPE;
  const CropRect c = usm_crop_rect(s, oh, ow);
  const long long gy0 = c.y - r > 0 ? c.y - r : 0, gy1 = static_cast<long long>(c.y) + c.h + r < s.H ? c.y + c.h + r : s.H;
  const long long gx0 = c.x - r > 0 ? c.x - r : 0, gx1 = static_cast<long long>(c.x) + c.w + r < s.W ? c.x + c.w + r : s.W;
  if (s.y0 > gy0 || s.x0 > gx0 || static_cast<long long>(s.y0) + s.h < gy1 || static_cast<long long>(s.x0) + s.w < gx1)
    return HDRNET_E_BAD_SHAPE;
  return HDRNET_OK;
}

// Bytes of one sample's workspace rows (256-byte aligned).
size_t usm_sample_bytes(const hdrnet_usm_sample& s, int oh, int ow, int r) {
  const CropRect c = usm_crop_rect(s, oh, ow);
  const long long gy0 = c.y - r > 0 ? c.y - r : 0, gy1 = static_cast<long long>(c.y) + c.h + r < s.H ? c.y + c.h + r : s.H;
  const size_t bytes = static_cast<size_t>(gy1 - gy0) * static_cast<size_t>(c.w) * 3 * sizeof(float);
  return (bytes + kUsmAlign - 1) / kUsmAlign * kUsmAlign;
}

// Workspace of the whole call: the largest launch's (launches run in stream order and reuse it).
size_t usm_workspace_bytes(const hdrnet_usm_sample* samples, int B, int oh, int ow, int r) {
  size_t most = 0;
  for (int b0 = 0; b0 < B; b0 += kUsmSamples) {
    size_t sum = 0;
    for (int b = b0; b < B && b < b0 + kUsmSamples; ++b) sum += usm_sample_bytes(samples[b], oh, ow, r);
    if (sum > most) most = sum;
  }
  return most;
}

}  // namespace hdrnet_b200

extern "C" size_t hdrnet_train_batch_usm_workspace_bytes(const hdrnet_usm_sample* samples, int B, int oh,
                                                          int ow, double sigma) {
  using namespace hdrnet_b200;
  if (B <= 0 || !samples || oh < 1 || ow < 1 || !usm_sigma_ok(sigma)) return 0;
  const int r = usm_radius(sigma);
  for (int b = 0; b < B; ++b)
    if (usm_check_sample(samples[b], oh, ow, r) != HDRNET_OK) return 0;
  return usm_workspace_bytes(samples, B, oh, ow, r);
}

extern "C" int hdrnet_train_batch_usm_f32(const hdrnet_usm_sample* samples, int B, float* fullres_in,
                                          float* fullres_out, float* lowres_in, int oh, int ow, int S,
                                          double sigma, double sharpen, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  using namespace hdrnet_b200;
  if (B < 0 || oh < 1 || ow < 1 || (lowres_in != nullptr && S < 1)) return HDRNET_E_BAD_SHAPE;
  if (!usm_sigma_ok(sigma) || !std::isfinite(sharpen)) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!samples || !fullres_out || !workspace) return HDRNET_E_NULL_POINTER;
  for (int b = 0; b < B; ++b)
    if (!samples[b].input) return HDRNET_E_NULL_POINTER;
  const int r = usm_radius(sigma);
  for (int b = 0; b < B; ++b) {
    const int rc = usm_check_sample(samples[b], oh, ow, r);
    if (rc != HDRNET_OK) return rc;
  }
  if (workspace_bytes < usm_workspace_bytes(samples, B, oh, ow, r)) return HDRNET_E_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(workspace) % 4 != 0) return HDRNET_E_BAD_SHAPE;
  const int lowres_S = lowres_in != nullptr ? S : 0;
  const int full_tiles_y = (oh + kUsmY - 1) / kUsmY;
  const long long tiles_y = static_cast<long long>(full_tiles_y) + (lowres_S + kUsmY - 1) / kUsmY;
  const long long tiles_x = (static_cast<long long>(ow > lowres_S ? ow : lowres_S) + kUsmX - 1) / kUsmX;
  if (tiles_y > 65535 || tiles_x > 0x7fffffffLL) return HDRNET_E_TOO_LARGE;
  // pass 1's grid: the launch's most workspace rows x its widest crop's column tiles
  int most_rows = 0, most_cols = 0;
  for (int b = 0; b < B; ++b) {
    const CropRect c = usm_crop_rect(samples[b], oh, ow);
    const int gy0 = c.y - r > 0 ? c.y - r : 0;
    const int gy1 = static_cast<long long>(c.y) + c.h + r < samples[b].H ? c.y + c.h + r : samples[b].H;
    most_rows = gy1 - gy0 > most_rows ? gy1 - gy0 : most_rows;
    most_cols = c.w > most_cols ? c.w : most_cols;
  }
  const int ctiles = (most_cols + kUsmRowTile - 1) / kUsmRowTile;
  if (static_cast<long long>(most_rows) * ctiles > 0x7fffffffLL) return HDRNET_E_TOO_LARGE;

  // scipy.ndimage._gaussian_kernel1d: exp(-0.5 / sigma^2 * k^2), normalised to sum 1
  UsmArgs a;
  std::vector<double> phi(2 * r + 1);
  double sum = 0.0;
  for (int k = -r; k <= r; ++k) sum += (phi[k + r] = std::exp(-0.5 / (sigma * sigma) * static_cast<double>(k) * k));
  for (int k = 0; k <= r; ++k) a.wt[k] = phi[k + r] / sum;
  a.ws = static_cast<float*>(workspace);
  a.fullres_in = fullres_in;
  a.fullres_out = fullres_out;
  a.lowres_in = lowres_in;
  a.sharpen = sharpen;
  a.radius = r;
  a.ctiles = ctiles;
  a.oh = oh;
  a.ow = ow;
  a.S = lowres_S;
  a.full_tiles_y = full_tiles_y;
  a.sy = lowres_S ? static_cast<float>(oh) / static_cast<float>(lowres_S) : 0.0f;
  a.sx = lowres_S ? static_cast<float>(ow) / static_cast<float>(lowres_S) : 0.0f;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kUsmSamples) {
    const int n = (B - b0 < kUsmSamples) ? B - b0 : kUsmSamples;
    long long off = 0;   // floats
    for (int k = 0; k < n; ++k) {
      const hdrnet_usm_sample& d = samples[b0 + k];
      const CropRect c = usm_crop_rect(d, oh, ow);
      UsmSample& s = a.s[k];
      s.input = static_cast<const unsigned char*>(d.input);
      s.ws = off;
      s.fmt = d.input_fmt;
      s.H = d.H;
      s.W = d.W;
      s.y0 = d.y0;
      s.x0 = d.x0;
      s.w = d.w;
      s.fliplr = d.fliplr != 0;
      s.flipud = d.flipud != 0;
      s.rot90 = d.rot90;
      s.crop_y = d.crop_y;
      s.crop_x = d.crop_x;
      s.cx0 = c.x;
      s.cw = c.w;
      s.gy0 = c.y - r > 0 ? c.y - r : 0;
      s.grows = (static_cast<long long>(c.y) + c.h + r < d.H ? c.y + c.h + r : d.H) - s.gy0;
      off += static_cast<long long>(usm_sample_bytes(d, oh, ow, r) / sizeof(float));
    }
    a.b0 = b0;
    usm_rows_kernel<<<dim3(static_cast<unsigned>(static_cast<long long>(most_rows) * ctiles), 1, n),
                      kUsmRowTile, 0, st>>>(a);
    usm_target_kernel<<<dim3(static_cast<unsigned>(tiles_x), static_cast<unsigned>(tiles_y), n),
                        dim3(kUsmX, kUsmY), 0, st>>>(a);
  }
  return static_cast<int>(cudaGetLastError());
}
