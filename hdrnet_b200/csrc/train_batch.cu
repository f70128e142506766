// train_batch.cu -- one training batch from decoded image pairs resident on the device: the
// augmentation and resizing of ImageFilesDataPipeline._augment_data (hdrnet/data_pipeline.py:126-171)
// as one gather per output pixel.
//
// Per sample: random_flip_left_right, random_flip_up_down, rot90(k) (counter-clockwise, = np.rot90),
// crop of oh x ow at (crop_y, crop_x) on the rotated extent; the resize to output_resolution after
// the crop is an identity.  The network input is TF1 resize_images(NEAREST_NEIGHBOR) of the crop:
// src = min(floor(dst * (float)in / out), in - 1), no half-pixel offset.  Integer pixels become
// float32 as tf.to_float(x) / wl (v / 255, v / 65535), through the same conversion as the model
// path's load_quad (px_to_float, slice_rows.cuh).
#include <cuda_runtime.h>

#include "hdrnet_b200.h"
#include "slice_rows.cuh"

namespace hdrnet_b200 {

constexpr int kTbSamples = 32;        // descriptors per launch (they travel in the parameter block)
constexpr int kTbX = 32, kTbY = 8;    // 2-D tiles: a rotated sample reads a compact source patch

struct TrainBatchArgs {
  hdrnet_train_sample s[kTbSamples];
  float* fullres_in;
  float* fullres_out;
  float* lowres_in;
  long long b0;       // batch index of s[0]
  int oh, ow, S;
  int full_tiles_y;   // blockIdx.y below this: a fullres tile; at or above: a lowres tile
  float sy, sx;       // (float)oh / S, (float)ow / S: TF1's nearest-neighbour scale
};

// Source pixel index (y * W + x) of crop pixel (i, j) of an augmented sample.
__device__ __forceinline__ long long source_pixel(const hdrnet_train_sample& s, int i, int j) {
  const int r = s.crop_y + i, c = s.crop_x + j;   // on the rotated extent
  int y, x;                                       // on the flipped source
  switch (s.rot90) {
    case 1: y = c; x = s.W - 1 - r; break;                  // np.rot90(m, 1)[r, c] = m[c, W-1-r]
    case 2: y = s.H - 1 - r; x = s.W - 1 - c; break;
    case 3: y = s.H - 1 - c; x = r; break;                  // np.rot90(m, 3)[r, c] = m[H-1-c, r]
    default: y = r; x = c; break;
  }
  if (s.flipud) y = s.H - 1 - y;
  if (s.fliplr) x = s.W - 1 - x;
  return static_cast<long long>(y) * s.W + x;
}

__device__ __forceinline__ void load_rgb(const void* img, int fmt, long long px, float* out) {
  const unsigned char* base = static_cast<const unsigned char*>(img);
  const long long e = px * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (fmt == kPxU8) out[c] = load_channel<kPxU8>(base, e + c);
    else if (fmt == kPxU16) out[c] = load_channel<kPxU16>(base, e + c);
    else out[c] = load_channel<kPxF32>(base, e + c);
  }
}

__device__ __forceinline__ void store_rgb(float* dst, const float* v) {
  dst[0] = v[0];
  dst[1] = v[1];
  dst[2] = v[2];
}

__global__ void __launch_bounds__(kTbX * kTbY) train_batch_kernel(const __grid_constant__ TrainBatchArgs a) {
  const hdrnet_train_sample& s = a.s[blockIdx.z];
  const long long b = a.b0 + blockIdx.z;
  const int j = blockIdx.x * kTbX + threadIdx.x;
  float v[3];
  if (static_cast<int>(blockIdx.y) < a.full_tiles_y) {
    const int i = blockIdx.y * kTbY + threadIdx.y;
    if (i >= a.oh || j >= a.ow) return;
    const long long px = source_pixel(s, i, j);
    const long long o = ((b * a.oh + i) * a.ow + j) * 3;
    load_rgb(s.input, s.input_fmt, px, v);
    store_rgb(a.fullres_in + o, v);
    load_rgb(s.target, s.target_fmt, px, v);
    store_rgb(a.fullres_out + o, v);
  } else {
    const int i = (blockIdx.y - a.full_tiles_y) * kTbY + threadIdx.y;
    if (i >= a.S || j >= a.S) return;
    const int ci = min(static_cast<int>(floorf(static_cast<float>(i) * a.sy)), a.oh - 1);
    const int cj = min(static_cast<int>(floorf(static_cast<float>(j) * a.sx)), a.ow - 1);
    load_rgb(s.input, s.input_fmt, source_pixel(s, ci, cj), v);
    store_rgb(a.lowres_in + ((b * a.S + i) * a.S + j) * 3, v);
  }
}

}  // namespace hdrnet_b200

extern "C" int hdrnet_train_batch_f32(const hdrnet_train_sample* samples, int B, float* fullres_in,
                                      float* fullres_out, float* lowres_in, int oh, int ow, int S,
                                      void* stream) {
  using namespace hdrnet_b200;
  if (B < 0 || oh < 1 || ow < 1 || S < 1) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!samples || !fullres_in || !fullres_out || !lowres_in) return HDRNET_E_NULL_POINTER;
  for (int b = 0; b < B; ++b) {
    const hdrnet_train_sample& s = samples[b];
    if (!s.input || !s.target) return HDRNET_E_NULL_POINTER;
  }
  for (int b = 0; b < B; ++b) {
    const hdrnet_train_sample& s = samples[b];
    if (s.H <= 0 || s.W <= 0 || s.rot90 < 0 || s.rot90 > 3) return HDRNET_E_BAD_SHAPE;
    const int rh = (s.rot90 & 1) ? s.W : s.H, rw = (s.rot90 & 1) ? s.H : s.W;
    if (s.crop_y < 0 || s.crop_x < 0 || s.crop_y > rh - oh || s.crop_x > rw - ow)
      return HDRNET_E_BAD_SHAPE;
    for (int fmt : {s.input_fmt, s.target_fmt})
      if (fmt != HDRNET_PX_F32 && fmt != HDRNET_PX_U8 && fmt != HDRNET_PX_U16) return HDRNET_E_UNSUPPORTED;
  }
  const int full_tiles_y = (oh + kTbY - 1) / kTbY;
  const long long tiles_y = static_cast<long long>(full_tiles_y) + (S + kTbY - 1) / kTbY;
  const long long tiles_x = (static_cast<long long>(ow > S ? ow : S) + kTbX - 1) / kTbX;
  if (tiles_y > 65535 || tiles_x > 0x7fffffffLL) return HDRNET_E_TOO_LARGE;

  TrainBatchArgs a;
  a.fullres_in = fullres_in;
  a.fullres_out = fullres_out;
  a.lowres_in = lowres_in;
  a.oh = oh;
  a.ow = ow;
  a.S = S;
  a.full_tiles_y = full_tiles_y;
  a.sy = static_cast<float>(oh) / static_cast<float>(S);
  a.sx = static_cast<float>(ow) / static_cast<float>(S);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int b0 = 0; b0 < B; b0 += kTbSamples) {
    const int n = (B - b0 < kTbSamples) ? B - b0 : kTbSamples;
    for (int k = 0; k < n; ++k) a.s[k] = samples[b0 + k];
    a.b0 = b0;
    train_batch_kernel<<<dim3(static_cast<unsigned>(tiles_x), static_cast<unsigned>(tiles_y), n),
                         dim3(kTbX, kTbY), 0, st>>>(a);
  }
  return static_cast<int>(cudaGetLastError());
}
