// slice_apply_ragged.cu -- the guide-fused slice-apply over a RAGGED batch: B images, each with its
// own H_i x W_i, its own buffers and its own grid row, in one launch (DESIGN.md section 3 and row
// f-13).
//
// slice_apply_ragged_kernel is a persistent kernel over one global row index: the rows of all the
// images, image after image, are cut into one contiguous range per CTA, so a small image does not
// leave SMs idle while a large one finishes.  Per image row a CTA stages the two grid rows the row
// touches (reloaded only when they change) and pre-blends them along y into a slab in shared memory,
// as the row kernels do; a thread then takes 4 consecutive pixels at a time with plain global loads
// (vector loads where the row's address allows them, scalar ones elsewhere and for the last pixels
// of a row) and runs the row kernels' per-pixel code on them (load_quad / blend_quad / store_quad).
// Images the single-image call sends to its per-pixel kernel (odd widths, unaligned buffers, narrow
// images) run that kernel's code instead (px_generic_pixel): every image's result is the single-image
// call's, bit for bit.  No bulk copies (a row of an image at an odd width or offset is not a whole
// number of 16-byte units) and no texture objects.
//
// The image descriptors travel in the kernel's parameter block (__grid_constant__), up to
// kRaggedMaxImages per launch: a CUDA graph that captures the call copies them into its node.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>

#include "slice_rows.cuh"

namespace hdrnet_b200 {

bool fused_call_runs_row_form(int H, int W, int gh, int gw, int gd, int mode, int in_fmt, int out_fmt,
                              bool aligned);
int pack_curves_params(CurvesGuideParams* p, const float* ccm, const float* ccm_bias,
                       const float* shifts, const float* slopes, const float* mix,
                       float mix_bias);
int pack_nn_params(NNGuideParams* p, const float* w1, const float* b1, const float* w2, float b2,
                   int feats);

constexpr int kRaggedMaxImages = HDRNET_RAGGED_MAX_IMAGES;
constexpr int kRaggedThreads = 256;

struct RaggedImage {
  const unsigned char* input;   // [H, W, 3] in the call's input format
  unsigned char* out;           // [H, W, 3] in the call's output format
  long long row0;               // global index of the image's first row
  int H, W;
  float scale_x, scale_y;       // make_geom's gw / W, gh / H
  int per_pixel;                // 1: the single-image call's per-pixel form, 0: its row-kernel form
};

template <class GuideFn>
struct RaggedArgs {
  const float* grid;            // [n, gh, gw, gd, 12], row i for image i
  long long total_rows;
  int n, gh, gw, gd, row_floats;
  GuideFn guide_fn;
  RaggedImage img[kRaggedMaxImages];
};

// One pixel of a row's tail (or of an unaligned row), in the output format.
template <int kOut>
__device__ __forceinline__ void store_pixel(unsigned char* row, int x, float r, float g, float b) {
  if constexpr (kOut == kPxF32) {
    float* o = reinterpret_cast<float*>(row) + 3 * x;
    o[0] = r; o[1] = g; o[2] = b;
  } else if constexpr (kOut == kPxU16) {
    unsigned short* o = reinterpret_cast<unsigned short*>(row) + 3 * x;
    o[0] = static_cast<unsigned short>(float_to_u16(r));
    o[1] = static_cast<unsigned short>(float_to_u16(g));
    o[2] = static_cast<unsigned short>(float_to_u16(b));
  } else {
    unsigned char* o = row + 3 * x;
    o[0] = static_cast<unsigned char>(float_to_u8(r));
    o[1] = static_cast<unsigned char>(float_to_u8(g));
    o[2] = static_cast<unsigned char>(float_to_u8(b));
  }
}

// Alignment of a quad (4 pixels) for load_quad / store_quad on global memory: 16 bytes for float32
// (float4), 8 for uint16 (uint2), 4 for uint8 (uint32).
__host__ __device__ constexpr unsigned quad_align(int fmt) { return fmt == kPxF32 ? 16u : (fmt == kPxU16 ? 8u : 4u); }

template <class GuideFn, int kIn, int kOut>
__global__ void __launch_bounds__(kRaggedThreads)
slice_apply_ragged_kernel(const __grid_constant__ RaggedArgs<GuideFn> a) {
  extern __shared__ __align__(16) float sm_ragged[];
  constexpr size_t kInBpp = 3u * px_bytes_per_channel(kIn), kOutBpp = 3u * px_bytes_per_channel(kOut);
  float* raw0 = sm_ragged;
  float* raw1 = raw0 + a.row_floats;
  float* slab = raw1 + a.row_floats;
  const int tid = threadIdx.x;
  const long long r_begin = a.total_rows * blockIdx.x / gridDim.x;
  const long long r_end = a.total_rows * (blockIdx.x + 1) / gridDim.x;
  if (r_begin >= r_end) return;
  // the image of the first row: the last one whose first row is <= r_begin
  int b = 0;
  for (int lo = 0, hi = a.n - 1; lo < hi;) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.img[mid].row0 <= r_begin) { lo = mid; b = mid; } else { hi = mid - 1; }
  }
  const long long grid_image = static_cast<long long>(a.gh) * a.row_floats;
  int cur_b = -1, cur_gy0 = INT_MIN;
  for (long long row = r_begin; row < r_end; ++row) {
    while (row >= a.img[b].row0 + a.img[b].H) ++b;
    const RaggedImage& im = a.img[b];
    SliceGeom g;
    g.B = 1; g.H = im.H; g.W = im.W; g.rows = im.H; g.y_off = 0;
    g.gh = a.gh; g.gw = a.gw; g.gd = a.gd;
    g.scale_x = im.scale_x; g.scale_y = im.scale_y;
    const int y = static_cast<int>(row - im.row0);
    const size_t row_px = static_cast<size_t>(y) * im.W;
    if (im.per_pixel) {   // slice_apply_px_generic_kernel's pixels
      for (int x = tid; x < im.W; x += kRaggedThreads)
        px_generic_pixel<GuideFn, kIn, kOut>(a.grid, grid_image, b, im.input, im.out, nullptr, g, x, y,
                                             static_cast<long long>(row_px + x), a.guide_fn);
      continue;
    }
    // the row kernels' pixels: grid rows + y pre-blend, then quads
    const Axis ay = spatial_axis(y, g.scale_y);
    __syncthreads();   // the previous row's pixels are done with the slab
    if (b != cur_b || ay.i0 != cur_gy0) {
      const float* gb = a.grid + static_cast<size_t>(b) * grid_image;
      const float* r0 = gb + static_cast<size_t>(clampi(ay.i0, 0, a.gh - 1)) * a.row_floats;
      const float* r1 = gb + static_cast<size_t>(clampi(ay.i0 + 1, 0, a.gh - 1)) * a.row_floats;
      for (int e = tid; e < a.row_floats; e += kRaggedThreads) { raw0[e] = __ldg(r0 + e); raw1[e] = __ldg(r1 + e); }
      cur_b = b;
      cur_gy0 = ay.i0;
      __syncthreads();
    }
    const float wy1 = ay.f, wy0 = 1.0f - ay.f;
    const float4* a4 = reinterpret_cast<const float4*>(raw0);
    const float4* b4 = reinterpret_cast<const float4*>(raw1);
    float4* s4 = reinterpret_cast<float4*>(slab);
    for (int e = tid; e < a.row_floats / 4; e += kRaggedThreads) s4[e] = lerp4(wy0, a4[e], wy1, b4[e]);
    __syncthreads();
    const unsigned char* rin = im.input + row_px * kInBpp;
    unsigned char* rout = im.out + row_px * kOutBpp;
    const bool vec_in = (reinterpret_cast<uintptr_t>(rin) % quad_align(kIn)) == 0;
    const bool vec_out = (reinterpret_cast<uintptr_t>(rout) % quad_align(kOut)) == 0;
    const int quads = (im.W + 3) / 4;
    for (int q = tid; q < quads; q += kRaggedThreads) {
      const int x = 4 * q;
      const int n = min(4, im.W - x);
      float pr[4], pg[4], pb[4];
      if (n == 4 && vec_in) {
        load_quad<kIn>(rin, q, pr, pg, pb);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const bool in_row = i < n;
          pr[i] = in_row ? load_channel<kIn>(rin, 3 * (x + i)) : 0.0f;
          pg[i] = in_row ? load_channel<kIn>(rin, 3 * (x + i) + 1) : 0.0f;
          pb[i] = in_row ? load_channel<kIn>(rin, 3 * (x + i) + 2) : 0.0f;
        }
      }
      float gv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) gv[i] = a.guide_fn(pr[i], pg[i], pb[i]);
      float o_r[4], o_g[4], o_b[4];
      blend_quad<0>(g, slab, 0, 0, x, gv, pr, pg, pb, o_r, o_g, o_b);
      if (n == 4 && vec_out) {
        store_quad<kOut>(rout, q, o_r, o_g, o_b);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (i < n) store_pixel<kOut>(rout, x + i, o_r[i], o_g[i], o_b[i]);
      }
    }
  }
}

static int ragged_device_attr(cudaDeviceAttr attr, int fallback) {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, attr, dev) != cudaSuccess || v <= 0) {
    (void)cudaGetLastError();
    return fallback;
  }
  return v;
}

static bool valid_px_fmt(int f) { return f == kPxF32 || f == kPxU8 || f == kPxU16; }

// The checks every ragged entry point makes before any launch (include/hdrnet_b200.h).
// need_out: descriptors' `out` is required; min_hw: smallest H and W an image may have.
int validate_ragged(const hdrnet_image_desc* images, int B, int in_fmt, int out_fmt, bool need_out, int min_hw) {
  if (B < 0) return HDRNET_E_BAD_SHAPE;
  if (B == 0) return HDRNET_OK;
  if (!images) return HDRNET_E_NULL_POINTER;
  if (!valid_px_fmt(in_fmt) || (need_out && !valid_px_fmt(out_fmt))) return HDRNET_E_UNSUPPORTED;
  for (int i = 0; i < B; ++i) {
    if (images[i].H <= 0 || images[i].W <= 0) return HDRNET_E_BAD_SHAPE;
    if (images[i].H < min_hw || images[i].W < min_hw) return HDRNET_E_BAD_SHAPE;
  }
  for (int i = 0; i < B; ++i)
    if (!images[i].image || (need_out && !images[i].out)) return HDRNET_E_NULL_POINTER;
  if (need_out && out_fmt == kPxU16) {
    // as the single-image forms: a uint16 result is not written over any input
    const size_t in_bpp = 3u * px_bytes_per_channel(in_fmt);
    for (int i = 0; i < B; ++i) {
      const uintptr_t o0 = reinterpret_cast<uintptr_t>(images[i].out);
      const uintptr_t o1 = o0 + static_cast<uintptr_t>(images[i].H) * images[i].W * 6u;
      for (int j = 0; j < B; ++j) {
        const uintptr_t i0 = reinterpret_cast<uintptr_t>(images[j].image);
        const uintptr_t i1 = i0 + static_cast<uintptr_t>(images[j].H) * images[j].W * in_bpp;
        if (o0 < i1 && i0 < o1) return HDRNET_E_UNSUPPORTED;
      }
    }
  }
  return HDRNET_OK;
}

template <class GuideFn, int kIn, int kOut>
static int launch_ragged_t(const RaggedArgs<GuideFn>& a, size_t smem, int sms, cudaStream_t stream) {
  auto kern = slice_apply_ragged_kernel<GuideFn, kIn, kOut>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kRaggedThreads, smem) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  const int ctas = static_cast<int>(std::min<long long>(a.total_rows, static_cast<long long>(sms) * per_sm));
  kern<<<ctas, kRaggedThreads, smem, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

template <class GuideFn>
static int launch_ragged_fmt(const RaggedArgs<GuideFn>& a, int in_fmt, int out_fmt, size_t smem, int sms,
                             cudaStream_t st) {
#define HDRNET_RAGGED_CASE(I, O) \
  if (in_fmt == I && out_fmt == O) return launch_ragged_t<GuideFn, I, O>(a, smem, sms, st);
  HDRNET_RAGGED_CASE(kPxU8, kPxU8)
  HDRNET_RAGGED_CASE(kPxU8, kPxU16)
  HDRNET_RAGGED_CASE(kPxU8, kPxF32)
  HDRNET_RAGGED_CASE(kPxU16, kPxU8)
  HDRNET_RAGGED_CASE(kPxU16, kPxU16)
  HDRNET_RAGGED_CASE(kPxU16, kPxF32)
  HDRNET_RAGGED_CASE(kPxF32, kPxU8)
  HDRNET_RAGGED_CASE(kPxF32, kPxU16)
  HDRNET_RAGGED_CASE(kPxF32, kPxF32)
#undef HDRNET_RAGGED_CASE
  return HDRNET_E_UNSUPPORTED;
}

// One launch per kRaggedMaxImages images; every check is made before the first launch.
template <class GuideFn>
static int launch_slice_apply_ragged(const float* grid, const hdrnet_image_desc* images, int B, int in_fmt,
                                     int out_fmt, int gh, int gw, int gd, int mode, const GuideFn& fn,
                                     cudaStream_t stream) {
  int rc = validate_ragged(images, B, in_fmt, out_fmt, true, 1);
  if (rc != HDRNET_OK || B == 0) return rc;
  if (gh < 1 || gw < 1 || gd < 1) return HDRNET_E_BAD_SHAPE;
  if (!grid) return HDRNET_E_NULL_POINTER;
  const long long row_floats = static_cast<long long>(gw) * gd * kGc;
  if (row_floats * gh > INT_MAX) return HDRNET_E_TOO_LARGE;
  if (out_fmt == kPxU16) {   // nor over the grid
    const uintptr_t g0 = reinterpret_cast<uintptr_t>(grid), g1 = g0 + static_cast<uintptr_t>(B) * gh * row_floats * 4u;
    for (int i = 0; i < B; ++i) {
      const uintptr_t o0 = reinterpret_cast<uintptr_t>(images[i].out);
      const uintptr_t o1 = o0 + static_cast<uintptr_t>(images[i].H) * images[i].W * 6u;
      if (o0 < g1 && g0 < o1) return HDRNET_E_UNSUPPORTED;
    }
  }
  const int sms = ragged_device_attr(cudaDevAttrMultiProcessorCount, 132);
  const size_t grid_image = static_cast<size_t>(gh) * row_floats;
  for (int c0 = 0; c0 < B; c0 += kRaggedMaxImages) {
    RaggedArgs<GuideFn> a;
    a.grid = grid + c0 * grid_image;
    a.n = std::min(kRaggedMaxImages, B - c0);
    a.gh = gh; a.gw = gw; a.gd = gd;
    a.row_floats = static_cast<int>(row_floats);
    a.guide_fn = fn;
    long long rows = 0;
    bool any_row_form = false;
    for (int i = 0; i < a.n; ++i) {
      const hdrnet_image_desc& d = images[c0 + i];
      RaggedImage& im = a.img[i];
      const SliceGeom g = make_geom(1, d.H, d.W, d.H, 0, gh, gw, gd);
      im.input = static_cast<const unsigned char*>(d.image);
      im.out = static_cast<unsigned char*>(d.out);
      im.row0 = rows;
      im.H = d.H;
      im.W = d.W;
      im.scale_x = g.scale_x;
      im.scale_y = g.scale_y;
      const bool aligned = (reinterpret_cast<uintptr_t>(a.grid + i * grid_image) % 16) == 0 &&
                           (reinterpret_cast<uintptr_t>(d.image) % 16) == 0 && (reinterpret_cast<uintptr_t>(d.out) % 16) == 0;
      im.per_pixel = fused_call_runs_row_form(d.H, d.W, gh, gw, gd, mode, in_fmt, out_fmt, aligned) ? 0 : 1;
      any_row_form |= im.per_pixel == 0;
      rows += d.H;
    }
    a.total_rows = rows;
    // the slab and its two grid rows, where an image runs the row kernels' form (the single-image
    // row kernels need more shared memory than this, so an image that runs them always fits)
    const size_t smem = any_row_form ? 3 * static_cast<size_t>(row_floats) * sizeof(float) : 0;
    rc = launch_ragged_fmt(a, in_fmt, out_fmt, smem, sms, stream);
    if (rc != HDRNET_OK) return rc;
  }
  return HDRNET_OK;
}

}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_slice_apply_ragged_workspace_bytes(const hdrnet_image_desc*, int, int, int, int) { return 0; }

int hdrnet_slice_apply_curves_ragged_px_ws(const float* grid, const hdrnet_image_desc* images, int B, int in_fmt,
                                           int out_fmt, int gh, int gw, int gd, const float* ccm,
                                           const float* ccm_bias, const float* shifts, const float* slopes,
                                           const float* mix, float mix_bias, void*, size_t, void* stream) {
  GuideCurves fn;
  const int rc = pack_curves_params(&fn.p, ccm, ccm_bias, shifts, slopes, mix, mix_bias);
  if (rc != HDRNET_OK) return rc;
  return launch_slice_apply_ragged(grid, images, B, in_fmt, out_fmt, gh, gw, gd, 1, fn,
                                   static_cast<cudaStream_t>(stream));
}

int hdrnet_slice_apply_nn_ragged_px_ws(const float* grid, const hdrnet_image_desc* images, int B, int in_fmt,
                                       int out_fmt, int gh, int gw, int gd, const float* w1, const float* b1,
                                       const float* w2, float b2, int feats, void*, size_t, void* stream) {
  NNGuideParams np;
  const int rc = pack_nn_params(&np, w1, b1, w2, b2, feats);
  if (rc != HDRNET_OK) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (np.feats <= 16) {
    GuideNN<16> fn; fn.p = np;
    return launch_slice_apply_ragged(grid, images, B, in_fmt, out_fmt, gh, gw, gd, 2, fn, st);
  }
  GuideNN<kMaxGuideFeats> fn; fn.p = np;
  return launch_slice_apply_ragged(grid, images, B, in_fmt, out_fmt, gh, gw, gd, 2, fn, st);
}

}  // extern "C"
