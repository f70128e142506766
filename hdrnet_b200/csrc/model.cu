// model.cu -- a whole trained model behind the C-ABI: the frozen model file (checkpoint.freeze_model)
// parsed and uploaded once, then one call per batch of images that runs what
// models.*.inference_image runs, kernel for kernel and chosen by the same rules, with every
// intermediate in a workspace the caller lends.  The run call allocates no memory, never synchronises
// and launches only on the caller's stream, so a CUDA graph can capture it.
//
// Frozen model file, version 1 (all integers little-endian uint32 / int32, floats IEEE float32 LE):
//   0   char[8]  magic "HDRNETFZ"
//   8   u32      format version (1)
//   12  u32      model kind (HDRNET_MODEL_*)
//   16  i32[5]   net_input_size, spatial_bin, luma_bins, channel_multiplier, guide width
//   36  u32      number of arrays
//   40  arrays, each: u32 ndim, u32 dims[ndim], float32 data[prod(dims)]
//   end u32      CRC-32C (Castagnoli) of every byte before it
// The arrays, in order, are exactly what the kernels consume (batch norm already folded):
//   every coefficient-network layer in chain order (splat conv1..n_ds, global conv1, conv2, fc1,
//   fc2, fc3, local conv1, conv2, prediction conv1) as its weights (conv HWIO, fc [in][out]) and
//   its bias ([cout]; dims [0] for local conv2, which has none); then the guide: ccm [3,3],
//   ccm_bias [3], shifts [3,16], slopes [3,16], mix [3], mix_bias [1] for the curves guide, or
//   w1 [3,F], b1 [F], w2 [F], b2 [1] for the pointwise-NN guide, once per pyramid level (0, 1, 2)
//   for the two pyramid kinds.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <new>
#include <unordered_set>
#include <vector>

#include "common.cuh"

namespace hdrnet_b200 {
int validate_ragged(const hdrnet_image_desc* images, int B, int in_fmt, int out_fmt, bool need_out, int min_hw);
int launch_image_to_float(const void* image, int fmt, float* out, long long total, cudaStream_t st);
int launch_resize_quantize(const float* in, const float* add, void* out, int out_fmt, int B, int H,
                           int W, int C, int OH, int OW, cudaStream_t st);
}  // namespace hdrnet_b200

namespace {

constexpr char kMagic[8] = {'H', 'D', 'R', 'N', 'E', 'T', 'F', 'Z'};
constexpr uint32_t kFormatVersion = 1;
constexpr size_t kHeaderBytes = 40;
constexpr int kMaxLayers = 16;        // n_ds <= 8 splat convs + 8 more layers
constexpr int kChainMaxBatch = 16;    // models.CHAIN_CNN_MAX_BATCH
constexpr int kPackedMinTiles = 64;   // models.PACKED_CONV_MIN_TILES
constexpr size_t kAlign = 512;        // workspace pieces start on the texture alignment
constexpr uint32_t kModelMagic = 0x48444d4cu;  // "HDML"

uint32_t crc32c(const unsigned char* p, size_t n) {
  static uint32_t table[256];
  static std::once_flag once;
  std::call_once(once, [] {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      table[i] = c;
    }
  });
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

uint32_t rd_u32(const unsigned char* p) {
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) |
         (static_cast<uint32_t>(p[2]) << 16) | (static_cast<uint32_t>(p[3]) << 24);
}

// One layer of the coefficient network: HWIO conv (k > 0) or fc (k == 0).
struct LayerSpec { int k, cin, cout, stride, relu, bias; };

struct Hyper { int kind, S, sb, gd, cm, feats; };

bool is_pyramid(int kind) { return kind == HDRNET_MODEL_GAUSSIAN_PYR_NN || kind == HDRNET_MODEL_GAUSSIAN_PYR; }
bool has_curves_guide(int kind) { return kind == HDRNET_MODEL_CURVES || kind == HDRNET_MODEL_GAUSSIAN_PYR; }
int n_out_of(int kind) { return is_pyramid(kind) ? 9 : 3; }

// models._coefficient_specs and init_weights' shapes; false when the hyperparameters are invalid.
bool layer_specs(const Hyper& h, std::vector<LayerSpec>* out, int* n_ds) {
  if (h.S < 2 || h.sb < 1 || h.gd < 1 || h.cm < 1 || h.S % h.sb) return false;
  if (h.gd > 256 || h.cm > 256 || h.S > 65536) return false;
  // every layer's weights, the widest being fc1's (sb / 4)^2 * 8 cm gd x 32 cm gd, fit 2^30 floats
  const long long c8l = 8LL * h.cm * h.gd, g2l = (h.sb + 3) / 4;
  if (g2l * g2l * c8l * 4 * c8l > (1LL << 30)) return false;
  int n = 0;
  for (int s = h.S; s > h.sb; s >>= 1) {
    if (s & 1) return false;
    ++n;
  }
  if (n < 1 || n > 8 || (h.sb << n) != h.S) return false;
  *n_ds = n;
  std::vector<LayerSpec>& L = *out;
  L.clear();
  int cin = 3;
  for (int i = 0; i < n; ++i) {
    const int c = h.cm * (1 << i) * h.gd;
    L.push_back({3, cin, c, 2, 1, 1});
    cin = c;
  }
  const int c8 = 8 * h.cm * h.gd, g2 = (((h.sb + 1) / 2) + 1) / 2;
  L.push_back({3, cin, c8, 2, 1, 1});                       // global conv1
  L.push_back({3, c8, c8, 2, 1, 1});                        // global conv2
  L.push_back({0, g2 * g2 * c8, 32 * h.cm * h.gd, 1, 1, 1});  // fc1
  L.push_back({0, 32 * h.cm * h.gd, 16 * h.cm * h.gd, 1, 1, 1});
  L.push_back({0, 16 * h.cm * h.gd, c8, 1, 0, 1});          // fc3
  L.push_back({3, cin, c8, 1, 1, 1});                       // local conv1
  L.push_back({3, c8, c8, 1, 0, 0});                        // local conv2: no bias
  L.push_back({1, c8, h.gd * n_out_of(h.kind) * 4, 1, 0, 1});  // prediction conv1
  return true;
}

// The shapes of every array of the file, in order.
void expected_shapes(const Hyper& h, const std::vector<LayerSpec>& L, std::vector<std::vector<uint32_t>>* s) {
  s->clear();
  for (const LayerSpec& l : L) {
    if (l.k) s->push_back({uint32_t(l.k), uint32_t(l.k), uint32_t(l.cin), uint32_t(l.cout)});
    else s->push_back({uint32_t(l.cin), uint32_t(l.cout)});
    s->push_back({uint32_t(l.bias ? l.cout : 0)});
  }
  const int levels = is_pyramid(h.kind) ? 3 : 1;
  const uint32_t F = static_cast<uint32_t>(h.feats);
  const std::vector<std::vector<uint32_t>> guide =
      has_curves_guide(h.kind) ? std::vector<std::vector<uint32_t>>{{3, 3}, {3}, {3, 16}, {3, 16}, {3}, {1}}
                               : std::vector<std::vector<uint32_t>>{{3, F}, {F}, {F}, {1}};
  for (int l = 0; l < levels; ++l)
    for (const auto& d : guide) s->push_back(d);
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct NNGuideHost { float w1[3 * 32], b1[32], w2[32], b2; int feats; };
struct CurvesGuideHost { float ccm[9], ccm_bias[3], shifts[48], slopes[48], mix[3], mix_bias; };

}  // namespace

struct hdrnet_model {
  uint32_t magic;
  int device;
  Hyper h;
  int n_ds;
  std::vector<LayerSpec> layers;
  void* dev_mem;                          // every device array below, one allocation
  const float* w[kMaxLayers];
  const float* b[kMaxLayers];             // NULL: no bias
  const float* packed[kMaxLayers];        // tensor-core packed conv weights, or NULL
  // guides, one per pyramid level: host arrays (the kernels take them in their argument block)
  CurvesGuideHost curves[3];
  NNGuideHost nn[3];
};

namespace {

std::mutex g_models_mutex;
std::unordered_set<const hdrnet_model*> g_models;   // live objects: a destroyed one is refused

bool is_live(const hdrnet_model* m) {
  std::lock_guard<std::mutex> lock(g_models_mutex);
  return m && g_models.count(m) && m->magic == kModelMagic;
}

// Parses and checks the whole blob without touching the device.  On success `arrays` points at each
// array's float data inside the blob.
int parse_blob(const unsigned char* p, size_t bytes, Hyper* h, std::vector<LayerSpec>* L, int* n_ds,
               std::vector<const unsigned char*>* arrays) {
  if (bytes < kHeaderBytes + 4 || std::memcmp(p, kMagic, 8) != 0) return HDRNET_E_BAD_MODEL;
  if (rd_u32(p + 8) != kFormatVersion) return HDRNET_E_BAD_MODEL;
  h->kind = static_cast<int>(rd_u32(p + 12));
  h->S = static_cast<int>(rd_u32(p + 16));
  h->sb = static_cast<int>(rd_u32(p + 20));
  h->gd = static_cast<int>(rd_u32(p + 24));
  h->cm = static_cast<int>(rd_u32(p + 28));
  h->feats = static_cast<int>(rd_u32(p + 32));
  if (h->kind != HDRNET_MODEL_CURVES && h->kind != HDRNET_MODEL_POINTWISE_NN &&
      h->kind != HDRNET_MODEL_GAUSSIAN_PYR_NN && h->kind != HDRNET_MODEL_GAUSSIAN_PYR)
    return HDRNET_E_BAD_MODEL;
  if (has_curves_guide(h->kind) ? h->feats != 16 : (h->feats < 1 || h->feats > 32)) return HDRNET_E_BAD_MODEL;
  if (!layer_specs(*h, L, n_ds)) return HDRNET_E_BAD_MODEL;
  std::vector<std::vector<uint32_t>> shapes;
  expected_shapes(*h, *L, &shapes);
  if (rd_u32(p + 36) != shapes.size()) return HDRNET_E_BAD_MODEL;
  if (crc32c(p, bytes - 4) != rd_u32(p + bytes - 4)) return HDRNET_E_BAD_MODEL;
  const size_t end = bytes - 4;
  size_t off = kHeaderBytes;
  arrays->clear();
  for (const auto& want : shapes) {
    if (end - off < 4 || rd_u32(p + off) != want.size()) return HDRNET_E_BAD_MODEL;
    off += 4;
    if ((end - off) / 4 < want.size()) return HDRNET_E_BAD_MODEL;
    size_t count = 1;
    for (uint32_t d : want) {
      if (rd_u32(p + off) != d) return HDRNET_E_BAD_MODEL;
      count *= d;
      off += 4;
    }
    if ((end - off) / 4 < count) return HDRNET_E_BAD_MODEL;
    arrays->push_back(p + off);
    off += count * 4;
  }
  return off == end ? HDRNET_OK : HDRNET_E_BAD_MODEL;
}

void read_floats(const unsigned char* src, float* dst, size_t n) { std::memcpy(dst, src, n * 4); }

// ---- workspace layout ---------------------------------------------------------------------------
// Every piece a run needs, carved from the lent workspace in this order, each at kAlign.  The same
// function sizes the workspace (base 0) and hands out the pointers, so the two cannot disagree.
struct Layout {
  float* lowres;        // [B, S, S, 3]
  float* grid;          // [B, sb, sb, gd, n_out, 4]
  float* acts;          // the coefficient network's activations (hdrnet_coefficients_scratch_bytes)
  size_t acts_bytes;
  float* gmap;          // curves / NN, float32 -> float32: the guide map the row kernel may need
  float* slab;          // curves / NN: the slab workspace of the texture-assisted forms, or NULL
  size_t slab_bytes;
  // pyramid
  float* full;          // [B, H, W, 3] img_as_float of an integer image
  float* lvl[3];        // levels 1, 2 ([0] is the float image)
  float* coef[3];       // the three levels' coefficient rows [B, sb, sb, gd, 12]
  float* lvl_out[3];    // each level's slice-apply result
  float* lvl_gmap[3];
  float* cur1;          // level 2's result upsampled and added to level 1's
  size_t end;
};

struct Carver {
  uintptr_t base, off = 0;
  float* take(size_t bytes) {
    off = align_up(off, kAlign);
    float* p = reinterpret_cast<float*>(base + off);
    off += bytes;
    return p;
  }
};

bool texture_form_runs(int B, int H, int W, int gd, int sb);

void layout(const hdrnet_model* m, int B, int H, int W, int in_fmt, int out_fmt, uintptr_t base,
            Layout* l) {
  const Hyper& h = m->h;
  const size_t npx = static_cast<size_t>(B) * H * W, f = sizeof(float);
  Carver c{base};
  *l = Layout{};
  l->lowres = c.take(static_cast<size_t>(B) * h.S * h.S * 3 * f);
  l->grid = c.take(static_cast<size_t>(B) * h.sb * h.sb * h.gd * n_out_of(h.kind) * 4 * f);
  l->acts_bytes = hdrnet_coefficients_scratch_bytes(B, h.S, h.sb, h.gd, h.cm, n_out_of(h.kind), 4);
  l->acts = c.take(l->acts_bytes);
  if (!is_pyramid(h.kind)) {
    if (in_fmt == HDRNET_PX_F32 && out_fmt == HDRNET_PX_F32) l->gmap = c.take(npx * f);
    if (texture_form_runs(B, H, W, h.gd, h.sb)) {
      l->slab_bytes = hdrnet_slice_apply_workspace_bytes(B, H, h.sb, h.gd);
      l->slab = c.take(l->slab_bytes);
    }
  } else {
    const int hs[3] = {H, H / 2, H / 4}, ws[3] = {W, W / 2, W / 4};
    if (in_fmt != HDRNET_PX_F32) l->full = c.take(npx * 3 * f);
    for (int i = 0; i < 3; ++i) {
      const size_t lp = static_cast<size_t>(B) * hs[i] * ws[i];
      if (i > 0) l->lvl[i] = c.take(lp * 3 * f);
      l->coef[i] = c.take(static_cast<size_t>(B) * h.sb * h.sb * h.gd * 12 * f);
      l->lvl_out[i] = c.take(lp * 3 * f);
      l->lvl_gmap[i] = c.take(lp * f);
    }
    l->cur1 = c.take(static_cast<size_t>(B) * hs[1] * ws[1] * 3 * f);
  }
  l->end = c.off;
}

// The workspace of a ragged batch (hdrnet_model_run_ragged_px): the network input, grids and
// activations for all B images; for the pyramid, each level's coefficient rows for all B images and
// the per-image intermediates of pyramid_fullres sized for the largest image at each level (the
// images run one after the other on the stream, so they share them).
void layout_ragged(const hdrnet_model* m, const hdrnet_image_desc* images, int B, int in_fmt, uintptr_t base,
                   Layout* l) {
  const Hyper& h = m->h;
  const size_t f = sizeof(float);
  Carver c{base};
  *l = Layout{};
  l->lowres = c.take(static_cast<size_t>(B) * h.S * h.S * 3 * f);
  l->grid = c.take(static_cast<size_t>(B) * h.sb * h.sb * h.gd * n_out_of(h.kind) * 4 * f);
  l->acts_bytes = hdrnet_coefficients_scratch_bytes(B, h.S, h.sb, h.gd, h.cm, n_out_of(h.kind), 4);
  l->acts = c.take(l->acts_bytes);
  if (is_pyramid(h.kind)) {
    size_t lp[3] = {0, 0, 0};
    for (int i = 0; i < B; ++i) {
      const int H = images[i].H, W = images[i].W;
      lp[0] = std::max(lp[0], static_cast<size_t>(H) * W);
      lp[1] = std::max(lp[1], static_cast<size_t>(H / 2) * (W / 2));
      lp[2] = std::max(lp[2], static_cast<size_t>(H / 4) * (W / 4));
    }
    if (in_fmt != HDRNET_PX_F32) l->full = c.take(lp[0] * 3 * f);
    for (int i = 0; i < 3; ++i) {
      if (i > 0) l->lvl[i] = c.take(lp[i] * 3 * f);
      l->coef[i] = c.take(static_cast<size_t>(B) * h.sb * h.sb * h.gd * 12 * f);
      l->lvl_out[i] = c.take(lp[i] * 3 * f);
      l->lvl_gmap[i] = c.take(lp[i] * f);
    }
    l->cur1 = c.take(lp[1] * 3 * f);
  }
  l->end = c.off;
}

// hdrnet_ops._texture_form_runs: AUTO runs a texture-assisted form from 2 Mi pixels on when lent
// the slab workspace, and only then does models' fused slice-apply lend it.
bool texture_form_runs(int B, int H, int W, int gd, int sb) {
  if (static_cast<long long>(B) * H * W < (1LL << 21) || W % 4) return false;
  int v = 0;
  if (hdrnet_slice_apply_plan_ws(B, H, W, sb, sb, gd, 3, 3, 1, 1, &v, nullptr, nullptr, nullptr) != HDRNET_OK)
    return false;
  return v == HDRNET_VARIANT_TEX || v == HDRNET_VARIANT_TEX_ASYNC;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// models._fused_row_kernel_takes
bool fused_row_kernel_takes(int W, const void* a, const void* b, const void* c) {
  return W % 4 == 0 && W >= 128 && aligned16(a) && aligned16(b) && aligned16(c);
}

// ---- the coefficient network (models.HDRNetCurves._coefficients) -----------------------------
int coefficients(const hdrnet_model* m, const float* lowres, float* grid, float* acts, size_t acts_bytes,
                 int B, cudaStream_t st) {
  const Hyper& h = m->h;
  const int n_out = n_out_of(h.kind), n_layers = static_cast<int>(m->layers.size());
  if (B <= kChainMaxBatch && acts_bytes != 0) {   // one call, the launch chain (csrc/cnn.cu)
    const int rc = hdrnet_coefficients_f32(lowres, grid, m->w, m->b, n_layers, acts, acts_bytes, B, h.S,
                                           h.sb, h.gd, h.cm, n_out, 4, st);
    if (rc != HDRNET_E_UNSUPPORTED) return rc;
  }
  // layer by layer (_coefficients_layers), each layer's output in the scratch in network order
  float* cur = acts;
  const auto take = [&](size_t n) { float* p = cur; cur += (n + 3) & ~static_cast<size_t>(3); return p; };
  const auto conv = [&](int li, const float* in, int H, int W, float* out) -> int {
    const LayerSpec& l = m->layers[li];
    const int oh = (H + l.stride - 1) / l.stride, ow = (W + l.stride - 1) / l.stride;
    if (m->packed[li] && (static_cast<long long>(B) * oh * ow + 127) / 128 >= kPackedMinTiles) {
      const int rc = hdrnet_conv2d_nhwc_tc_f32(in, m->packed[li], m->b[li], out, B, H, W, l.cin, l.cout, l.k,
                                               l.stride, l.relu, st);
      if (rc != HDRNET_E_UNSUPPORTED) return rc;
    }
    return hdrnet_conv2d_nhwc_f32(in, m->w[li], m->b[li], out, B, H, W, l.cin, l.cout, l.k, l.stride, l.relu, st);
  };
  int rc = HDRNET_OK, H = h.S, li = 0;
  const float* x = lowres;
  for (; li < m->n_ds && rc == HDRNET_OK; ++li) {
    float* out = take(static_cast<size_t>(B) * (H / 2) * (H / 2) * m->layers[li].cout);
    rc = conv(li, x, H, H, out);
    x = out;
    H /= 2;
  }
  const float* splat = x;
  const int sb = h.sb, g1 = (sb + 1) / 2, g2 = (g1 + 1) / 2, c8 = 8 * h.cm * h.gd;
  float* gb1 = take(static_cast<size_t>(B) * g1 * g1 * c8);
  float* gb2 = take(static_cast<size_t>(B) * g2 * g2 * c8);
  float* lb1 = take(static_cast<size_t>(B) * sb * sb * c8);
  float* lb2 = take(static_cast<size_t>(B) * sb * sb * c8);
  float* f1 = take(static_cast<size_t>(B) * m->layers[li + 2].cout);
  float* f2 = take(static_cast<size_t>(B) * m->layers[li + 3].cout);
  float* f3 = take(static_cast<size_t>(B) * c8);
  if (!rc) rc = conv(li, splat, sb, sb, gb1);
  if (!rc) rc = conv(li + 1, gb1, g1, g1, gb2);
  const float* fin[3] = {gb2, f1, f2};
  float* fout[3] = {f1, f2, f3};
  for (int i = 0; i < 3 && !rc; ++i) {
    const LayerSpec& l = m->layers[li + 2 + i];
    rc = hdrnet_fc_f32(fin[i], m->w[li + 2 + i], m->b[li + 2 + i], fout[i], B, l.cin, l.cout, l.relu, st);
  }
  if (!rc) rc = conv(li + 5, splat, sb, sb, lb1);
  if (!rc) rc = conv(li + 6, lb1, sb, sb, lb2);
  if (!rc) rc = hdrnet_fuse_predict_f32(lb2, f3, m->w[li + 7], m->b[li + 7], grid, B, sb, sb, c8, h.gd, n_out, 4, st);
  return rc;
}

// One fused guide + slice-apply call (models._slice_apply_fused).
int slice_apply(const hdrnet_model* m, int level, const float* grid, const void* in, int in_fmt, void* out,
                int out_fmt, float* gmap, int B, int H, int W, float* slab, size_t slab_bytes, cudaStream_t st) {
  const Hyper& h = m->h;
  if (has_curves_guide(h.kind)) {
    const CurvesGuideHost& g = m->curves[level];
    return hdrnet_slice_apply_curves_px_ws(grid, in, in_fmt, out, out_fmt, gmap, B, H, W, h.sb, h.sb, h.gd, g.ccm,
                                           g.ccm_bias, g.shifts, g.slopes, g.mix, g.mix_bias, slab, slab_bytes, st);
  }
  const NNGuideHost& g = m->nn[level];
  return hdrnet_slice_apply_nn_px_ws(grid, in, in_fmt, out, out_fmt, gmap, B, H, W, h.sb, h.sb, h.gd, g.w1, g.b1,
                                     g.w2, g.b2, g.feats, slab, slab_bytes, st);
}

// coeffs [cells, 9, 4] -> the three levels' [cells, 3, 4] (coeffs[..., 3l:3l+3, :])
__global__ void __launch_bounds__(256)
split_level_rows_kernel(const float* __restrict__ coeffs, float* __restrict__ c0, float* __restrict__ c1,
                        float* __restrict__ c2, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long cell = e / 36;
    const int r = static_cast<int>(e % 36), level = r / 12;
    float* dst = level == 0 ? c0 : (level == 1 ? c1 : c2);
    dst[cell * 12 + r % 12] = coeffs[e];
  }
}

// HDRNetGaussianPyrNN.inference_image (and HDRNetGaussianPyr's) after the coefficients: the float image, its two smaller
// levels, one fused slice-apply per level with its three coefficient rows `coef` (level il's rows
// [B, sb, sb, gd, 12]), coarse-to-fine upsample-and-add.  `l` holds the intermediates for B x H x W.
int pyramid_fullres(const hdrnet_model* m, const Layout& l, const float* const coef[3], const void* image,
                    int in_fmt, void* out, int out_fmt, int B, int H, int W, cudaStream_t st) {
  const long long npx = static_cast<long long>(B) * H * W;
  int rc = HDRNET_OK;
  const float* lvl[3] = {static_cast<const float*>(image), l.lvl[1], l.lvl[2]};
  if (in_fmt != HDRNET_PX_F32) {
    rc = hdrnet_b200::launch_image_to_float(image, in_fmt, l.full, npx * 3, st);
    lvl[0] = l.full;
  }
  const int hs[3] = {H, H / 2, H / 4}, ws[3] = {W, W / 2, W / 4};
  for (int i = 1; i < 3 && !rc; ++i)
    rc = hdrnet_resize_bilinear_f32(lvl[i - 1], nullptr, l.lvl[i], B, hs[i - 1], ws[i - 1], 3, hs[i], ws[i], st);
  for (int il = 0; il < 3 && !rc; ++il) {
    const int src = 2 - il;   // reversed(zip(lvls, guides)): the coarsest level takes rows 0..2
    float* gmap = fused_row_kernel_takes(ws[src], lvl[src], l.lvl_out[src], coef[il]) ? nullptr : l.lvl_gmap[src];
    rc = slice_apply(m, src, coef[il], lvl[src], HDRNET_PX_F32, l.lvl_out[src], HDRNET_PX_F32, gmap, B, hs[src],
                     ws[src], nullptr, 0, st);
    if (rc || il == 0) continue;
    const float* current = il == 1 ? l.lvl_out[2] : l.cur1;
    if (il == 1)
      rc = hdrnet_resize_bilinear_f32(current, l.lvl_out[1], l.cur1, B, hs[2], ws[2], 3, hs[1], ws[1], st);
    else if (out_fmt == HDRNET_PX_F32)
      rc = hdrnet_resize_bilinear_f32(current, l.lvl_out[0], static_cast<float*>(out), B, hs[1], ws[1], 3, H, W, st);
    else
      rc = hdrnet_b200::launch_resize_quantize(current, l.lvl_out[0], out, out_fmt, B, hs[1], ws[1], 3, H, W, st);
  }
  return rc;
}

bool valid_fmt(int f) { return f == HDRNET_PX_F32 || f == HDRNET_PX_U8 || f == HDRNET_PX_U16; }
size_t px_bytes(int f) { return f == HDRNET_PX_U8 ? 1 : (f == HDRNET_PX_U16 ? 2 : 4); }

}  // namespace

extern "C" {

int hdrnet_model_create(const void* blob, size_t bytes, hdrnet_model** out) {
  if (!out) return HDRNET_E_NULL_POINTER;
  *out = nullptr;
  if (!blob) return HDRNET_E_NULL_POINTER;
  const unsigned char* p = static_cast<const unsigned char*>(blob);
  Hyper h;
  std::vector<LayerSpec> L;
  int n_ds = 0;
  std::vector<const unsigned char*> arrays;
  int rc = parse_blob(p, bytes, &h, &L, &n_ds, &arrays);
  if (rc != HDRNET_OK) return rc;

  hdrnet_model* m = new (std::nothrow) hdrnet_model();
  if (!m) return static_cast<int>(cudaErrorMemoryAllocation);
  m->h = h;
  m->n_ds = n_ds;
  m->layers = L;
  const int n_layers = static_cast<int>(L.size());
  // device layout: weights, biases, then the packed conv weights (models.pack_conv_weights: the
  // convs whose shape the packed tensor-core kernel takes, Cout <= 128; not the prediction layer)
  size_t off = 0, w_off[kMaxLayers], b_off[kMaxLayers], pk_off[kMaxLayers], pk_bytes[kMaxLayers];
  for (int i = 0; i < n_layers; ++i) {
    const LayerSpec& l = L[i];
    const size_t wn = static_cast<size_t>(l.k ? l.k * l.k : 1) * l.cin * l.cout;
    w_off[i] = off; off = align_up(off + wn * 4, 256);
    b_off[i] = off; off = align_up(off + static_cast<size_t>(l.bias ? l.cout : 0) * 4, 256);
    pk_bytes[i] = (l.k && i != n_layers - 1 && l.cout <= 128) ? hdrnet_conv2d_tc_packed_bytes(l.k, l.cin, l.cout) : 0;
    pk_off[i] = off; off = align_up(off + pk_bytes[i], 256);
  }
  cudaError_t e = cudaGetDevice(&m->device);
  cudaStream_t st = nullptr;
  if (e == cudaSuccess) e = cudaMalloc(&m->dev_mem, off);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  unsigned char* d = static_cast<unsigned char*>(m->dev_mem);
  for (int i = 0; i < n_layers && e == cudaSuccess; ++i) {
    const LayerSpec& l = L[i];
    const size_t wn = static_cast<size_t>(l.k ? l.k * l.k : 1) * l.cin * l.cout;
    m->w[i] = reinterpret_cast<const float*>(d + w_off[i]);
    m->b[i] = l.bias ? reinterpret_cast<const float*>(d + b_off[i]) : nullptr;
    e = cudaMemcpyAsync(d + w_off[i], arrays[2 * i], wn * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && l.bias)
      e = cudaMemcpyAsync(d + b_off[i], arrays[2 * i + 1], static_cast<size_t>(l.cout) * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && pk_bytes[i]) {
      float* pk = reinterpret_cast<float*>(d + pk_off[i]);
      rc = hdrnet_conv2d_tc_pack_f32(m->w[i], pk, l.k, l.cin, l.cout, st);
      if (rc > 0) e = static_cast<cudaError_t>(rc);
      m->packed[i] = rc == HDRNET_OK ? pk : nullptr;
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (st) cudaStreamDestroy(st);
  if (e != cudaSuccess) {
    if (m->dev_mem) cudaFree(m->dev_mem);
    delete m;
    return static_cast<int>(e);
  }
  // guides: host copies
  size_t a = 2 * n_layers;
  const int levels = is_pyramid(h.kind) ? 3 : 1;
  if (has_curves_guide(h.kind)) {
    for (int l = 0; l < levels; ++l, a += 6) {
      CurvesGuideHost& g = m->curves[l];
      read_floats(arrays[a], g.ccm, 9);
      read_floats(arrays[a + 1], g.ccm_bias, 3);
      read_floats(arrays[a + 2], g.shifts, 48);
      read_floats(arrays[a + 3], g.slopes, 48);
      read_floats(arrays[a + 4], g.mix, 3);
      read_floats(arrays[a + 5], &g.mix_bias, 1);
    }
  } else {
    for (int l = 0; l < levels; ++l, a += 4) {
      NNGuideHost& g = m->nn[l];
      g.feats = h.feats;
      read_floats(arrays[a], g.w1, 3 * static_cast<size_t>(h.feats));
      read_floats(arrays[a + 1], g.b1, h.feats);
      read_floats(arrays[a + 2], g.w2, h.feats);
      read_floats(arrays[a + 3], &g.b2, 1);
    }
  }
  m->magic = kModelMagic;
  {
    std::lock_guard<std::mutex> lock(g_models_mutex);
    g_models.insert(m);
  }
  *out = m;
  return HDRNET_OK;
}

int hdrnet_model_destroy(hdrnet_model* m) {
  {
    std::lock_guard<std::mutex> lock(g_models_mutex);
    if (!m || !g_models.erase(m)) return HDRNET_E_BAD_CONTEXT;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != m->device) cudaSetDevice(m->device);
  cudaFree(m->dev_mem);   // waits for work still reading the weights
  if (dev != m->device) cudaSetDevice(dev);
  m->magic = 0;
  delete m;
  return HDRNET_OK;
}

int hdrnet_model_info(const hdrnet_model* m, int* kind, int* net_input_size, int* spatial_bin, int* luma_bins,
                      int* channel_multiplier, int* guide_width) {
  if (!is_live(m)) return HDRNET_E_BAD_CONTEXT;
  if (kind) *kind = m->h.kind;
  if (net_input_size) *net_input_size = m->h.S;
  if (spatial_bin) *spatial_bin = m->h.sb;
  if (luma_bins) *luma_bins = m->h.gd;
  if (channel_multiplier) *channel_multiplier = m->h.cm;
  if (guide_width) *guide_width = m->h.feats;
  return HDRNET_OK;
}

size_t hdrnet_model_workspace_bytes(const hdrnet_model* m, int B, int H, int W, int in_fmt, int out_fmt) {
  if (!is_live(m) || B < 0 || H < 0 || W < 0 || !valid_fmt(in_fmt) || !valid_fmt(out_fmt)) return 0;
  Layout l;
  layout(m, B, H, W, in_fmt, out_fmt, 0, &l);
  return l.end + kAlign;   // + kAlign: any base is aligned up to kAlign
}

int hdrnet_model_run_px(const hdrnet_model* m, const void* image, int in_fmt, const void* lowres_image,
                        int lowres_fmt, int SH, int SW, void* out, int out_fmt, int B, int H, int W,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (!is_live(m)) return HDRNET_E_BAD_CONTEXT;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev != m->device) return HDRNET_E_BAD_CONTEXT;
  if (!valid_fmt(in_fmt) || !valid_fmt(out_fmt) || (lowres_image && !valid_fmt(lowres_fmt)))
    return HDRNET_E_UNSUPPORTED;
  const bool pyr = is_pyramid(m->h.kind);
  if (B < 0 || H < 0 || W < 0 || (lowres_image && (SH < 1 || SW < 1))) return HDRNET_E_BAD_SHAPE;
  const long long npx = static_cast<long long>(B) * H * W;
  if (npx == 0) return HDRNET_OK;
  if (pyr && (H < 4 || W < 4)) return HDRNET_E_BAD_SHAPE;   // three levels of floor(size / 2)
  if (!image || !out || !workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_model_workspace_bytes(m, B, H, W, in_fmt, out_fmt)) return HDRNET_E_BAD_SHAPE;
  if (out_fmt == HDRNET_PX_U16) {   // as the fused kernels: a uint16 result is not written over its input
    const uintptr_t o0 = reinterpret_cast<uintptr_t>(out), o1 = o0 + static_cast<uintptr_t>(npx) * 6u;
    const uintptr_t i0 = reinterpret_cast<uintptr_t>(image), i1 = i0 + static_cast<uintptr_t>(npx) * 3u * px_bytes(in_fmt);
    if (o0 < i1 && i0 < o1) return HDRNET_E_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Hyper& h = m->h;
  Layout l;
  layout(m, B, H, W, in_fmt, out_fmt, align_up(reinterpret_cast<uintptr_t>(workspace), kAlign), &l);

  const void* low_src = lowres_image ? lowres_image : image;
  int rc = hdrnet_lowres_nearest_f32(low_src, lowres_image ? lowres_fmt : in_fmt, l.lowres, B,
                                     lowres_image ? SH : H, lowres_image ? SW : W, h.S, h.S, st);
  if (!rc) rc = coefficients(m, l.lowres, l.grid, l.acts, l.acts_bytes, B, st);
  if (rc) return rc;

  if (!pyr) {
    const bool f32 = in_fmt == HDRNET_PX_F32 && out_fmt == HDRNET_PX_F32;
    float* gmap = (f32 && !fused_row_kernel_takes(W, image, out, l.grid)) ? l.gmap : nullptr;
    return slice_apply(m, 0, l.grid, image, in_fmt, out, out_fmt, gmap, B, H, W, l.slab, l.slab_bytes, st);
  }

  // the pyramids' inference_image: the float image, its two smaller levels, one fused
  // slice-apply per level with its three coefficient rows, coarse-to-fine upsample-and-add
  const long long cells = static_cast<long long>(B) * h.sb * h.sb * h.gd;
  split_level_rows_kernel<<<static_cast<unsigned>(std::min<long long>((cells * 36 + 255) / 256, 132LL * 32)), 256, 0,
                            st>>>(l.grid, l.coef[0], l.coef[1], l.coef[2], cells * 36);
  rc = static_cast<int>(cudaGetLastError());
  if (rc) return rc;
  const float* coef[3] = {l.coef[0], l.coef[1], l.coef[2]};
  return pyramid_fullres(m, l, coef, image, in_fmt, out, out_fmt, B, H, W, st);
}

size_t hdrnet_model_workspace_bytes_ragged(const hdrnet_model* m, const hdrnet_image_desc* images, int B, int in_fmt,
                                           int out_fmt) {
  if (!is_live(m) || !valid_fmt(in_fmt) || !valid_fmt(out_fmt) || B < 0 || (B > 0 && !images)) return 0;
  for (int i = 0; i < B; ++i)
    if (images[i].H <= 0 || images[i].W <= 0) return 0;
  Layout l;
  layout_ragged(m, images, B, in_fmt, 0, &l);
  return l.end + kAlign;   // + kAlign: any base is aligned up to kAlign
}

int hdrnet_model_run_ragged_px(const hdrnet_model* m, const hdrnet_image_desc* images, int B, int in_fmt,
                               int out_fmt, const hdrnet_image_desc* lowres, int lowres_fmt, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (!is_live(m)) return HDRNET_E_BAD_CONTEXT;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev != m->device) return HDRNET_E_BAD_CONTEXT;
  if (!valid_fmt(in_fmt) || !valid_fmt(out_fmt) || (lowres && !valid_fmt(lowres_fmt))) return HDRNET_E_UNSUPPORTED;
  const bool pyr = is_pyramid(m->h.kind);
  int rc = hdrnet_b200::validate_ragged(images, B, in_fmt, out_fmt, true, pyr ? 4 : 1);
  if (rc != HDRNET_OK || B == 0) return rc;
  if (lowres && (rc = hdrnet_b200::validate_ragged(lowres, B, lowres_fmt, out_fmt, false, 1)) != HDRNET_OK) return rc;
  if (!workspace) return HDRNET_E_NULL_POINTER;
  if (workspace_bytes < hdrnet_model_workspace_bytes_ragged(m, images, B, in_fmt, out_fmt)) return HDRNET_E_BAD_SHAPE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Hyper& h = m->h;
  Layout l;
  layout_ragged(m, images, B, in_fmt, align_up(reinterpret_cast<uintptr_t>(workspace), kAlign), &l);

  rc = hdrnet_lowres_nearest_ragged_f32(lowres ? lowres : images, B, lowres ? lowres_fmt : in_fmt, l.lowres, h.S,
                                        h.S, st);
  if (!rc) rc = coefficients(m, l.lowres, l.grid, l.acts, l.acts_bytes, B, st);
  if (rc) return rc;
  if (!pyr) {
    if (h.kind == HDRNET_MODEL_CURVES) {
      const CurvesGuideHost& g = m->curves[0];
      return hdrnet_slice_apply_curves_ragged_px_ws(l.grid, images, B, in_fmt, out_fmt, h.sb, h.sb, h.gd, g.ccm,
                                                    g.ccm_bias, g.shifts, g.slopes, g.mix, g.mix_bias, nullptr, 0, st);
    }
    const NNGuideHost& g = m->nn[0];
    return hdrnet_slice_apply_nn_ragged_px_ws(l.grid, images, B, in_fmt, out_fmt, h.sb, h.sb, h.gd, g.w1, g.b1, g.w2,
                                              g.b2, g.feats, nullptr, 0, st);
  }
  // the pyramid: its coefficient network ran on the whole batch; its full-resolution stages run image
  // by image on hdrnet_model_run_px's kernels (there is no ragged form of the resizes)
  const long long cells = static_cast<long long>(B) * h.sb * h.sb * h.gd;
  split_level_rows_kernel<<<static_cast<unsigned>(std::min<long long>((cells * 36 + 255) / 256, 132LL * 32)), 256, 0,
                            st>>>(l.grid, l.coef[0], l.coef[1], l.coef[2], cells * 36);
  rc = static_cast<int>(cudaGetLastError());
  const size_t image_cells = static_cast<size_t>(h.sb) * h.sb * h.gd * 12;
  for (int i = 0; i < B && !rc; ++i) {
    const float* coef[3] = {l.coef[0] + i * image_cells, l.coef[1] + i * image_cells, l.coef[2] + i * image_cells};
    rc = pyramid_fullres(m, l, coef, images[i].image, in_fmt, images[i].out, out_fmt, 1, images[i].H, images[i].W,
                         st);
  }
  return rc;
}

}  // extern "C"
