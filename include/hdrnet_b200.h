/*
 * hdrnet_b200.h -- C-ABI of libhdrnet_b200.so: the H100 (sm_90a) implementation of
 * google/hdrnet's bilateral-slice hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / TF types.  Each entry
 * point cites the reference interface it replaces.  All tensors use the reference op's
 * layout (TF row-major NHWC, last index fastest; hdrnet/ops/bilateral_slice_apply_op.cc:
 * 201-227):
 *
 *     grid   [B, gh, gw, gd, gc]   float32   gc = n_out * (n_in + has_offset), c = i*J + j
 *     guide  [B, H, W]             float32   expected in [0, 1], not enforced
 *     input  [B, H, W, n_in]       float32
 *     out    [B, H, W, n_out]      float32   (slice-apply)   /  [B, H, W, gc]  (slice)
 *
 * Conventions (replacing TF's OpKernel contract, SURVEY.md section 8b):
 *   - the caller owns and allocates every buffer, including outputs;
 *   - `*_f32` device entry points take DEVICE pointers valid on the current CUDA device and
 *     launch asynchronously on `stream` (a cudaStream_t passed as void*; NULL = default
 *     stream); they never allocate, never synchronise, and are re-entrant;
 *   - every function returns 0 on success, a negative HDRNET_E_* code for a contract
 *     violation (the conditions the reference raises InvalidArgument for), or a positive
 *     cudaError_t if a launch failed (the reference's Internal("... kernel failed."));
 *   - empty outputs (B*H*W == 0) succeed without launching (bilateral_slice_apply.cu.cc:
 *     373-379).
 */
#ifndef HDRNET_B200_H_
#define HDRNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HDRNET_B200_ABI_VERSION 1

/* Exported from libhdrnet_b200.so (the library is built with -fvisibility=hidden). */
#if defined(__GNUC__)
#define HDRNET_API __attribute__((visibility("default")))
#else
#define HDRNET_API
#endif

/* Contract violations (negative; positive return values are cudaError_t). */
#define HDRNET_OK 0
#define HDRNET_E_NULL_POINTER (-1)   /* a required pointer is NULL                         */
#define HDRNET_E_BAD_SHAPE (-2)      /* a dimension is negative, or gh/gw/gd/gc/n_* is < 1 */
#define HDRNET_E_BAD_CHANNELS (-3)   /* gc != n_out * (n_in + has_offset)                  */
#define HDRNET_E_TOO_LARGE (-4)      /* an extent does not fit the kernels' 32-bit indices */
#define HDRNET_E_UNSUPPORTED (-5)    /* the requested variant cannot run these shapes      */
#define HDRNET_E_BAD_CONTEXT (-6)    /* invalid / destroyed context or model, wrong device */
#define HDRNET_E_BAD_MODEL (-7)      /* malformed frozen model file                        */

/* Kernel selection for the *_variant debug entry points. */
#define HDRNET_VARIANT_AUTO 0    /* what the plain entry points use                        */
#define HDRNET_VARIANT_GENERIC 1 /* one thread per pixel, any shape / alignment            */
#define HDRNET_VARIANT_TMA 2     /* persistent TMA-staged row kernel (needs W % 4 == 0,    */
                                 /* 16-byte aligned buffers; n_in == 3, n_out == 3,        */
                                 /* has_offset for slice-apply)                            */
#define HDRNET_VARIANT_TEX 4     /* texture-assisted TMA kernel: a pre-pass writes the      */
                                 /* y-pre-blended slab rows to a caller workspace; the row  */
                                 /* kernel then fetches part of each pixel's corner data    */
                                 /* through the texture pipe, which does not share the      */
                                 /* shared-memory crossbar.  Needs hdrnet_slice_apply_f32_ws*/
#define HDRNET_VARIANT_TEX_ASYNC 7 /* the texture-assisted kernel with an ISSUER warp: math      */
                                 /* warps that never wait for each other (mbarrier arrive    */
                                 /* instead of block barriers) + one warp that issues every  */
                                 /* bulk copy; per-quad index arithmetic.  Same requirements */
                                 /* as HDRNET_VARIANT_TEX.  (Values 3, 5, 6, 8-11 named forms */
                                 /* that measured slower; they are not part of the library.) */
HDRNET_API int hdrnet_b200_abi_version(void);

/* Human-readable text for a return code of this library (static storage). */
HDRNET_API const char* hdrnet_b200_error_string(int code);

/*
 * Fused slice + affine apply.  Replaces the BilateralSliceApply op:
 *   Python   hdrnet/hdrnet_ops.py:31          hdrnet_ops.bilateral_slice_apply
 *   OpKernel hdrnet/ops/bilateral_slice_apply_op.cc:140-235  (Compute, GpuDevice)
 *   kernel   hdrnet/ops/bilateral_slice_apply.cu.cc:36-126, launcher :368-382
 * out[b,y,x,i] = sum_j trilerp(grid[..., i*J + j]) * (j < n_in ? input[b,y,x,j] : 1).
 */
HDRNET_API int hdrnet_slice_apply_f32(const float* grid, const float* guide, const float* input,
                           float* out, int B, int H, int W, int gh, int gw, int gd, int n_in,
                           int n_out, int has_offset, void* stream);

/* Same, with the kernel variant forced (tests exercise every variant on the same inputs). */
HDRNET_API int hdrnet_slice_apply_f32_variant(const float* grid, const float* guide, const float* input,
                                   float* out, int B, int H, int W, int gh, int gw, int gd,
                                   int n_in, int n_out, int has_offset, int variant,
                                   void* stream);

/*
 * Same op with a caller-provided device workspace (the library itself never allocates):
 * required by HDRNET_VARIANT_TEX, ignored by the other variants.
 * hdrnet_slice_apply_workspace_bytes() = B * H * gw * gd * 48.  The texture-assisted forms read
 * the workspace through a texture object, so they need it aligned to the device's texture alignment
 * (512 bytes on H100; cudaMalloc and torch's allocator return such blocks): with any other base AUTO
 * runs the TMA row kernel and a forced TEX / TEX_ASYNC returns HDRNET_E_UNSUPPORTED.
 * The workspace is scratch: its contents are undefined after a call (the kernels may drop rows
 * they are done with from L2 without writing them back), and a call never reads what an earlier
 * call left there.
 */
HDRNET_API size_t hdrnet_slice_apply_workspace_bytes(int B, int H, int gw, int gd);
HDRNET_API int hdrnet_slice_apply_f32_ws(const float* grid, const float* guide,
                                         const float* input, float* out, int B, int H, int W,
                                         int gh, int gw, int gd, int n_in, int n_out,
                                         int has_offset, int variant, void* workspace,
                                         size_t workspace_bytes, void* stream);

/*
 * Row band of the same op: guide / input / out hold `rows` image rows per image, starting at
 * image row `y_off` of images that are H rows tall ([B, rows, W(, c)] dense); the grid is whole.
 * The op is pointwise in (x, y) -- the kernel's only use of y is the grid coordinate
 * (y + 0.5) * gh / H, hdrnet/ops/bilateral_slice_apply.cu.cc:52, :75, :80, :88-90 -- so bands need no halo
 * and the bands of an image, computed anywhere, are bit for bit the rows of the whole-image call
 * by the same kernel.  This is the multi-GPU fallback when there are fewer images than GPUs
 * (SURVEY.md section 8e: each rank takes a row band and a copy of the 98 KB grid) and what the
 * host path streams.  workspace (optional, may be NULL / 0): hdrnet_slice_apply_workspace_bytes(B,
 * rows, gw, gd) bytes.  rows == H, y_off == 0 is hdrnet_slice_apply_f32_ws.
 */
HDRNET_API int hdrnet_slice_apply_rows_f32_ws(const float* grid, const float* guide,
                                              const float* input, float* out, int B, int H, int W,
                                              int rows, int y_off, int gh, int gw, int gd, int n_in,
                                              int n_out, int has_offset, int variant,
                                              void* workspace, size_t workspace_bytes, void* stream);

/*
 * Un-fused slice.  Replaces the BilateralSlice op:
 *   Python   hdrnet/hdrnet_ops.py:30          hdrnet_ops.bilateral_slice
 *   OpKernel hdrnet/ops/bilateral_slice_op.cc:120-174
 *   kernel   hdrnet/ops/bilateral_slice.cu.cc:34-91, launcher :230-244
 * out[b,y,x,c] = trilerp(grid[..., c]) at ((x+.5)*gw/W, (y+.5)*gh/H, guide*gd).
 */
HDRNET_API int hdrnet_slice_f32(const float* grid, const float* guide, float* out, int B, int H, int W,
                     int gh, int gw, int gd, int gc, void* stream);

HDRNET_API int hdrnet_slice_f32_variant(const float* grid, const float* guide, float* out, int B, int H,
                             int W, int gh, int gw, int gd, int gc, int variant, void* stream);

/*
 * Vector-Jacobian products (training).  Replace the BilateralSliceApplyGrad / BilateralSliceGrad
 * ops: Python registration hdrnet/hdrnet_ops.py:34-48; OpKernels
 * hdrnet/ops/bilateral_slice_apply_op.cc:249-362 and bilateral_slice_op.cc:183-256; kernels
 * hdrnet/ops/bilateral_slice_apply.cu.cc:128-364 (+ launcher :384-417) and
 * bilateral_slice.cu.cc:93-227 (+ :246-272).  codomain_tangent has the forward output's shape;
 * grid_vjp / guide_vjp / input_vjp have the shapes of grid / guide / input.  Semantics follow
 * the reference exactly (mirror boundary of the grid-VJP footprint, wz = 1 at the depth
 * borders, dwz = gd * SmoothedLerpWeightGrad); results are deterministic (no atomics).
 */
HDRNET_API int hdrnet_slice_apply_grad_f32(const float* grid, const float* guide,
                                           const float* input, const float* codomain_tangent,
                                           float* grid_vjp, float* guide_vjp, float* input_vjp,
                                           int B, int H, int W, int gh, int gw, int gd, int n_in,
                                           int n_out, int has_offset, void* stream);

HDRNET_API int hdrnet_slice_grad_f32(const float* grid, const float* guide,
                                     const float* codomain_tangent, float* grid_vjp,
                                     float* guide_vjp, int B, int H, int W, int gh, int gw,
                                     int gd, int gc, void* stream);

/*
 * Debug: the unclamped lower cell indices (gx0, gy0, gz0) the kernels use, written as
 * idx[b,y,x,0..2] int32.  It runs the same device functions as the slice kernels, so the
 * bit-exactness of the index arithmetic (bilateral_slice_apply.cu.cc:73-80;
 * jax/bilateral_slice.py:317-327) can be asserted against the oracle.
 */
HDRNET_API int hdrnet_slice_indices_i32(const float* guide, int32_t* idx, int B, int H, int W, int gh,
                             int gw, int gd, void* stream);

/*
 * Kernel-introspection for benchmarks: the variant AUTO runs for these shapes with 16-byte aligned
 * buffers, and the launch geometry of its main kernel (CTAs, threads, dynamic shared memory bytes).
 * The same planner decides the launches, so the report is what the call runs.
 */
HDRNET_API int hdrnet_slice_apply_plan(int B, int H, int W, int gh, int gw, int gd, int n_in, int n_out,
                            int has_offset, int* variant, int* ctas, int* threads,
                            int* smem_bytes);
/* Same, for a call that lends a workspace (hdrnet_slice_apply_f32_ws) of
 * hdrnet_slice_apply_workspace_bytes at the device's texture alignment. */
HDRNET_API int hdrnet_slice_apply_plan_ws(int B, int H, int W, int gh, int gw, int gd, int n_in,
                                          int n_out, int has_offset, int with_workspace,
                                          int* variant, int* ctas, int* threads, int* smem_bytes);

/*
 * Full-resolution guidance maps (input [npix, 3] float32 RGB -> guide [npix] float32).
 * Coefficient arrays are HOST pointers, read before the call returns (they travel in the
 * kernel argument block).
 *
 * Curves guide.  Replaces HDRNetCurves._guide, hdrnet/models.py:145-190:
 *   t = rgb . ccm + ccm_bias;  u_c = sum_k slopes[c][k] * relu(t_c - shifts[c][k]);
 *   guide = clip(sum_c mix[c] * u_c + mix_bias, 0, 1)
 * ccm[3][3] is indexed [in][out] (tf.matmul(x, ccm), :156); shifts/slopes are [3][16]
 * (the reference's variables `shifts` [1,1,3,16] and `slopes` [1,1,1,3,16] flattened).
 */
HDRNET_API int hdrnet_guide_curves_f32(const float* input, float* guide, long long npix,
                                       const float* ccm, const float* ccm_bias,
                                       const float* shifts, const float* slopes,
                                       const float* mix, float mix_bias, void* stream);

/*
 * Pointwise-NN guide.  Replaces HDRNetPointwiseNNGuide._guide, hdrnet/models.py:199-210:
 *   h_f = relu(sum_c x_c * w1[c][f] + b1[f]);  guide = sigmoid(sum_f h_f * w2[f] + b2)
 * with conv1's batch norm already folded into w1[3][feats] / b1[feats] by the caller
 * (inference form, hdrnet/bin/freeze_graph.py:141-142).  feats <= 32.
 */
HDRNET_API int hdrnet_guide_nn_f32(const float* input, float* guide, long long npix,
                                   const float* w1, const float* b1, const float* w2, float b2,
                                   int feats, void* stream);

/*
 * Curves-guide VJP: the backward of hdrnet_guide_curves_f32 (training the guide; the gradient TF
 * gives HDRNetCurves._guide, hdrnet/models.py:145-190).  dguide [npix] is the gradient of the
 * guide; the clip passes it where 0 <= a <= 1 (equality included, as tf.clip_by_value) and each
 * relu where t > shift (0 at equality, as TF's ReluGrad), both decided on the forward's own floats.
 *   dinput [npix, 3]  gradient of the input; NULL: not computed.
 *   dparams [112]     DEVICE array, the gradients of the variables summed over all npix pixels, in
 *                     the order ccm 9 ([in][out]), ccm_bias 3, shifts 48 ([3][16]), slopes 48
 *                     ([3][16]), mix 3, mix_bias 1; NULL: not computed.
 * The coefficient arrays are HOST pointers, as for hdrnet_guide_curves_f32.  Gradients are written,
 * not accumulated.  The parameter sums go through per-CTA partial sums of fixed pixel chunks (the
 * chunk size depends on npix alone) in a caller-lent workspace of
 * hdrnet_guide_curves_grad_workspace_bytes(npix) bytes (needed when dparams is not NULL; smaller:
 * HDRNET_E_BAD_SHAPE), then a second pass adds the chunks in a fixed order: no atomics, bitwise
 * reproducible.  The workspace is scratch, undefined after the call.  npix == 0 writes zero
 * parameter gradients.
 */
HDRNET_API size_t hdrnet_guide_curves_grad_workspace_bytes(long long npix);
HDRNET_API int hdrnet_guide_curves_grad_f32(const float* input, const float* dguide, float* dinput,
                                            long long npix, const float* ccm,
                                            const float* ccm_bias, const float* shifts,
                                            const float* slopes, const float* mix, float mix_bias,
                                            float* dparams, void* workspace,
                                            size_t workspace_bytes, void* stream);

/*
 * Pointwise-NN guide in training mode (HDRNetPointwiseNNGuide._guide with is_training=True,
 * hdrnet/models.py:203-210): conv1's batch norm normalises with the batch's statistics.  conv1 is
 * 1x1 and linear from 3 channels, so the mean and variance of every feature follow from the mean m
 * and the biased covariance C of the input's three channels:
 *   mu_f = m . w1[:, f],  var_f = w1[:, f]' C w1[:, f],  s_f = 1 / sqrt(var_f + 1e-3)
 * and the layer is hdrnet_guide_nn_f32 with w1'[c][f] = w1[c][f] s_f, b1'[f] = beta[f] - mu_f s_f.
 *
 * hdrnet_guide_nn_stats_f32: moments [9], a DEVICE array of doubles, receives m (3) and C
 * (c00, c01, c02, c11, c12, c22) over npix pixels of input [npix, 3].  Per-CTA partials of fixed
 * pixel chunks (the chunking depends on npix alone), each centred on its chunk, go to a caller-lent
 * workspace of hdrnet_guide_nn_stats_workspace_bytes(npix) bytes (smaller: HDRNET_E_BAD_SHAPE) and
 * are merged in float64 in a fixed order: no atomics, bitwise reproducible.  npix == 0 writes zeros.
 *
 * hdrnet_guide_nn_batch_fold: HOST arithmetic in float64, no device work.  From w1 [3][feats]
 * (conv1/weights), beta [feats] (BatchNorm/beta) and HOST moments [9] it writes the folded
 * w1_folded [3][feats] and b1_folded [feats] (float32, for hdrnet_guide_nn_f32) and, when not NULL,
 * batch_mean [feats] and batch_var [feats] (the biased variance that normalises).
 *
 * hdrnet_guide_nn_grad_f32: the VJP of that guide, batch statistics included (the gradient flows
 * through mu and var).  dguide [npix] is the gradient of the guide; relu masks are TF's
 * (ReluGrad: y > 0), decided on the floats hdrnet_guide_nn_f32 computes with the folded weights.
 *   dinput [npix, 3]     gradient of the input; NULL: not computed.
 *   dparams [5 feats + 1] DEVICE array, the gradients of conv1/weights [3][feats], BatchNorm/beta
 *                        [feats], conv2/weights [feats] and conv2/biases [1], in that order; NULL:
 *                        not computed.
 * w1, beta, w2 and moments are HOST pointers (the moments the forward used).  Gradients are
 * written, not accumulated.  Per-CTA partial sums of fixed pixel chunks go to a caller-lent
 * workspace of hdrnet_guide_nn_grad_workspace_bytes(npix, feats) bytes (needed when either output
 * is wanted: dinput needs the sums too; smaller: HDRNET_E_BAD_SHAPE), added in a fixed order: no
 * atomics, bitwise reproducible.  The workspace is scratch, undefined after the call.  npix == 0
 * writes zero parameter gradients.  feats <= 32.
 */
HDRNET_API size_t hdrnet_guide_nn_stats_workspace_bytes(long long npix);
HDRNET_API int hdrnet_guide_nn_stats_f32(const float* input, long long npix, double* moments,
                                         void* workspace, size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_guide_nn_batch_fold(const float* w1, const float* beta, const double* moments,
                                          int feats, float* w1_folded, float* b1_folded,
                                          double* batch_mean, double* batch_var);
HDRNET_API size_t hdrnet_guide_nn_grad_workspace_bytes(long long npix, int feats);
HDRNET_API int hdrnet_guide_nn_grad_f32(const float* input, const float* dguide, float* dinput,
                                        long long npix, const float* w1, const float* beta,
                                        const float* w2, float b2, int feats,
                                        const double* moments, float* dparams, void* workspace,
                                        size_t workspace_bytes, void* stream);

/*
 * Training-mode batch norm of the coefficient network's layers (hdrnet/layers.py:47-54 with
 * is_training=True, center=True, scale=False, epsilon 1e-3, decay 0.999).  z is the layer's conv
 * or fc output WITHOUT bias or relu (hdrnet_conv2d_nhwc_f32 / hdrnet_fc_f32 with bias NULL and
 * relu 0), an [N, C] row-major float32 view (NHWC flattened; an fc layer has N = B).  Every
 * pointer is a DEVICE pointer; nothing is read back to the host.  N >= 1 and
 * 1 <= C <= HDRNET_BN_MAX_CHANNELS (larger: HDRNET_E_UNSUPPORTED).  Float arrays must be 4-byte
 * and double arrays and workspaces 8-byte aligned (HDRNET_E_BAD_SHAPE otherwise).
 *
 * moments [3][C] (float64) holds per channel the row count n, the mean and the sum of squared
 * deviations M2, so that the moments of several ranks' shards merge exactly (Chan et al.).
 *
 * hdrnet_bn_stats_f32: the moments of z over its N rows (n = N).  Per-CTA partials of fixed row
 * chunks (chosen from N and C alone), each centred on its first row, go to a caller-lent
 * workspace of hdrnet_bn_stats_workspace_bytes(N, C) bytes (smaller: HDRNET_E_BAD_SHAPE) and are
 * merged in float64 in a fixed order: no atomics, bitwise reproducible.
 *
 * hdrnet_bn_relu_f32: y [N, C] = relu((z - mean) / sqrt(M2 / n + 1e-3) + beta [C]).  When
 * moving_mean and moving_var [C] are given (both or neither) they move toward the batch's
 * statistics in place, as TF's moving-average update does without zero-debias:
 * v -= (1 - 0.999) (v - batch), the variance fed to it Bessel-corrected, M2 / n * n / (n - 1)
 * (0 for n = 1).
 *
 * hdrnet_bn_relu_grad_sums_f32: with dy [N, C] the gradient of y and dyh = dy [y > 0] (TF's
 * ReluGrad on the y hdrnet_bn_relu_f32 computes), sums [2][C] (float64) receives
 * A = sum dyh and B = sum dyh (z - mean) s over this call's N rows, and dbeta [C] (optional) A as
 * float32.  The workspace is that of hdrnet_bn_stats_f32 (hdrnet_bn_stats_workspace_bytes), the
 * same fixed chunks summed in a fixed order.
 *
 * hdrnet_bn_relu_grad_f32: dz [N, C] = s (dyh - A / n - (z - mean) s B / n), with n, A and B
 * from moments and sums.  Split from the sums so that the sums of several ranks can be added
 * between the two calls, as their moments are merged before hdrnet_bn_relu_f32.
 * The workspaces are scratch, undefined after the call.
 */
#define HDRNET_BN_MAX_CHANNELS 8192
HDRNET_API size_t hdrnet_bn_stats_workspace_bytes(long long N, int C);
HDRNET_API int hdrnet_bn_stats_f32(const float* z, long long N, int C, double* moments,
                                   void* workspace, size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_bn_relu_f32(const float* z, long long N, int C, const double* moments,
                                  const float* beta, float* y, float* moving_mean,
                                  float* moving_var, void* stream);
HDRNET_API int hdrnet_bn_relu_grad_sums_f32(const float* z, const float* dy, long long N, int C,
                                            const double* moments, const float* beta,
                                            double* sums, float* dbeta, void* workspace,
                                            size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_bn_relu_grad_f32(const float* z, const float* dy, long long N, int C,
                                       const double* moments, const float* beta,
                                       const double* sums, float* dz, void* stream);

/*
 * Model-path forms of slice-apply: the guide is computed per pixel INSIDE the kernel from the
 * full-res RGB (the guide map never touches HBM: 24 B/px instead of 28 B/px + a guide pass).
 * Replaces HDRNetCurves.inference / HDRNetPointwiseNNGuide.inference's `_guide` + `_output`
 * (hdrnet/models.py:43-59, :145-196, :199-210).  n_in = 3, n_out = 3, has_offset.
 * guide_out: optional [B,H,W] dump of the guide (run.py --debug); may be NULL when the
 * shapes suit the fused kernel (W % 4 == 0, W >= 128, 16-byte aligned buffers); other shapes
 * run guide kernel + generic slice-apply and then REQUIRE guide_out as the intermediate.
 * Coefficient arrays are host pointers, as for hdrnet_guide_*_f32.
 */
HDRNET_API int hdrnet_slice_apply_curves_f32(const float* grid, const float* input, float* out,
                                             float* guide_out, int B, int H, int W, int gh,
                                             int gw, int gd, const float* ccm,
                                             const float* ccm_bias, const float* shifts,
                                             const float* slopes, const float* mix,
                                             float mix_bias, void* stream);

HDRNET_API int hdrnet_slice_apply_nn_f32(const float* grid, const float* input, float* out,
                                         float* guide_out, int B, int H, int W, int gh, int gw,
                                         int gd, const float* w1, const float* b1,
                                         const float* w2, float b2, int feats, void* stream);

/*
 * Coefficient network layers (device pointers; activations NHWC, float32).  Replace the TF
 * layers of HDRNetCurves._coefficients, hdrnet/models.py:62-142 / hdrnet/layers.py:25-93.
 * Batch norm (inference) is folded into w / bias by the caller.
 *
 * conv2d: k in {1, 3}, stride in {1, 2}, TF 'SAME' padding (total = max((ceil(in/s)-1)*s +
 * k - in, 0), floor(total/2) before, rest after), weights HWIO [k][k][Cin][Cout], optional
 * bias (NULL = none), optional ReLU.  out is [B, ceil(H/s), ceil(W/s), Cout].
 */
HDRNET_API int hdrnet_conv2d_nhwc_f32(const float* in, const float* w, const float* bias,
                                      float* out, int B, int H, int W, int Cin, int Cout, int k,
                                      int stride, int relu, void* stream);

/*
 * Tensor-core form of conv2d (wgmma.mma_async .tf32 with 3xTF32 operand splitting, fp32
 * accumulator; float32-grade results).  Weights are packed ONCE per model into per-chunk hi/lo tiles
 * in the MMA's shared-memory layout (hdrnet_conv2d_tc_packed_bytes() bytes, 16-byte aligned device
 * memory owned by the caller: HDRNET_E_UNSUPPORTED otherwise); the layer call then needs
 * Cin % 4 == 0, Cout % 16 == 0, 16 <= Cout <= 128.
 * hdrnet_conv2d_nhwc_f32 runs an unpacked tensor-core kernel on its own when the layer has
 * >= 96 tiles of 128 output pixels and its shape suits that kernel.
 */
HDRNET_API size_t hdrnet_conv2d_tc_packed_bytes(int k, int Cin, int Cout);
HDRNET_API int hdrnet_conv2d_tc_pack_f32(const float* w, float* packed, int k, int Cin, int Cout,
                                         void* stream);
HDRNET_API int hdrnet_conv2d_nhwc_tc_f32(const float* in, const float* packed_w, const float* bias,
                                         float* out, int B, int H, int W, int Cin, int Cout,
                                         int k, int stride, int relu, void* stream);

/*
 * conv2d on the CUDA cores alone (float32 FMAs rounded to nearest), at every shape: what
 * hdrnet_conv2d_nhwc_f32 runs below 96 tiles.  Its tensor-core form from 96 tiles up (3xTF32)
 * is float32-grade to about 1e-6 of a product; training-mode batch norm divides a conv's error by
 * the channel's spread, and runs its convs here.
 */
HDRNET_API int hdrnet_conv2d_nhwc_fp32_f32(const float* in, const float* w, const float* bias,
                                           float* out, int B, int H, int W, int Cin, int Cout,
                                           int k, int stride, int relu, void* stream);

/* fully_connected: out[B,O] = in[B,I] @ w[I,O] + bias (+ReLU). */
HDRNET_API int hdrnet_fc_f32(const float* in, const float* w, const float* bias, float* out,
                             int B, int I, int O, int relu, void* stream);

/*
 * Fusion + prediction + unroll_grid (models.py:122-139) in one pass:
 *   f = relu(local[b,y,x,:] + global[b,:]);  p[o] = sum_c f[c] * w[c][o] + bias[o]
 *   grid[b,y,x,z,i,j] = p[(j*n_out + i)*gd + z]        (n_in counts the offset column)
 * local [B,gh,gw,C], global [B,C], w [C][gd*n_out*n_in], grid [B,gh,gw,gd,n_out*n_in].
 */
HDRNET_API int hdrnet_fuse_predict_f32(const float* local, const float* global_feat,
                                       const float* w, const float* bias, float* grid, int B,
                                       int gh, int gw, int C, int gd, int n_out, int n_in,
                                       void* stream);

/*
 * Vector-Jacobian products of the coefficient network's layers (fine-tuning the network through
 * the slice-apply VJP; the backward of hdrnet/models.py:62-142 that TF's gradients give).  Same
 * layouts and the same TF 'SAME' geometry as the forwards above.  `dout` is the gradient of the
 * layer's output; for a ReLU layer it is masked by `out > 0` (TF's ReluGrad masks on the layer's
 * output), so `out` is required when relu != 0 and may be NULL otherwise.  Any of din / dw / db
 * may be NULL when that gradient is not wanted (din of the first layer, db of a layer without
 * bias); `w` may be NULL when din is, `in` when dw and db are.  Gradients are written, not
 * accumulated.  The weight and bias VJPs sum over output pixels in per-CTA chunks whose partial
 * sums go to a caller-lent workspace (*_workspace_bytes; the library never allocates), then a
 * second pass adds the chunks in a fixed order.  No floating-point atomics: results are
 * bitwise reproducible.  The workspace is scratch, undefined after the call.
 *
 * conv2d VJP: the backward of hdrnet_conv2d_nhwc_f32 (and of its tensor-core form).
 */
HDRNET_API size_t hdrnet_conv2d_grad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int k,
                                                     int stride);
HDRNET_API int hdrnet_conv2d_grad_f32(const float* in, const float* w, const float* out,
                                      const float* dout, float* din, float* dw, float* db, int B,
                                      int H, int W, int Cin, int Cout, int k, int stride, int relu,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* fully_connected VJP: the backward of hdrnet_fc_f32 (din = dout' w^T, dw = in^T dout',
 * db = sum_b dout'). */
HDRNET_API size_t hdrnet_fc_grad_workspace_bytes(int B, int I, int O);
HDRNET_API int hdrnet_fc_grad_f32(const float* in, const float* w, const float* out,
                                  const float* dout, float* din, float* dw, float* db, int B, int I,
                                  int O, int relu, void* workspace, size_t workspace_bytes,
                                  void* stream);

/*
 * Fusion + prediction + unroll_grid VJP: the backward of hdrnet_fuse_predict_f32.  dgrid has the
 * grid's shape; dpred[o] = dgrid[b,y,x,z,i,j] for o = (j*n_out + i)*gd + z.  fused =
 * relu(local + global) is recomputed from the saved local / global, not stored:
 *   dw[c][o] = sum_{b,y,x} fused * dpred,  db[o] = sum dpred,
 *   dlocal = (dpred w^T) * (fused > 0),   dglobal[b,c] = sum_{y,x} dlocal[b,y,x,c].
 */
HDRNET_API size_t hdrnet_fuse_predict_grad_workspace_bytes(int B, int gh, int gw, int C, int gd,
                                                           int n_out, int n_in);
HDRNET_API int hdrnet_fuse_predict_grad_f32(const float* local, const float* global_feat,
                                            const float* w, const float* dgrid, float* dlocal,
                                            float* dglobal, float* dw, float* db, int B, int gh,
                                            int gw, int C, int gd, int n_out, int n_in,
                                            void* workspace, size_t workspace_bytes, void* stream);

/*
 * The WHOLE coefficient network (splat convs, global convs + fcs, local convs, fusion, prediction,
 * unroll_grid) behind one call: replaces HDRNetCurves._coefficients, hdrnet/models.py:62-142, with
 * batch norm folded by the caller.  At small batch the twelve layers are 8 launches -- the global
 * and the local branch (both read the splat features) share a launch per depth, fc1-fc3 run in one
 * 8-CTA cluster with activations in distributed shared memory -- chained with programmatic
 * dependent launch so that each layer's launch and weight fetch overlap the previous layer's tail
 * (tools/time_cnn.py compares it with twelve per-layer calls).
 *   lowres [B, S, S, 3] float32 -> grid [B, sb, sb, gd, n_out, n_in] float32
 *   weights / biases: HOST arrays of n_layers = n_ds + 8 DEVICE pointers (n_ds = log2(S / sb)), in
 *     the order splat conv1..n_ds, global conv1, conv2, fc1, fc2, fc3, local conv1, conv2,
 *     prediction conv1; conv weights HWIO, fc / prediction weights [in][out]; a bias may be NULL;
 *   scratch: hdrnet_coefficients_scratch_bytes(...) bytes of device memory, 16-byte aligned (every
 *     layer's activations, each in a buffer of its own; the library never allocates).  0 bytes =
 *     S / sb is not a power of two >= 2 (HDRNET_E_UNSUPPORTED from the call).
 * Layers whose shape a fast form does not take (channels % 4, fc widths not powers of two, large
 * batches) run the general kernels inside the same call.
 */
HDRNET_API size_t hdrnet_coefficients_scratch_bytes(int B, int net_input_size, int spatial_bin,
                                                    int luma_bins, int channel_multiplier, int n_out,
                                                    int n_in);
HDRNET_API int hdrnet_coefficients_f32(const float* lowres, float* grid, const float* const* weights,
                                       const float* const* biases, int n_layers, void* scratch,
                                       size_t scratch_bytes, int B, int net_input_size,
                                       int spatial_bin, int luma_bins, int channel_multiplier,
                                       int n_out, int n_in, void* stream);

/*
 * Bilinear resize, align_corners=True, NHWC, with an optional fused add (`add` has the output's
 * shape, or NULL).  Replaces tf.image.resize_images(BILINEAR, align_corners=True) in
 * HDRNetGaussianPyrNN._multiscale_input / ._output (hdrnet/models.py:249-289).
 */
HDRNET_API int hdrnet_resize_bilinear_f32(const float* in, const float* add, float* out, int B,
                                          int H, int W, int C, int OH, int OW, void* stream);

/*
 * VJP of hdrnet_resize_bilinear_f32 (the fused add's VJP is the identity): din [B, H, W, C], the
 * input-shaped gradient, from dout [B, OH, OW, C].  Each din element gathers the output pixels
 * whose taps (the forward's own float32 lo / hi / frac) reach it, weighted (1-fy)(1-fx),
 * (1-fy)fx, fy(1-fx) and fy fx, in a fixed order: no atomics, bitwise reproducible.  Every din
 * element is written.  Same argument checks and return codes as the forward.
 */
HDRNET_API int hdrnet_resize_bilinear_grad_f32(const float* dout, float* din, int B, int H, int W,
                                               int C, int OH, int OW, void* stream);

/* The model-path forms with a lent workspace (B*H*gw*gd*48 bytes, as for
 * hdrnet_slice_apply_f32_ws): large images then run the texture-assisted kernel. */
HDRNET_API int hdrnet_slice_apply_curves_f32_ws(const float* grid, const float* input, float* out,
                                                float* guide_out, int B, int H, int W, int gh,
                                                int gw, int gd, const float* ccm,
                                                const float* ccm_bias, const float* shifts,
                                                const float* slopes, const float* mix,
                                                float mix_bias, void* workspace,
                                                size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_slice_apply_nn_f32_ws(const float* grid, const float* input, float* out,
                                            float* guide_out, int B, int H, int W, int gh, int gw,
                                            int gd, const float* w1, const float* b1,
                                            const float* w2, float b2, int feats, void* workspace,
                                            size_t workspace_bytes, void* stream);

/*
 * Pixel storage formats of the model-path forms below (SURVEY.md section 8 row f-3).  The
 * reference's CLI decodes an image to uint8 / uint16, converts it on the host with
 * skimage.img_as_float (v / 255, v / 65535; hdrnet/bin/run.py:156-164), feeds float32 to the
 * graph and casts the prediction with tf.cast(255 * clip(x, 0, 1), tf.uint8) (run.py:95).  These
 * entry points keep the full-resolution image in its integer format on both sides: 3 + 3 bytes
 * per pixel cross PCIe and HBM instead of 12 + 12.
 */
#define HDRNET_PX_F32 0 /* float32 [B,H,W,3]                                              */
#define HDRNET_PX_U8 1  /* uint8   [B,H,W,3]; as input: img_as_float; as output: the cast  */
#define HDRNET_PX_U16 2 /* uint16  [B,H,W,3]; as input: img_as_float; as output: rint(65535 * clip) */

/*
 * hdrnet_slice_apply_{curves,nn}_f32_ws with `input` in in_fmt and `out` in out_fmt
 * (HDRNET_PX_F32, HDRNET_PX_U8 or HDRNET_PX_U16).  The conversion of a code value is bit-exact with
 * float32(float64(v) / 255) (resp. 65535); the uint8 cast truncates like tf.cast; the uint16 result
 * is rint(65535 * clip(x, 0, 1)), rounded to nearest even, so an identity model returns every
 * uint16 code unchanged; NaN gives 0 in both.  (u8 | u16) -> (u8 | u16) with W % 16 == 0 (W % 8
 * when both sides are u16) and 16-byte aligned buffers runs the persistent row kernel; every other
 * combination runs a one-thread-per-pixel fused kernel.  A uint16 `out` must not overlap `input`
 * or `grid` (HDRNET_E_UNSUPPORTED).  guide_out (optional) receives the float32 guide map.
 * f32 -> f32 is hdrnet_slice_apply_{curves,nn}_f32_ws itself.
 */
HDRNET_API int hdrnet_slice_apply_curves_px_ws(const float* grid, const void* input, int in_fmt,
                                               void* out, int out_fmt, float* guide_out, int B,
                                               int H, int W, int gh, int gw, int gd,
                                               const float* ccm, const float* ccm_bias,
                                               const float* shifts, const float* slopes,
                                               const float* mix, float mix_bias, void* workspace,
                                               size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_slice_apply_nn_px_ws(const float* grid, const void* input, int in_fmt,
                                           void* out, int out_fmt, float* guide_out, int B, int H,
                                           int W, int gh, int gw, int gd, const float* w1,
                                           const float* b1, const float* w2, float b2, int feats,
                                           void* workspace, size_t workspace_bytes, void* stream);

/*
 * Low-resolution network input straight from the decoded image: nearest-neighbour resize of
 * image [B,H,W,3] (fmt) to lowres [B,SH,SW,3] float32, img_as_float applied on the fly.
 * Replaces skimage.transform.resize(im, [S, S], order=0) on the float image (run.py:168-169):
 * output sample i reads input floor((i + 0.5) * H / SH).
 */
HDRNET_API int hdrnet_lowres_nearest_f32(const void* image, int fmt, float* lowres, int B, int H,
                                         int W, int SH, int SW, void* stream);

/*
 * One training batch from decoded image pairs resident on the device: the augmentation of the
 * reference's ImageFilesDataPipeline (hdrnet/data_pipeline.py:126-171) as one gather per output
 * pixel, no workspace.  Per sample, in this order: flip left-right, flip up-down, rot90(k)
 * counter-clockwise (equal to np.rot90(m, k)), then the oh x ow crop at (crop_y, crop_x) of the
 * ROTATED extent ([W, H] for odd k).  Writes
 *   fullres_in, fullres_out [B, oh, ow, 3] float32   the crop of input / target
 *   lowres_in               [B, S, S, 3]   float32   TF1 resize_images(NEAREST_NEIGHBOR) of the
 *                                                    input crop: src = min(floor(dst * (float)oh / S),
 *                                                    oh - 1) (same for x), no half-pixel offset
 * Integer pixels are converted as tf.to_float(v) / 255 (resp. 65535) in IEEE float32, the same
 * bits as the model path's conversion.  The batch is ragged: each sample has its own source extent
 * and each image its own format.  `samples` is a HOST array of B descriptors, read before the call
 * returns; the image pointers in it are device pointers.  Errors: HDRNET_E_NULL_POINTER for a NULL
 * output, descriptor array or image; HDRNET_E_BAD_SHAPE for B < 0, oh / ow / S < 1, H or W <= 0,
 * k outside 0..3 or a crop outside the rotated source; HDRNET_E_UNSUPPORTED for an unknown format.
 */
typedef struct hdrnet_train_sample {
  const void* input;    /* [H, W, 3] in input_fmt (HDRNET_PX_*), device memory  */
  const void* target;   /* [H, W, 3] in target_fmt, the same extent              */
  int input_fmt, target_fmt;
  int H, W;             /* source extent                                          */
  int fliplr, flipud;   /* nonzero: flip                                          */
  int rot90;            /* k in 0..3                                              */
  int crop_y, crop_x;   /* crop origin on the rotated extent                      */
} hdrnet_train_sample;

HDRNET_API int hdrnet_train_batch_f32(const hdrnet_train_sample* samples, int B, float* fullres_in,
                                      float* fullres_out, float* lowres_in, int oh, int ow, int S,
                                      void* stream);

/*
 * One training batch of UnsharpMaskDataPipeline: the target is computed from the input.  The
 * reference's usm/ scripts name this pipeline but its sources do not define it; this is the
 * project's definition.  With x the float32 input pixel (converted as hdrnet_train_batch_f32 does)
 *   b = G_sigma * x   per channel: the separable Gaussian of scipy.ndimage.gaussian_filter1d
 *                     (truncate 4.0: radius r = int(4 sigma + 0.5), weights exp(-k^2 / 2 sigma^2)
 *                     normalised to sum 1) along source x, then source y, with half-sample
 *                     symmetric reflection (d c b a | a b c d, repeated) at the SOURCE's edges
 *   fullres_out = clip(x + sharpen (x - b), 0, 1)
 * computed in source coordinates: a source pixel's target does not depend on the draw, and the
 * flips, rot90 and crop (hdrnet_train_batch_f32's) only move pixels.  fullres_in and lowres_in are
 * hdrnet_train_batch_f32's, bit for bit; either may be NULL (not written; S is then ignored).
 *
 * A sample's buffer holds a window of its source: rows [y0, y0 + h), columns [x0, x0 + w) of the
 * full H x W source, row pitch w pixels.  It must cover the crop's source rectangle grown by r on
 * each side and clipped to [0, H) x [0, W) (the whole source always does).  The flips, rot90 and
 * crop origin are given on the full source's rotated extent.  Sums run in float64 in a fixed tap
 * order, no atomics: bitwise the same from run to run.  0 < sigma <= 32 (so r <= 128); sharpen
 * finite.  The workspace (4-byte aligned) holds float32 rows of the horizontal pass; its size is
 * hdrnet_train_batch_usm_workspace_bytes (0 for B = 0 or arguments the call refuses).  `samples`
 * is a HOST array read before the call returns.  Errors, all before any launch:
 * HDRNET_E_NULL_POINTER for a NULL descriptor array, input, fullres_out or workspace;
 * HDRNET_E_BAD_SHAPE for B < 0, oh / ow < 1, S < 1 with lowres_in, a bad sigma or sharpen, H or
 * W <= 0, k outside 0..3, a crop outside the rotated source, a window outside the source or not
 * covering the grown crop rectangle, or a short or misaligned workspace; HDRNET_E_UNSUPPORTED for
 * an unknown format; HDRNET_E_TOO_LARGE for grids past the launch limits.  B = 0 succeeds.
 */
typedef struct hdrnet_usm_sample {
  const void* input;    /* the window [h, w, 3] in input_fmt (HDRNET_PX_*), device memory */
  int input_fmt;
  int H, W;             /* the full source's extent                                      */
  int y0, x0, h, w;     /* the window the buffer holds, in source pixels                 */
  int fliplr, flipud;   /* nonzero: flip                                                 */
  int rot90;            /* k in 0..3                                                     */
  int crop_y, crop_x;   /* crop origin on the full source's rotated extent               */
} hdrnet_usm_sample;

HDRNET_API size_t hdrnet_train_batch_usm_workspace_bytes(const hdrnet_usm_sample* samples, int B, int oh,
                                                          int ow, double sigma);
HDRNET_API int hdrnet_train_batch_usm_f32(const hdrnet_usm_sample* samples, int B, float* fullres_in,
                                          float* fullres_out, float* lowres_in, int oh, int ow, int S,
                                          double sigma, double sharpen, void* workspace,
                                          size_t workspace_bytes, void* stream);

/*
 * Host-buffer path (what a CPU-tensor caller of the reference op gets: TF copies feeds to
 * the GPU and fetches back, hdrnet/bin/run.py:185).  A context owns device staging buffers
 * and streams; the call splits the batch into row bands, and pipelines H2D copy -> kernel
 * -> D2H copy across streams.  Host buffers should be page-locked for the copies to
 * overlap (pageable memory works but serialises).  Blocks until `out` is complete.
 */
typedef struct hdrnet_host_ctx hdrnet_host_ctx;

/* max_band_pixels: staging capacity per pipeline slot, in pixels (0 = default 4 Mi px). */
HDRNET_API int hdrnet_host_ctx_create(hdrnet_host_ctx** ctx, size_t max_band_pixels);
HDRNET_API int hdrnet_host_ctx_destroy(hdrnet_host_ctx* ctx);

HDRNET_API int hdrnet_slice_apply_host_f32(hdrnet_host_ctx* ctx, const float* grid, const float* guide,
                                const float* input, float* out, int B, int H, int W, int gh,
                                int gw, int gd, int n_in, int n_out, int has_offset);

/*
 * A whole trained model (HDRNetCurves, HDRNetPointwiseNNGuide, HDRNetGaussianPyrNN or
 * HDRNetGaussianPyr) from its frozen model file (hdrnet_b200.checkpoint.freeze_model; the layout is
 * documented in csrc/model.cu and DESIGN.md row f-12): the C counterpart of models.*.inference_image,
 * running the same kernels chosen by the same rules, so its results are bit for bit that path's --
 * except the pyramids from uint8 / uint16 pixels, whose full-resolution image is converted with the
 * bit-exact img_as_float here where models.image_to_float divides through torch (DESIGN.md row f-11):
 * there the results are bit for bit the pyramid's inference on the host's img_as_float, quantised as
 * inference_image quantises.
 *
 * hdrnet_model_create: checks the whole host blob (magic, format version, lengths, every array's
 *   shape against the hyperparameters, CRC-32C) before any CUDA call -- HDRNET_E_BAD_MODEL for any
 *   fault -- then uploads the weights to the CURRENT device and packs the tensor-core conv weights
 *   once.  The only call that allocates device memory (and it synchronises).  The blob may be freed
 *   after the call.
 * hdrnet_model_destroy: frees the object (after work still reading its weights); any later use of
 *   the handle returns HDRNET_E_BAD_CONTEXT.
 * hdrnet_model_info: the model kind (HDRNET_MODEL_*) and hyperparameters; NULL outputs are skipped.
 * hdrnet_model_workspace_bytes: the workspace hdrnet_model_run_px needs for B images of H x W in
 *   in_fmt -> out_fmt (any base address; 0 for a bad handle or format).
 * hdrnet_model_run_px: image [B,H,W,3] in in_fmt -> out [B,H,W,3] in out_fmt (HDRNET_PX_*, device
 *   pointers): the network input is lowres_image [B,SH,SW,3] in lowres_fmt when not NULL, else the
 *   image itself, resized nearest-neighbour to net_input_size (hdrnet_lowres_nearest_f32).  Every
 *   intermediate lives in the lent workspace, which is scratch (undefined after the call, never read
 *   before being written).  The call allocates no memory, never synchronises and launches only on
 *   `stream`, so it can be captured in a CUDA graph; calls on different streams with different
 *   workspaces may run concurrently.  The texture-assisted forms (from 2 Mi pixels per call) fetch the
 *   slab through a texture object over the workspace: outside a capture the library creates it on a
 *   workspace's first use and caches it; under a capture the call creates one that the graph owns and
 *   that is destroyed only after the graph and its executable graphs are gone, so a graph replays
 *   correctly however many other workspaces are lent meanwhile.  Errors, all before any launch:
 *   HDRNET_E_BAD_CONTEXT for a
 *   destroyed handle or a current device other than the one the model was created on;
 *   HDRNET_E_BAD_SHAPE for a workspace smaller than hdrnet_model_workspace_bytes, negative extents,
 *   or a pyramid image under 4 x 4; HDRNET_E_UNSUPPORTED for an unknown format or a uint16 `out`
 *   overlapping `image`.  B * H * W == 0 succeeds without launching.
 */
#define HDRNET_MODEL_CURVES 0
#define HDRNET_MODEL_POINTWISE_NN 1
#define HDRNET_MODEL_GAUSSIAN_PYR_NN 2
#define HDRNET_MODEL_GAUSSIAN_PYR 3     /* the pyramid with a curves guide per level */

typedef struct hdrnet_model hdrnet_model;

HDRNET_API int hdrnet_model_create(const void* blob, size_t bytes, hdrnet_model** model);
HDRNET_API int hdrnet_model_destroy(hdrnet_model* model);
HDRNET_API int hdrnet_model_info(const hdrnet_model* model, int* kind, int* net_input_size,
                                 int* spatial_bin, int* luma_bins, int* channel_multiplier,
                                 int* guide_width);
HDRNET_API size_t hdrnet_model_workspace_bytes(const hdrnet_model* model, int B, int H, int W,
                                               int in_fmt, int out_fmt);
HDRNET_API int hdrnet_model_run_px(const hdrnet_model* model, const void* image, int in_fmt,
                                   const void* lowres_image, int lowres_fmt, int SH, int SW,
                                   void* out, int out_fmt, int B, int H, int W, void* workspace,
                                   size_t workspace_bytes, void* stream);

/*
 * Ragged batches: B images of different sizes in one call (a photo collection: 4032 x 3024 next to
 * 3024 x 4032 next to a 1080p frame).  `images` is a HOST array of B descriptors of device buffers
 * [H, W, 3]; the library reads it before the call returns and passes it to the kernels in their
 * parameter blocks, so a CUDA graph that captures the call keeps its own copy and a replay never
 * reads host memory.  One kernel launch takes at most HDRNET_RAGGED_MAX_IMAGES images; a longer
 * call is split into launches of that many inside the library.  The pixel format is one per call.
 * Errors, all before any launch: HDRNET_E_NULL_POINTER for a NULL descriptor array (B > 0), image,
 * output or grid; HDRNET_E_BAD_SHAPE for B < 0, H or W <= 0, gh / gw / gd < 1 or a short
 * workspace; HDRNET_E_UNSUPPORTED for an unknown format or a uint16 output overlapping any input
 * (or the grid).  B == 0 succeeds without launching.
 *
 * hdrnet_lowres_nearest_ragged_f32: hdrnet_lowres_nearest_f32 per image (out unused) into one
 *   lowres [B, SH, SW, 3]: image i's rows are bit for bit that call on image i alone.
 * hdrnet_slice_apply_{curves,nn}_ragged_px_ws: hdrnet_slice_apply_{curves,nn}_px_ws per image, in
 *   one launch: image i reads grid row i of grid [B, gh, gw, gd, 12] and has its own cell scales
 *   (gw / W_i, gh / H_i); the launch's rows are handed out across the GPU as one range, so a small
 *   image does not leave SMs idle behind a large one.  Each image runs the per-pixel arithmetic of
 *   the form the single-image call takes for it (the row kernels' 4-corner blend of the slab, or the
 *   per-pixel kernel's 8-corner gather), so its result is bit for bit that call's -- except a
 *   float32 -> float32 image the row kernels do not take at W >= 64, where the single-image call runs
 *   the guide kernel and then the any-shape row kernel, whose apply sums in another order (equal to
 *   within float32 rounding; DESIGN.md row f-13).  No guide map is written.
 * hdrnet_slice_apply_ragged_workspace_bytes: the workspace those calls need: 0 (the slab rows stay
 *   in shared memory; no texture objects); the workspace arguments are accepted and unused.
 * hdrnet_model_workspace_bytes_ragged / hdrnet_model_run_ragged_px: hdrnet_model_run_px for a
 *   ragged batch (each descriptor's `out` receives that image's result).  `lowres` is NULL or B
 *   descriptors of network-input images (their `out` unused) in lowres_fmt.  The coefficient network
 *   runs once on the whole batch; curves and pointwise-NN models then run one ragged lowres launch
 *   and one ragged slice-apply launch per HDRNET_RAGGED_MAX_IMAGES images; the pyramid runs its
 *   full-resolution stages image by image on the kernels of hdrnet_model_run_px.  Same rules as
 *   hdrnet_model_run_px: no allocation, no synchronisation, capturable, every error before any
 *   launch (HDRNET_E_BAD_SHAPE also for a pyramid image under 4 x 4).
 */
#define HDRNET_RAGGED_MAX_IMAGES 256

typedef struct hdrnet_image_desc {
  const void* image;   /* [H, W, 3] input pixels, device memory */
  void* out;           /* [H, W, 3] result, device memory       */
  int H, W;
} hdrnet_image_desc;

HDRNET_API int hdrnet_lowres_nearest_ragged_f32(const hdrnet_image_desc* images, int B, int fmt,
                                                float* lowres, int SH, int SW, void* stream);
HDRNET_API size_t hdrnet_slice_apply_ragged_workspace_bytes(const hdrnet_image_desc* images, int B,
                                                            int gh, int gw, int gd);
HDRNET_API int hdrnet_slice_apply_curves_ragged_px_ws(const float* grid,
                                                      const hdrnet_image_desc* images, int B,
                                                      int in_fmt, int out_fmt, int gh, int gw,
                                                      int gd, const float* ccm,
                                                      const float* ccm_bias, const float* shifts,
                                                      const float* slopes, const float* mix,
                                                      float mix_bias, void* workspace,
                                                      size_t workspace_bytes, void* stream);
HDRNET_API int hdrnet_slice_apply_nn_ragged_px_ws(const float* grid, const hdrnet_image_desc* images,
                                                  int B, int in_fmt, int out_fmt, int gh, int gw,
                                                  int gd, const float* w1, const float* b1,
                                                  const float* w2, float b2, int feats,
                                                  void* workspace, size_t workspace_bytes,
                                                  void* stream);
HDRNET_API size_t hdrnet_model_workspace_bytes_ragged(const hdrnet_model* model,
                                                      const hdrnet_image_desc* images, int B,
                                                      int in_fmt, int out_fmt);
HDRNET_API int hdrnet_model_run_ragged_px(const hdrnet_model* model,
                                          const hdrnet_image_desc* images, int B, int in_fmt,
                                          int out_fmt, const hdrnet_image_desc* lowres,
                                          int lowres_fmt, void* workspace, size_t workspace_bytes,
                                          void* stream);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* HDRNET_B200_H_ */
