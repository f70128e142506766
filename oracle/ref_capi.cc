// ref_capi.cc -- C entry points around the REFERENCE's own CPU loops.
//
// TEST INFRASTRUCTURE ONLY (oracle/).  oracle/Makefile compiles this file together with
// the reference checkout's hdrnet/ops/bilateral_slice.cc and bilateral_slice_apply.cc -- taken where
// they lie, UNMODIFIED, never copied into this repo -- against oracle/nda_standin (a
// stand-in for the un-vendored nda header) into oracle/_ref/libhdrnet_ref.so.
//
// The wrappers below reinterpret TF-layout (row-major NHWC) buffers as column-major nda
// refs exactly the way the reference's OpKernels do:
//   slice-apply : hdrnet/ops/bilateral_slice_apply_op.cc:201-227
//   slice       : hdrnet/ops/bilateral_slice_op.cc:151-169
// The reference loops are single-threaded (nda::for_all_indices); the only parallelism
// added here is over the batch index (each image is an independent call on a B=1 view),
// which cannot change any result.
#include <cstddef>

#include "bilateral_slice.h"
#include "bilateral_slice_apply.h"

#ifdef _OPENMP
#include <omp.h>
#endif

#define HDRNET_REF_API extern "C" __attribute__((visibility("default")))

namespace {

template <size_t N>
using shape = nda::shape_of_rank<N>;

}  // namespace

HDRNET_REF_API int hdrnet_ref_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

HDRNET_REF_API void hdrnet_ref_slice(const float* grid, const float* guide, float* out, int B,
                                     int H, int W, int gh, int gw, int gd, int gc) {
  const size_t grid_b = (size_t)gh * gw * gd * gc;
  const size_t px_b = (size_t)H * W;
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < B; ++b) {
    auto grid_ref = nda::make_array_ref(grid + b * grid_b, shape<5>(gc, gd, gw, gh, 1));
    auto guide_ref = nda::make_array_ref(guide + b * px_b, shape<3>(W, H, 1));
    auto out_ref = nda::make_array_ref(out + b * px_b * gc, shape<4>(gc, W, H, 1));
    hdrnet::BilateralSlice(grid_ref, guide_ref, out_ref);
  }
}

HDRNET_REF_API void hdrnet_ref_slice_apply(const float* grid, const float* guide,
                                           const float* input, float* out, int B, int H, int W,
                                           int gh, int gw, int gd, int n_in, int n_out,
                                           int has_offset) {
  const int J = n_in + (has_offset ? 1 : 0);
  const size_t grid_b = (size_t)gh * gw * gd * n_out * J;
  const size_t px_b = (size_t)H * W;
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < B; ++b) {
    auto grid_ref = nda::make_array_ref(grid + b * grid_b, shape<6>(J, n_out, gd, gw, gh, 1));
    auto guide_ref = nda::make_array_ref(guide + b * px_b, shape<3>(W, H, 1));
    auto in_ref = nda::make_array_ref(input + b * px_b * n_in, shape<4>(n_in, W, H, 1));
    auto out_ref = nda::make_array_ref(out + b * px_b * n_out, shape<4>(n_out, W, H, 1));
    hdrnet::BilateralSliceApply(grid_ref, guide_ref, in_ref, out_ref);
  }
}

// VJPs (bilateral_slice_apply_op.cc:249-362, bilateral_slice_op.cc:183-256).
HDRNET_REF_API void hdrnet_ref_slice_apply_grad(const float* grid, const float* guide,
                                                const float* input, const float* ct,
                                                float* grid_vjp, float* guide_vjp,
                                                float* input_vjp, int B, int H, int W, int gh,
                                                int gw, int gd, int n_in, int n_out,
                                                int has_offset) {
  const int J = n_in + (has_offset ? 1 : 0);
  const size_t grid_b = (size_t)gh * gw * gd * n_out * J;
  const size_t px_b = (size_t)H * W;
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < B; ++b) {
    nda::array_ref_of_rank<const float, 6> grid_ref(grid + b * grid_b,
                                                    shape<6>(J, n_out, gd, gw, gh, 1));
    nda::array_ref_of_rank<const float, 3> guide_ref(guide + b * px_b, shape<3>(W, H, 1));
    nda::array_ref_of_rank<const float, 4> in_ref(input + b * px_b * n_in,
                                                  shape<4>(n_in, W, H, 1));
    nda::array_ref_of_rank<const float, 4> ct_ref(ct + b * px_b * n_out,
                                                  shape<4>(n_out, W, H, 1));
    nda::array_ref_of_rank<float, 6> gv(grid_vjp + b * grid_b, shape<6>(J, n_out, gd, gw, gh, 1));
    nda::array_ref_of_rank<float, 3> uv(guide_vjp + b * px_b, shape<3>(W, H, 1));
    nda::array_ref_of_rank<float, 4> iv(input_vjp + b * px_b * n_in, shape<4>(n_in, W, H, 1));
    hdrnet::BilateralSliceApplyGridGrad(guide_ref, in_ref, ct_ref, gv);
    hdrnet::BilateralSliceApplyGuideGrad(grid_ref, guide_ref, in_ref, ct_ref, uv);
    hdrnet::BilateralSliceApplyInputGrad(grid_ref, guide_ref, ct_ref, iv);
  }
}

HDRNET_REF_API void hdrnet_ref_slice_grad(const float* grid, const float* guide, const float* ct,
                                          float* grid_vjp, float* guide_vjp, int B, int H, int W,
                                          int gh, int gw, int gd, int gc) {
  const size_t grid_b = (size_t)gh * gw * gd * gc;
  const size_t px_b = (size_t)H * W;
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < B; ++b) {
    nda::array_ref_of_rank<const float, 5> grid_ref(grid + b * grid_b,
                                                    shape<5>(gc, gd, gw, gh, 1));
    nda::array_ref_of_rank<const float, 3> guide_ref(guide + b * px_b, shape<3>(W, H, 1));
    nda::array_ref_of_rank<const float, 4> ct_ref(ct + b * px_b * gc, shape<4>(gc, W, H, 1));
    nda::array_ref_of_rank<float, 5> gv(grid_vjp + b * grid_b, shape<5>(gc, gd, gw, gh, 1));
    nda::array_ref_of_rank<float, 3> uv(guide_vjp + b * px_b, shape<3>(W, H, 1));
    hdrnet::BilateralSliceGridGrad(guide_ref, ct_ref, gv);
    hdrnet::BilateralSliceGuideGrad(grid_ref, guide_ref, ct_ref, uv);
  }
}
