"""ctypes binding of libhdrnet_b200.so (the C-ABI declared in include/hdrnet_b200.h).

The library is built in-tree (``hdrnet_b200/lib/``) by ``hdrnet_b200/csrc/Makefile`` for
sm_90a.  There is NO fallback: if the library is missing or an op is called without a CUDA
device, the call raises -- a silent CPU path would void every parity claim.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libhdrnet_b200.so")
CSRC_DIR = os.path.join(_HERE, "csrc")
HEADER_PATH = os.path.normpath(os.path.join(_HERE, "..", "include", "hdrnet_b200.h"))

# Return codes (include/hdrnet_b200.h)
OK = 0
E_NULL_POINTER, E_BAD_SHAPE, E_BAD_CHANNELS, E_TOO_LARGE, E_UNSUPPORTED, E_BAD_CONTEXT, E_BAD_MODEL = (
    -1, -2, -3, -4, -5, -6, -7)
VARIANT_AUTO, VARIANT_GENERIC, VARIANT_TMA, VARIANT_TEX, VARIANT_TEX_ASYNC = 0, 1, 2, 4, 7

_c_int = ctypes.c_int
_vp = ctypes.c_void_p

# name -> (restype, argtypes); must list every function the header declares
# (tests/test_boundary.py cross-checks this table against the header and the .so).
SIGNATURES = {
    "hdrnet_b200_abi_version": (_c_int, []),
    "hdrnet_b200_error_string": (ctypes.c_char_p, [_c_int]),
    "hdrnet_slice_apply_f32": (_c_int, [_vp] * 4 + [_c_int] * 9 + [_vp]),
    "hdrnet_slice_apply_f32_variant": (_c_int, [_vp] * 4 + [_c_int] * 10 + [_vp]),
    "hdrnet_slice_apply_workspace_bytes": (ctypes.c_size_t, [_c_int] * 4),
    "hdrnet_slice_apply_f32_ws": (_c_int, [_vp] * 4 + [_c_int] * 10 + [_vp, ctypes.c_size_t, _vp]),
    # (grid, guide, input, out, B,H,W, rows,y_off, gh,gw,gd, n_in,n_out,has_offset, variant, ws, bytes, stream)
    "hdrnet_slice_apply_rows_f32_ws": (_c_int, [_vp] * 4 + [_c_int] * 12 + [_vp, ctypes.c_size_t, _vp]),
    "hdrnet_slice_f32": (_c_int, [_vp] * 3 + [_c_int] * 7 + [_vp]),
    "hdrnet_slice_f32_variant": (_c_int, [_vp] * 3 + [_c_int] * 8 + [_vp]),
    "hdrnet_slice_apply_grad_f32": (_c_int, [_vp] * 7 + [_c_int] * 9 + [_vp]),
    "hdrnet_slice_grad_f32": (_c_int, [_vp] * 5 + [_c_int] * 7 + [_vp]),
    "hdrnet_slice_indices_i32": (_c_int, [_vp] * 2 + [_c_int] * 6 + [_vp]),
    "hdrnet_slice_apply_plan": (_c_int, [_c_int] * 9 + [ctypes.POINTER(_c_int)] * 4),
    "hdrnet_slice_apply_plan_ws": (_c_int, [_c_int] * 10 + [ctypes.POINTER(_c_int)] * 4),
    "hdrnet_guide_curves_f32": (_c_int, [_vp, _vp, ctypes.c_longlong] + [_vp] * 5 + [ctypes.c_float, _vp]),
    "hdrnet_guide_nn_f32": (_c_int, [_vp, _vp, ctypes.c_longlong] + [_vp] * 3 + [ctypes.c_float, _c_int, _vp]),
    # (input, dguide, dinput, npix, ccm, ccm_bias, shifts, slopes, mix, mix_bias, dparams, ws, bytes, stream)
    "hdrnet_guide_curves_grad_workspace_bytes": (ctypes.c_size_t, [ctypes.c_longlong]),
    "hdrnet_guide_curves_grad_f32": (_c_int, [_vp] * 3 + [ctypes.c_longlong] + [_vp] * 5
                                     + [ctypes.c_float, _vp, _vp, ctypes.c_size_t, _vp]),
    # (input, npix, moments, ws, bytes, stream); (w1, beta, moments, feats, w1_folded, b1_folded, mean, var)
    "hdrnet_guide_nn_stats_workspace_bytes": (ctypes.c_size_t, [ctypes.c_longlong]),
    "hdrnet_guide_nn_stats_f32": (_c_int, [_vp, ctypes.c_longlong, _vp, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_guide_nn_batch_fold": (_c_int, [_vp] * 3 + [_c_int] + [_vp] * 4),
    # (input, dguide, dinput, npix, w1, beta, w2, b2, feats, moments, dparams, ws, bytes, stream)
    "hdrnet_guide_nn_grad_workspace_bytes": (ctypes.c_size_t, [ctypes.c_longlong, _c_int]),
    "hdrnet_guide_nn_grad_f32": (_c_int, [_vp] * 3 + [ctypes.c_longlong] + [_vp] * 3
                                 + [ctypes.c_float, _c_int, _vp, _vp, _vp, ctypes.c_size_t, _vp]),
    # coefficient-network batch norm in training mode: (z, N, C, moments, ws, bytes, stream);
    # (z, N, C, moments, beta, y, moving_mean, moving_var, stream);
    # (z, dy, N, C, moments, beta, sums, dbeta, ws, bytes, stream); (z, dy, N, C, moments, beta, sums, dz, stream)
    "hdrnet_bn_stats_workspace_bytes": (ctypes.c_size_t, [ctypes.c_longlong, _c_int]),
    "hdrnet_bn_stats_f32": (_c_int, [_vp, ctypes.c_longlong, _c_int, _vp, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_bn_relu_f32": (_c_int, [_vp, ctypes.c_longlong, _c_int] + [_vp] * 6),
    "hdrnet_bn_relu_grad_sums_f32": (_c_int, [_vp, _vp, ctypes.c_longlong, _c_int] + [_vp] * 5
                                     + [ctypes.c_size_t, _vp]),
    "hdrnet_bn_relu_grad_f32": (_c_int, [_vp, _vp, ctypes.c_longlong, _c_int] + [_vp] * 5),
    "hdrnet_slice_apply_curves_f32": (_c_int, [_vp] * 4 + [_c_int] * 6 + [_vp] * 5 + [ctypes.c_float, _vp]),
    "hdrnet_slice_apply_nn_f32": (_c_int, [_vp] * 4 + [_c_int] * 6 + [_vp] * 3 + [ctypes.c_float, _c_int, _vp]),
    "hdrnet_slice_apply_curves_f32_ws": (_c_int, [_vp] * 4 + [_c_int] * 6 + [_vp] * 5
                                         + [ctypes.c_float, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_slice_apply_nn_f32_ws": (_c_int, [_vp] * 4 + [_c_int] * 6 + [_vp] * 3
                                     + [ctypes.c_float, _c_int, _vp, ctypes.c_size_t, _vp]),
    # (grid, input, in_fmt, out, out_fmt, guide_out, B,H,W,gh,gw,gd, guide params..., ws, bytes, stream)
    "hdrnet_slice_apply_curves_px_ws": (_c_int, [_vp, _vp, _c_int, _vp, _c_int, _vp] + [_c_int] * 6
                                        + [_vp] * 5 + [ctypes.c_float, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_slice_apply_nn_px_ws": (_c_int, [_vp, _vp, _c_int, _vp, _c_int, _vp] + [_c_int] * 6
                                    + [_vp] * 3 + [ctypes.c_float, _c_int, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_lowres_nearest_f32": (_c_int, [_vp, _c_int, _vp] + [_c_int] * 5 + [_vp]),
    "hdrnet_conv2d_nhwc_f32": (_c_int, [_vp] * 4 + [_c_int] * 8 + [_vp]),
    "hdrnet_conv2d_nhwc_fp32_f32": (_c_int, [_vp] * 4 + [_c_int] * 8 + [_vp]),
    "hdrnet_conv2d_tc_packed_bytes": (ctypes.c_size_t, [_c_int] * 3),
    "hdrnet_conv2d_tc_pack_f32": (_c_int, [_vp, _vp] + [_c_int] * 3 + [_vp]),
    "hdrnet_conv2d_nhwc_tc_f32": (_c_int, [_vp] * 4 + [_c_int] * 8 + [_vp]),
    "hdrnet_fc_f32": (_c_int, [_vp] * 4 + [_c_int] * 4 + [_vp]),
    "hdrnet_fuse_predict_f32": (_c_int, [_vp] * 5 + [_c_int] * 7 + [_vp]),
    # (in, w, out, dout, din, dw, db, B,H,W,Cin,Cout,k,stride,relu, ws, bytes, stream)
    "hdrnet_conv2d_grad_workspace_bytes": (ctypes.c_size_t, [_c_int] * 7),
    "hdrnet_conv2d_grad_f32": (_c_int, [_vp] * 7 + [_c_int] * 8 + [_vp, ctypes.c_size_t, _vp]),
    "hdrnet_fc_grad_workspace_bytes": (ctypes.c_size_t, [_c_int] * 3),
    "hdrnet_fc_grad_f32": (_c_int, [_vp] * 7 + [_c_int] * 4 + [_vp, ctypes.c_size_t, _vp]),
    # (local, global, w, dgrid, dlocal, dglobal, dw, db, B,gh,gw,C,gd,n_out,n_in, ws, bytes, stream)
    "hdrnet_fuse_predict_grad_workspace_bytes": (ctypes.c_size_t, [_c_int] * 7),
    "hdrnet_fuse_predict_grad_f32": (_c_int, [_vp] * 8 + [_c_int] * 7 + [_vp, ctypes.c_size_t, _vp]),
    "hdrnet_resize_bilinear_f32":(_c_int, [_vp] * 3 + [_c_int] * 6 + [_vp]),
    # (dout, din, B, H, W, C, OH, OW, stream)
    "hdrnet_resize_bilinear_grad_f32": (_c_int, [_vp] * 2 + [_c_int] * 6 + [_vp]),
    "hdrnet_coefficients_scratch_bytes": (ctypes.c_size_t, [_c_int] * 7),
    "hdrnet_coefficients_f32": (_c_int, [_vp] * 4 + [_c_int, _vp, ctypes.c_size_t] + [_c_int] * 7 + [_vp]),
    # (samples, B, fullres_in, fullres_out, lowres_in, oh, ow, S, stream)
    "hdrnet_train_batch_f32": (_c_int, [_vp, _c_int] + [_vp] * 3 + [_c_int] * 3 + [_vp]),
    # (samples, B, oh, ow, sigma); (samples, B, fullres_in, fullres_out, lowres_in, oh, ow, S, sigma,
    # sharpen, ws, bytes, stream)
    "hdrnet_train_batch_usm_workspace_bytes": (ctypes.c_size_t, [_vp] + [_c_int] * 3 + [ctypes.c_double]),
    "hdrnet_train_batch_usm_f32": (_c_int, [_vp, _c_int] + [_vp] * 3 + [_c_int] * 3
                                   + [ctypes.c_double] * 2 + [_vp, ctypes.c_size_t, _vp]),
    "hdrnet_host_ctx_create": (_c_int, [ctypes.POINTER(_vp), ctypes.c_size_t]),
    "hdrnet_host_ctx_destroy": (_c_int, [_vp]),
    "hdrnet_slice_apply_host_f32": (_c_int, [_vp] * 5 + [_c_int] * 9),
    # the whole-model object (frozen model file -> hdrnet_model*)
    "hdrnet_model_create": (_c_int, [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(_vp)]),
    "hdrnet_model_destroy": (_c_int, [_vp]),
    "hdrnet_model_info": (_c_int, [_vp] + [ctypes.POINTER(_c_int)] * 6),
    "hdrnet_model_workspace_bytes": (ctypes.c_size_t, [_vp] + [_c_int] * 5),
    # (model, image, in_fmt, lowres, lowres_fmt, SH, SW, out, out_fmt, B, H, W, ws, bytes, stream)
    "hdrnet_model_run_px": (_c_int, [_vp, _vp, _c_int, _vp] + [_c_int] * 3 + [_vp] + [_c_int] * 4
                            + [_vp, ctypes.c_size_t, _vp]),
    # ragged batches: (descs, B, fmt, lowres, SH, SW, stream); (descs, B, gh, gw, gd)
    "hdrnet_lowres_nearest_ragged_f32": (_c_int, [_vp, _c_int, _c_int, _vp, _c_int, _c_int, _vp]),
    "hdrnet_slice_apply_ragged_workspace_bytes": (ctypes.c_size_t, [_vp] + [_c_int] * 4),
    # (grid, descs, B, in_fmt, out_fmt, gh, gw, gd, guide params..., ws, bytes, stream)
    "hdrnet_slice_apply_curves_ragged_px_ws": (_c_int, [_vp, _vp] + [_c_int] * 6 + [_vp] * 5
                                               + [ctypes.c_float, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_slice_apply_nn_ragged_px_ws": (_c_int, [_vp, _vp] + [_c_int] * 6 + [_vp] * 3
                                           + [ctypes.c_float, _c_int, _vp, ctypes.c_size_t, _vp]),
    "hdrnet_model_workspace_bytes_ragged": (ctypes.c_size_t, [_vp, _vp] + [_c_int] * 3),
    # (model, descs, B, in_fmt, out_fmt, lowres descs, lowres_fmt, ws, bytes, stream)
    "hdrnet_model_run_ragged_px": (_c_int, [_vp, _vp] + [_c_int] * 3 + [_vp, _c_int, _vp, ctypes.c_size_t, _vp]),
}

# pixel storage formats (include/hdrnet_b200.h HDRNET_PX_*)
PX_F32, PX_U8, PX_U16 = 0, 1, 2

# images per launch of the ragged kernels (HDRNET_RAGGED_MAX_IMAGES): longer calls are split
RAGGED_MAX_IMAGES = 256


class ImageDesc(ctypes.Structure):
    """hdrnet_image_desc: one image of a ragged batch (device pointers to [H, W, 3] buffers)."""
    _fields_ = [("image", _vp), ("out", _vp), ("H", _c_int), ("W", _c_int)]


def image_descs(images, outs=None):
    """A ctypes array of hdrnet_image_desc for CUDA tensors [H_i, W_i, 3] (and their outputs)."""
    arr = (ImageDesc * max(len(images), 1))()
    for i, im in enumerate(images):
        arr[i] = ImageDesc(im.data_ptr(), 0 if outs is None else outs[i].data_ptr(), im.shape[0], im.shape[1])
    return arr


class TrainSample(ctypes.Structure):
    """hdrnet_train_sample: one sample's descriptor for hdrnet_train_batch_f32."""
    _fields_ = [("input", _vp), ("target", _vp), ("input_fmt", _c_int), ("target_fmt", _c_int),
                ("H", _c_int), ("W", _c_int), ("fliplr", _c_int), ("flipud", _c_int),
                ("rot90", _c_int), ("crop_y", _c_int), ("crop_x", _c_int)]


class UsmSample(ctypes.Structure):
    """hdrnet_usm_sample: one sample's descriptor for hdrnet_train_batch_usm_f32 (a window of the
    full H x W source, and the draw on the full source's rotated extent)."""
    _fields_ = [("input", _vp), ("input_fmt", _c_int), ("H", _c_int), ("W", _c_int),
                ("y0", _c_int), ("x0", _c_int), ("h", _c_int), ("w", _c_int),
                ("fliplr", _c_int), ("flipud", _c_int), ("rot90", _c_int), ("crop_y", _c_int), ("crop_x", _c_int)]

_lock = threading.Lock()
_lib = None


class HdrnetLibraryError(RuntimeError):
    """The CUDA library is missing / unloadable, or a kernel launch failed."""


def build(verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into hdrnet_b200/lib/ (nvcc cross-compiles
    without a GPU).  Returns the library path."""
    proc = subprocess.run(["make", "-C", CSRC_DIR, "-j8"], capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        print(proc.stdout, proc.stderr)
    if proc.returncode != 0:
        raise HdrnetLibraryError("building libhdrnet_b200.so failed:\n" + proc.stdout + proc.stderr)
    return LIB_PATH


def load() -> ctypes.CDLL:
    """Load the library (once) and attach the signatures.  Raises if it is not built."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise HdrnetLibraryError(
                    f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; "
                    "g.build()'` or `make -C hdrnet_b200/csrc`. hdrnet_b200 has no CPU fallback.")
            lib = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            if lib.hdrnet_b200_abi_version() != 1:
                raise HdrnetLibraryError("libhdrnet_b200.so ABI version mismatch")
            _lib = lib
    return _lib


def error_string(code: int) -> str:
    return load().hdrnet_b200_error_string(int(code)).decode()


def check(code: int, what: str) -> None:
    """Map a library return code onto the reference's error convention
    (InvalidArgument -> ValueError, Internal -> RuntimeError; SURVEY.md section 8b)."""
    if code == OK:
        return
    msg = f"{what}: {error_string(code)} (code {code})"
    if code < 0:
        raise ValueError(msg)
    raise HdrnetLibraryError(f"{what} kernel failed. {msg}")
