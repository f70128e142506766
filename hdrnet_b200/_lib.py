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
E_NULL_POINTER, E_BAD_SHAPE, E_BAD_CHANNELS, E_TOO_LARGE, E_UNSUPPORTED, E_BAD_CONTEXT = (
    -1, -2, -3, -4, -5, -6)
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
    "hdrnet_conv2d_tc_packed_bytes": (ctypes.c_size_t, [_c_int] * 3),
    "hdrnet_conv2d_tc_pack_f32": (_c_int, [_vp, _vp] + [_c_int] * 3 + [_vp]),
    "hdrnet_conv2d_nhwc_tc_f32": (_c_int, [_vp] * 4 + [_c_int] * 8 + [_vp]),
    "hdrnet_fc_f32": (_c_int, [_vp] * 4 + [_c_int] * 4 + [_vp]),
    "hdrnet_fuse_predict_f32": (_c_int, [_vp] * 5 + [_c_int] * 7 + [_vp]),
    "hdrnet_resize_bilinear_f32": (_c_int, [_vp] * 3 + [_c_int] * 6 + [_vp]),
    "hdrnet_coefficients_scratch_bytes": (ctypes.c_size_t, [_c_int] * 7),
    "hdrnet_coefficients_f32": (_c_int, [_vp] * 4 + [_c_int, _vp, ctypes.c_size_t] + [_c_int] * 7 + [_vp]),
    "hdrnet_host_ctx_create": (_c_int, [ctypes.POINTER(_vp), ctypes.c_size_t]),
    "hdrnet_host_ctx_destroy": (_c_int, [_vp]),
    "hdrnet_slice_apply_host_f32": (_c_int, [_vp] * 5 + [_c_int] * 9),
}

# pixel storage formats (include/hdrnet_b200.h HDRNET_PX_*)
PX_F32, PX_U8, PX_U16 = 0, 1, 2

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
