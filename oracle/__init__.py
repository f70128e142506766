"""Parity oracle for hdrnet_b200 -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package ``hdrnet_b200``
never does (tests/test_boundary.py greps for it) and fails loudly when its CUDA library is
missing instead of falling back to anything here.

Three independent CPU implementations of the reference's hot path live here; they are
cross-checked against each other and against the reference's known-answer tests in
``tests/test_oracle.py``:

``port``      ``hdrnet_oracle.c`` -- plain-C float32 restatement of
              hdrnet/ops/bilateral_slice{,_apply}.cc + numerics.h, OpenMP over rows.
``ref``       the reference's own .cc files compiled unmodified into ``oracle/_ref/``
              (``oracle/Makefile``; needs a google/hdrnet checkout -- HDRNET_REFERENCE, default
              /root/reference -- at build time only; the .so then travels with the tree).
``jax_shim``  the reference's own jax/bilateral_slice.py imported under a numpy stand-in
              for jax (works only where that checkout is readable; it generated the fixtures in
              tests/golden/).
``model_np``  numpy restatement of hdrnet/models.py + layers.py (coefficient CNN, guides).
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_SO = os.path.join(_HERE, "_build", "libhdrnet_oracle.so")
_REF_SO = os.path.join(_HERE, "_ref", "libhdrnet_ref.so")

_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int32)


def build(verbose: bool = False) -> None:
    """Compile the C restatement and, where the reference checkout is readable, ``oracle/_ref``."""
    out = subprocess.run(["make", "-C", _HERE, "all"], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout, out.stderr)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout + out.stderr)


def _as_f32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(_f32p)


def _slice_shapes(grid, guide):
    if grid.ndim != 5 or guide.ndim != 3:
        raise ValueError("grid must be [B,gh,gw,gd,gc], guide [B,H,W]")
    B, gh, gw, gd, gc = grid.shape
    Bg, H, W = guide.shape
    if Bg != B:
        raise ValueError("Batch sizes should match.")
    return B, H, W, gh, gw, gd, gc


def _apply_shapes(grid, guide, inp, has_offset):
    B, H, W, gh, gw, gd, gc = _slice_shapes(grid, guide)
    if inp.ndim != 4 or inp.shape[:3] != guide.shape:
        raise ValueError("Input and guide size should match.")
    n_in = inp.shape[3]
    J = n_in + (1 if has_offset else 0)
    if gc % J != 0:
        raise ValueError("grid channels not divisible by input channels (+offset)")
    return B, H, W, gh, gw, gd, n_in, gc // J


class _Lib:
    """ctypes view of one of the two C libraries (same entry-point shapes, different prefix)."""

    def __init__(self, path: str, prefix: str):
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.path = path
        self.prefix = prefix
        self.lib = ctypes.CDLL(path)
        self.kind = "reference" if prefix == "hdrnet_ref" else "port"

    def _fn(self, name, argtypes):
        fn = getattr(self.lib, f"{self.prefix}_{name}")
        fn.argtypes = argtypes
        fn.restype = None
        return fn

    def num_threads(self) -> int:
        fn = getattr(self.lib, f"{self.prefix}_num_threads")
        fn.restype = ctypes.c_int
        return int(fn())

    def bilateral_slice(self, grid, guide) -> np.ndarray:
        grid, guide = _as_f32(grid), _as_f32(guide)
        B, H, W, gh, gw, gd, gc = _slice_shapes(grid, guide)
        out = np.empty((B, H, W, gc), np.float32)
        fn = self._fn("slice", [_f32p, _f32p, _f32p] + [ctypes.c_int] * 7)
        fn(_ptr(grid), _ptr(guide), _ptr(out), B, H, W, gh, gw, gd, gc)
        return out

    def bilateral_slice_apply(self, grid, guide, inp, has_offset: bool) -> np.ndarray:
        grid, guide, inp = _as_f32(grid), _as_f32(guide), _as_f32(inp)
        B, H, W, gh, gw, gd, n_in, n_out = _apply_shapes(grid, guide, inp, has_offset)
        out = np.empty((B, H, W, n_out), np.float32)
        fn = self._fn("slice_apply", [_f32p] * 4 + [ctypes.c_int] * 9)
        fn(_ptr(grid), _ptr(guide), _ptr(inp), _ptr(out), B, H, W, gh, gw, gd, n_in, n_out,
           int(bool(has_offset)))
        return out


class _Port(_Lib):
    def __init__(self):
        super().__init__(_PORT_SO, "hdrnet_oracle")

    def slice_indices(self, guide, gh: int, gw: int, gd: int) -> np.ndarray:
        """(gx0, gy0, gz0) per pixel, unclamped, int32 [B,H,W,3]."""
        guide = _as_f32(guide)
        B, H, W = guide.shape
        idx = np.empty((B, H, W, 3), np.int32)
        fn = self._fn("slice_indices", [_f32p, _i32p] + [ctypes.c_int] * 6)
        fn(_ptr(guide), idx.ctypes.data_as(_i32p), B, H, W, gh, gw, gd)
        return idx

    def bilateral_slice_apply_grad(self, grid, guide, inp, ct, has_offset: bool):
        grid, guide, inp, ct = _as_f32(grid), _as_f32(guide), _as_f32(inp), _as_f32(ct)
        B, H, W, gh, gw, gd, n_in, n_out = _apply_shapes(grid, guide, inp, has_offset)
        ho = int(bool(has_offset))
        ints = [ctypes.c_int] * 9
        gv = np.empty_like(grid)
        uv = np.empty_like(guide)
        iv = np.empty_like(inp)
        self._fn("slice_apply_grid_grad", [_f32p] * 4 + ints)(
            _ptr(guide), _ptr(inp), _ptr(ct), _ptr(gv), B, H, W, gh, gw, gd, n_in, n_out, ho)
        self._fn("slice_apply_guide_grad", [_f32p] * 5 + ints)(
            _ptr(grid), _ptr(guide), _ptr(inp), _ptr(ct), _ptr(uv), B, H, W, gh, gw, gd, n_in,
            n_out, ho)
        self._fn("slice_apply_input_grad", [_f32p] * 4 + ints)(
            _ptr(grid), _ptr(guide), _ptr(ct), _ptr(iv), B, H, W, gh, gw, gd, n_in, n_out, ho)
        return gv, uv, iv

    def bilateral_slice_grad(self, grid, guide, ct):
        grid, guide, ct = _as_f32(grid), _as_f32(guide), _as_f32(ct)
        B, H, W, gh, gw, gd, gc = _slice_shapes(grid, guide)
        ints = [ctypes.c_int] * 7
        gv = np.empty_like(grid)
        uv = np.empty_like(guide)
        self._fn("slice_grid_grad", [_f32p] * 3 + ints)(
            _ptr(guide), _ptr(ct), _ptr(gv), B, H, W, gh, gw, gd, gc)
        self._fn("slice_guide_grad", [_f32p] * 4 + ints)(
            _ptr(grid), _ptr(guide), _ptr(ct), _ptr(uv), B, H, W, gh, gw, gd, gc)
        return gv, uv


class _Ref(_Lib):
    def __init__(self):
        super().__init__(_REF_SO, "hdrnet_ref")

    def bilateral_slice_apply_grad(self, grid, guide, inp, ct, has_offset: bool):
        grid, guide, inp, ct = _as_f32(grid), _as_f32(guide), _as_f32(inp), _as_f32(ct)
        B, H, W, gh, gw, gd, n_in, n_out = _apply_shapes(grid, guide, inp, has_offset)
        gv, uv, iv = np.empty_like(grid), np.empty_like(guide), np.empty_like(inp)
        fn = self._fn("slice_apply_grad", [_f32p] * 7 + [ctypes.c_int] * 9)
        fn(_ptr(grid), _ptr(guide), _ptr(inp), _ptr(ct), _ptr(gv), _ptr(uv), _ptr(iv), B, H, W,
           gh, gw, gd, n_in, n_out, int(bool(has_offset)))
        return gv, uv, iv

    def bilateral_slice_grad(self, grid, guide, ct):
        grid, guide, ct = _as_f32(grid), _as_f32(guide), _as_f32(ct)
        B, H, W, gh, gw, gd, gc = _slice_shapes(grid, guide)
        gv, uv = np.empty_like(grid), np.empty_like(guide)
        fn = self._fn("slice_grad", [_f32p] * 5 + [ctypes.c_int] * 7)
        fn(_ptr(grid), _ptr(guide), _ptr(ct), _ptr(gv), _ptr(uv), B, H, W, gh, gw, gd, gc)
        return gv, uv


_port = None
_ref = None


def port() -> _Port:
    """The C restatement (builds it on first use if the .so is missing)."""
    global _port
    if _port is None:
        if not os.path.exists(_PORT_SO):
            build()
        _port = _Port()
    return _port


def have_ref() -> bool:
    return os.path.exists(_REF_SO)


def ref() -> _Ref:
    """The reference's own compiled loops (oracle/_ref). Raises if it was never built."""
    global _ref
    if _ref is None:
        _ref = _Ref()
    return _ref


def best():
    """The strongest available checker: compiled reference if present, else the port."""
    return ref() if have_ref() else port()
