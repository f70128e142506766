"""Run the reference's own ``jax/bilateral_slice.py`` without JAX -- TEST INFRASTRUCTURE ONLY.

The parity target BASELINE.json names is the reference's ``jax/bilateral_slice.py``
(``bilateral_slice`` :299-380, numerics in ``jax/numerics.py``), found in the google/hdrnet
checkout that the environment variable ``HDRNET_REFERENCE`` points to (default: ``DEFAULT_REFERENCE``,
where the build environment mounts it).  JAX need not be
installed: this module injects a small numpy stand-in for ``jax`` / ``jax.numpy`` into
``sys.modules`` and then imports the two reference files UNMODIFIED from where they lie.
Nothing is copied; without a checkout ``load()`` raises, and the tests use the fixtures that
``tests/golden/make_golden.py`` stored from it.

Stand-in semantics that matter for parity:
* ``jnp.arange`` returns int32 (as JAX does with x64 disabled);
* ``int_array + 0.5`` must be float32 in JAX but is float64 in numpy.  ``_F32Int`` keeps
  index arrays in a thin ndarray subclass whose arithmetic with python floats yields
  float32, so coordinates ``(ii + 0.5) * scale`` are computed in float32 exactly as JAX
  does (weak-typed python scalars), which is what makes the cell indices bit-comparable;
* ``x.at[idx].add(v)`` -> ``np.add.at`` on a copy;
* ``jax.custom_vjp`` -> identity decorator with a no-op ``defvjp``.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np

DEFAULT_REFERENCE = "/root/reference"   # same default as oracle/Makefile
REFERENCE_JAX_DIR = os.path.join(os.environ.get("HDRNET_REFERENCE") or DEFAULT_REFERENCE, "jax")


class _F32Int(np.ndarray):
    """int32 ndarray whose +,-,* with python floats produce float32 (JAX weak typing)."""

    def _weak(self, other, op):
        if isinstance(other, float):
            return op(np.asarray(self).astype(np.float32), np.float32(other))
        res = op(np.asarray(self), np.asarray(other) if isinstance(other, _F32Int) else other)
        if isinstance(res, np.ndarray) and res.dtype.kind in "iu":
            return res.astype(np.int32).view(_F32Int)
        return res

    def __add__(self, o):
        return self._weak(o, np.add)

    __radd__ = __add__

    def __sub__(self, o):
        return self._weak(o, np.subtract)

    def __mul__(self, o):
        return self._weak(o, np.multiply)

    __rmul__ = __mul__

    def clip(self, lo, hi):  # keeps int32 for fancy indexing
        return np.clip(np.asarray(self), lo, hi).astype(np.int32)


class _At:
    def __init__(self, arr):
        self._arr = arr

    def __getitem__(self, idx):
        arr = self._arr

        class _Upd:
            def add(self_inner, val):
                out = np.array(arr, copy=True)
                np.add.at(out, idx, val)
                return out.view(_Arr)

        return _Upd()


class _Arr(np.ndarray):
    """float ndarray with a JAX-style ``.at`` property."""

    @property
    def at(self):
        return _At(self)


def _make_jnp() -> types.ModuleType:
    jnp = types.ModuleType("jax.numpy")

    def arange(*a, **k):
        return np.arange(*a, **k).astype(np.int32).view(_F32Int)

    def meshgrid(*xs, **k):
        # integer coordinates stay weak-typed int32; float arguments (the VJP helpers mesh float grid
        # coordinates with integer cell indices, bilateral_slice.py:153-154) keep their values
        return [m.astype(np.int32).view(_F32Int) if m.dtype.kind in "iu" else m
                for m in np.meshgrid(*[np.asarray(x) for x in xs], **k)]

    def zeros(shape, dtype=np.float32):
        return np.zeros(shape, dtype).view(_Arr)

    def floor(x):
        return np.floor(np.asarray(x))

    def ceil(x):
        return np.ceil(np.asarray(x))

    jnp.arange = arange
    jnp.meshgrid = meshgrid
    jnp.zeros = zeros
    jnp.floor = floor
    jnp.ceil = ceil
    jnp.int32 = np.int32
    jnp.float32 = np.float32
    for name in ("atleast_3d", "divide", "einsum", "maximum", "multiply", "pad", "sqrt", "sum",
                 "where", "abs", "clip", "asarray", "array"):
        setattr(jnp, name, getattr(np, name))
    return jnp


def _make_jax(jnp) -> types.ModuleType:
    jax = types.ModuleType("jax")

    def custom_vjp(fn):
        fn.defvjp = lambda fwd, bwd: None
        return fn

    jax.custom_vjp = custom_vjp
    jax.numpy = jnp
    return jax


_loaded = None


def available() -> bool:
    return os.access(os.path.join(REFERENCE_JAX_DIR, "bilateral_slice.py"), os.R_OK)


def load():
    """Import the reference's jax package under the stand-in; returns the bilateral_slice module."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not available():
        raise FileNotFoundError(f"no readable google/hdrnet checkout at {os.path.dirname(REFERENCE_JAX_DIR)} "
                                "(HDRNET_REFERENCE); the tests use tests/golden fixtures")
    saved = {k: sys.modules.get(k) for k in ("jax", "jax.numpy")}
    jnp = _make_jnp()
    jax = _make_jax(jnp)
    sys.modules["jax"] = jax
    sys.modules["jax.numpy"] = jnp
    try:
        pkg = types.ModuleType("_hdrnet_ref_jax")
        pkg.__path__ = [REFERENCE_JAX_DIR]
        sys.modules["_hdrnet_ref_jax"] = pkg
        mods = {}
        for name in ("numerics", "bilateral_slice"):
            spec = importlib.util.spec_from_file_location(
                f"_hdrnet_ref_jax.{name}", os.path.join(REFERENCE_JAX_DIR, f"{name}.py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules[spec.name] = mod
            spec.loader.exec_module(mod)
            mods[name] = mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    _loaded = mods["bilateral_slice"]
    return _loaded


def bilateral_slice(grid, guide) -> np.ndarray:
    """Batched reference slice: vmap of jax/bilateral_slice.py:299-380 over axis 0
    (as hdrnet/hdrnet_ops_jax_tf2_test.py:23-24 does with jax.vmap)."""
    mod = load()
    grid = np.asarray(grid, np.float32)
    guide = np.asarray(guide, np.float32)
    outs = [np.asarray(mod.bilateral_slice(grid[b], guide[b])) for b in range(grid.shape[0])]
    return np.stack(outs).astype(np.float32)


def bilateral_slice_vjp(grid, guide, codomain_tangent):
    """Batched reference VJPs of the slice: (grid_vjp, guide_vjp) from the reference's own
    ``bilateral_slice_grid_vjp`` (jax/bilateral_slice.py:257-295: mirror-padded footprint, einsum of
    the spatial and range weights) and ``bilateral_slice_guide_vjp`` (:26-108), one image at a time
    -- what ``_bilateral_slice_bwd`` (:387-392) returns under ``jax.vmap``."""
    mod = load()
    grid = np.asarray(grid, np.float32)
    guide = np.asarray(guide, np.float32)
    ct = np.asarray(codomain_tangent, np.float32)
    gv = [np.asarray(mod.bilateral_slice_grid_vjp(guide[b], ct[b], grid.shape[1:])) for b in range(grid.shape[0])]
    uv = [np.asarray(mod.bilateral_slice_guide_vjp(grid[b], guide[b], ct[b])) for b in range(grid.shape[0])]
    return np.stack(gv).astype(np.float32), np.stack(uv).astype(np.float32)


def bilateral_slice_apply(grid, guide, inp, has_offset: bool) -> np.ndarray:
    """Reference slice (JAX file) followed by the reference's pure-TF ``apply`` semantics
    (hdrnet/layers.py:153-198): out[i] = sum_j sliced[i,j]*in[j] (+ sliced[i,n_in])."""
    inp = np.asarray(inp, np.float32)
    sliced = bilateral_slice(grid, guide).astype(np.float64)
    n_in = inp.shape[-1]
    J = n_in + (1 if has_offset else 0)
    n_out = sliced.shape[-1] // J
    s = sliced.reshape(sliced.shape[:3] + (n_out, J))
    out = np.einsum("bhwij,bhwj->bhwi", s[..., :n_in], inp.astype(np.float64))
    if has_offset:
        out = out + s[..., n_in]
    return out.astype(np.float32)


def slice_indices(guide, gh: int, gw: int, gd: int) -> np.ndarray:
    """(gj0, gi0, gk0) = (gx0, gy0, gz0) as jax/bilateral_slice.py:314-327 computes them."""
    load()
    jnp = _make_jnp()
    guide = np.asarray(guide, np.float32)
    B, H, W = guide.shape
    ii, jj = jnp.meshgrid(jnp.arange(H), jnp.arange(W), indexing="ij")
    gif = (ii + 0.5) * (gh / H)
    gjf = (jj + 0.5) * (gw / W)
    assert gif.dtype == np.float32 and gjf.dtype == np.float32
    gi0 = np.floor(gif - np.float32(0.5)).astype(np.int32)
    gj0 = np.floor(gjf - np.float32(0.5)).astype(np.int32)
    out = np.empty((B, H, W, 3), np.int32)
    for b in range(B):
        gkf = guide[b] * gd
        out[b, ..., 0] = gj0
        out[b, ..., 1] = gi0
        out[b, ..., 2] = np.floor(gkf - np.float32(0.5)).astype(np.int32)
    return out
