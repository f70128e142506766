"""Float64 reference of the bilateral-slice ops and their VJPs -- TEST INFRASTRUCTURE ONLY.

numpy, float64 throughout.  It restates the semantics of the reference's C++ loops
(hdrnet/ops/bilateral_slice.cc:26-168, bilateral_slice_apply.cc:25-259, numerics.h) but not their
form: every quantity is written per pixel, over the pixel's 8 grid corners, and the grid VJP is
SCATTERED into the grid with ``np.bincount`` instead of gathered over each cell's mirrored pixel
footprint as the reference does (bilateral_slice_apply.cc:95-125).  The two forms are equal in
exact arithmetic, so agreement with the float32 loops (tests/test_slice_f64.py) checks both, and
this one does not share their float32 accumulation: at training sizes a grid-VJP element sums
~10^4-10^5 terms, and only a float64 sum tells whether a float32 kernel's result is accurate.

Semantics (reference file:line):
  * x / y: tent weights max(1 - |dx|, 0) of the two cells around the pixel's cell coordinate
    (x + 0.5) * gw / W, corner cells clamped to the grid (bilateral_slice.cc:35-58,
    numerics.h:53-57).
  * depth: the smoothed weight max(1 - sqrt(d^2 + 1e-8), 0) of cells floor(gd*g - 0.5) and the
    next, clamped (numerics.h:83-113); gd*g is the float32 product for a float32 guide (_depth).  Where gd*g - 0.5 is an integer k the cells are k and
    k + 1 (the C++ floor; DESIGN.md section 2 has how the JAX helper differs).
  * grid VJP: the same weights, except that where both depth corners clamp to one border cell
    (gd*g < 0.5 or gd*g > gd - 0.5) that cell's depth weight is 1
    (bilateral_slice_apply.cc:115-118, oracle/hdrnet_oracle.c:236).  Inside (0.5, gd - 0.5) the
    grid VJP is exactly the adjoint of the forward.
  * guide VJP: sum over corners of wx * wy * gd * SmoothedLerpWeightGrad(d) * grid * tangent,
    no override (bilateral_slice_apply.cc:140-206).  SmoothedLerpWeightGrad is 0 where the
    smoothed |d| exceeds 1 (numerics.h:116-126).  In float32, sqrt(d^2 + 1e-8) rounds to |d| for
    |d| near 1 (1e-8 is below half an ulp of 1), so that test is |d| > 1 and |d| == 1 takes the
    gradient path, as numerics.h:101-103 says it should; this module uses |d| > 1 so that an
    exact cell centre (d = 0 and d = 1 at once) gets the reference's value.
  * input VJP: sum over outputs i of tangent[i] * sliced[i, j] (bilateral_slice_apply.cc:208-259).

Besides each grid / guide VJP element, ``*_grad`` returns the sum of the absolute values of the
terms that make it up: the scale a float32 sum of those terms can be held to element by element.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np

EPS = 1.0e-8                 # numerics.h:83 (SmoothedAbs eps)
_CHUNK = 1 << 18             # pixels per step: bounds the working set to ~100 MB at gc = 36


class SliceVjps(NamedTuple):
    grid: np.ndarray                 # [B, gh, gw, gd, gc]
    guide: np.ndarray                # [B, H, W]
    input: Optional[np.ndarray]      # [B, H, W, n_in]; None for bilateral_slice
    grid_abs: np.ndarray             # sum of |terms| of each grid VJP element
    guide_abs: np.ndarray            # sum of |terms| of each guide VJP element


def _axis(n_px: int, n_cells: int):
    """Per pixel of one spatial axis: the two clamped corner cells and their tent weights."""
    c = (np.arange(n_px, dtype=np.float64) + 0.5) * n_cells / n_px
    i0 = np.floor(c - 0.5).astype(np.int64)
    w0 = np.maximum(1.0 - np.abs(i0 + 0.5 - c), 0.0)
    w1 = np.maximum(1.0 - np.abs(i0 + 1.5 - c), 0.0)
    return (np.clip(i0, 0, n_cells - 1), np.clip(i0 + 1, 0, n_cells - 1)), (w0, w1)


def _depth(g: np.ndarray, gd: int):
    """Per pixel: clamped depth corners, forward weights, grid-VJP weights, guide-VJP weights.

    The depth coordinate is guide * gd formed in the guide's own precision: for a float32 guide
    the float32 product, as every float32 implementation forms it (bilateral_slice.cc:49).  Near
    a cell centre d / sqrt(d^2 + 1e-8) amplifies an error in d by up to 1e4, so the exact product
    would move a float32 guide VJP by up to ~1e-3 of its terms at pixels within 1e-4 of a centre:
    an error of the input's quantisation, not of the arithmetic under test.  Everything after this
    product is float64.  A float64 guide (finite differences) uses the exact product."""
    if g.dtype == np.float32:
        z = (g * np.float32(gd)).astype(np.float64)
    else:
        z = np.asarray(g, np.float64) * gd
    z0 = np.floor(z - 0.5)
    cells, w, wv, dw = [], [], [], []
    lo, hi = z < 0.5, z > gd - 0.5
    for k in (0, 1):
        d = (z0 + k + 0.5) - z
        a = np.sqrt(d * d + EPS)
        wk = np.maximum(1.0 - a, 0.0)
        cells.append(np.clip(z0 + k, 0, gd - 1).astype(np.int64))
        w.append(wk)
        # border override: corner 0 carries the whole weight, corner 1 none (both clamp to it)
        wv.append(np.where(lo | hi, 1.0 if k == 0 else 0.0, wk))
        dw.append(np.where(np.abs(d) > 1.0, 0.0, gd * d / a))
    return cells, w, wv, dw


def _shapes(grid, guide, inp, has_offset):
    if grid.ndim != 5 or guide.ndim != 3 or grid.shape[0] != guide.shape[0]:
        raise ValueError("grid must be [B,gh,gw,gd,gc], guide [B,H,W]")
    B, gh, gw, gd, gc = grid.shape
    _, H, W = guide.shape
    if inp is None:
        return B, H, W, gh, gw, gd, gc, 0, gc, 1
    if inp.ndim != 4 or inp.shape[:3] != guide.shape:
        raise ValueError("input must be [B,H,W,n_in]")
    n_in = inp.shape[3]
    J = n_in + (1 if has_offset else 0)
    if gc % J:
        raise ValueError("grid channels not divisible by input channels (+offset)")
    return B, H, W, gh, gw, gd, gc, n_in, gc // J, J


def _run(grid, guide, inp, ct, has_offset, want_grads, y_off=0, height=None):
    """The one pass behind every entry point.  apply mode when ``inp`` is given.  ``guide`` / ``inp``
    hold image rows ``y_off ..`` of images ``height`` rows tall (default: the whole image)."""
    grid = np.asarray(grid, np.float64)
    guide = np.asarray(guide)
    inp = None if inp is None else np.asarray(inp, np.float64)
    B, H, W, gh, gw, gd, gc, n_in, n_out, J = _shapes(grid, guide, inp, has_offset)
    apply = inp is not None
    ncell = gh * gw * gd
    out = np.zeros((B, H, W, n_out if apply else gc))
    if want_grads:
        ct = np.asarray(ct, np.float64).reshape(B, H * W, -1)
        gv = np.zeros((B, ncell * gc))
        gv_abs = np.zeros((B, ncell * gc))
        uv = np.zeros((B, H * W))
        uv_abs = np.zeros((B, H * W))
        iv = np.zeros((B, H * W, n_in)) if apply else None
    if height is None:
        height = H
    if y_off < 0 or y_off + H > height:
        raise ValueError(f"rows [{y_off}, {y_off + H}) do not fit an image of {height} rows")
    (ys, wys) = _axis(height, gh)
    (xs, wxs) = _axis(W, gw)
    guide_f = guide.reshape(B, H * W)
    for b in range(B):
        gflat = grid[b].reshape(ncell, gc)
        for p0 in range(0, H * W, _CHUNK):
            p = np.arange(p0, min(p0 + _CHUNK, H * W))
            y, x = p // W + y_off, p % W
            zc, zw, zwv, zdw = _depth(guide_f[b, p], gd)
            if apply:
                ext = inp[b].reshape(H * W, n_in)[p]
                if J > n_in:
                    ext = np.concatenate([ext, np.ones((len(p), 1))], 1)
            if want_grads:
                ctp = ct[b, p]
                # tangent of each grid channel c = i * J + j: ct[i] * (input[j] or 1)
                v = (ctp[:, :, None] * ext[:, None, :]).reshape(len(p), gc) if apply else ctp
                av = np.abs(v)
                ds = np.zeros(len(p))
                ds_abs = np.zeros(len(p))
            sliced = np.zeros((len(p), gc))
            for ky in (0, 1):
                for kx in (0, 1):
                    wxy = wys[ky][y] * wxs[kx][x]
                    col = (ys[ky][y] * gw + xs[kx][x]) * gd
                    for kz in (0, 1):
                        cell = col + zc[kz]
                        G = gflat[cell]
                        sliced += (wxy * zw[kz])[:, None] * G
                        if not want_grads:
                            continue
                        idx = (cell[:, None] * gc + np.arange(gc)).ravel()
                        wgt = wxy * zwv[kz]
                        gv[b] += np.bincount(idx, (wgt[:, None] * v).ravel(), ncell * gc)
                        gv_abs[b] += np.bincount(idx, (np.abs(wgt)[:, None] * av).ravel(), ncell * gc)
                        dwk = wxy * zdw[kz]
                        ds += dwk * (G * v).sum(1)
                        ds_abs += np.abs(dwk) * (np.abs(G) * av).sum(1)
            if apply:
                s = sliced.reshape(len(p), n_out, J)
                out[b].reshape(H * W, n_out)[p] = np.einsum("pij,pj->pi", s, ext)
                if want_grads:
                    iv[b, p] = np.einsum("pi,pij->pj", ctp, s)[:, :n_in]
            else:
                out[b].reshape(H * W, gc)[p] = sliced
            if want_grads:
                uv[b, p] = ds
                uv_abs[b, p] = ds_abs
    if not want_grads:
        return out
    return SliceVjps(gv.reshape(grid.shape), uv.reshape(guide.shape),
                     None if iv is None else iv.reshape(inp.shape),
                     gv_abs.reshape(grid.shape), uv_abs.reshape(guide.shape))


def bilateral_slice(grid, guide) -> np.ndarray:
    """[B,gh,gw,gd,gc] x [B,H,W] -> [B,H,W,gc], float64."""
    return _run(grid, guide, None, None, False, False)


def bilateral_slice_apply(grid, guide, inp, has_offset: bool, y_off: int = 0, height=None) -> np.ndarray:
    """-> [B,H,W,n_out], float64; grid channel c = i * (n_in + has_offset) + j.  With ``height``,
    ``guide`` / ``inp`` are the row band ``y_off .. y_off + H - 1`` of images ``height`` rows tall
    (what ``hdrnet_ops.bilateral_slice_apply_rows`` computes): a few rows of a large image cost
    only their own pixels."""
    return _run(grid, guide, inp, None, has_offset, False, y_off, height)


def bilateral_slice_grad(grid, guide, ct) -> SliceVjps:
    """VJPs of bilateral_slice for the tangent ``ct`` [B,H,W,gc] (``input`` is None)."""
    return _run(grid, guide, None, ct, False, True)


def bilateral_slice_apply_grad(grid, guide, inp, ct, has_offset: bool, y_off: int = 0, height=None) -> SliceVjps:
    """VJPs of bilateral_slice_apply for the tangent ``ct`` [B,H,W,n_out].  ``y_off`` / ``height`` as in
    bilateral_slice_apply; the grid VJP is then the band's pixels' share of it."""
    return _run(grid, guide, inp, ct, has_offset, True, y_off, height)
