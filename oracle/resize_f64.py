"""Float64 reference of the align-corners bilinear resize and its VJP -- TEST INFRASTRUCTURE ONLY.

tf.image.resize_images(x, [oh, ow], BILINEAR, align_corners=True), TF1 legacy semantics, as
HDRNetGaussianPyrNN uses it (hdrnet/models.py:249-289).  The tap coordinates are formed in float32,
as the kernels form them (csrc/resize.cu): s = float32(n - 1) / float32(on - 1) (0 when on = 1),
src = float32(o) * s, lo = floor(src), hi = min(lo + 1, n - 1), f = src - lo.  Everything after
that is float64.

The VJP is written in SCATTER form: each output pixel adds its 4 weighted corner terms into the
input-shaped gradient (``np.bincount`` over the corners' flat indices).  The kernel gathers over
each input pixel's candidate output pixels instead; the two are equal in exact arithmetic, so agreement checks the kernel's
choice of candidates and weights.  Besides the gradient, ``resize_vjp`` returns Σ|terms| per
element: the scale a float32 sum of those terms can be held to.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np


def taps(n: int, on: int):
    """(lo, hi, frac) of each of the `on` output coordinates over an input axis of `n`: int arrays
    lo and hi, float64 frac (computed in float32, as the kernels do)."""
    s = np.float32(n - 1) / np.float32(on - 1) if on > 1 else np.float32(0.0)
    src = np.arange(on).astype(np.float32) * s
    lo = np.floor(src).astype(np.int64)
    hi = np.minimum(lo + 1, n - 1)
    frac = (src - lo.astype(np.float32)).astype(np.float64)
    return lo, hi, frac


def resize(x, oh: int, ow: int) -> np.ndarray:
    """The forward, float64: x [B, H, W, C] -> [B, oh, ow, C]."""
    x = np.asarray(x, np.float64)
    _, H, W, _ = x.shape
    y0, y1, fy = taps(H, oh)
    x0, x1, fx = taps(W, ow)
    fy, fx = fy[None, :, None, None], fx[None, None, :, None]
    top = x[:, y0][:, :, x0] * (1.0 - fx) + x[:, y0][:, :, x1] * fx
    bot = x[:, y1][:, :, x0] * (1.0 - fx) + x[:, y1][:, :, x1] * fx
    return top * (1.0 - fy) + bot * fy


class ResizeVjp(NamedTuple):
    din: np.ndarray        # [B, H, W, C] float64
    din_abs: np.ndarray    # Σ|terms| of each element


def resize_vjp(dout, H: int, W: int) -> ResizeVjp:
    """The VJP of ``resize`` to an input of H x W, from dout [B, oh, ow, C], scattered: each output
    pixel's 4 corner terms w * dout are added into din (np.bincount over the corners' indices);
    corners that coincide, lo == hi on the last row or column, get both terms."""
    dout = np.asarray(dout, np.float64)
    B, oh, ow, C = dout.shape
    y0, y1, fy = taps(H, oh)
    x0, x1, fx = taps(W, ow)
    din = np.zeros((B, H * W, C))
    din_abs = np.zeros((B, H * W, C))
    oy, ox = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    oy, ox = oy.reshape(-1), ox.reshape(-1)
    d = dout.reshape(B, oh * ow, C)
    for ys, wy in ((y0, 1.0 - fy), (y1, fy)):
        for xs, wx in ((x0, 1.0 - fx), (x1, fx)):
            target = ys[oy] * W + xs[ox]
            w = wy[oy] * wx[ox]
            for b in range(B):
                for c in range(C):
                    t = w * d[b, :, c]
                    din[b, :, c] += np.bincount(target, weights=t, minlength=H * W)
                    din_abs[b, :, c] += np.bincount(target, weights=np.abs(t), minlength=H * W)
    return ResizeVjp(din.reshape(B, H, W, C), din_abs.reshape(B, H, W, C))
