"""Float64 reference of the curves guide and its VJP -- TEST INFRASTRUCTURE ONLY.

numpy, float64 throughout.  HDRNetCurves._guide (hdrnet/models.py:145-190) per pixel, with x the
RGB input and g the gradient of the guide:

    t_c = sum_i x_i ccm[i][c] + ccm_bias[c]
    u_c = sum_k slope_ck relu(t_c - s_ck)
    a = sum_c mix_c u_c + mix_bias,   guide = clip(a, 0, 1)

and the gradients TF gives that graph, with its tie rules:

  * clip: g^ = g [0 <= a <= 1]; tf.clip_by_value (like torch.clamp) passes the gradient at equality;
  * relu: [t_c > s_ck]; TF's ReluGrad is `features > 0`, 0 at t = s.

    d mix_bias = g^,  d mix_c = g^ u_c,  d slope_ck = g^ mix_c relu(t_c - s_ck),
    d s_ck = -g^ mix_c slope_ck [t_c > s_ck],  d ccm_bias_c = g^ mix_c u'_c,
    d ccm[i][c] = x_i g^ mix_c u'_c,  dx_i = sum_c ccm[i][c] g^ mix_c u'_c,
    u'_c = sum_k slope_ck [t_c > s_ck]

Parameter gradients are summed over every pixel.  Besides each gradient element the VJP returns
the sum of the absolute values of the terms that make it up, with every factor expanded into its
own terms: u'_c as sum_k |slope_ck| [t_c > s_ck], and relu(t_c - s_ck) = x . ccm[:, c] + ccm_bias_c
- s_ck (where positive) as sum_i |x_i ccm[i][c]| + |ccm_bias_c| + |s_ck|.  That is the scale a
float32 computation of those terms, and a float32 sum of them, can be held to.

Variables are taken in the shapes the model stores them (ccm [3,3], ccm_bias [3], shifts
[1,1,3,16], slopes [1,1,1,3,16], channel_mixing/weights [1,1,3,1], channel_mixing/biases [1]) or
any shape with the same element order; gradients come back in those shapes.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

_CHUNK = 1 << 18             # pixels per step: bounds the [n, 3, 16] temporaries
NAMES = ("ccm", "ccm_bias", "shifts", "slopes", "channel_mixing/weights", "channel_mixing/biases")
SIZES = (9, 3, 48, 48, 3, 1)          # the library's 112-float parameter gradient, in this order


class GuideVjp(NamedTuple):
    dinput: np.ndarray       # x's shape
    dinput_abs: np.ndarray   # Σ|terms| of every dinput element
    dparams: dict            # name (NAMES) -> gradient, in the variable's shape
    dparams_abs: dict        # name -> Σ|terms| of every gradient element


def _vars(wts, prefix="inference/guide"):
    return [np.asarray(wts[f"{prefix}/{n}"], np.float64) for n in NAMES]


def _split(v):
    ccm, ccm_bias, shifts, slopes, mix, mix_bias = v
    return (ccm.reshape(3, 3), ccm_bias.reshape(3), shifts.reshape(3, 16), slopes.reshape(3, 16),
            mix.reshape(3), float(mix_bias.reshape(-1)[0]))


def preclip(x, wts, prefix="inference/guide"):
    """(a, t) in float64: a [...] before the clip, t [..., 3]."""
    ccm, ccm_bias, shifts, slopes, mix, mix_bias = _split(_vars(wts, prefix))
    x = np.asarray(x, np.float64)
    t = x @ ccm + ccm_bias
    u = (slopes * np.maximum(t[..., None] - shifts, 0.0)).sum(-1)
    return u @ mix + mix_bias, t


def guide(x, wts, prefix="inference/guide"):
    return np.clip(preclip(x, wts, prefix)[0], 0.0, 1.0)


def vjp(x, dguide, wts, prefix="inference/guide") -> GuideVjp:
    """The VJP of guide(x) for the upstream gradient dguide (x's shape without the last axis)."""
    v = _vars(wts, prefix)
    ccm, ccm_bias, shifts, slopes, mix, mix_bias = _split(v)
    x = np.asarray(x, np.float64)
    shape = x.shape
    xs = x.reshape(-1, 3)
    gs = np.asarray(dguide, np.float64).reshape(-1)
    dx, dx_abs = np.empty_like(xs), np.empty_like(xs)
    acc = {n: np.zeros(s) for n, s in zip(NAMES, SIZES)}
    acc_abs = {n: np.zeros(s) for n, s in zip(NAMES, SIZES)}
    for s0 in range(0, xs.shape[0], _CHUNK):
        xc, g = xs[s0:s0 + _CHUNK], gs[s0:s0 + _CHUNK]
        t = xc @ ccm + ccm_bias                                   # [n, 3]
        d = t[:, :, None] - shifts                                # [n, 3, 16]
        r = np.maximum(d, 0.0)
        on = d > 0.0
        u = (slopes * r).sum(-1)                                  # [n, 3]
        r_abs = (np.abs(xc) @ np.abs(ccm) + np.abs(ccm_bias))[:, :, None] + np.abs(shifts)
        r_abs = np.where(on, r_abs, 0.0)                          # Σ|terms| of r
        u_abs = (np.abs(slopes) * r_abs).sum(-1)
        a = u @ mix + mix_bias
        gh = np.where((a >= 0.0) & (a <= 1.0), g, 0.0)            # [n]
        gc = gh[:, None] * mix                                    # [n, 3]
        up = (slopes * on).sum(-1)                                # u'
        up_abs = (np.abs(slopes) * on).sum(-1)
        w, w_abs = gc * up, np.abs(gc) * up_abs                   # [n, 3]
        dx[s0:s0 + _CHUNK] = w @ ccm.T
        dx_abs[s0:s0 + _CHUNK] = w_abs @ np.abs(ccm).T
        for n, val, val_abs in (
                ("ccm", xc.T @ w, np.abs(xc).T @ w_abs),
                ("ccm_bias", w.sum(0), w_abs.sum(0)),
                ("shifts", -(gc[:, :, None] * on).sum(0) * slopes,
                 (np.abs(gc)[:, :, None] * on).sum(0) * np.abs(slopes)),
                ("slopes", (gc[:, :, None] * r).sum(0), (np.abs(gc)[:, :, None] * r_abs).sum(0)),
                ("channel_mixing/weights", gh @ u, np.abs(gh) @ u_abs),
                ("channel_mixing/biases", gh.sum(keepdims=True), np.abs(gh).sum(keepdims=True))):
            acc[n] += val.reshape(-1)
            acc_abs[n] += val_abs.reshape(-1)
    shapes = {n: np.shape(a) for n, a in zip(NAMES, v)}
    return GuideVjp(dx.reshape(shape), dx_abs.reshape(shape),
                    {n: acc[n].reshape(shapes[n]) for n in NAMES},
                    {n: acc_abs[n].reshape(shapes[n]) for n in NAMES})


def flat(d: dict) -> np.ndarray:
    """A name -> array dict (dparams / dparams_abs) as the library's 112-float vector."""
    return np.concatenate([np.asarray(d[n], np.float64).reshape(-1) for n in NAMES])
