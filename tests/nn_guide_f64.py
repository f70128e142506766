"""Float64 reference of the pointwise-NN guide in training mode, its moving-average update and its
VJP -- TEST INFRASTRUCTURE ONLY.

numpy, float64 throughout.  HDRNetPointwiseNNGuide._guide (hdrnet/models.py:203-210) with
is_training=True, over N = B*H*W pixels x_p in R^3 and F features:

    z_pf = x_p . W1[:, f]                         (conv1, 1x1, no bias)
    mu_f = mean_p z_pf,  var_f = mean_p (z_pf - mu_f)^2      (from z itself, not the input moments)
    xh_pf = (z_pf - mu_f) / sqrt(var_f + 1e-3),  y_pf = xh_pf + beta_f,  h_pf = relu(y_pf)
    guide_p = sigmoid(sum_f h_pf w2_f + b2)

tf.contrib.layers.batch_norm's defaults: center=True, scale=False, epsilon=1e-3, decay=0.999.  The
moving averages move as TF's assign_moving_average without zero-debias,
    mm -= (1 - 0.999) (mm - mu),   mv -= (1 - 0.999) (mv - var N / (N - 1))
with the Bessel-corrected variance TF's fused batch norm feeds them (N / (N - 1) taken as 1 at N = 1).

The VJP is TF's gradient of that graph, with ReluGrad's tie rule (y > 0), through the batch
statistics: dz_pf = s_f (dy_pf - A_f / N - xh_pf B_f / N), dW1_if = sum_p x_pi dz_pf, dx = dz W1'.
It is summed directly over the pixels, not through the closed form the kernel uses.  Besides each
parameter-gradient element it returns the sum of the absolute values of the terms that make it up,
every factor expanded into its own terms (h as |x . W1| s + |mu| s + |beta|, dz as
s (|dy| + |A| / N + |xh| |B| / N)): the scale a float32 computation can be held to.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

EPS = 1e-3
DECAY = 0.999
NAMES = ("conv1/weights", "conv1/BatchNorm/beta", "conv2/weights", "conv2/biases")
_CHUNK = 1 << 18             # pixels per step: bounds the [n, F] temporaries


class NNGuideVjp(NamedTuple):
    dinput: np.ndarray       # x's shape
    dparams: dict            # name (NAMES) -> gradient, in the variable's shape
    dparams_abs: dict        # name -> sum |terms| of every gradient element


def _vars(wts, prefix="inference/guide"):
    w1 = np.asarray(wts[f"{prefix}/conv1/weights"], np.float64)
    beta = np.asarray(wts[f"{prefix}/conv1/BatchNorm/beta"], np.float64)
    w2 = np.asarray(wts[f"{prefix}/conv2/weights"], np.float64)
    b2 = np.asarray(wts[f"{prefix}/conv2/biases"], np.float64)
    return w1, beta, w2, b2


def _flat(x):
    return np.asarray(x, np.float64).reshape(-1, 3)


def batch_stats(x, wts, prefix="inference/guide"):
    """(mu [F], var [F]): conv1's batch mean and biased variance, from z directly (two passes)."""
    w1 = _vars(wts, prefix)[0].reshape(3, -1)
    xs = _flat(x)
    n = xs.shape[0]
    s = np.zeros(w1.shape[1])
    for s0 in range(0, n, _CHUNK):
        s += (xs[s0:s0 + _CHUNK] @ w1).sum(0)
    mu = s / n
    q = np.zeros(w1.shape[1])
    for s0 in range(0, n, _CHUNK):
        q += ((xs[s0:s0 + _CHUNK] @ w1 - mu) ** 2).sum(0)
    return mu, q / n


def guide(x, wts, prefix="inference/guide", stats=None):
    """The training-mode guide [x.shape[:-1]] in float64."""
    w1, beta, w2, b2 = _vars(wts, prefix)
    w1, beta, w2 = w1.reshape(3, -1), beta.reshape(-1), w2.reshape(-1)
    mu, var = batch_stats(x, wts, prefix) if stats is None else stats
    s = 1.0 / np.sqrt(var + EPS)
    xs = _flat(x)
    out = np.empty(xs.shape[0])
    for s0 in range(0, xs.shape[0], _CHUNK):
        y = (xs[s0:s0 + _CHUNK] @ w1 - mu) * s + beta
        out[s0:s0 + _CHUNK] = 1.0 / (1.0 + np.exp(-(np.maximum(y, 0.0) @ w2 + b2.reshape(-1)[0])))
    return out.reshape(np.shape(x)[:-1])


def moving_average_update(moving_mean, moving_variance, x, wts, prefix="inference/guide"):
    """One step of the moving averages after a training-mode forward over x."""
    mu, var = batch_stats(x, wts, prefix)
    n = _flat(x).shape[0]
    unbiased = var * (n / (n - 1.0) if n > 1 else 1.0)
    mm = np.asarray(moving_mean, np.float64)
    mv = np.asarray(moving_variance, np.float64)
    return mm - (1.0 - DECAY) * (mm - mu), mv - (1.0 - DECAY) * (mv - unbiased)


def vjp(x, dguide, wts, prefix="inference/guide") -> NNGuideVjp:
    """The VJP of guide(x) for the upstream gradient dguide (x's shape without the last axis)."""
    w1v, betav, w2v, b2v = _vars(wts, prefix)
    w1, beta, w2, b2 = w1v.reshape(3, -1), betav.reshape(-1), w2v.reshape(-1), b2v.reshape(-1)[0]
    F = beta.size
    xs = _flat(x)
    gs = np.asarray(dguide, np.float64).reshape(-1)
    n = xs.shape[0]
    mu, var = batch_stats(x, wts, prefix)
    s = 1.0 / np.sqrt(var + EPS)

    def chunk(s0):
        xc, g = xs[s0:s0 + _CHUNK], gs[s0:s0 + _CHUNK]
        xh = (xc @ w1 - mu) * s
        y = xh + beta
        h = np.maximum(y, 0.0)
        sg = 1.0 / (1.0 + np.exp(-(h @ w2 + b2)))
        do = g * sg * (1.0 - sg)
        dy = np.where(y > 0.0, do[:, None] * w2, 0.0)
        h_abs = np.where(y > 0.0, (np.abs(xc) @ np.abs(w1) + np.abs(mu)) * s + np.abs(beta), 0.0)
        return xc, xh, h, h_abs, do, dy

    # pass 1: the sums the batch statistics' gradient needs, and the conv2 / beta gradients
    A, B = np.zeros(F), np.zeros(F)
    dw2, dw2_abs, db2, db2_abs, dbeta_abs = np.zeros(F), np.zeros(F), 0.0, 0.0, np.zeros(F)
    for s0 in range(0, n, _CHUNK):
        _, xh, h, h_abs, do, dy = chunk(s0)
        A += dy.sum(0)
        B += (dy * xh).sum(0)
        dw2 += do @ h
        dw2_abs += np.abs(do) @ h_abs
        db2 += do.sum()
        db2_abs += np.abs(do).sum()
        dbeta_abs += np.abs(dy).sum(0)
    # pass 2: dz, then dW1 and dx from it directly
    dx = np.empty_like(xs)
    dw1, dw1_abs = np.zeros((3, F)), np.zeros((3, F))
    for s0 in range(0, n, _CHUNK):
        xc, xh, _, _, _, dy = chunk(s0)
        dz = s * (dy - A / n - xh * B / n)
        dz_abs = s * (np.abs(dy) + np.abs(A) / n + np.abs(xh) * np.abs(B) / n)
        dw1 += xc.T @ dz
        dw1_abs += np.abs(xc).T @ dz_abs
        dx[s0:s0 + _CHUNK] = dz @ w1.T
    shapes = dict(zip(NAMES, (w1v.shape, betav.shape, w2v.shape, b2v.shape)))
    grads = dict(zip(NAMES, (dw1, A, dw2, np.array([db2]))))
    grads_abs = dict(zip(NAMES, (dw1_abs, dbeta_abs, dw2_abs, np.array([db2_abs]))))
    return NNGuideVjp(dx.reshape(np.shape(x)), {k: v.reshape(shapes[k]) for k, v in grads.items()},
                      {k: v.reshape(shapes[k]) for k, v in grads_abs.items()})


def flat(d: dict) -> np.ndarray:
    """A name -> array dict as the library's 5 F + 1 parameter gradient (conv1/weights [3][F], beta,
    conv2/weights, conv2/biases)."""
    return np.concatenate([np.asarray(d[n], np.float64).reshape(-1) for n in NAMES])
