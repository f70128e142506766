"""float64 restatement of the coefficient network with its batch norm in training mode -- TEST ONLY.

``params['batch_norm']`` puts a batch norm after splat conv2..conv_n, global conv1, conv2, fc1, fc2 and
local conv1 (hdrnet/models.py:73-117); in the reference's training graph (is_training=True,
hdrnet/layers.py:47-54: center=True, scale=False, epsilon 1e-3, decay 0.999) each such layer computes,
per output channel c over the N rows of the whole batch (B H W, or B for an fc layer):

    z = conv(x, W) or x @ W (no bias),  mu_c, var_c = mean and biased variance of z[:, c]
    s_c = 1 / sqrt(var_c + 1e-3),  zh = (z - mu_c) s_c,  y = relu(zh + beta_c)

and its VJP, with dyh = dy [y > 0] (TF's ReluGrad), A_c = sum dyh (= d beta_c), B_c = sum dyh zh:

    dz = s_c (dyh - A_c / N - zh B_c / N)

This module writes both out in numpy float64 (``bn_relu``, ``bn_relu_vjp``), gives the moving-average
update (``moving_update``), and chains them with the layer VJPs of ``cnn_grad_f64`` into a whole
network (``TrainingNetwork``): ``forward(lowres)`` and ``backward(dgrid)``.  ``cnn_grad_f64.Network``
keeps restating the batch_norm=False network only.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import cnn_grad_f64 as G

P = G.P
BN_EPS = 1e-3
BN_DECAY = 0.999


def batch_norm_scopes(params):
    """The layers with batch norm when params['batch_norm'] is set (models._coefficient_specs)."""
    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    return ([f"{P}/splat/conv{i + 1}" for i in range(1, n_ds)] +
            [f"{P}/global/conv1", f"{P}/global/conv2", f"{P}/global/fc1", f"{P}/global/fc2", f"{P}/local/conv1"])


def variable_names(params):
    """The trainable variables: weights, biases of the layers without batch norm, BatchNorm/beta."""
    bn = set(batch_norm_scopes(params))
    names = []
    for scope, _, _, _, bias in G.layer_specs(params):
        names.append(scope + "/weights")
        if scope in bn:
            names.append(scope + "/BatchNorm/beta")
        elif bias:
            names.append(scope + "/biases")
    return names


def bn_relu(z, beta):
    """(y, mean, biased variance) of one layer over z [..., C], float64."""
    z = np.asarray(z, np.float64)
    C = z.shape[-1]
    z2 = z.reshape(-1, C)
    mean = z2.mean(0)
    var = ((z2 - mean) ** 2).mean(0)
    zh = (z2 - mean) / np.sqrt(var + BN_EPS)
    y = np.maximum(zh + np.asarray(beta, np.float64), 0.0)
    return y.reshape(z.shape), mean, var


class BnVjp(NamedTuple):
    dz: np.ndarray
    dbeta: np.ndarray       # A
    dbeta_abs: np.ndarray   # sum |dyh|, the scale a float32 sum of A's terms is rounded against
    b: np.ndarray           # B


def bn_relu_vjp(z, beta, dy, mask=None) -> BnVjp:
    """The VJP of bn_relu at z for dy.  ``mask`` (y > 0, e.g. the CUDA forward's own) decides the relu;
    by default it is this module's float64 forward's."""
    z = np.asarray(z, np.float64)
    C = z.shape[-1]
    z2, dy2 = z.reshape(-1, C), np.asarray(dy, np.float64).reshape(-1, C)
    n = z2.shape[0]
    mean = z2.mean(0)
    var = ((z2 - mean) ** 2).mean(0)
    s = 1.0 / np.sqrt(var + BN_EPS)
    zh = (z2 - mean) * s
    m = (zh + np.asarray(beta, np.float64) > 0) if mask is None else np.asarray(mask).reshape(-1, C)
    g = dy2 * m
    A, B = g.sum(0), (g * zh).sum(0)
    dz = s * (g - A / n - zh * B / n)
    return BnVjp(dz.reshape(z.shape), A, np.abs(g).sum(0), B)


def moving_update(moving_mean, moving_var, mean, var, n):
    """TF's assign_moving_average without zero-debias, v -= (1 - decay) (v - batch), the variance fed to
    it Bessel-corrected, var n / (n - 1) (n = 1 feeds 0: its variance is 0), in float64."""
    unbiased = np.asarray(var, np.float64) * (n / (n - 1.0) if n > 1 else 1.0)
    mm = np.asarray(moving_mean, np.float64)
    mv = np.asarray(moving_var, np.float64)
    return mm - (1.0 - BN_DECAY) * (mm - mean), mv - (1.0 - BN_DECAY) * (mv - unbiased)


def _conv(x, w, stride):
    with torch.no_grad():
        return G.conv_same(G._t(x), G._t(w), stride).numpy()


class TrainingNetwork:
    """The coefficient network with batch_norm=True in training mode, float64.  ``forward`` keeps every
    layer's input, pre-activation and output and each batch-norm layer's (mean, variance, N) in
    ``stats``; ``backward(dgrid)`` returns {variable name: gradient} plus "lowres_input", through
    cnn_grad_f64's conv / fc / fusion VJPs and bn_relu_vjp."""

    def __init__(self, wts, params, n_out: int = 3, n_in: int = 4):
        if not params.get("batch_norm"):
            raise ValueError("TrainingNetwork restates batch_norm=True; cnn_grad_f64.Network the rest")
        self.params, self.n_out, self.n_in = params, n_out, n_in
        self.v = {k: np.asarray(wts[k], np.float64) for k in variable_names(params)}
        self.bn = set(batch_norm_scopes(params))
        self.specs = {s[0]: s for s in G.layer_specs(params)}
        self.acts, self.stats = {}, {}

    def _layer(self, scope, x):
        _, kind, stride, relu, bias = self.specs[scope]
        w = self.v[scope + "/weights"]
        z = _conv(x, w, stride) if kind == "conv" else x @ w
        if scope in self.bn:
            y, mean, var = bn_relu(z, self.v[scope + "/BatchNorm/beta"])
            self.stats[scope] = (mean, var, z.size // z.shape[-1])
        else:
            y = z + self.v[scope + "/biases"] if bias else z
            y = np.maximum(y, 0.0) if relu else y
        self.acts[scope] = (x, z, y)
        return y

    def forward(self, lowres) -> np.ndarray:
        self.x = x = np.asarray(lowres, np.float64)
        n_ds = int(np.log2(self.params["net_input_size"] / self.params["spatial_bin"]))
        for i in range(n_ds):
            x = self._layer(f"{P}/splat/conv{i + 1}", x)
        self.splat = splat = x
        g = self._layer(f"{P}/global/conv2", self._layer(f"{P}/global/conv1", splat))
        self.g_shape = g.shape
        g = g.reshape(g.shape[0], -1)
        g = self._layer(f"{P}/global/fc3", self._layer(f"{P}/global/fc2", self._layer(f"{P}/global/fc1", g)))
        loc = self._layer(f"{P}/local/conv2", self._layer(f"{P}/local/conv1", splat))
        s = f"{P}/prediction/conv1"
        self.fuse_in = (loc, g)
        with torch.no_grad():
            grid = G.fuse_predict(G._t(loc), G._t(g), G._t(self.v[s + "/weights"][0, 0]),
                                  G._t(self.v[s + "/biases"]), self.params["luma_bins"], self.n_out, self.n_in)
        return grid.numpy()

    def _back(self, scope, dy, grads):
        """dy of the layer's output -> dx of its input; the layer's variable gradients into grads."""
        _, kind, stride, relu, bias = self.specs[scope]
        x, z, y = self.acts[scope]
        w = self.v[scope + "/weights"]
        if scope in self.bn:
            bv = bn_relu_vjp(z, self.v[scope + "/BatchNorm/beta"], dy)
            grads[scope + "/BatchNorm/beta"] = bv.dbeta
            dy, relu = bv.dz, False
        vj = G.conv_vjp(x, w, y, dy, stride, relu) if kind == "conv" else G.fc_vjp(x, w, y, dy, relu)
        grads[scope + "/weights"] = vj.dw
        if bias and scope not in self.bn:
            grads[scope + "/biases"] = vj.db
        return vj.dx

    def backward(self, dgrid) -> dict:
        grads = {}
        s = f"{P}/prediction/conv1"
        loc, g = self.fuse_in
        fv = G.fuse_predict_vjp(loc, g, self.v[s + "/weights"][0, 0], dgrid, self.params["luma_bins"],
                                self.n_out, self.n_in)
        grads[s + "/weights"] = fv.dw[None, None]
        grads[s + "/biases"] = fv.db
        dl = self._back(f"{P}/local/conv1", self._back(f"{P}/local/conv2", fv.dlocal, grads), grads)
        dg = fv.dglobal
        for name in ("fc3", "fc2", "fc1"):
            dg = self._back(f"{P}/global/{name}", dg, grads)
        dg = dg.reshape(self.g_shape)
        dg = self._back(f"{P}/global/conv1", self._back(f"{P}/global/conv2", dg, grads), grads)
        dx = dl + dg
        n_ds = int(np.log2(self.params["net_input_size"] / self.params["spatial_bin"]))
        for i in reversed(range(n_ds)):
            dx = self._back(f"{P}/splat/conv{i + 1}", dx, grads)
        grads["lowres_input"] = dx
        return grads
