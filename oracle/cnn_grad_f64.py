"""float64 torch-autograd restatement of the coefficient network and its VJPs -- TEST ONLY.

``oracle/model_torch.py`` passes numpy between layers, so it cannot be differentiated.  This module
restates HDRNetCurves._coefficients (hdrnet/models.py:62-142, hdrnet/layers.py:25-93) in float64
torch with autograd, with the same explicit asymmetric SAME pads (``model_torch.same_pad_amounts``)
and the same NHWC flatten / ``unroll_grid`` map, and gives

  * per-layer VJPs that take GIVEN activations (the CUDA forward's own, so that a ReLU mask flipped
    by float32 rounding cannot decide a comparison): ``conv_vjp``, ``fc_vjp``, ``fuse_predict_vjp``;
  * a whole network (``Network``): ``forward(lowres)`` and ``backward(dgrid)``.

Every weight / bias VJP also comes with Σ|terms| per element: the same VJP of |x| and |dy'|, the
scale a float32 sum of those terms is rounded against.  Inference-form layers only: batch norm is
not restated here (its training form is a different forward).
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F

from .model_torch import same_pad_amounts

P = "inference/coefficients"


def _t(a, grad=False) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64)))
    return t.requires_grad_(grad)


def conv_same(x: torch.Tensor, w: torch.Tensor, stride: int) -> torch.Tensor:
    """x [B,H,W,Cin], w HWIO -> [B,ceil(H/s),ceil(W/s),Cout] (no bias), float64, differentiable."""
    xt = x.permute(0, 3, 1, 2)
    k = w.shape[0]
    pt, pb = same_pad_amounts(xt.shape[2], k, stride)
    pl, pr = same_pad_amounts(xt.shape[3], k, stride)
    y = F.conv2d(F.pad(xt, (pl, pr, pt, pb)), w.permute(3, 2, 0, 1), stride=stride)
    return y.permute(0, 2, 3, 1)


class Vjp(NamedTuple):
    dx: np.ndarray
    dw: np.ndarray
    db: np.ndarray
    dw_abs: np.ndarray   # Σ|terms| of every dw element
    db_abs: np.ndarray


def _masked(dy, out, relu):
    dy = np.asarray(dy, np.float64)
    return dy * (np.asarray(out) > 0) if relu else dy


def conv_vjp(x, w, out, dy, stride, relu) -> Vjp:
    """VJPs of out = act(conv_same(x, w) + b) at the given x and (for the ReLU mask) out."""
    dyp = _t(_masked(dy, out, relu))
    xt, wt = _t(x, True), _t(w, True)
    dx, dw = torch.autograd.grad(conv_same(xt, wt, stride), (xt, wt), dyp)
    xa, wa = _t(np.abs(np.asarray(x, np.float64))), _t(w, True)
    (dw_abs,) = torch.autograd.grad(conv_same(xa, wa, stride), (wa,), dyp.abs())
    return Vjp(dx.numpy(), dw.numpy(), dyp.sum(dim=(0, 1, 2)).numpy(), dw_abs.numpy(),
               dyp.abs().sum(dim=(0, 1, 2)).numpy())


def fc_vjp(x, w, out, dy, relu) -> Vjp:
    """VJPs of out = act(x @ w + b)."""
    dyp = np.asarray(_masked(dy, out, relu))
    x64, w64 = np.asarray(x, np.float64), np.asarray(w, np.float64)
    return Vjp(dyp @ w64.T, x64.T @ dyp, dyp.sum(0), np.abs(x64).T @ np.abs(dyp), np.abs(dyp).sum(0))


def _unroll(pred: torch.Tensor, gd: int, n_out: int, n_in: int) -> torch.Tensor:
    """unroll_grid (models.py:134-139): [B,gh,gw,gd*n_out*n_in] -> [B,gh,gw,gd,n_out,n_in]."""
    cur = torch.stack(torch.split(pred, gd, dim=3), dim=4)
    return torch.stack(torch.split(cur, n_out, dim=4), dim=5)


def fuse_predict(local, glob, w, b, gd, n_out, n_in):
    """relu(local + global) -> 1x1 prediction conv -> unroll_grid, differentiable torch."""
    fused = F.relu(local + glob[:, None, None, :])
    pred = torch.einsum("bhwc,co->bhwo", fused, w)
    if b is not None:
        pred = pred + b
    return _unroll(pred, gd, n_out, n_in)


class FuseVjp(NamedTuple):
    dlocal: np.ndarray
    dglobal: np.ndarray
    dw: np.ndarray
    db: np.ndarray
    dw_abs: np.ndarray
    db_abs: np.ndarray


def fuse_predict_vjp(local, glob, w, dgrid, gd, n_out, n_in) -> FuseVjp:
    lt, gt, wt, bt = _t(local, True), _t(glob, True), _t(w, True), _t(np.zeros(w.shape[1]), True)
    dg = _t(dgrid)
    dl, dgl, dw, db = torch.autograd.grad(fuse_predict(lt, gt, wt, bt, gd, n_out, n_in), (lt, gt, wt, bt), dg)
    # Σ|terms|: fused >= 0 already, so |fused| = fused; |dpred| through the same unroll map
    wa, ba = _t(w, True), _t(np.zeros(w.shape[1]), True)
    dw_abs, db_abs = torch.autograd.grad(
        fuse_predict(_t(local), _t(glob), wa, ba, gd, n_out, n_in), (wa, ba), dg.abs())
    return FuseVjp(dl.numpy(), dgl.numpy(), dw.numpy(), db.numpy(), dw_abs.numpy(), db_abs.numpy())


def layer_specs(params):
    """(scope, kind, stride, relu, bias) in network order (models.py:62-142)."""
    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    s = [(f"{P}/splat/conv{i + 1}", "conv", 2, True, True) for i in range(n_ds)]
    s += [(f"{P}/global/conv1", "conv", 2, True, True), (f"{P}/global/conv2", "conv", 2, True, True),
          (f"{P}/global/fc1", "fc", 1, True, True), (f"{P}/global/fc2", "fc", 1, True, True),
          (f"{P}/global/fc3", "fc", 1, False, True), (f"{P}/local/conv1", "conv", 1, True, True),
          (f"{P}/local/conv2", "conv", 1, False, False), (f"{P}/prediction/conv1", "pred", 1, False, True)]
    return s


def variable_names(params):
    names = []
    for scope, _, _, _, bias in layer_specs(params):
        names.append(scope + "/weights")
        if bias:
            names.append(scope + "/biases")
    return names


class Network:
    """The coefficient network in float64 autograd.  ``forward`` keeps the graph; ``backward(dgrid)``
    returns {variable name: gradient} plus "lowres_input"."""

    def __init__(self, wts, params, n_out: int = 3, n_in: int = 4):
        if params.get("batch_norm"):
            raise NotImplementedError("the float64 gradient reference restates batch_norm=False only")
        self.params, self.n_out, self.n_in = params, n_out, n_in
        self.vars = {k: _t(wts[k], True) for k in variable_names(params)}
        self.acts = {}

    def forward(self, lowres) -> np.ndarray:
        v, gd = self.vars, self.params["luma_bins"]
        self.x = x = _t(lowres, True)
        specs = {s[0]: s for s in layer_specs(self.params)}

        def layer(scope, inp):
            _, kind, stride, relu, bias = specs[scope]
            y = conv_same(inp, v[scope + "/weights"], stride) if kind == "conv" else inp @ v[scope + "/weights"]
            if bias:
                y = y + v[scope + "/biases"]
            y = F.relu(y) if relu else y
            self.acts[scope] = y
            return y

        n_ds = int(np.log2(self.params["net_input_size"] / self.params["spatial_bin"]))
        for i in range(n_ds):
            x = layer(f"{P}/splat/conv{i + 1}", x)
        splat = x
        g = layer(f"{P}/global/conv2", layer(f"{P}/global/conv1", splat))
        g = g.reshape(g.shape[0], -1)
        g = layer(f"{P}/global/fc3", layer(f"{P}/global/fc2", layer(f"{P}/global/fc1", g)))
        loc = layer(f"{P}/local/conv2", layer(f"{P}/local/conv1", splat))
        s = f"{P}/prediction/conv1"
        self.grid = fuse_predict(loc, g, v[s + "/weights"][0, 0], v[s + "/biases"], gd, self.n_out, self.n_in)
        return self.grid.detach().numpy()

    def backward(self, dgrid) -> dict:
        names = list(self.vars)
        grads = torch.autograd.grad(self.grid, [self.vars[k] for k in names] + [self.x], _t(dgrid),
                                    allow_unused=True)
        out = {k: g.numpy() for k, g in zip(names, grads[:-1])}
        out["lowres_input"] = grads[-1].numpy()
        return out
