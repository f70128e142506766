"""Layer helpers: drop-in for the slicing part of the reference's ``hdrnet/layers.py``.

Same names, argument order and shapes as the reference (hdrnet/layers.py:99-198) over
``torch.Tensor``:

    bilateral_slice(grid, guide)                                   layers.py:99-121
    bilateral_slice_apply(grid, guide, input_image, has_offset)    layers.py:125-148
    apply(sliced, input_image, has_affine_term)                    layers.py:153-198

    conv(inputs, num_outputs, kernel_size, stride, ..., scope)     layers.py:25-59
    fc(inputs, num_outputs, ..., scope)                            layers.py:62-93

``conv`` / ``fc`` are the INFERENCE form of the reference's layer constructors: TensorFlow creates
the layer's variables under ``scope``; here the variables already exist -- a dict keyed by the
reference's variable names (``<scope>/weights``, ``<scope>/biases``, ``<scope>/BatchNorm/beta`` ...;
``weights=`` or the dict given to ``models.set_weights``) -- and ``scope`` is the full variable scope
(e.g. ``inference/coefficients/splat/conv1``).  The variables may be CUDA float32 tensors: with
grad enabled and the input or a variable requiring grad, the layer is an autograd Function whose
backward runs the VJP kernels (csrc/cnn_grad.cu); batch-norm layers are not differentiated.
The models call the same kernels through ``hdrnet_b200.models`` with device-resident, pre-folded
weights.
"""
from __future__ import annotations

import torch

from . import hdrnet_ops

__all__ = ["conv", "fc", "bilateral_slice", "bilateral_slice_apply", "apply", "relu"]


def relu(x: torch.Tensor) -> torch.Tensor:
    """``tf.nn.relu``: the default ``activation_fn`` of conv / fc (fused into the layer's kernel)."""
    return torch.relu(x)


def _layer_variables(scope, weights, use_bias, batch_norm, device):
    """(weights, bias-or-None) on `device`, as the models prepare a layer (models._layer_weights)."""
    from . import models
    if scope is None:
        raise ValueError("scope is required: it names the layer's variables (<scope>/weights, ...)")
    wts = weights if weights is not None else models._resolve_weights({})
    return models._layer_weights(wts, scope, bool(batch_norm), bool(use_bias), device)


def _refuse_batch_norm(scope, weights, batch_norm) -> None:
    from . import models
    wts = weights if weights is not None else models._weights
    if batch_norm and scope is not None and wts is not None:
        models._refuse_batch_norm_scope(wts, scope)


def _differentiable(*ts) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def _activation(activation_fn):
    """(fused_relu, post_fn): tf.nn.relu / torch.relu / layers.relu fuse into the kernel, None is
    linear, any other callable runs on the layer's output."""
    if activation_fn is None:
        return False, None
    if activation_fn in (relu, torch.relu, torch.nn.functional.relu) or activation_fn == "relu":
        return True, None
    if not callable(activation_fn):
        raise TypeError("activation_fn must be None or a callable")
    return False, activation_fn


def conv(inputs: torch.Tensor, num_outputs: int, kernel_size: int, stride: int = 1, rate: int = 1,
         use_bias: bool = True, batch_norm: bool = False, is_training: bool = False,
         activation_fn=relu, scope: str | None = None, reuse: bool = False, *,
         weights: dict | None = None) -> torch.Tensor:
    """hdrnet/layers.py:25-59 (``tf.contrib.layers.convolution2d``, padding='SAME' incl. the
    asymmetric stride-2 padding, HWIO weights, batch norm with center and no scale; with
    ``batch_norm`` the layer has no bias of its own, :30-32).  inputs [B, H, W, Cin] float32 CUDA;
    returns [B, ceil(H / stride), ceil(W / stride), num_outputs]."""
    del reuse
    from . import models
    if is_training:
        raise NotImplementedError("hdrnet_b200 implements the inference path only")
    _refuse_batch_norm(scope, weights, batch_norm)
    if rate != 1:
        raise NotImplementedError("dilated convolutions (rate != 1) are not used by the reference models")
    if not isinstance(inputs, torch.Tensor) or inputs.dtype != torch.float32 or inputs.dim() != 4:
        raise ValueError("inputs must be a float32 tensor [B, H, W, C]")
    if inputs.device.type != "cuda":
        from . import _lib
        raise _lib.HdrnetLibraryError("inputs must be a CUDA tensor; hdrnet_b200 has no CPU path")
    w, b = _layer_variables(scope, weights, use_bias, batch_norm, inputs.device)
    if w.dim() != 4 or w.shape[0] != kernel_size or w.shape[1] != kernel_size or w.shape[3] != num_outputs:
        raise ValueError(f"{scope}/weights has shape {tuple(w.shape)}, expected "
                         f"[{kernel_size}, {kernel_size}, Cin, {num_outputs}]")
    fused, post = _activation(activation_fn)
    with torch.cuda.device(inputs.device):
        if _differentiable(inputs, w, b):
            out = models._ConvFn.apply(inputs, w, b, stride, fused)
        else:
            out = models._conv(inputs.contiguous(), (w, b), stride=stride, relu=fused)
    return out if post is None else post(out)


def fc(inputs: torch.Tensor, num_outputs: int, use_bias: bool = True, batch_norm: bool = False,
       is_training: bool = False, activation_fn=relu, scope: str | None = None, *,
       weights: dict | None = None) -> torch.Tensor:
    """hdrnet/layers.py:62-93 (``tf.contrib.layers.fully_connected``).  inputs [B, I] float32 CUDA;
    returns [B, num_outputs]."""
    from . import models
    if is_training:
        raise NotImplementedError("hdrnet_b200 implements the inference path only")
    _refuse_batch_norm(scope, weights, batch_norm)
    if not isinstance(inputs, torch.Tensor) or inputs.dtype != torch.float32 or inputs.dim() != 2:
        raise ValueError("inputs must be a float32 tensor [B, I]")
    if inputs.device.type != "cuda":
        from . import _lib
        raise _lib.HdrnetLibraryError("inputs must be a CUDA tensor; hdrnet_b200 has no CPU path")
    w, b = _layer_variables(scope, weights, use_bias, batch_norm, inputs.device)
    if w.dim() != 2 or w.shape[1] != num_outputs:
        raise ValueError(f"{scope}/weights has shape {tuple(w.shape)}, expected [I, {num_outputs}]")
    fused, post = _activation(activation_fn)
    with torch.cuda.device(inputs.device):
        if _differentiable(inputs, w, b):
            out = models._FcFn.apply(inputs, w, b, fused)
        else:
            out = models._fc(inputs.contiguous(), (w, b), relu=fused)
    return out if post is None else post(out)


# pylint: disable=redefined-builtin
def bilateral_slice(grid: torch.Tensor, guide: torch.Tensor, name=None) -> torch.Tensor:
    """Slices into a bilateral grid using the guide map (hdrnet/layers.py:99-121).

    grid:  [B, gh, gw, gd, n_outputs] or the 6-D [B, gh, gw, gd, n_out, n_in];
    guide: [B, H, W].  Returns [B, H, W, n_outputs] or, for a 6-D grid, [B, H, W, n_out, n_in].
    A 6-D grid is packed input-channel-major, c = j * n_out + i, exactly as the reference's
    ``tf.concat(tf.unstack(grid, axis=5), 4)`` (layers.py:113-120).
    """
    del name
    six_d = grid.dim() == 6
    if six_d:
        B, gh, gw, gd, n_out, n_in = grid.shape
        grid = grid.permute(0, 1, 2, 3, 5, 4).reshape(B, gh, gw, gd, n_in * n_out)
    sliced = hdrnet_ops.bilateral_slice(grid, guide)
    if six_d:
        b, h, w, _ = sliced.shape
        sliced = sliced.reshape(b, h, w, n_in, n_out).permute(0, 1, 2, 4, 3)
    return sliced


def bilateral_slice_apply(grid: torch.Tensor, guide: torch.Tensor, input_image: torch.Tensor,
                          has_offset: bool = True, name=None) -> torch.Tensor:
    """Slices into a bilateral grid and applies the sliced affine model to ``input_image``
    in one fused pass (hdrnet/layers.py:125-148).

    grid: [B, gh, gw, gd, n_out * (n_in + has_offset)] or 6-D [B, gh, gw, gd, n_out, n_in(+1)]
    (flattened output-major, c = i * (n_in+1) + j, as ``tf.reshape`` does at layers.py:141-144);
    guide: [B, H, W]; input_image: [B, H, W, n_in].  Returns [B, H, W, n_out].
    """
    del name
    if grid.dim() == 6:
        B, gh, gw, gd, n_out, n_in = grid.shape
        grid = grid.reshape(B, gh, gw, gd, n_out * n_in)
    return hdrnet_ops.bilateral_slice_apply(grid, guide, input_image, has_offset=has_offset)


def apply(sliced: torch.Tensor, input_image: torch.Tensor, has_affine_term: bool = True,
          name=None) -> torch.Tensor:
    """Applies a sliced affine model to the input image (hdrnet/layers.py:153-198): the
    un-fused second half of bilateral_slice_apply, kept in plain torch ops as the reference
    keeps it in plain TF ops.

    sliced: [B, H, W, n_out, n_in(+1)]; input_image: [B, H, W, n_in].  Returns [B, H, W, n_out].
    """
    del name
    if input_image.dim() != 4:
        raise ValueError("input image should have dims [b,h,w,n_in].")
    in_shape = list(input_image.shape)
    sliced_shape = list(sliced.shape)
    if in_shape[:-1] != sliced_shape[:-2]:
        raise ValueError("input image and affine coefficients"
                         " dimensions do not match: {} and {}".format(in_shape, sliced_shape))
    n_in = sliced_shape[-1]
    if has_affine_term:
        n_in -= 1
    scale = sliced[..., :n_in]
    ret = (scale * input_image[:, :, :, None, :n_in]).sum(dim=-1)
    if has_affine_term:
        ret = ret + sliced[..., n_in]
    return ret
# pylint: enable=redefined-builtin
