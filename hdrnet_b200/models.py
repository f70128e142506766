"""Model graphs: drop-in for the reference's ``hdrnet/models.py`` (inference).

Same class names, classmethods and call signature as the reference
(hdrnet/models.py:30-210; selected by name in hdrnet/bin/run.py:82-85):

    mdl = getattr(models, params['model_name'])
    out = mdl.inference(lowres_input, fullres_input, params, is_training=False)

over ``torch.Tensor`` (CUDA, float32, NHWC).  ``params`` carries the reference's model
hyper-parameters (hdrnet/bin/train.py:224-236): ``luma_bins, channel_multiplier, spatial_bin,
net_input_size, batch_norm, guide_complexity``.

Where TF keeps variables in the graph (restored from a checkpoint), this module keeps a
flat dict of numpy arrays keyed by the SAME variable names under ``inference/``
(``inference/coefficients/splat/conv1/weights`` ...): pass it as ``params['weights']`` or
install it once with ``set_weights`` / ``load_weights``.  Conv weights are HWIO, FC weights
[in, out], exactly as TF stores them.

The values may also be CUDA float32 ``torch.Tensor``s.  With grad enabled and any coefficient-network
variable (or ``lowres_input``) requiring grad, ``_coefficients`` runs layer by layer through
autograd Functions over the same forward kernels and the VJP kernels of ``csrc/cnn_grad.cu``, so
``torch.optim`` can fine-tune the network through the slice-apply VJP with the guide held fixed.
A dict holding tensors is never cached: every call reads the current values.  The gradients are
those of the inference-form graph; with ``batch_norm=False`` (the reference's default,
hdrnet/bin/train.py:224-236) that is the coefficient network's training graph.  With
``params['guide_grad']`` truthy, ``HDRNetCurves``'s guide variables (``ccm``, ``ccm_bias``,
``shifts``, ``slopes``, ``channel_mixing/*``) and ``fullres_input`` are differentiated too, through
``_CurvesGuideFn`` and the VJP of ``csrc/guide_grad.cu``; without the key, asking for their gradient
raises ``NotImplementedError`` as before.  The pointwise-NN guide's conv1 has batch norm, which
training runs in training mode: ``HDRNetPointwiseNNGuide.inference(..., is_training=True)`` is the
reference's training graph, with conv1 normalised by the batch's statistics
(``csrc/guide_nn_grad.cu``), its moving averages updated in place on every call, and, with
``params['guide_grad']``, gradients for the guide's variables and ``fullres_input`` through
``_NNGuideFn``.  In the inference form (``is_training=False``) that guide is not differentiated.
Under a process group of several ranks (data-parallel training, each rank holding a shard of the
batch) the training-mode statistics are those of the whole batch: the ranks' input moments are
merged before the fold (``parallel.moments_over_ranks``).  ``HDRNetGaussianPyrNN`` has one such guide per
pyramid level (``inference/guide/level_{0,1,2}``): ``inference(..., is_training=True)`` normalises each
level with its own batch statistics and moves that level's moving averages, and differentiates the
coefficient network and, with ``params['guide_grad']``, every level's guide and ``fullres_input``,
through ``_ResizeFn``, whose backward is the VJP of the align-corners resize (``csrc/resize.cu``); its
inference form is not differentiated.  ``HDRNetGaussianPyr`` is that pyramid with a curves guide per
level (DESIGN.md row f-17); with ``params['guide_grad']`` each level's curves variables and
``fullres_input`` are differentiated through ``_CurvesGuideFn`` and ``_ResizeFn``.  Batch-norm layers of the coefficient network are not
differentiated in their folded inference form: asking for their gradient raises
``NotImplementedError``.  With ``params['coefficient_batch_stats']`` (and ``batch_norm``),
``inference(..., is_training=True)`` runs them in training mode (``_coefficients_training``, the kernels
of ``csrc/bn_train.cu``): batch statistics, moving averages moved in place, and gradients for their
``weights`` and ``BatchNorm/beta``.

Execution (all hand-written sm_90a kernels through the C-ABI, no torch math on the path):
  coefficients  4 splat convs, 2 global convs + 3 FCs, 2 local convs (conv2d / fc kernels),
                then fusion + prediction + unroll_grid in one kernel -> grid [B,gh,gw,gd,12]
  guide+output  ONE kernel: per-pixel guide (curves or pointwise NN) computed in registers
                and fed straight into the fused slice-apply (the guide never touches HBM).
"""
from __future__ import annotations

import collections
import ctypes
import math

import numpy as np
import torch

from . import _lib, layers, parallel
from .hdrnet_ops import _slice_apply_workspace, _workspace
from .layers import bilateral_slice_apply

__all__ = ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN", "HDRNetGaussianPyr", "set_weights",
           "load_weights", "init_weights", "DEFAULT_PARAMS"]

BN_EPS = 1e-3   # tf.contrib.layers.batch_norm default epsilon (hdrnet/layers.py:47-54)
BN_DECAY = 0.999  # ... and its moving-average decay

DEFAULT_PARAMS = dict(  # hdrnet/bin/train.py:224-236
    model_name="HDRNetCurves", net_input_size=256, output_resolution=[512, 512],
    batch_norm=False, channel_multiplier=1, guide_complexity=16, luma_bins=8, spatial_bin=16)

_weights: dict | None = None


def set_weights(weights: dict) -> None:
    """Install the variable store (reference variable names -> numpy arrays)."""
    global _weights
    _weights = {k: np.asarray(v) for k, v in weights.items()}
    _prepared.clear()


def load_weights(path: str) -> dict:
    """Load a ``.npz`` keyed by the reference's variable names and install it."""
    with np.load(path) as z:
        w = {k.replace("__", "/"): z[k] for k in z.files}
    set_weights(w)
    return w


def _resolve_weights(params) -> dict:
    w = params.get("weights") if isinstance(params, dict) else None
    if w is None:
        w = _weights
    if w is None:
        raise ValueError("no weights: pass params['weights'] or call models.set_weights()")
    return w


def _weights_or_none(params):
    w = params.get("weights") if isinstance(params, dict) else None
    return _weights if w is None else w


def init_weights(params, seed: int = 0, model_name: str | None = None) -> dict:
    """Fresh variables with the reference's initialisers: variance-scaling (fan-in, factor 2,
    truncated normal) for conv/fc weights and zero biases (hdrnet/layers.py:22-23), identity
    ccm / linspace shifts / unit first slope / 1/3 mixing for the curves guide
    (hdrnet/models.py:150-186), one curves guide per level for HDRNetGaussianPyr, each ccm with its own
    jitter.  Used for synthetic-weight benchmarks."""
    rng = np.random.RandomState(seed)
    gd, cm = params["luma_bins"], params["channel_multiplier"]
    bn = bool(params["batch_norm"])
    model_name = model_name or params.get("model_name", "HDRNetCurves")
    w = {}

    def vs(shape, fan_in):
        std = math.sqrt(1.3 * 2.0 / fan_in)   # tf.contrib variance_scaling_initializer
        v = rng.randn(*shape)
        v = np.clip(v, -2.0, 2.0)             # truncated normal
        return (v * std).astype(np.float32)

    def post(scope, cout, use_bias, use_bn):
        if use_bn:
            w[scope + "/BatchNorm/beta"] = np.zeros(cout, np.float32)
            w[scope + "/BatchNorm/moving_mean"] = np.zeros(cout, np.float32)
            w[scope + "/BatchNorm/moving_variance"] = np.ones(cout, np.float32)
        elif use_bias:
            w[scope + "/biases"] = np.zeros(cout, np.float32)

    def conv(scope, k, cin, cout, use_bias=True, use_bn=False):
        w[scope + "/weights"] = vs((k, k, cin, cout), k * k * cin)
        post(scope, cout, use_bias, use_bn)

    def fc(scope, cin, cout, use_bias=True, use_bn=False):
        w[scope + "/weights"] = vs((cin, cout), cin)
        post(scope, cout, use_bias, use_bn)

    p = "inference/coefficients"
    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    cin = 3
    for i in range(n_ds):
        conv(f"{p}/splat/conv{i + 1}", 3, cin, cm * (2 ** i) * gd, use_bn=bn and i > 0)
        cin = cm * (2 ** i) * gd
    c8 = 8 * cm * gd
    conv(f"{p}/global/conv1", 3, cin, c8, use_bn=bn)
    conv(f"{p}/global/conv2", 3, c8, c8, use_bn=bn)
    sb = params["spatial_bin"]
    flat = int(math.ceil(sb / 4)) ** 2 * c8
    fc(f"{p}/global/fc1", flat, 32 * cm * gd, use_bn=bn)
    fc(f"{p}/global/fc2", 32 * cm * gd, 16 * cm * gd, use_bn=bn)
    fc(f"{p}/global/fc3", 16 * cm * gd, c8)
    conv(f"{p}/local/conv1", 3, cin, c8, use_bn=bn)
    conv(f"{p}/local/conv2", 3, c8, c8, use_bias=False)
    n_out = 9 if model_name in ("HDRNetGaussianPyrNN", "HDRNetGaussianPyr") else 3
    conv(f"{p}/prediction/conv1", 1, c8, gd * n_out * 4)
    g = "inference/guide"

    def curves(scope):   # models.py:152 draws the ccm's jitter once per call
        w[scope + "/ccm"] = (np.identity(3) + rng.randn(1) * 1e-4).astype(np.float32)
        w[scope + "/ccm_bias"] = np.zeros(3, np.float32)
        w[scope + "/shifts"] = np.tile(np.linspace(0, 1, 16, endpoint=False, dtype=np.float32)
                                       [None, None, None, :], (1, 1, 3, 1))
        slopes = np.zeros((1, 1, 1, 3, 16), np.float32)
        slopes[..., 0] = 1.0
        w[scope + "/slopes"] = slopes
        w[scope + "/channel_mixing/weights"] = np.full((1, 1, 3, 1), 1.0 / 3.0, np.float32)
        w[scope + "/channel_mixing/biases"] = np.zeros(1, np.float32)

    if model_name == "HDRNetGaussianPyrNN":
        nf = params["guide_complexity"]
        for lvl in range(3):
            conv(f"{g}/level_{lvl}/conv1", 1, 3, nf, use_bn=True)
            conv(f"{g}/level_{lvl}/conv2", 1, nf, 1)
    elif model_name == "HDRNetGaussianPyr":
        for lvl in range(3):
            curves(f"{g}/level_{lvl}")
    elif model_name == "HDRNetCurves":
        curves(g)
    else:
        nf = params["guide_complexity"]
        conv(g + "/conv1", 1, 3, nf, use_bn=True)
        conv(g + "/conv2", 1, nf, 1)
    return w


# Batches up to this size run the coefficient network through ONE library call
# (hdrnet_coefficients_f32, csrc/cnn.cu: 8 launches chained with programmatic dependent launch, the
# global and local branches sharing launches, fc1-fc3 in one cluster) instead of twelve per-layer
# calls from Python; larger batches go layer by layer so that the convs can use the packed
# tensor-core weights (tools/time_cnn.py times both).  Tests set this to force either path.
CHAIN_CNN_MAX_BATCH = 16

_host_pipelines = {}   # (model class, device, out dtype) -> HostImagePipeline (inference_image_host)

# ---- prepared (device-resident, BN-folded) weights ---------------------------------------------
# Keyed by the identity of the weights dict: an entry keeps a reference to its dict (so the id
# cannot be recycled while the entry lives), the cache holds the most recent kPreparedMax entries,
# and a dict UPDATED IN PLACE must be announced with invalidate_prepared().
_prepared: "collections.OrderedDict" = collections.OrderedDict()
kPreparedMax = 8


def invalidate_prepared() -> None:
    """Drop every cached device copy of model weights (call after mutating a weights dict in place)."""
    _prepared.clear()


def _fold(wts, scope, use_bn, use_bias):
    """Returns (weights, bias-or-None) as float32 numpy with inference batch norm folded in:
    y = (conv - mean) / sqrt(var + eps) + beta  (center=True, scale=False; layers.py:47-54;
    the fold freeze_graph.py:141-142 applies).  Tensor variables are read through host copies."""
    def var(name, dtype):
        return np.asarray(_host(wts[f"{scope}/{name}"]), dtype)

    w = var("weights", np.float32)
    if use_bn:
        s = 1.0 / np.sqrt(var("BatchNorm/moving_variance", np.float64) + BN_EPS)
        b = var("BatchNorm/beta", np.float64) - var("BatchNorm/moving_mean", np.float64) * s
        return (w.astype(np.float64) * s).astype(np.float32), b.astype(np.float32)
    if use_bias:
        return w, var("biases", np.float32)
    return w, None


def _host(v):
    """A variable as the host sees it: a tensor's detached host copy, anything else as it is."""
    return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v


def _host_f32(v) -> np.ndarray:
    return np.ascontiguousarray(_host(v), np.float32).reshape(-1)


def _has_tensors(wts) -> bool:
    return any(isinstance(v, torch.Tensor) for v in wts.values())


def _device_var(v, device) -> torch.Tensor:
    """A variable as a contiguous float32 tensor on `device`: a tensor already there is used as is
    (it keeps its autograd identity), anything else is copied."""
    if isinstance(v, torch.Tensor):
        return v.to(device=device, dtype=torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(v, np.float32))).to(device)


def _coefficient_specs(params):
    """(scope, batch norm, bias) of every coefficient-network layer, in network order."""
    bn = bool(params["batch_norm"])
    p = "inference/coefficients"
    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    specs = [(f"{p}/splat/conv{i + 1}", bn and i > 0, True) for i in range(n_ds)]
    specs += [(f"{p}/global/conv1", bn, True), (f"{p}/global/conv2", bn, True),
              (f"{p}/global/fc1", bn, True), (f"{p}/global/fc2", bn, True),
              (f"{p}/global/fc3", False, True), (f"{p}/local/conv1", bn, True),
              (f"{p}/local/conv2", False, False), (f"{p}/prediction/conv1", False, True)]
    return specs


def _layer_weights(wts, scope, use_bn, use_bias, device):
    """(weights, bias-or-None) of one layer as float32 tensors on `device`.  A batch-norm layer is
    folded (_fold) into copies; any other layer runs on its variables as they are, so that a tensor
    variable already on `device` is used without a copy and its gradient reaches it."""
    if use_bn:
        w, b = _fold(wts, scope, True, False)
    else:
        w, b = wts[scope + "/weights"], (wts[scope + "/biases"] if use_bias else None)
    return _device_var(w, device), (None if b is None else _device_var(b, device))


_CURVES_VARS = ("ccm", "ccm_bias", "shifts", "slopes", "channel_mixing/weights", "channel_mixing/biases")


class _CurvesGuide:
    """The curves guide (hdrnet/models.py:145-190) as its kernels take it: float32 host arrays ccm
    [3, 3] ([in][out]), ccm_bias [3], shifts and slopes [3, 16], mix [3], the float mix_bias, and
    `args`, the trailing arguments of hdrnet_guide_curves_f32 and hdrnet_slice_apply_curves_px_ws
    (host pointers into the arrays this object keeps)."""

    def __init__(self, ccm, ccm_bias, shifts, slopes, mix, mix_bias):
        self.ccm = _host_f32(ccm).reshape(3, 3)
        self.ccm_bias = _host_f32(ccm_bias).reshape(3)
        self.shifts = _host_f32(shifts).reshape(3, 16)
        self.slopes = _host_f32(slopes).reshape(3, 16)
        self.mix = _host_f32(mix).reshape(3)
        self.mix_bias = float(_host_f32(mix_bias)[0])
        arrays = (self.ccm, self.ccm_bias, self.shifts, self.slopes, self.mix)
        self.args = (*[_hp(a) for a in arrays], self.mix_bias)

    @classmethod
    def from_weights(cls, wts, scope="inference/guide"):
        return cls(*[wts[f"{scope}/{n}"] for n in _CURVES_VARS])

    def run(self, x: torch.Tensor) -> torch.Tensor:
        """The standalone guide kernel over x [B, H, W, 3] (float32, contiguous) -> [B, H, W]."""
        B, H, W, _ = x.shape
        guide = torch.empty((B, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.load().hdrnet_guide_curves_f32(x.data_ptr(), guide.data_ptr(), B * H * W, *self.args,
                                                     _stream(x.device))
        _lib.check(rc, "guide_curves")
        return guide


class _NNGuide:
    """The pointwise-NN guide (hdrnet/models.py:199-210) with conv1's batch norm folded in: float32
    host arrays w1 [3, F], b1 [F], w2 [F], the float b2 and the int feats F, and `args`, the trailing
    arguments of hdrnet_guide_nn_f32 and hdrnet_slice_apply_nn_px_ws."""

    def __init__(self, w1, b1, w2, b2):
        self.w1 = _host_f32(w1).reshape(3, -1)
        self.b1 = _host_f32(b1)
        self.w2 = _host_f32(w2)
        self.b2 = float(_host_f32(b2)[0])
        self.feats = int(self.w1.shape[1])
        self.args = (_hp(self.w1), _hp(self.b1), _hp(self.w2), self.b2, self.feats)

    @classmethod
    def folded(cls, wts, scope):
        """The inference form: conv1's batch norm folded from the moving averages."""
        w1, b1 = _fold(wts, scope + "/conv1", True, False)
        return cls(w1, b1, wts[scope + "/conv2/weights"], wts[scope + "/conv2/biases"])

    def run(self, x: torch.Tensor) -> torch.Tensor:
        """The standalone guide kernel over x [B, H, W, 3] (float32, contiguous) -> [B, H, W]."""
        B, H, W, _ = x.shape
        guide = torch.empty((B, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.load().hdrnet_guide_nn_f32(x.data_ptr(), guide.data_ptr(), B * H * W, *self.args,
                                                 _stream(x.device))
        _lib.check(rc, "guide_nn")
        return guide


class _Prepared:
    """Device copies of the coefficient-network weights + the guide's host parameters: `guides`, one
    _CurvesGuide or _NNGuide, or one per level of a pyramid model.  `nn_guide` is the model's
    _nn_guide: False (curves), True (pointwise NN), "pyramid" (an NN guide per level) or
    "curves_pyramid" (a curves guide per level)."""

    def __init__(self, wts, params, device, nn_guide):
        self.device = device
        self.source = wts   # keeps the dict alive: the cache is keyed by id(wts)
        self.layers = {}
        for scope, use_bn, use_bias in _coefficient_specs(params):
            wd, bd = _layer_weights(wts, scope, use_bn, use_bias, device)
            # tensor variables change between optimizer steps: packed per call (this object is)
            packed = pack_conv_weights(wd.detach()) if (wd.dim() == 4 and device.type == "cuda") else None
            self.layers[scope] = (wd, bd, packed)
        g = "inference/guide"
        if nn_guide == "pyramid":     # HDRNetGaussianPyrNN: one pointwise NN per level
            self.guides = [_NNGuide.folded(wts, f"{g}/level_{lvl}") for lvl in range(3)]
        elif nn_guide == "curves_pyramid":     # HDRNetGaussianPyr: one curves guide per level
            self.guides = [_CurvesGuide.from_weights(wts, f"{g}/level_{lvl}") for lvl in range(3)]
        elif nn_guide:
            self.guides = [_NNGuide.folded(wts, g)]
        else:
            self.guides = [_CurvesGuide.from_weights(wts)]


def _prepare(wts, params, device, nn_guide) -> _Prepared:
    if _has_tensors(wts):
        # tensor variables may be updated in place (optimizer steps): never served from the cache
        return _Prepared(wts, params, device, nn_guide)
    key = (id(wts), str(device), str(nn_guide), bool(params["batch_norm"]),
           params["net_input_size"], params["spatial_bin"])
    prep = _prepared.get(key)
    if prep is None:
        prep = _Prepared(wts, params, device, nn_guide)
        prep.source = wts                      # pins id(wts) for the lifetime of the entry
        _prepared[key] = prep
        while len(_prepared) > kPreparedMax:
            _prepared.popitem(last=False)
    else:
        _prepared.move_to_end(key)
    return prep


def _hp(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def _check_input(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError(f"{what} must be a float32 tensor [B, H, W, 3]")
    if t.device.type != "cuda":
        raise _lib.HdrnetLibraryError(f"{what} must be a CUDA tensor; hdrnet_b200 has no CPU path")
    return t.contiguous()


# ---- layer wrappers (hdrnet/layers.py:25-93 over the C-ABI) ------------------------------------
_PX_FMT = {torch.float32: _lib.PX_F32, torch.uint8: _lib.PX_U8, torch.uint16: _lib.PX_U16}


def _check_image(t: torch.Tensor, what: str) -> torch.Tensor:
    """A decoded image batch [B,H,W,3], uint8 / uint16 / float32, on a CUDA device."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if t.dtype not in _PX_FMT:
        raise TypeError(f"{what} must be uint8, uint16 or float32, got {t.dtype}")
    if t.dim() != 4 or t.shape[-1] != 3:
        raise ValueError(f"{what} must be [B,H,W,3], got {tuple(t.shape)}")
    if not t.is_cuda:
        raise _lib.HdrnetLibraryError(f"{what} is on {t.device}: hdrnet_b200 has no CPU path")
    return t.contiguous()


def _fused_row_kernel_takes(W: int, *bufs: torch.Tensor) -> bool:
    """Whether the float32 guide-fused slice-apply can run without a guide buffer: its row kernel
    takes W % 4 == 0, W >= 128 and 16-byte aligned buffers (include/hdrnet_b200.h); anything else
    runs the guide kernel into the caller's buffer first.  A contiguous view at an offset (a frame
    carved out of a packed buffer, an ``out`` from a pool) is not aligned."""
    return W % 4 == 0 and W >= 128 and all(t.data_ptr() % 16 == 0 for t in bufs)


def _slice_apply_fused(coeffs, x, guide, out_dtype, want_guide: bool, lend_workspace: bool):
    """Guide + slice + apply in one kernel (hdrnet_slice_apply_{curves,nn}_px_ws): x [B,H,W,3]
    (uint8 / uint16 / float32, contiguous), the coefficients [B,gh,gw,gd,3,4] and a _CurvesGuide or
    _NNGuide -> (out [B,H,W,3] of `out_dtype`, the guide map [B,H,W] or None).  The map is written
    when `want_guide` asks for it, and always where the float32 form runs the guide kernel into it
    first (_fused_row_kernel_takes).  `lend_workspace`: lend the slab workspace with which AUTO runs
    the texture-assisted kernel on large images."""
    B, H, W, _ = x.shape
    _, gh, gw, gd = coeffs.shape[:4]
    in_fmt, out_fmt = _PX_FMT[x.dtype], _PX_FMT[out_dtype]
    out = torch.empty((B, H, W, 3), dtype=out_dtype, device=x.device)
    f32 = in_fmt == _lib.PX_F32 and out_fmt == _lib.PX_F32
    gmap = torch.empty((B, H, W), dtype=torch.float32, device=x.device) \
        if want_guide or (f32 and not _fused_row_kernel_takes(W, x, out, coeffs)) else None
    lib = _lib.load()
    launch = lib.hdrnet_slice_apply_nn_px_ws if isinstance(guide, _NNGuide) else lib.hdrnet_slice_apply_curves_px_ws
    with torch.cuda.device(x.device):
        ws = _slice_apply_workspace(x.device, B, H, W, gh, gw, gd) if lend_workspace else None
        rc = launch(coeffs.data_ptr(), x.data_ptr(), in_fmt, out.data_ptr(), out_fmt, _ptr(gmap), B, H, W,
                    gh, gw, gd, *guide.args, _ptr(ws), 0 if ws is None else ws.numel() * 4, _stream(x.device))
    _lib.check(rc, "BilateralSliceApply(fused guide)")
    return out, gmap


def lowres_from_image(image: torch.Tensor, size: int) -> torch.Tensor:
    """[B,H,W,3] uint8 / uint16 / float32 -> [B,size,size,3] float32: img_as_float +
    skimage.transform.resize(order=0) of hdrnet/bin/run.py:156-169 in one gather kernel."""
    image = _check_image(image, "image")
    B, H, W, _ = image.shape
    low = torch.empty((B, size, size, 3), dtype=torch.float32, device=image.device)
    with torch.cuda.device(image.device):
        rc = _lib.load().hdrnet_lowres_nearest_f32(
            image.data_ptr(), _PX_FMT[image.dtype], low.data_ptr(), B, H, W, size, size,
            torch.cuda.current_stream(image.device).cuda_stream)
    _lib.check(rc, "lowres_nearest")
    return low


def _check_images(images, what: str) -> list:
    """A ragged batch: a list of [H_i, W_i, 3] tensors of one dtype (uint8 / uint16 / float32) on one
    CUDA device -> the list with every tensor contiguous.  Refuses before any device work."""
    if not isinstance(images, (list, tuple)):
        raise TypeError(f"{what} must be a list of tensors [H, W, 3]")
    for t in images:
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{what} must hold torch.Tensors, got {type(t).__name__}")
        if t.dtype not in _PX_FMT:
            raise TypeError(f"{what} must be uint8, uint16 or float32, got {t.dtype}")
        if t.dim() != 3 or t.shape[-1] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"{what} must hold non-empty [H, W, 3] images, got {tuple(t.shape)}")
    if len({t.dtype for t in images}) > 1:
        raise TypeError(f"{what} mixes dtypes {sorted({str(t.dtype) for t in images})}: one call takes one pixel format")
    if len({t.device for t in images}) > 1:
        raise ValueError(f"{what} spans devices {sorted({str(t.device) for t in images})}: one call runs on one device")
    if images and not images[0].is_cuda:
        raise _lib.HdrnetLibraryError(f"{what} are on {images[0].device}: hdrnet_b200 has no CPU path")
    return [t.contiguous() for t in images]


def lowres_from_images(images: list, size: int) -> torch.Tensor:
    """lowres_from_image of each image of a ragged batch (a list of [H_i, W_i, 3] tensors, checked by
    _check_images) into one [B, size, size, 3] float32 batch, one launch per RAGGED_MAX_IMAGES images;
    row i is bit for bit lowres_from_image(images[i][None], size)."""
    dev = images[0].device
    low = torch.empty((len(images), size, size, 3), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().hdrnet_lowres_nearest_ragged_f32(
            _lib.image_descs(images), len(images), _PX_FMT[images[0].dtype], low.data_ptr(), size, size, _stream(dev))
    _lib.check(rc, "lowres_nearest (ragged)")
    return low


def _slice_apply_fused_ragged(coeffs, images, guide, out_dtype):
    """_slice_apply_fused over a ragged batch (hdrnet_slice_apply_{curves,nn}_ragged_px_ws): image i
    with grid row i of coeffs [B,gh,gw,gd,3,4] -> a list of [H_i, W_i, 3] tensors of `out_dtype`."""
    _, gh, gw, gd = coeffs.shape[:4]
    dev = images[0].device
    outs = [torch.empty(im.shape, dtype=out_dtype, device=dev) for im in images]
    lib = _lib.load()
    launch = lib.hdrnet_slice_apply_nn_ragged_px_ws if isinstance(guide, _NNGuide) \
        else lib.hdrnet_slice_apply_curves_ragged_px_ws
    with torch.cuda.device(dev):
        rc = launch(coeffs.data_ptr(), _lib.image_descs(images, outs), len(images), _PX_FMT[images[0].dtype],
                    _PX_FMT[out_dtype], gh, gw, gd, *guide.args, None, 0, _stream(dev))
    _lib.check(rc, "BilateralSliceApply(fused guide, ragged)")
    return outs


def _ragged_inputs(images, lowres_images, out_dtype, params):
    """The checks of inference_images: (images, network-input images) as contiguous lists."""
    _check_out_dtype(out_dtype)
    images = _check_images(images, "images")
    if params.get("debug"):
        raise ValueError("params['debug'] stores one batch's collections: run inference_image per image for them")
    if lowres_images is None:
        return images, images
    lowres_images = _check_images(lowres_images, "lowres_images")
    if len(lowres_images) != len(images):
        raise ValueError("lowres_images must hold one image per image")
    if images and lowres_images[0].device != images[0].device:
        raise ValueError("lowres_images must be on the images' device")
    return images, lowres_images

def image_to_float(image: torch.Tensor) -> torch.Tensor:
    """skimage.img_as_float of a uint8 / uint16 tensor (IEEE division: the same float32)."""
    if image.dtype == torch.uint8:
        return image.to(torch.float32) / 255.0
    if image.dtype == torch.uint16:
        return image.to(torch.int32).to(torch.float32) / 65535.0
    return image.to(torch.float32)


def quantize_u8(x: torch.Tensor) -> torch.Tensor:
    """tf.cast(255.0 * tf.clip_by_value(x, 0, 1), tf.uint8) (hdrnet/bin/run.py:95)."""
    return (255.0 * x.clamp(0.0, 1.0)).to(torch.uint8)


def quantize_u16(x: torch.Tensor) -> torch.Tensor:
    """rint(65535 * clip(x, 0, 1)) in float32, round half to even, NaN -> 0: the uint16 epilogue of
    the fused slice-apply kernels (csrc/slice_rows.cuh float_to_u16), for results computed in float."""
    y = torch.round(65535.0 * x.nan_to_num(nan=0.0).clamp(0.0, 1.0))
    return y.to(torch.int32).to(torch.uint16)


# What inference_image / inference_image_host return: the reference's uint8 cast, the 16-bit result
# (rint(65535 * clip)), or the unquantised prediction.
OUT_DTYPES = (torch.uint8, torch.uint16, torch.float32)


def _check_out_dtype(out_dtype) -> None:
    if out_dtype not in OUT_DTYPES:
        raise TypeError(f"out_dtype must be torch.uint8, torch.uint16 or torch.float32, got {out_dtype}")


def pack_conv_weights(w: torch.Tensor):
    """Pre-pack HWIO conv weights for the pipelined tensor-core (wgmma) kernel (once per model); returns a
    device buffer, or None when the layer's shape does not suit that kernel."""
    lib = _lib.load()
    k, _, cin, cout = w.shape
    nbytes = int(lib.hdrnet_conv2d_tc_packed_bytes(k, cin, cout))
    if nbytes == 0 or cout > 128:
        return None
    packed = torch.empty(nbytes // 4, dtype=torch.float32, device=w.device)
    with torch.cuda.device(w.device):
        rc = lib.hdrnet_conv2d_tc_pack_f32(w.data_ptr(), packed.data_ptr(), k, cin, cout,
                                           torch.cuda.current_stream(w.device).cuda_stream)
    _lib.check(rc, "conv weight packing")
    return packed


# Layers given packed weights take the packed tensor-core form from this many tiles of 128 output
# pixels up.  Measured on an H100 (tools/conv_bench.py, the network's conv shapes): at 16 tiles the
# CUDA-core kernels were 3-15 % faster, at 64 the two were even, at 128 the packed tensor-core
# kernel was 1.7-5x faster.
PACKED_CONV_MIN_TILES = 64


def _conv(x: torch.Tensor, wb, stride=1, relu=True, tensor_cores=True) -> torch.Tensor:
    """One conv layer.  `tensor_cores=False` runs the CUDA-core forms alone
    (hdrnet_conv2d_nhwc_fp32_f32, float32 rounded to nearest) at every size."""
    w, b = wb[0], wb[1]
    packed = wb[2] if len(wb) > 2 else None
    B, H, W, cin = x.shape
    k, _, wcin, cout = w.shape
    if wcin != cin:
        raise ValueError(f"conv: input has {cin} channels, weights expect {wcin}")
    oh, ow = -(-H // stride), -(-W // stride)
    out = torch.empty((B, oh, ow, cout), dtype=torch.float32, device=x.device)
    lib = _lib.load()
    if not tensor_cores:
        rc = lib.hdrnet_conv2d_nhwc_fp32_f32(x.data_ptr(), w.data_ptr(), 0 if b is None else b.data_ptr(),
                                             out.data_ptr(), B, H, W, cin, cout, k, stride, int(relu),
                                             torch.cuda.current_stream(x.device).cuda_stream)
        _lib.check(rc, "conv2d (CUDA cores)")
        return out
    if packed is not None and (B * oh * ow + 127) // 128 >= PACKED_CONV_MIN_TILES:
        rc = lib.hdrnet_conv2d_nhwc_tc_f32(x.data_ptr(), packed.data_ptr(),
                                           0 if b is None else b.data_ptr(), out.data_ptr(), B, H,
                                           W, cin, cout, k, stride, int(relu),
                                           torch.cuda.current_stream(x.device).cuda_stream)
        if rc != _lib.E_UNSUPPORTED:
            _lib.check(rc, "conv2d(tensor cores)")
            return out
    rc = lib.hdrnet_conv2d_nhwc_f32(x.data_ptr(), w.data_ptr(), 0 if b is None else b.data_ptr(),
                                    out.data_ptr(), B, H, W, cin, cout, k, stride, int(relu),
                                    torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "conv2d")
    return out


def _fc(x: torch.Tensor, wb, relu=True) -> torch.Tensor:
    w, b = wb[0], wb[1]
    B, I = x.shape
    if w.shape[0] != I:
        raise ValueError(f"fc: input has {I} features, weights expect {w.shape[0]}")
    O = w.shape[1]
    out = torch.empty((B, O), dtype=torch.float32, device=x.device)
    lib = _lib.load()
    rc = lib.hdrnet_fc_f32(x.data_ptr(), w.data_ptr(), 0 if b is None else b.data_ptr(),
                           out.data_ptr(), B, I, O, int(relu),
                           torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "fc")
    return out


# ---- autograd over the layer kernels (backward: csrc/cnn_grad.cu) ------------------------------
def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


# Each layer Function's `run` is its forward alone, on the current device, for calls that want no
# gradient: Function.apply costs host time on every layer, and a setup_context split would make
# apply itself slower (it binds the arguments through inspect.signature on every call).
class _ConvFn(torch.autograd.Function):
    """One conv layer (hdrnet/layers.py:25-59, inference batch norm already folded): forward _conv
    (given `packed`, pack_conv_weights of w, the packed tensor-core form from PACKED_CONV_MIN_TILES
    up), backward hdrnet_conv2d_grad_f32."""

    @staticmethod
    def run(x, w, b, stride, relu, packed=None, tensor_cores=True):
        b = None if b is None else b.contiguous()
        return _conv(x.contiguous(), (w.contiguous(), b, packed), stride=stride, relu=relu, tensor_cores=tensor_cores)

    @staticmethod
    def forward(ctx, x, w, b, stride, relu, packed=None, tensor_cores=True):
        x, w = x.contiguous(), w.contiguous()
        with torch.cuda.device(x.device):
            out = _ConvFn.run(x, w, b, stride, relu, packed, tensor_cores)
        ctx.save_for_backward(x, w, out)
        ctx.stride, ctx.relu, ctx.has_bias = stride, bool(relu), b is not None
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w, out = ctx.saved_tensors
        dy = dy.contiguous()
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        B, H, W, cin = x.shape
        k, cout = w.shape[0], w.shape[3]
        dx = torch.empty_like(x) if need_x else None
        dw = torch.empty_like(w) if need_w else None
        db = torch.empty(cout, dtype=torch.float32, device=x.device) if (need_b and ctx.has_bias) else None
        lib = _lib.load()
        ws = None
        if dw is not None or db is not None:
            ws = _workspace(x.device, lib.hdrnet_conv2d_grad_workspace_bytes(B, H, W, cin, cout, k, ctx.stride))
        with torch.cuda.device(x.device):
            rc = lib.hdrnet_conv2d_grad_f32(
                x.data_ptr(), w.data_ptr(), out.data_ptr(), dy.data_ptr(), _ptr(dx), _ptr(dw), _ptr(db),
                B, H, W, cin, cout, k, ctx.stride, int(ctx.relu), _ptr(ws),
                0 if ws is None else ws.numel() * 4, _stream(x.device))
        _lib.check(rc, "conv2d VJP")
        return dx, dw, db, None, None, None, None


class _FcFn(torch.autograd.Function):
    """One fully connected layer (hdrnet/layers.py:62-93): forward hdrnet_fc_f32, backward
    hdrnet_fc_grad_f32."""

    @staticmethod
    def run(x, w, b, relu):
        b = None if b is None else b.contiguous()
        return _fc(x.contiguous(), (w.contiguous(), b), relu=relu)

    @staticmethod
    def forward(ctx, x, w, b, relu):
        x, w = x.contiguous(), w.contiguous()
        with torch.cuda.device(x.device):
            out = _FcFn.run(x, w, b, relu)
        ctx.save_for_backward(x, w, out)
        ctx.relu, ctx.has_bias = bool(relu), b is not None
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w, out = ctx.saved_tensors
        dy = dy.contiguous()
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        B, I = x.shape
        O = w.shape[1]
        dx = torch.empty_like(x) if need_x else None
        dw = torch.empty_like(w) if need_w else None
        db = torch.empty(O, dtype=torch.float32, device=x.device) if (need_b and ctx.has_bias) else None
        lib = _lib.load()
        ws = None
        if dw is not None or db is not None:
            ws = _workspace(x.device, lib.hdrnet_fc_grad_workspace_bytes(B, I, O))
        with torch.cuda.device(x.device):
            rc = lib.hdrnet_fc_grad_f32(
                x.data_ptr(), w.data_ptr(), out.data_ptr(), dy.data_ptr(), _ptr(dx), _ptr(dw), _ptr(db),
                B, I, O, int(ctx.relu), _ptr(ws), 0 if ws is None else ws.numel() * 4, _stream(x.device))
        _lib.check(rc, "fc VJP")
        return dx, dw, db, None


class _FusePredictFn(torch.autograd.Function):
    """Fusion + prediction + unroll_grid (models.py:122-139): forward hdrnet_fuse_predict_f32,
    backward hdrnet_fuse_predict_grad_f32 (fused = relu(local + global) is recomputed there from the
    saved local and global)."""

    @staticmethod
    def run(local, glob, w, b, gd, n_out, n_in):
        local, glob, w = local.contiguous(), glob.contiguous(), w.contiguous()
        b = None if b is None else b.contiguous()
        bs, gh, gw, C = local.shape
        grid = torch.empty((bs, gh, gw, gd, n_out, n_in), dtype=torch.float32, device=local.device)
        rc = _lib.load().hdrnet_fuse_predict_f32(
            local.data_ptr(), glob.data_ptr(), w.data_ptr(), _ptr(b), grid.data_ptr(), bs, gh, gw,
            C, gd, n_out, n_in, _stream(local.device))
        _lib.check(rc, "fuse_predict")
        return grid

    @staticmethod
    def forward(ctx, local, glob, w, b, gd, n_out, n_in):
        local, glob, w = local.contiguous(), glob.contiguous(), w.contiguous()
        with torch.cuda.device(local.device):
            grid = _FusePredictFn.run(local, glob, w, b, gd, n_out, n_in)
        ctx.save_for_backward(local, glob, w)
        ctx.dims, ctx.has_bias = (gd, n_out, n_in), b is not None
        return grid

    @staticmethod
    def backward(ctx, dgrid):
        local, glob, w = ctx.saved_tensors
        dgrid = dgrid.contiguous()
        gd, n_out, n_in = ctx.dims
        need_l, need_g, need_w, need_b = ctx.needs_input_grad[:4]
        bs, gh, gw, C = local.shape
        dl = torch.empty_like(local) if need_l else None
        dg = torch.empty_like(glob) if need_g else None
        dw = torch.empty_like(w) if need_w else None
        db = torch.empty(w.shape[1], dtype=torch.float32, device=w.device) if (need_b and ctx.has_bias) else None
        lib = _lib.load()
        ws = None
        if dw is not None or db is not None:
            ws = _workspace(local.device, lib.hdrnet_fuse_predict_grad_workspace_bytes(
                bs, gh, gw, C, gd, n_out, n_in))
        with torch.cuda.device(local.device):
            rc = lib.hdrnet_fuse_predict_grad_f32(
                local.data_ptr(), glob.data_ptr(), w.data_ptr(), dgrid.data_ptr(), _ptr(dl), _ptr(dg),
                _ptr(dw), _ptr(db), bs, gh, gw, C, gd, n_out, n_in, _ptr(ws),
                0 if ws is None else ws.numel() * 4, _stream(local.device))
        _lib.check(rc, "fuse_predict VJP")
        return dl, dg, dw, db, None, None, None


# [start, end) of each variable in the library's 112-float parameter gradient (include/hdrnet_b200.h)
_CURVES_GRAD_SLICES = ((0, 9), (9, 12), (12, 60), (60, 108), (108, 111), (111, 112))


def _var_shapes(variables):
    """(shape, device) of each tensor variable, None for the others: what _split_param_grad needs."""
    return [(v.shape, v.device) if isinstance(v, torch.Tensor) else None for v in variables]


def _split_param_grad(dp, needs, shapes, slices):
    """The gradient of each variable out of a guide VJP's flat parameter gradient `dp`: [start, end)
    in `slices`, None where it is not needed or the variable is no tensor.  A copy per variable:
    optimizers may update a .grad in place."""
    return [dp[a:b].reshape(s[0]).to(s[1], copy=True) if need and s is not None else None
            for need, s, (a, b) in zip(needs, shapes, slices)]


class _CurvesGuideFn(torch.autograd.Function):
    """The curves guide (hdrnet/models.py:145-190) over its six variables (_CURVES_VARS order):
    forward hdrnet_guide_curves_f32, the standalone guide kernel (the guide keeps its bits),
    backward hdrnet_guide_curves_grad_f32 with the host copies of the variables the forward used."""

    @staticmethod
    def forward(ctx, x, ccm, ccm_bias, shifts, slopes, mix, mix_bias):
        x = x.contiguous()
        ctx.guide = _CurvesGuide(ccm, ccm_bias, shifts, slopes, mix, mix_bias)
        ctx.save_for_backward(x)
        ctx.vars = _var_shapes((ccm, ccm_bias, shifts, slopes, mix, mix_bias))
        return ctx.guide.run(x)

    @staticmethod
    def backward(ctx, dguide):
        (x,) = ctx.saved_tensors
        dguide = dguide.contiguous()
        need_x = ctx.needs_input_grad[0]
        need_p = any(ctx.needs_input_grad[1:])
        B, H, W, _ = x.shape
        npix = B * H * W
        dx = torch.empty_like(x) if need_x else None
        dp = torch.empty(112, dtype=torch.float32, device=x.device) if need_p else None
        lib = _lib.load()
        ws = _workspace(x.device, lib.hdrnet_guide_curves_grad_workspace_bytes(npix)) if need_p else None
        with torch.cuda.device(x.device):
            rc = lib.hdrnet_guide_curves_grad_f32(
                x.data_ptr(), dguide.data_ptr(), _ptr(dx), npix, *ctx.guide.args,
                _ptr(dp), _ptr(ws), 0 if ws is None else ws.numel() * 4, _stream(x.device))
        _lib.check(rc, "guide_curves VJP")
        return (dx, *_split_param_grad(dp, ctx.needs_input_grad[1:], ctx.vars, _CURVES_GRAD_SLICES))


GUIDE = "inference/guide"   # the guide's variable scope; the pyramid's levels are GUIDE/level_{l}
_NN_GUIDE_VARS = ("conv1/weights", "conv1/BatchNorm/beta", "conv2/weights", "conv2/biases")
_NN_MOVING = ("conv1/BatchNorm/moving_mean", "conv1/BatchNorm/moving_variance")


def _guide_grad(wts, params, x, names, scope=GUIDE) -> bool:
    """Whether a guide goes through autograd: grad enabled, params['guide_grad'] truthy, and the input
    or one of the guide's variables `names` (under `scope`) requiring grad."""
    if not (torch.is_grad_enabled() and isinstance(params, dict) and params.get("guide_grad")):
        return False
    return _requires_grad(x) or (wts is not None and
                                 any(_requires_grad(wts.get(f"{scope}/{n}")) for n in names))


class _BatchStats(collections.namedtuple("_BatchStats", "npix moments guide mean var host count")):
    """conv1's batch statistics of one training-mode call: this call's pixel count, the input's
    moments (float64 [9]), the _NNGuide on the folded weights the guide kernel runs with, the
    features' batch mean and biased variance (float64), the host copies (_host_f32) of the four
    variables they were folded from, and the pixel count the statistics cover (npix, or the whole
    batch's under a process group)."""


def _nn_batch_stats(x, host) -> _BatchStats:
    """hdrnet_guide_nn_stats_f32 over x [B,H,W,3] (contiguous), one device-to-host copy of the 9
    moments, under a process group of several ranks their merge with the other ranks' moments
    (parallel.moments_over_ranks), then hdrnet_guide_nn_batch_fold in float64 on the host."""
    lib = _lib.load()
    npix = x.numel() // 3
    w1, beta = host[0], host[1]
    feats = beta.size
    moments = torch.empty(9, dtype=torch.float64, device=x.device)
    ws = _workspace(x.device, lib.hdrnet_guide_nn_stats_workspace_bytes(npix))
    rc = lib.hdrnet_guide_nn_stats_f32(x.data_ptr(), npix, moments.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                                       _stream(x.device))
    _lib.check(rc, "guide_nn batch statistics")
    mom, count = parallel.moments_over_ranks(moments.cpu().numpy(), npix)
    mom = np.ascontiguousarray(mom, np.float64)
    w1f, b1f = np.empty(3 * feats, np.float32), np.empty(feats, np.float32)
    mean, var = np.empty(feats, np.float64), np.empty(feats, np.float64)
    rc = lib.hdrnet_guide_nn_batch_fold(_hp(w1), _hp(beta), _hp(mom), feats, _hp(w1f), _hp(b1f), _hp(mean), _hp(var))
    _lib.check(rc, "guide_nn batch-norm fold")
    return _BatchStats(npix, mom, _NNGuide(w1f, b1f, host[2], host[3]), mean, var, host, count)


def _update_moving_averages(moving, stats: _BatchStats) -> None:
    """moving_mean and moving_variance toward the batch's statistics, in place, as TF's
    assign_moving_average without zero-debias: v -= (1 - decay) (v - batch).  The variance fed to it
    is Bessel-corrected, var N / (N - 1) (1 for N = 1), as TF's fused batch norm does (DESIGN.md §5),
    with N the pixel count of the whole batch the statistics cover."""
    n = stats.count
    unbiased = stats.var * (n / (n - 1.0) if n > 1 else 1.0)
    with torch.no_grad():
        for v, batch in zip(moving, (stats.mean, unbiased)):
            b = torch.from_numpy(batch.astype(np.float32)).to(v.device).reshape(v.shape)
            v.sub_((v - b) * (1.0 - BN_DECAY))


def _moving_averages(wts, scope=GUIDE, names=_NN_MOVING):
    """The moving averages of the NN guide under `scope` (or `names` under it), which training mode
    updates in place: float32 tensors that do not require grad (TF does not train them)."""
    out = []
    for n in names:
        key = f"{scope}/{n}"
        v = wts.get(key) if isinstance(wts, dict) else None
        if not isinstance(v, torch.Tensor) or v.dtype != torch.float32:
            raise TypeError(f"{key} must be a float32 torch.Tensor: is_training=True updates it in place "
                            f"(got {type(v).__name__ if not isinstance(v, torch.Tensor) else v.dtype})")
        if v.requires_grad:
            raise ValueError(f"{key} requires grad: moving averages are not trainable; is_training=True "
                             "updates them in place")
        out.append(v)
    return out


# ---- the coefficient network's batch norm in training mode (csrc/bn_train.cu) -------------------
_BN_MOVING = ("BatchNorm/moving_mean", "BatchNorm/moving_variance")


def _coefficient_batch_stats(params) -> bool:
    """Whether the coefficient network's batch-norm layers run in training mode when is_training is
    set: params['coefficient_batch_stats'] truthy with params['batch_norm'].  The key without
    batch_norm is a ValueError (there is no such layer to run)."""
    if not (isinstance(params, dict) and params.get("coefficient_batch_stats")):
        return False
    if not params.get("batch_norm"):
        raise ValueError("params['coefficient_batch_stats'] runs the coefficient network's batch-norm layers in "
                         "training mode; params['batch_norm'] is not set, so it has none")
    return True


def _bn_relu(z: torch.Tensor, beta: torch.Tensor, moving) -> tuple:
    """One batch-norm layer in training mode over z [..., C] (the conv or fc output without bias or
    relu, contiguous): (y, moments).  moments [3, C] float64 (count, mean, M2) are those of the whole
    batch, merged over the ranks under a process group (parallel.bn_moments_over_ranks); the moving
    averages `moving` (mean, variance) move toward them in place.  No host synchronisation."""
    lib = _lib.load()
    C = z.shape[-1]
    N = z.numel() // C
    moments = torch.empty((3, C), dtype=torch.float64, device=z.device)
    ws = _workspace(z.device, lib.hdrnet_bn_stats_workspace_bytes(N, C))
    rc = lib.hdrnet_bn_stats_f32(z.data_ptr(), N, C, moments.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                                 _stream(z.device))
    _lib.check(rc, "batch-norm statistics")
    moments = parallel.bn_moments_over_ranks(moments)
    y = torch.empty_like(z)
    rc = lib.hdrnet_bn_relu_f32(z.data_ptr(), N, C, moments.data_ptr(), beta.data_ptr(), y.data_ptr(),
                                moving[0].data_ptr(), moving[1].data_ptr(), _stream(z.device))
    _lib.check(rc, "batch norm + relu")
    return y, moments


class _BatchNormReluFn(torch.autograd.Function):
    """relu(batch_norm(z) + beta) in training mode over z and beta (hdrnet/layers.py:47-54,
    center=True, scale=False); `moving` is the pair of moving averages it updates, not
    differentiated.  Backward: hdrnet_bn_relu_grad_sums_f32, the sums merged over the ranks
    (parallel.bn_sums_over_ranks), then hdrnet_bn_relu_grad_f32.  d beta is this rank's own sum, its
    share of the whole batch's."""

    @staticmethod
    def run(z, beta, moving):
        return _bn_relu(z.contiguous(), beta.contiguous(), moving)[0]

    @staticmethod
    def forward(ctx, z, beta, moving):
        z, beta = z.contiguous(), beta.contiguous()
        with torch.cuda.device(z.device):
            y, moments = _bn_relu(z, beta, moving)
        ctx.save_for_backward(z, beta, moments)
        return y

    @staticmethod
    def backward(ctx, dy):
        z, beta, moments = ctx.saved_tensors
        dy = dy.contiguous()
        C = z.shape[-1]
        N = z.numel() // C
        lib = _lib.load()
        dbeta = torch.empty(C, dtype=torch.float32, device=z.device) if ctx.needs_input_grad[1] else None
        dz = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        sums = torch.empty((2, C), dtype=torch.float64, device=z.device)
        with torch.cuda.device(z.device):
            ws = _workspace(z.device, lib.hdrnet_bn_stats_workspace_bytes(N, C))
            rc = lib.hdrnet_bn_relu_grad_sums_f32(z.data_ptr(), dy.data_ptr(), N, C, moments.data_ptr(),
                                                  beta.data_ptr(), sums.data_ptr(), _ptr(dbeta), ws.data_ptr(),
                                                  ws.numel() * 4, _stream(z.device))
            _lib.check(rc, "batch-norm VJP sums")
            sums = parallel.bn_sums_over_ranks(sums)    # every rank joins, whatever it needs
            if dz is not None:
                rc = lib.hdrnet_bn_relu_grad_f32(z.data_ptr(), dy.data_ptr(), N, C, moments.data_ptr(),
                                                 beta.data_ptr(), sums.data_ptr(), dz.data_ptr(), _stream(z.device))
                _lib.check(rc, "batch-norm VJP")
        return dz, dbeta, None


class _NNGuideFn(torch.autograd.Function):
    """The pointwise-NN guide in training mode (hdrnet/models.py:203-210, batch norm with the batch's
    statistics) over x and its four variables (_NN_GUIDE_VARS order); `stats` is _nn_batch_stats of
    x.  Forward: the existing guide kernel on the folded weights.  Backward:
    hdrnet_guide_nn_grad_f32, whose gradients include the paths through the batch mean and variance."""

    @staticmethod
    def forward(ctx, x, w1, beta, w2, b2, stats):
        x = x.contiguous()
        ctx.save_for_backward(x)
        ctx.stats = stats
        ctx.vars = _var_shapes((w1, beta, w2, b2))
        return stats.guide.run(x)

    @staticmethod
    def backward(ctx, dguide):
        (x,) = ctx.saved_tensors
        dguide = dguide.contiguous()
        need_x = ctx.needs_input_grad[0]
        need_p = any(ctx.needs_input_grad[1:5])
        st = ctx.stats
        w1, beta, w2, b2 = st.host
        F = beta.size
        npix = st.npix
        dx = torch.empty_like(x) if need_x else None
        dp = torch.empty(5 * F + 1, dtype=torch.float32, device=x.device) if need_p else None
        lib = _lib.load()
        ws = _workspace(x.device, lib.hdrnet_guide_nn_grad_workspace_bytes(npix, F))
        with torch.cuda.device(x.device):
            rc = lib.hdrnet_guide_nn_grad_f32(
                x.data_ptr(), dguide.data_ptr(), _ptr(dx), npix, _hp(w1), _hp(beta), _hp(w2), float(b2[0]), F,
                _hp(st.moments), _ptr(dp), ws.data_ptr(), ws.numel() * 4, _stream(x.device))
        _lib.check(rc, "guide_nn VJP")
        slices = ((0, 3 * F), (3 * F, 4 * F), (4 * F, 5 * F), (5 * F, 5 * F + 1))
        return (dx, *_split_param_grad(dp, ctx.needs_input_grad[1:5], ctx.vars, slices), None)


def _requires_grad(t) -> bool:
    return isinstance(t, torch.Tensor) and t.requires_grad


def _trainable_keys(wts, prefix: str):
    return sorted(k for k, v in wts.items() if k.startswith(prefix) and _requires_grad(v))


def _refuse_untrained(wts, params, lowres_input=None, fullres_input=None, what=None, nn_guide=False,
                      is_training=False, bn_training=False, curves_model="HDRNetCurves") -> None:
    """NotImplementedError for every gradient this package does not compute (checked before any
    device work).  `what`: refuse the whole model's gradient (HDRNetGaussianPyrNN's inference form).
    The curves guide's variables and fullres_input are differentiated only with params['guide_grad'], the
    pointwise-NN guide's only with params['guide_grad'] and `is_training` (training-mode batch norm).
    `bn_training`: the coefficient network's batch-norm layers run in training mode
    (_coefficient_batch_stats), so their variables may require grad.  `curves_model`: the curves-guide
    model the messages name."""
    if not torch.is_grad_enabled() or wts is None:
        return
    if what is not None:
        wanted = _trainable_keys(wts, "inference/") + \
            [n for n, t in (("lowres_input", lowres_input), ("fullres_input", fullres_input)) if _requires_grad(t)]
        if wanted:
            raise NotImplementedError(f"{what}: the inference form, with batch norm folded from the moving "
                                      f"averages, is not differentiated (a gradient was requested for {wanted[0]}); "
                                      "inference(..., is_training=True), the training graph, is")
        return
    guide = _trainable_keys(wts, "inference/guide")
    guide_grad = bool(params.get("guide_grad")) if isinstance(params, dict) else False
    if guide_grad and nn_guide and not is_training and (guide or _requires_grad(fullres_input)):
        wanted = guide[0] if guide else "fullres_input"
        raise NotImplementedError(
            f"gradients for the pointwise-NN guide variables and its fullres_input are not implemented ({wanted} "
            "requires grad): its conv1 has batch norm, which training runs in training mode with batch "
            "statistics, a different forward; inference(..., is_training=True) runs that forward and "
            "differentiates it")
    hint = f"; params['guide_grad'] computes them for {curves_model}"
    if guide and not guide_grad:
        raise NotImplementedError(f"gradients for the guide variables are not implemented ({guide[0]} requires "
                                  "grad): the guide is held fixed; set requires_grad=False on its variables"
                                  + ("" if nn_guide else hint))
    if _requires_grad(fullres_input) and not guide_grad:
        raise NotImplementedError("gradients for fullres_input are not implemented: they need the guide's "
                                  "backward; pass it with requires_grad=False" + ("" if nn_guide else hint))
    if not bn_training:
        _refuse_batch_norm(wts, params)


def _refuse_batch_norm(wts, params) -> None:
    if not torch.is_grad_enabled() or wts is None:
        return
    for scope, use_bn, _ in _coefficient_specs(params):
        if use_bn:
            _refuse_batch_norm_scope(wts, scope)


def _refuse_batch_norm_scope(wts, scope) -> None:
    """A batch-norm layer is folded in its inference form: its variables get no gradient."""
    keys = _trainable_keys(wts, scope + "/") if torch.is_grad_enabled() else []
    if keys:
        raise NotImplementedError(
            f"gradients through a batch-norm layer are not implemented ({keys[0]} requires grad): "
            "training-mode batch norm uses batch statistics, a different forward")


class HDRNetCurves(object):
    """Main model, as submitted in January 2017 (hdrnet/models.py:30-196)."""

    _nn_guide = False

    @classmethod
    def n_out(cls):
        return 3

    @classmethod
    def n_in(cls):
        return 3 + 1

    @classmethod
    def inference(cls, lowres_input, fullres_input, params, is_training=False):
        """models.py:43-59.  lowres_input [B,S,S,3], fullres_input [B,H,W,3] -> [B,H,W,3].
        With params['debug'] truthy also stores the coefficients and guide on
        ``cls.last_debug`` (the collections run.py --debug reads, run.py:98-133).

        With coefficient-network variables (or lowres_input) requiring grad, the coefficients come
        from autograd and the output from the standalone guide kernel and
        hdrnet_ops.bilateral_slice_apply, whose VJP carries the gradient back to the grid.  The guide
        is a constant there unless params['guide_grad'] is truthy and a curves-guide variable or
        fullres_input requires grad: then it is _CurvesGuideFn, whose VJP takes the slice-apply's
        guide gradient to the guide variables and adds its input gradient to the slice-apply's.

        ``is_training=True`` needs params['coefficient_batch_stats'] with params['batch_norm'] (else
        NotImplementedError): the coefficient network's batch-norm layers then normalise with the
        batch's statistics and move their moving averages, as _coefficients(..., is_training=True)."""
        bn_training = _coefficient_batch_stats(params)
        if is_training and not bn_training:
            raise NotImplementedError("hdrnet_b200 implements the inference path only")
        wts = _weights_or_none(params)
        _refuse_untrained(wts, params, fullres_input=fullres_input, nn_guide=bool(cls._nn_guide),
                          bn_training=bool(is_training))
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, is_training)
        if coeffs.requires_grad or (not cls._nn_guide and _guide_grad(wts, params, fullres_input, _CURVES_VARS)):
            return cls._output(fullres_input, cls._guide(fullres_input, params, is_training), coeffs)
        return cls._fullres(coeffs, fullres_input, params, torch.float32)

    @classmethod
    def inference_image(cls, image, params, lowres_image=None, out_dtype=torch.uint8):
        """The reference CLI's per-image path (hdrnet/bin/run.py:145-190) with the decoded image
        kept in its storage format on the device: ``image`` [B,H,W,3] uint8 / uint16 / float32
        -> nearest-neighbour S x S float32 network input (img_as_float on the fly, run.py:156-169)
        -> coefficients -> guide + slice + apply in one full-resolution pass that reads the
        integer pixels and writes ``uint8(255 * clip(out, 0, 1))`` (run.py:95).  3 + 3 bytes per
        pixel cross PCIe / HBM instead of 12 + 12.  ``lowres_image`` replaces the resized input
        (run.py --lowres_input); ``out_dtype=torch.float32`` returns the unquantised prediction and
        ``out_dtype=torch.uint16`` the 16-bit one, ``rint(65535 * clip(out, 0, 1))`` written by the
        same kernel (6 bytes per pixel).  Any other ``out_dtype`` is a TypeError."""
        _check_out_dtype(out_dtype)
        image = _check_image(image, "image")
        src = image if lowres_image is None else _check_image(lowres_image, "lowres_image")
        lowres = lowres_from_image(src, int(params["net_input_size"]))
        coeffs = cls._coefficients(lowres, params, False)
        return cls._fullres(coeffs, image, params, out_dtype)

    @classmethod
    def inference_images(cls, images, params, lowres_images=None, out_dtype=torch.uint8):
        """``inference_image`` over a ragged batch: ``images`` is a list of CUDA [H_i, W_i, 3] tensors
        of one dtype (uint8 / uint16 / float32), each of its own size -> a list of [H_i, W_i, 3]
        tensors of ``out_dtype``.  The coefficient network runs once on the whole batch; the network
        inputs and the full-resolution pass are one launch each over all the images (per
        RAGGED_MAX_IMAGES images).  Image i's result is ``_fullres`` of grid row i, bit for bit
        (DESIGN.md row f-13 names the one exception, float32 -> float32 images the row kernels do not
        take).  ``lowres_images`` (a list of as many images) replaces the resized inputs.  Mixed dtypes
        raise TypeError and mixed devices ValueError, before any device work; [] returns []."""
        images, sources = _ragged_inputs(images, lowres_images, out_dtype, params)
        if not images:
            return []
        lowres = lowres_from_images(sources, int(params["net_input_size"]))
        coeffs = cls._coefficients(lowres, params, False)
        return cls._fullres_images(coeffs, images, params, out_dtype)

    @classmethod
    def _fullres_images(cls, coeffs, images, params, out_dtype):
        """_fullres over a ragged batch: one guide + slice + apply launch for all the images."""
        prep = _prepare(_resolve_weights(params), params, images[0].device, cls._nn_guide)
        return _slice_apply_fused_ragged(coeffs, images, prep.guides[0], out_dtype)

    @classmethod
    def inference_image_host(cls, frames, params, out=None, device=None, out_dtype=torch.uint8):
        """``inference_image`` for frames that live in HOST memory (what hdrnet/bin/run.py does per
        file: load, ``sess.run``, save): uploads, the model and downloads of consecutive frames
        overlap on three streams (hdrnet_b200/host_pipeline.py).  ``frames`` [N,H,W,3] uint8 /
        uint16 / float32 CPU tensor (pinned for asynchronous copies) -> CPU tensor of ``out_dtype``
        (uint8, uint16 or float32).  One pipeline (streams + two frame buffers) is kept per (class,
        device, out_dtype)."""
        _check_out_dtype(out_dtype)
        from .host_pipeline import HostImagePipeline
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        key = (cls, dev, out_dtype)
        pipe = _host_pipelines.get(key)
        if pipe is None:
            pipe = _host_pipelines.setdefault(key, HostImagePipeline(cls, params, dev, out_dtype=out_dtype))
        pipe.params = params
        return pipe(frames, out)

    @classmethod
    def _fullres(cls, coeffs, fullres_input, params, out_dtype):
        """Guide + slice + apply over the full-resolution image (models.py:53-58), one kernel."""
        prep = _prepare(_resolve_weights(params), params, fullres_input.device, cls._nn_guide)
        debug = bool(params.get("debug"))
        out, guide = _slice_apply_fused(coeffs, fullres_input, prep.guides[0], out_dtype, debug, True)
        if debug:
            cls.last_debug = {"bilateral_coefficients": coeffs, "guide": guide, "output": out}
        return out

    @classmethod
    def _coefficients(cls, input_tensor, params, is_training=False):
        """models.py:62-142 -> [B, gh, gw, gd, n_out, n_in].  ``is_training=True`` runs the batch-norm
        layers in training mode (_coefficients_training) when _coefficient_batch_stats says so, and
        raises NotImplementedError otherwise."""
        if is_training:
            if not _coefficient_batch_stats(params):
                raise NotImplementedError("hdrnet_b200 implements the inference path only")
            return cls._coefficients_training(input_tensor, params)
        _coefficient_batch_stats(params)
        _refuse_batch_norm(_weights_or_none(params), params)
        x = _check_input(input_tensor, "lowres_input")
        prep = _prepare(_resolve_weights(params), params, x.device, cls._nn_guide)
        grad = torch.is_grad_enabled() and (x.requires_grad or any(
            _requires_grad(t) for wb in prep.layers.values() for t in wb[:2]))
        # small batches: the whole network behind one library call (launch chain, csrc/cnn.cu)
        if not grad and x.shape[0] <= CHAIN_CNN_MAX_BATCH:
            grid = cls._coefficients_chain(x, prep, params)
            if grid is not None:
                return grid
        n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
        return cls._coefficients_layers(x, prep.layers, params["luma_bins"], n_ds, grad)

    @classmethod
    def _coefficients_layers(cls, x, L, gd, n_ds, grad, bn=None):
        """Layer by layer over the prepared weights: with `grad` every layer an autograd Function
        (backward through csrc/cnn_grad.cu), else only its forward (`run`).  `bn` maps the scope of
        each layer that runs batch norm in training mode to its (beta, moving averages): that layer
        runs without bias or relu, then _BatchNormReluFn, and every conv of the network then runs on the
        CUDA cores (float32 rounded to nearest): batch norm divides a conv's rounding error by the
        channel's spread, and the 3xTF32 tensor-core form's error, about 1e-6 of a product, would
        reach the gradients at 1e-3 to 1e-2 of their range (DESIGN.md row f-14)."""
        conv_fn, fc_fn, fuse_fn, bn_fn = (f.apply if grad else f.run
                                          for f in (_ConvFn, _FcFn, _FusePredictFn, _BatchNormReluFn))
        p = "inference/coefficients"
        bs = x.shape[0]
        bn = bn or {}

        tc = not bn

        def conv(x, scope, stride, relu=True):
            w, b, packed = L[f"{p}/{scope}"]
            if f"{p}/{scope}" in bn:
                return bn_fn(conv_fn(x, w, None, stride, False, packed, tc), *bn[f"{p}/{scope}"])
            return conv_fn(x, w, b, stride, relu, packed, tc)

        def fc(x, scope, relu=True):
            w, b = L[f"{p}/{scope}"][:2]
            if f"{p}/{scope}" in bn:
                return bn_fn(fc_fn(x, w, None, False), *bn[f"{p}/{scope}"])
            return fc_fn(x, w, b, relu)

        with torch.cuda.device(x.device):
            for i in range(n_ds):                                   # splat, :69-82
                x = conv(x, f"splat/conv{i + 1}", 2)
            splat = x
            g = conv(splat, "global/conv1", 2)                      # global, :86-105
            g = conv(g, "global/conv2", 2)
            g = g.reshape(bs, -1)                                   # NHWC flatten, :94-95
            g = fc(g, "global/fc1")
            g = fc(g, "global/fc2")
            g = fc(g, "global/fc3", False)
            loc = conv(splat, "local/conv1", 1)                     # local, :109-118
            loc = conv(loc, "local/conv2", 1, relu=False)
            wp, bp = L[f"{p}/prediction/conv1"][:2]                 # HWIO [1, 1, C, O] -> [C, O]
            # fusion + prediction + unroll, :122-139
            return fuse_fn(loc, g, wp.reshape(wp.shape[-2:]), bp, gd, cls.n_out(), cls.n_in())

    @classmethod
    def _coefficients_training(cls, input_tensor, params):
        """The coefficient network with its batch-norm layers in training mode (hdrnet/layers.py:47-54,
        is_training=True): each normalises with the batch's statistics (the whole batch's under a
        process group) and moves its ``BatchNorm/moving_mean`` and ``moving_variance`` (float32 tensors
        on the input's device that do not require grad) in place, once per call.  Layer by layer on
        the raw variables, nothing folded and no host synchronisation; ``weights``, ``BatchNorm/beta``,
        the other layers' variables and ``lowres_input`` are differentiated where they require grad."""
        wts = _resolve_weights(params)
        specs = _coefficient_specs(params)
        moving = {scope: _moving_averages(wts, scope, _BN_MOVING) for scope, use_bn, _ in specs if use_bn}
        x = _check_input(input_tensor, "lowres_input")
        if x.shape[0] == 0:
            raise ValueError("lowres_input is empty: batch statistics need at least one image")
        for scope, pair in moving.items():
            for name, v in zip(_BN_MOVING, pair):
                if v.device != x.device or not v.is_contiguous():
                    raise ValueError(f"{scope}/{name} must be a contiguous tensor on {x.device}: is_training=True "
                                     "updates it in place there")
        dev = x.device
        layers_, bn = {}, {}
        with torch.cuda.device(dev):
            for scope, use_bn, use_bias in specs:
                w = _device_var(wts[scope + "/weights"], dev)
                b = _device_var(wts[scope + "/biases"], dev) if use_bias and not use_bn else None
                layers_[scope] = (w, b, None)      # the convs run on the CUDA cores (_coefficients_layers)
                if use_bn:
                    bn[scope] = (_device_var(wts[scope + "/BatchNorm/beta"], dev), moving[scope])
        grad = torch.is_grad_enabled() and (x.requires_grad or any(
            _requires_grad(t) for wb in layers_.values() for t in wb[:2]) or
            any(_requires_grad(beta) for beta, _ in bn.values()))
        n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
        return cls._coefficients_layers(x, layers_, params["luma_bins"], n_ds, grad, bn)

    @classmethod
    def _coefficients_chain(cls, x, prep, params):
        """One library call for all layers; None when the library does not take the shape."""
        lib = _lib.load()
        bs, S = x.shape[0], x.shape[1]
        gd, cm, sb = params["luma_bins"], params["channel_multiplier"], params["spatial_bin"]
        nbytes = lib.hdrnet_coefficients_scratch_bytes(bs, S, sb, gd, cm, cls.n_out(), cls.n_in())
        if nbytes == 0 or x.shape[2] != S:
            return None
        order = [scope for scope, _, _ in _coefficient_specs(params)]
        ptrs = getattr(prep, "_pc_ptrs", None)
        if ptrs is None:     # host arrays of device pointers, built once per prepared model
            n = len(order)
            wa, ba = (ctypes.c_void_p * n)(), (ctypes.c_void_p * n)()
            for i, scope in enumerate(order):
                w, b = prep.layers[scope][:2]
                wa[i] = w.data_ptr()
                ba[i] = None if b is None else b.data_ptr()
            ptrs = prep._pc_ptrs = (wa, ba)
        scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=x.device)
        grid = torch.empty((bs, sb, sb, gd, cls.n_out(), cls.n_in()), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = lib.hdrnet_coefficients_f32(x.data_ptr(), grid.data_ptr(), ptrs[0], ptrs[1], len(order),
                                             scratch.data_ptr(), nbytes, bs, S, sb, gd, cm, cls.n_out(),
                                             cls.n_in(), torch.cuda.current_stream(x.device).cuda_stream)
        if rc == _lib.E_UNSUPPORTED:
            return None
        _lib.check(rc, "coefficients (launch chain)")
        return grid

    @classmethod
    def _guide(cls, input_tensor, params, is_training=False, scope=GUIDE):
        """models.py:145-190 as a standalone kernel -> [B, H, W].  Differentiable (_CurvesGuideFn)
        when _guide_grad says so.  ``scope``: the guide's variable scope (the pyramid's
        GUIDE/level_{l})."""
        x = _check_input(input_tensor, "fullres_input")
        wts = _resolve_weights(params)
        if _guide_grad(wts, params, x, _CURVES_VARS, scope):
            with torch.cuda.device(x.device):
                return _CurvesGuideFn.apply(x, *[wts[f"{scope}/{n}"] for n in _CURVES_VARS])
        if is_training or scope != GUIDE:   # the coefficient layers are not prepared (folded, packed) for the guide alone
            return _CurvesGuide.from_weights(wts, scope).run(x)
        return _prepare(wts, params, x.device, False).guides[0].run(x)

    @classmethod
    def _output(cls, im, guide, coeffs):
        """models.py:193-196."""
        return bilateral_slice_apply(coeffs, guide, im, has_offset=True, name="slice")


class HDRNetPointwiseNNGuide(HDRNetCurves):
    """Replaces the pointwise curves in the guide by a pointwise neural net
    (hdrnet/models.py:199-210)."""

    _nn_guide = True

    @classmethod
    def inference(cls, lowres_input, fullres_input, params, is_training=False):
        """models.py:43-59.  With ``is_training=True`` the reference's training graph
        (hdrnet/bin/train.py:89-115): the guide's conv1 batch norm normalises with the batch's
        statistics and its ``moving_mean`` / ``moving_variance`` (float32 tensors in the weights dict)
        move toward them in place, once per call (decay 0.999).  The coefficient network is the
        inference graph, which is its training graph without batch norm; ``params['batch_norm']``
        raises ``NotImplementedError``.  The output comes from hdrnet_ops.bilateral_slice_apply, and
        with ``params['guide_grad']`` the guide's variables (``conv1/weights``,
        ``conv1/BatchNorm/beta``, ``conv2/*``) and ``fullres_input`` are differentiated through
        _NNGuideFn; without it they are held fixed, while batch norm still uses the batch's
        statistics."""
        if not is_training:
            return super().inference(lowres_input, fullres_input, params)
        wts = _resolve_weights(params)
        bn_training = _coefficient_batch_stats(params)
        if params.get("batch_norm") and not bn_training:
            raise NotImplementedError(
                "training-mode batch norm in the coefficient network (params['batch_norm']) is not "
                "implemented: only the guide's conv1 batch norm runs in training mode; "
                "params['coefficient_batch_stats'] runs the coefficient network's in training mode too")
        _moving_averages(wts)
        _refuse_untrained(wts, params, fullres_input=fullres_input, nn_guide=True, is_training=True,
                          bn_training=bn_training)
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, bn_training)
        return cls._output(fullres_input, cls._guide(fullres_input, params, is_training=True), coeffs)

    @classmethod
    def _guide(cls, input_tensor, params, is_training=False, scope=GUIDE):
        """models.py:199-210 -> [B, H, W].  Inference form: conv1's batch norm folded from the moving
        averages.  ``is_training=True``: normalised with the batch's statistics (_nn_batch_stats), the
        moving averages updated in place, and differentiable (_NNGuideFn) when _guide_grad says so.
        Under a process group of several ranks the statistics are the whole batch's, every rank's
        shard included; the parameter gradients are then this rank's share of the whole batch's
        (their sum over the ranks), and ``fullres_input`` requiring grad raises NotImplementedError.
        ``scope``: the training branch's variable scope (the pyramid's GUIDE/level_{l})."""
        if is_training:
            wts = _resolve_weights(params)
            moving = _moving_averages(wts, scope)
            _refuse_untrained(wts, params, fullres_input=input_tensor, nn_guide=True, is_training=True,
                              bn_training=_coefficient_batch_stats(params))
            x = _check_input(input_tensor, "fullres_input")
            if x.numel() == 0:
                raise ValueError("fullres_input is empty: batch statistics need at least one pixel")
            variables = [wts[f"{scope}/{n}"] for n in _NN_GUIDE_VARS]
            if parallel.world_size() > 1 and _requires_grad(x) and _guide_grad(wts, params, x, _NN_GUIDE_VARS, scope):
                # each pixel's dinput depends on sums over the whole batch, which the VJP has for its own rank only
                raise NotImplementedError(
                    "the gradient of fullres_input through batch statistics taken over several ranks is not "
                    "implemented: the guide's variables are differentiated, fullres_input must not require grad")
            with torch.cuda.device(x.device):
                x = x.contiguous()
                stats = _nn_batch_stats(x, [_host_f32(v) for v in variables])
                _update_moving_averages(moving, stats)
                if _guide_grad(wts, params, x, _NN_GUIDE_VARS, scope):
                    return _NNGuideFn.apply(x, *variables, stats)
                return stats.guide.run(x)
        x = _check_input(input_tensor, "fullres_input")
        return _prepare(_resolve_weights(params), params, x.device, True).guides[0].run(x)


def _resize(x: torch.Tensor, oh: int, ow: int, add: torch.Tensor | None = None) -> torch.Tensor:
    """tf.image.resize_images(x, [oh, ow], BILINEAR, align_corners=True) (+ fused add)."""
    B, H, W, C = x.shape
    out = torch.empty((B, oh, ow, C), dtype=torch.float32, device=x.device)
    rc = _lib.load().hdrnet_resize_bilinear_f32(
        x.data_ptr(), 0 if add is None else add.data_ptr(), out.data_ptr(), B, H, W, C, oh, ow,
        torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "resize_bilinear")
    return out


class _ResizeFn(torch.autograd.Function):
    """_resize (+ fused add) over x and add: forward hdrnet_resize_bilinear_f32, the same kernel, so
    the output keeps its bits; backward hdrnet_resize_bilinear_grad_f32 for x, and the identity for
    add."""

    @staticmethod
    def forward(ctx, x, oh, ow, add=None):
        x = x.contiguous()
        ctx.in_hw = x.shape[1:3]
        with torch.cuda.device(x.device):
            return _resize(x, oh, ow, None if add is None else add.contiguous())

    @staticmethod
    def backward(ctx, dout):
        dout = dout.contiguous()
        din = None
        if ctx.needs_input_grad[0]:
            B, OH, OW, C = dout.shape
            H, W = ctx.in_hw
            din = torch.empty((B, H, W, C), dtype=torch.float32, device=dout.device)
            with torch.cuda.device(dout.device):
                rc = _lib.load().hdrnet_resize_bilinear_grad_f32(dout.data_ptr(), din.data_ptr(), B, H, W, C,
                                                                 OH, OW, _stream(dout.device))
            _lib.check(rc, "resize_bilinear VJP")
        return din, None, None, (dout if ctx.needs_input_grad[3] else None)


def _resize_maybe_grad(x, oh, ow, add=None):
    """_resize, through _ResizeFn when grad is enabled and x or add requires it."""
    if torch.is_grad_enabled() and (_requires_grad(x) or _requires_grad(add)):
        return _ResizeFn.apply(x, oh, ow, add)
    return _resize(x, oh, ow, add)


class _GaussianPyramid:
    """The pyramid of hdrnet/models.py:213-289, shared by HDRNetGaussianPyrNN and HDRNetGaussianPyr,
    which differ only in the guide each level runs (their _nn_guide and _guide): 3-level bilinear
    (align_corners) pyramid of the full-res image, one guide per level, one slice-apply per level
    with its own 3 of the 9 output rows of the coefficient grid, coarse-to-fine upsample-and-add.
    The reference file is Python-2 only here (`reversed(zip(...))`, :278); the semantics restated:
    the COARSEST level uses output rows 0..2, the finest rows 6..8."""

    @classmethod
    def n_scales(cls):
        return 3

    @classmethod
    def n_out(cls):
        return 3 * cls.n_scales()

    @classmethod
    def n_in(cls):
        return 3 + 1

    @classmethod
    def _guide_scopes(cls):
        return [f"{GUIDE}/level_{il}" for il in range(cls.n_scales())]

    @classmethod
    def inference_image(cls, image, params, lowres_image=None, out_dtype=torch.uint8):
        """Same contract as HDRNetCurves.inference_image.  The pyramid needs the float image at
        three scales, so only the network input is taken straight from the integer pixels; the
        full-resolution image is converted once on the device.  The float result of the three
        levels' sum is quantised once, on the device (quantize_u8 / quantize_u16)."""
        _check_out_dtype(out_dtype)
        image = _check_image(image, "image")
        src = image if lowres_image is None else _check_image(lowres_image, "lowres_image")
        lowres = lowres_from_image(src, int(params["net_input_size"]))
        out = cls.inference(lowres, image_to_float(image), params, False)
        if out_dtype == torch.uint8:
            return quantize_u8(out)
        return quantize_u16(out) if out_dtype == torch.uint16 else out

    @classmethod
    def _fullres_images(cls, coeffs, images, params, out_dtype):
        """The pyramid over a ragged batch: the coefficients of all the images come from one network
        call; the full-resolution stages (float image, level resizes, three slice-applies, upsample
        and add) run image by image, as inference_image runs them on one image (there is no ragged
        form of the resizes)."""
        outs = []
        with torch.cuda.device(images[0].device):
            for i, image in enumerate(images):
                out = cls._output(cls._multiscale_input(image_to_float(image[None])), None, coeffs[i:i + 1], params)
                if out_dtype == torch.uint8:
                    out = quantize_u8(out)
                elif out_dtype == torch.uint16:
                    out = quantize_u16(out)
                outs.append(out[0])
        return outs

    @classmethod
    def _multiscale_input(cls, fullres_input):
        """models.py:249-262: each level is the previous one resized to floor(size / 2);
        differentiable (_ResizeFn) when fullres_input requires grad."""
        lvls = [fullres_input]
        h, w = fullres_input.shape[1:3]
        for _ in range(cls.n_scales() - 1):
            h, w = h // 2, w // 2
            lvls.append(_resize_maybe_grad(lvls[-1], h, w))
        return lvls

    @classmethod
    def _output(cls, lvls, guide_lvls, coeffs, params=None):
        """models.py:274-289, coarse to fine.  With guide_lvls=None (the fast path) each level's
        guide is computed inside its slice-apply kernel; given the guides, hdrnet_ops' slice-apply
        runs on them, and the upsample-and-add is differentiable (_ResizeFn) where grad is on."""
        prep = _prepare(_resolve_weights(params), params, lvls[0].device, cls._nn_guide) \
            if guide_lvls is None else None
        B, gh, gw, gd = coeffs.shape[:4]
        current = None
        for il in range(cls.n_scales()):
            src = cls.n_scales() - 1 - il                       # reversed(zip(lvls, guides))
            lvl = lvls[src]
            c = coeffs[:, :, :, :, il * 3:(il + 1) * 3, :].contiguous().reshape(B, gh, gw, gd, 12)
            _, H, W, _ = lvl.shape
            if guide_lvls is not None:
                out_lvl = bilateral_slice_apply(c, guide_lvls[src], lvl, has_offset=True)
            else:
                out_lvl = _slice_apply_fused(c, lvl, prep.guides[src], torch.float32, False, False)[0]
            current = out_lvl if il == 0 else _resize_maybe_grad(current, H, W, add=out_lvl)
        return current


class HDRNetGaussianPyrNN(_GaussianPyramid, HDRNetPointwiseNNGuide):
    """Replace input to the affine model by a pyramid (hdrnet/models.py:213-289): the pyramid of
    _GaussianPyramid with one pointwise-NN guide per level."""

    _nn_guide = "pyramid"

    @classmethod
    def inference(cls, lowres_input, fullres_input, params, is_training=False):
        """models.py:213-247.  The inference form (``is_training=False``) folds each level's conv1
        batch norm from its moving averages and runs each level's guide inside its slice-apply; it
        is not differentiated.  ``is_training=True`` is the reference's training graph
        (hdrnet/bin/train.py:89-115), as HDRNetPointwiseNNGuide's: each level's guide normalises
        conv1 with that level's batch statistics and moves ``level_{l}/conv1/BatchNorm/moving_mean``
        and ``moving_variance`` toward them in place, once per call.  The coefficient variables and
        ``lowres_input`` are differentiated; with ``params['guide_grad']`` so are each level's guide
        variables and ``fullres_input``, through _NNGuideFn and the resize VJP (_ResizeFn)."""
        if is_training:
            return cls._inference_training(lowres_input, fullres_input, params)
        _refuse_untrained(_weights_or_none(params), params, lowres_input, fullres_input,
                          what="HDRNetGaussianPyrNN.inference (needs the VJP of the align-corners resize)")
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, is_training)       # [B,gh,gw,gd,9,4]
        with torch.cuda.device(fullres_input.device):
            multiscale = cls._multiscale_input(fullres_input)
            guides = cls._guide(multiscale, params, is_training) if params.get("debug") else None
            out = cls._output(multiscale, guides, coeffs, params)
        if params.get("debug"):
            cls.last_debug = {"bilateral_coefficients": coeffs, "guide": guides,
                              "multiscale": multiscale, "output": out}
        return out

    @classmethod
    def _inference_training(cls, lowres_input, fullres_input, params):
        """inference(..., is_training=True): every refusal on the CPU first, then the coefficients,
        the pyramid, the three levels' guides (level 0 first, on every rank) and the coarse-to-fine
        output through hdrnet_ops' slice-apply."""
        wts = _resolve_weights(params)
        bn_training = _coefficient_batch_stats(params)
        if params.get("batch_norm") and not bn_training:
            raise NotImplementedError(
                "training-mode batch norm in the coefficient network (params['batch_norm']) is not "
                "implemented: only the guides' conv1 batch norm runs in training mode; "
                "params['coefficient_batch_stats'] runs the coefficient network's in training mode too")
        for scope in cls._guide_scopes():
            _moving_averages(wts, scope)
        _refuse_untrained(wts, params, fullres_input=fullres_input, nn_guide=True, is_training=True,
                          bn_training=bn_training)
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, bn_training)
        with torch.cuda.device(fullres_input.device):
            multiscale = cls._multiscale_input(fullres_input)
            guides = cls._guide(multiscale, params, is_training=True)
            return cls._output(multiscale, guides, coeffs, params)

    @classmethod
    def _guide(cls, multiscale, params, is_training=False):
        """models.py:264-272: HDRNetPointwiseNNGuide._guide per level (scope level_{il}).  In training
        mode each level is normalised with its own batch statistics and updates its own moving
        averages, the levels called in order."""
        if is_training:
            return [HDRNetPointwiseNNGuide._guide(lvl, params, True, scope)
                    for lvl, scope in zip(multiscale, cls._guide_scopes())]
        prep = _prepare(_resolve_weights(params), params, multiscale[0].device, "pyramid")
        return [guide.run(lvl) for lvl, guide in zip(multiscale, prep.guides)]


class HDRNetGaussianPyr(_GaussianPyramid, HDRNetCurves):
    """HDRNetGaussianPyrNN with HDRNetCurves' guide in place of the pointwise NN: the pyramid of
    _GaussianPyramid with one curves guide per level (``inference/guide/level_{0,1,2}/{ccm, ccm_bias,
    shifts, slopes, channel_mixing/*}``).  The reference's gpyr recipes name this model
    (scripts/ll/train_gpyr.sh, scripts/usm/train_gpyr.sh, scripts/ll_strong/train_gpyrnn*.sh), but its
    models.py never defines it; this definition is the project's own (DESIGN.md row f-17).  The curves
    guide has no batch norm, so the inference form is also the training form, as for HDRNetCurves."""

    _nn_guide = "curves_pyramid"

    @classmethod
    def inference(cls, lowres_input, fullres_input, params, is_training=False):
        """lowres_input [B,S,S,3], fullres_input [B,H,W,3] (H, W >= 4) -> [B,H,W,3].  Without
        gradients each level's curves guide runs inside its slice-apply.  With coefficient-network
        variables (or lowres_input) requiring grad, the guides come from the standalone kernel and
        the output from hdrnet_ops' slice-apply and the resize, whose VJPs carry the gradient back to
        the grid; with params['guide_grad'] each level's curves variables and fullres_input are
        differentiated too, through _CurvesGuideFn and _ResizeFn.  With params['debug'] the
        coefficients, the three guide maps and the levels go to ``cls.last_debug``.

        ``is_training=True`` needs params['coefficient_batch_stats'] with params['batch_norm'] (else
        NotImplementedError): the coefficient network's batch-norm layers then normalise with the
        batch's statistics, as in HDRNetCurves.inference."""
        bn_training = _coefficient_batch_stats(params)
        if is_training and not bn_training:
            raise NotImplementedError("hdrnet_b200 implements the inference path only")
        wts = _weights_or_none(params)
        _refuse_untrained(wts, params, fullres_input=fullres_input, bn_training=bool(is_training),
                          curves_model=cls.__name__)
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, is_training)       # [B,gh,gw,gd,9,4]
        debug = bool(params.get("debug"))
        with torch.cuda.device(fullres_input.device):
            multiscale = cls._multiscale_input(fullres_input)
            grad = coeffs.requires_grad or any(_guide_grad(wts, params, lvl, _CURVES_VARS, scope)
                                               for lvl, scope in zip(multiscale, cls._guide_scopes()))
            guides = cls._guide(multiscale, params) if grad or debug else None
            out = cls._output(multiscale, guides, coeffs, params)
        if debug:
            cls.last_debug = {"bilateral_coefficients": coeffs, "guide": guides,
                              "multiscale": multiscale, "output": out}
        return out

    @classmethod
    def _guide(cls, multiscale, params, is_training=False):
        """models.py:264-272 with HDRNetCurves' guide: HDRNetCurves._guide per level (scope
        level_{il}), each differentiable (_CurvesGuideFn) when _guide_grad says so."""
        return [HDRNetCurves._guide(lvl, params, is_training, scope)
                for lvl, scope in zip(multiscale, cls._guide_scopes())]


del layers  # imported for the side effect of the public surface only
