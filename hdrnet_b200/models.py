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

Execution (all hand-written sm_90a kernels through the C-ABI, no torch math on the path):
  coefficients  4 splat convs, 2 global convs + 3 FCs, 2 local convs (conv2d / fc kernels),
                then fusion + prediction + unroll_grid in one kernel -> grid [B,gh,gw,gd,12]
  guide+output  ONE kernel: per-pixel guide (curves or pointwise NN) computed in registers
                and fed straight into the fused slice-apply (the guide never touches HBM).
"""
from __future__ import annotations

import collections
import ctypes
import os
import math

import numpy as np
import torch

from . import _lib, layers
from .layers import bilateral_slice_apply

__all__ = ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN", "set_weights", "load_weights",
           "init_weights", "DEFAULT_PARAMS"]

BN_EPS = 1e-3   # tf.contrib.layers.batch_norm default epsilon (hdrnet/layers.py:47-54)

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


def init_weights(params, seed: int = 0, model_name: str | None = None) -> dict:
    """Fresh variables with the reference's initialisers: variance-scaling (fan-in, factor 2,
    truncated normal) for conv/fc weights and zero biases (hdrnet/layers.py:22-23), identity
    ccm / linspace shifts / unit first slope / 1/3 mixing for the curves guide
    (hdrnet/models.py:150-186).  Used for synthetic-weight benchmarks."""
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
    n_out = 9 if model_name == "HDRNetGaussianPyrNN" else 3
    conv(f"{p}/prediction/conv1", 1, c8, gd * n_out * 4)
    g = "inference/guide"
    if model_name == "HDRNetGaussianPyrNN":
        nf = params["guide_complexity"]
        for lvl in range(3):
            conv(f"{g}/level_{lvl}/conv1", 1, 3, nf, use_bn=True)
            conv(f"{g}/level_{lvl}/conv2", 1, nf, 1)
    elif model_name == "HDRNetCurves":
        w[g + "/ccm"] = (np.identity(3) + rng.randn(1) * 1e-4).astype(np.float32)
        w[g + "/ccm_bias"] = np.zeros(3, np.float32)
        w[g + "/shifts"] = np.tile(np.linspace(0, 1, 16, endpoint=False, dtype=np.float32)
                                   [None, None, None, :], (1, 1, 3, 1))
        slopes = np.zeros((1, 1, 1, 3, 16), np.float32)
        slopes[..., 0] = 1.0
        w[g + "/slopes"] = slopes
        w[g + "/channel_mixing/weights"] = np.full((1, 1, 3, 1), 1.0 / 3.0, np.float32)
        w[g + "/channel_mixing/biases"] = np.zeros(1, np.float32)
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
    the fold freeze_graph.py:141-142 applies)."""
    w = np.asarray(wts[scope + "/weights"], np.float32)
    if use_bn:
        s = 1.0 / np.sqrt(np.asarray(wts[scope + "/BatchNorm/moving_variance"], np.float64) + BN_EPS)
        b = np.asarray(wts[scope + "/BatchNorm/beta"], np.float64) - \
            np.asarray(wts[scope + "/BatchNorm/moving_mean"], np.float64) * s
        return (w.astype(np.float64) * s).astype(np.float32), b.astype(np.float32)
    if use_bias:
        return w, np.asarray(wts[scope + "/biases"], np.float32)
    return w, None


class _Prepared:
    """Device copies of the coefficient-network weights + host copies of the guide params."""

    def __init__(self, wts, params, device, nn_guide):
        self.device = device
        self.source = wts   # keeps the dict alive: the cache is keyed by id(wts)
        bn = bool(params["batch_norm"])
        self.layers = {}
        p = "inference/coefficients"
        n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
        specs = [(f"{p}/splat/conv{i + 1}", bn and i > 0, True) for i in range(n_ds)]
        specs += [(f"{p}/global/conv1", bn, True), (f"{p}/global/conv2", bn, True),
                  (f"{p}/global/fc1", bn, True), (f"{p}/global/fc2", bn, True),
                  (f"{p}/global/fc3", False, True), (f"{p}/local/conv1", bn, True),
                  (f"{p}/local/conv2", False, False), (f"{p}/prediction/conv1", False, True)]
        for scope, use_bn, use_bias in specs:
            w, b = _fold(wts, scope, use_bn, use_bias)
            wd = torch.from_numpy(np.ascontiguousarray(w)).to(device)
            bd = None if b is None else torch.from_numpy(np.ascontiguousarray(b)).to(device)
            packed = pack_conv_weights(wd) if (wd.dim() == 4 and device.type == "cuda") else None
            self.layers[scope] = (wd, bd, packed)
        g = "inference/guide"
        f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float32))  # noqa: E731

        def nn_params(scope):
            w1, b1 = _fold(wts, scope + "/conv1", True, False)
            w1 = f32(w1.reshape(3, -1))
            return (w1, f32(b1), f32(np.asarray(wts[scope + "/conv2/weights"]).reshape(-1)),
                    float(np.asarray(wts[scope + "/conv2/biases"]).reshape(-1)[0]), int(w1.shape[1]))

        if nn_guide == "pyramid":     # HDRNetGaussianPyrNN: one pointwise NN per level
            self.nn_levels = [nn_params(f"{g}/level_{lvl}") for lvl in range(3)]
        elif nn_guide:
            self.nn_w1, self.nn_b1, self.nn_w2, self.nn_b2, self.nn_feats = nn_params(g)
        else:
            self.ccm = f32(wts[g + "/ccm"])
            self.ccm_bias = f32(wts[g + "/ccm_bias"])
            self.shifts = f32(np.asarray(wts[g + "/shifts"]).reshape(3, 16))
            self.slopes = f32(np.asarray(wts[g + "/slopes"]).reshape(3, 16))
            self.mix = f32(np.asarray(wts[g + "/channel_mixing/weights"]).reshape(3))
            self.mix_bias = float(np.asarray(wts[g + "/channel_mixing/biases"]).reshape(-1)[0])


def _prepare(wts, params, device, nn_guide) -> _Prepared:
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


def _use_packed_tc(tiles: int) -> bool:
    """HDRNET_CONV_TCGEN05: '1' = tensor-core convs wherever weights were packed, '0' = never.
    Default: from 64 tiles of 128 output pixels up.  Measured on an H100 (tools/conv_bench.py, the
    network's conv shapes): at 16 tiles the CUDA-core kernels were 3-15 % faster, at 64 the two
    were even, at 128 the packed tensor-core kernel was 1.7-5x faster."""
    import os
    flag = os.environ.get("HDRNET_CONV_TCGEN05")
    if flag is not None:
        return flag == "1"
    return tiles >= 64


def _conv(x: torch.Tensor, wb, stride=1, relu=True) -> torch.Tensor:
    w, b = wb[0], wb[1]
    packed = wb[2] if len(wb) > 2 else None
    B, H, W, cin = x.shape
    k, _, wcin, cout = w.shape
    if wcin != cin:
        raise ValueError(f"conv: input has {cin} channels, weights expect {wcin}")
    oh, ow = -(-H // stride), -(-W // stride)
    out = torch.empty((B, oh, ow, cout), dtype=torch.float32, device=x.device)
    lib = _lib.load()
    if packed is not None and _use_packed_tc((B * oh * ow + 127) // 128):
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
        ``cls.last_debug`` (the collections run.py --debug reads, run.py:98-133)."""
        if is_training:
            raise NotImplementedError("hdrnet_b200 implements the inference path only")
        fullres_input = _check_input(fullres_input, "fullres_input")
        coeffs = cls._coefficients(lowres_input, params, is_training)
        return cls._fullres(coeffs, fullres_input, params, torch.float32)

    @classmethod
    def inference_image(cls, image, params, lowres_image=None, out_dtype=torch.uint8):
        """The reference CLI's per-image path (hdrnet/bin/run.py:145-190) with the decoded image
        kept in its storage format on the device: ``image`` [B,H,W,3] uint8 / uint16 / float32
        -> nearest-neighbour S x S float32 network input (img_as_float on the fly, run.py:156-169)
        -> coefficients -> guide + slice + apply in one full-resolution pass that reads the
        integer pixels and writes ``uint8(255 * clip(out, 0, 1))`` (run.py:95).  3 + 3 bytes per
        pixel cross PCIe / HBM instead of 12 + 12.  ``lowres_image`` replaces the resized input
        (run.py --lowres_input); ``out_dtype=torch.float32`` returns the unquantised prediction."""
        image = _check_image(image, "image")
        src = image if lowres_image is None else _check_image(lowres_image, "lowres_image")
        lowres = lowres_from_image(src, int(params["net_input_size"]))
        coeffs = cls._coefficients(lowres, params, False)
        return cls._fullres(coeffs, image, params, out_dtype)

    @classmethod
    def inference_image_host(cls, frames, params, out=None, device=None, out_dtype=torch.uint8):
        """``inference_image`` for frames that live in HOST memory (what hdrnet/bin/run.py does per
        file: load, ``sess.run``, save): uploads, the model and downloads of consecutive frames
        overlap on three streams (hdrnet_b200/host_pipeline.py).  ``frames`` [N,H,W,3] uint8 /
        uint16 / float32 CPU tensor (pinned for asynchronous copies) -> CPU tensor of ``out_dtype``.
        One pipeline (streams + two frame buffers) is kept per (class, device, out_dtype)."""
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
        B, H, W, _ = fullres_input.shape
        _, gh, gw, gd = coeffs.shape[:4]
        in_fmt, out_fmt = _PX_FMT[fullres_input.dtype], _PX_FMT[out_dtype]
        out = torch.empty((B, H, W, 3), dtype=out_dtype, device=fullres_input.device)
        debug = bool(params.get("debug"))
        f32 = in_fmt == _lib.PX_F32 and out_fmt == _lib.PX_F32
        # the float32 form needs the guide buffer for shapes its row kernel cannot take
        need_guide = debug or (f32 and ((W % 4 != 0) or W < 128))
        guide = torch.empty((B, H, W), dtype=torch.float32, device=fullres_input.device) \
            if need_guide else None
        lib = _lib.load()
        with torch.cuda.device(fullres_input.device):
            stream = torch.cuda.current_stream(fullres_input.device).cuda_stream
            gptr = 0 if guide is None else guide.data_ptr()
            # workspace lent to the library (it never allocates): texture-assisted kernel for
            # large images, exactly as hdrnet_ops.bilateral_slice_apply does
            ws_ptr, ws_bytes = 0, 0
            if B * H * W >= (1 << 21) and W % 4 == 0:
                from .hdrnet_ops import _workspace
                ws = _workspace(fullres_input.device,
                                lib.hdrnet_slice_apply_workspace_bytes(B, H, gw, gd))
                ws_ptr, ws_bytes = ws.data_ptr(), ws.numel() * 4
            if cls._nn_guide:
                rc = lib.hdrnet_slice_apply_nn_px_ws(
                    coeffs.data_ptr(), fullres_input.data_ptr(), in_fmt, out.data_ptr(), out_fmt,
                    gptr, B, H, W, gh, gw, gd, _hp(prep.nn_w1), _hp(prep.nn_b1), _hp(prep.nn_w2),
                    prep.nn_b2, prep.nn_feats, ws_ptr, ws_bytes, stream)
            else:
                rc = lib.hdrnet_slice_apply_curves_px_ws(
                    coeffs.data_ptr(), fullres_input.data_ptr(), in_fmt, out.data_ptr(), out_fmt,
                    gptr, B, H, W, gh, gw, gd, _hp(prep.ccm), _hp(prep.ccm_bias), _hp(prep.shifts),
                    _hp(prep.slopes), _hp(prep.mix), prep.mix_bias, ws_ptr, ws_bytes, stream)
        _lib.check(rc, "BilateralSliceApply(fused guide)")
        if debug:
            cls.last_debug = {"bilateral_coefficients": coeffs, "guide": guide, "output": out}
        return out

    @classmethod
    def _coefficients(cls, input_tensor, params, is_training=False):
        """models.py:62-142 -> [B, gh, gw, gd, n_out, n_in]."""
        if is_training:
            raise NotImplementedError("hdrnet_b200 implements the inference path only")
        x = _check_input(input_tensor, "lowres_input")
        prep = _prepare(_resolve_weights(params), params, x.device, cls._nn_guide)
        L = prep.layers
        gd = params["luma_bins"]
        p = "inference/coefficients"
        n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
        bs = x.shape[0]
        # small batches: the whole network behind one library call (launch chain, csrc/cnn.cu)
        if bs <= CHAIN_CNN_MAX_BATCH and os.environ.get("HDRNET_CONV_TCGEN05") != "1":
            grid = cls._coefficients_chain(x, prep, params, n_ds)
            if grid is not None:
                return grid
        with torch.cuda.device(x.device):
            for i in range(n_ds):                                   # splat, :69-82
                x = _conv(x, L[f"{p}/splat/conv{i + 1}"], stride=2)
            splat = x
            g = _conv(splat, L[f"{p}/global/conv1"], stride=2)      # global, :86-105
            g = _conv(g, L[f"{p}/global/conv2"], stride=2)
            g = g.reshape(bs, -1)                                   # NHWC flatten, :94-95
            g = _fc(g, L[f"{p}/global/fc1"])
            g = _fc(g, L[f"{p}/global/fc2"])
            g = _fc(g, L[f"{p}/global/fc3"], relu=False)
            loc = _conv(splat, L[f"{p}/local/conv1"])               # local, :109-118
            loc = _conv(loc, L[f"{p}/local/conv2"], relu=False)
            wp, bp = L[f"{p}/prediction/conv1"][:2]
            _, gh, gw, C = loc.shape
            grid = torch.empty((bs, gh, gw, gd, cls.n_out(), cls.n_in()), dtype=torch.float32,
                               device=x.device)
            rc = _lib.load().hdrnet_fuse_predict_f32(           # fusion+prediction+unroll, :122-139
                loc.data_ptr(), g.data_ptr(), wp.data_ptr(), 0 if bp is None else bp.data_ptr(),
                grid.data_ptr(), bs, gh, gw, C, gd, cls.n_out(), cls.n_in(),
                torch.cuda.current_stream(x.device).cuda_stream)
        _lib.check(rc, "fuse_predict")
        return grid

    @classmethod
    def _coefficients_chain(cls, x, prep, params, n_ds):
        """One library call for all layers; None when the library does not take the shape."""
        lib = _lib.load()
        bs, S = x.shape[0], x.shape[1]
        gd, cm, sb = params["luma_bins"], params["channel_multiplier"], params["spatial_bin"]
        nbytes = lib.hdrnet_coefficients_scratch_bytes(bs, S, sb, gd, cm, cls.n_out(), cls.n_in())
        if nbytes == 0 or x.shape[2] != S:
            return None
        p = "inference/coefficients"
        order = [f"{p}/splat/conv{i + 1}" for i in range(n_ds)] + \
                [f"{p}/global/conv1", f"{p}/global/conv2", f"{p}/global/fc1", f"{p}/global/fc2",
                 f"{p}/global/fc3", f"{p}/local/conv1", f"{p}/local/conv2", f"{p}/prediction/conv1"]
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
    def _guide(cls, input_tensor, params, is_training=False):
        """models.py:145-190 as a standalone kernel -> [B, H, W]."""
        x = _check_input(input_tensor, "fullres_input")
        prep = _prepare(_resolve_weights(params), params, x.device, False)
        B, H, W, _ = x.shape
        guide = torch.empty((B, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.load().hdrnet_guide_curves_f32(
                x.data_ptr(), guide.data_ptr(), B * H * W, _hp(prep.ccm), _hp(prep.ccm_bias),
                _hp(prep.shifts), _hp(prep.slopes), _hp(prep.mix), prep.mix_bias,
                torch.cuda.current_stream(x.device).cuda_stream)
        _lib.check(rc, "guide_curves")
        return guide

    @classmethod
    def _output(cls, im, guide, coeffs):
        """models.py:193-196."""
        return bilateral_slice_apply(coeffs, guide, im, has_offset=True, name="slice")


class HDRNetPointwiseNNGuide(HDRNetCurves):
    """Replaces the pointwise curves in the guide by a pointwise neural net
    (hdrnet/models.py:199-210)."""

    _nn_guide = True

    @classmethod
    def _guide(cls, input_tensor, params, is_training=False):
        x = _check_input(input_tensor, "fullres_input")
        prep = _prepare(_resolve_weights(params), params, x.device, True)
        B, H, W, _ = x.shape
        guide = torch.empty((B, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.load().hdrnet_guide_nn_f32(
                x.data_ptr(), guide.data_ptr(), B * H * W, _hp(prep.nn_w1), _hp(prep.nn_b1),
                _hp(prep.nn_w2), prep.nn_b2, prep.nn_feats,
                torch.cuda.current_stream(x.device).cuda_stream)
        _lib.check(rc, "guide_nn")
        return guide


def _resize(x: torch.Tensor, oh: int, ow: int, add: torch.Tensor | None = None) -> torch.Tensor:
    """tf.image.resize_images(x, [oh, ow], BILINEAR, align_corners=True) (+ fused add)."""
    B, H, W, C = x.shape
    out = torch.empty((B, oh, ow, C), dtype=torch.float32, device=x.device)
    rc = _lib.load().hdrnet_resize_bilinear_f32(
        x.data_ptr(), 0 if add is None else add.data_ptr(), out.data_ptr(), B, H, W, C, oh, ow,
        torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "resize_bilinear")
    return out


class HDRNetGaussianPyrNN(HDRNetPointwiseNNGuide):
    """Replace input to the affine model by a pyramid (hdrnet/models.py:213-289): 3-level
    bilinear (align_corners) pyramid of the full-res image, one pointwise-NN guide per level,
    one slice-apply per level with its own 3 of the 9 output rows of the coefficient grid,
    coarse-to-fine upsample-and-add.  The reference file is Python-2 only here
    (`reversed(zip(...))`, :278); the semantics restated: the COARSEST level uses output rows
    0..2, the finest rows 6..8."""

    _nn_guide = "pyramid"

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
    def inference(cls, lowres_input, fullres_input, params, is_training=False):
        if is_training:
            raise NotImplementedError("hdrnet_b200 implements the inference path only")
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
    def inference_image(cls, image, params, lowres_image=None, out_dtype=torch.uint8):
        """Same contract as HDRNetCurves.inference_image.  The pyramid needs the float image at
        three scales, so only the network input is taken straight from the integer pixels; the
        full-resolution image is converted once on the device."""
        image = _check_image(image, "image")
        src = image if lowres_image is None else _check_image(lowres_image, "lowres_image")
        lowres = lowres_from_image(src, int(params["net_input_size"]))
        out = cls.inference(lowres, image_to_float(image), params, False)
        return quantize_u8(out) if out_dtype == torch.uint8 else out

    @classmethod
    def _multiscale_input(cls, fullres_input):
        """models.py:249-262: each level is the previous one resized to floor(size / 2)."""
        lvls = [fullres_input]
        h, w = fullres_input.shape[1:3]
        for _ in range(cls.n_scales() - 1):
            h, w = h // 2, w // 2
            lvls.append(_resize(lvls[-1], h, w))
        return lvls

    @classmethod
    def _guide(cls, multiscale, params, is_training=False):
        """models.py:264-272: HDRNetPointwiseNNGuide._guide per level (scope level_{il})."""
        prep = _prepare(_resolve_weights(params), params, multiscale[0].device, "pyramid")
        lib = _lib.load()
        guides = []
        for lvl, (w1, b1, w2, b2, feats) in zip(multiscale, prep.nn_levels):
            B, H, W, _ = lvl.shape
            g = torch.empty((B, H, W), dtype=torch.float32, device=lvl.device)
            rc = lib.hdrnet_guide_nn_f32(lvl.data_ptr(), g.data_ptr(), B * H * W, _hp(w1), _hp(b1),
                                         _hp(w2), b2, feats,
                                         torch.cuda.current_stream(lvl.device).cuda_stream)
            _lib.check(rc, "guide_nn")
            guides.append(g)
        return guides

    @classmethod
    def _output(cls, lvls, guide_lvls, coeffs, params=None):
        """models.py:274-289, coarse to fine.  With guide_lvls=None (the fast path) each level's
        guide is computed inside its slice-apply kernel."""
        prep = _prepare(_resolve_weights(params), params, lvls[0].device, "pyramid") \
            if guide_lvls is None else None
        lib = _lib.load()
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
                w1, b1, w2, b2, feats = prep.nn_levels[src]
                out_lvl = torch.empty_like(lvl)
                need_guide = (W % 4 != 0) or W < 128
                scratch = torch.empty((B, H, W), dtype=torch.float32, device=lvl.device) \
                    if need_guide else None
                rc = lib.hdrnet_slice_apply_nn_f32(
                    c.data_ptr(), lvl.data_ptr(), out_lvl.data_ptr(),
                    0 if scratch is None else scratch.data_ptr(), B, H, W, gh, gw, gd, _hp(w1),
                    _hp(b1), _hp(w2), b2, feats, torch.cuda.current_stream(lvl.device).cuda_stream)
                _lib.check(rc, "BilateralSliceApply(fused NN guide)")
            current = out_lvl if il == 0 else _resize(current, H, W, add=out_lvl)
        return current


del layers  # imported for the side effect of the public surface only
