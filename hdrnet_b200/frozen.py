"""A frozen model (``checkpoint.freeze_model``) run through the whole-model C-ABI
(``hdrnet_model_*``, include/hdrnet_b200.h): the object a C or C++ caller would hold, owned from
Python.  Its results are bit for bit those of ``models.*.inference_image`` on the same weights, with one
exception: the pyramids from uint8 / uint16 pixels convert the image with the bit-exact img_as_float,
where ``inference_image`` divides through torch (``models.image_to_float``, DESIGN.md row f-11); their
results are bit for bit ``HDRNetGaussianPyrNN.inference`` (or ``HDRNetGaussianPyr.inference``) on the
host's img_as_float, then ``quantize_u8`` / ``quantize_u16``.

    model = FrozenModel("frozen_model.hdrnet")            # weights uploaded to the current device
    out = model(image_u8)                                  # [B,H,W,3] uint8 -> uint8, current stream
    model.run(image_u8, out, workspace)                    # caller-lent buffers: CUDA-graph capturable

``__call__`` takes the output and the workspace from torch's caching allocator on the current
stream; ``run`` takes them from the caller and does nothing else on the host, so a
``torch.cuda.CUDAGraph`` can capture it.  A list of images of different sizes (a ragged batch,
``hdrnet_model_run_ragged_px``) goes the same two ways:

    outs = model([im_4032x3024, im_3024x4032, im_1080p])   # list in, list out
    model.run_images(images, outs, workspace)              # caller-lent buffers: capturable
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from .checkpoint import FROZEN_MODEL_NAMES
from .models import OUT_DTYPES, _PX_FMT, _check_image, _check_images, _check_out_dtype


class FrozenModel:
    """Owner of one ``hdrnet_model`` on one device (``device``; default the current one)."""

    _handle = None

    def __init__(self, path: str, device=None):
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise _lib.HdrnetLibraryError(f"FrozenModel needs a CUDA device, got {self.device}")
        with open(path, "rb") as f:
            blob = f.read()
        lib = _lib.load()
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            rc = lib.hdrnet_model_create(blob, len(blob), ctypes.byref(handle))
        _lib.check(rc, f"loading frozen model {path}")
        self._handle = handle
        vals = [ctypes.c_int() for _ in range(6)]
        _lib.check(lib.hdrnet_model_info(handle, *[ctypes.byref(v) for v in vals]), "model info")
        kind, self.net_input_size, self.spatial_bin, self.luma_bins, self.channel_multiplier, self.guide_width = (
            v.value for v in vals)
        self.model_name = FROZEN_MODEL_NAMES[kind]

    @property
    def handle(self) -> ctypes.c_void_p:
        if self._handle is None:
            raise ValueError("the FrozenModel is closed")
        return self._handle

    def workspace_bytes(self, B: int, H: int, W: int, in_dtype=torch.uint8, out_dtype=torch.uint8) -> int:
        """Bytes of workspace ``run`` needs for B images of H x W from `in_dtype` to `out_dtype`."""
        _check_out_dtype(out_dtype)
        if in_dtype not in _PX_FMT:
            raise TypeError(f"in_dtype must be uint8, uint16 or float32, got {in_dtype}")
        return int(_lib.load().hdrnet_model_workspace_bytes(self.handle, B, H, W, _PX_FMT[in_dtype],
                                                            _PX_FMT[out_dtype]))

    def workspace_bytes_images(self, images, out_dtype=torch.uint8) -> int:
        """Bytes of workspace ``run_images`` needs for this list of [H_i, W_i, 3] images."""
        _check_out_dtype(out_dtype)
        images = _check_images(images, "images")
        fmt = _PX_FMT[images[0].dtype] if images else _PX_FMT[torch.uint8]
        return int(_lib.load().hdrnet_model_workspace_bytes_ragged(self.handle, _lib.image_descs(images), len(images),
                                                                   fmt, _PX_FMT[out_dtype]))

    def __call__(self, image, lowres_image=None, out_dtype=torch.uint8):
        """image [B,H,W,3] uint8 / uint16 / float32 on the model's device -> [B,H,W,3] `out_dtype`
        (uint8, uint16 or float32), as ``inference_image(image, params, lowres_image, out_dtype)``.
        A list of [H_i, W_i, 3] images of one dtype (and `lowres_image` a list of as many, or None)
        -> a list of [H_i, W_i, 3] results, as ``inference_images``."""
        _check_out_dtype(out_dtype)
        if isinstance(image, (list, tuple)):
            images = _check_images(image, "images")
            outs = [torch.empty(im.shape, dtype=out_dtype, device=im.device) for im in images]
            if not images:
                return outs
            ws = torch.empty(self.workspace_bytes_images(images, out_dtype), dtype=torch.uint8,
                             device=images[0].device)
            return self.run_images(images, outs, ws, lowres_image)
        image = _check_image(image, "image")
        B, H, W, _ = image.shape
        out = torch.empty((B, H, W, 3), dtype=out_dtype, device=image.device)
        ws = torch.empty(self.workspace_bytes(B, H, W, image.dtype, out_dtype), dtype=torch.uint8,
                         device=image.device)
        self.run(image, out, ws, lowres_image)
        return out

    def run(self, image: torch.Tensor, out: torch.Tensor, workspace: torch.Tensor,
            lowres_image: torch.Tensor | None = None) -> torch.Tensor:
        """One ``hdrnet_model_run_px`` on the current stream into the caller's `out` (contiguous
        [B,H,W,3] of an OUT_DTYPES dtype) with the caller's `workspace` (any contiguous tensor of at
        least ``workspace_bytes`` bytes).  Returns `out`."""
        image = _check_image(image, "image")
        if out.dtype not in OUT_DTYPES or out.shape != image.shape or not out.is_contiguous():
            raise ValueError("out must be a contiguous uint8 / uint16 / float32 tensor of the image's shape")
        if not workspace.is_contiguous():
            raise ValueError("workspace must be contiguous")
        B, H, W, _ = image.shape
        low, lfmt, SH, SW = None, 0, 0, 0
        if lowres_image is not None:
            lowres_image = _check_image(lowres_image, "lowres_image")
            low, lfmt, SH, SW = lowres_image.data_ptr(), _PX_FMT[lowres_image.dtype], *lowres_image.shape[1:3]
            if lowres_image.shape[0] != B:
                raise ValueError("lowres_image must hold as many images as image")
        with torch.cuda.device(image.device):
            rc = _lib.load().hdrnet_model_run_px(
                self.handle, image.data_ptr(), _PX_FMT[image.dtype], low, lfmt, SH, SW, out.data_ptr(),
                _PX_FMT[out.dtype], B, H, W, workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                torch.cuda.current_stream(image.device).cuda_stream)
        _lib.check(rc, f"{self.model_name} (frozen)")
        return out

    def run_images(self, images, outs, workspace: torch.Tensor, lowres_images=None) -> list:
        """One ``hdrnet_model_run_ragged_px`` on the current stream: `images` a list of [H_i, W_i, 3]
        tensors of one dtype, `outs` a list of contiguous tensors of the same shapes and one
        OUT_DTYPES dtype, `workspace` any contiguous tensor of at least ``workspace_bytes_images``
        bytes.  The descriptors are passed to the kernels by value, so a ``torch.cuda.CUDAGraph``
        that captures this call replays it on whatever pixels those buffers then hold.  Returns
        `outs`."""
        images = _check_images(images, "images")
        if len(outs) != len(images) or any(
                o.dtype != outs[0].dtype or o.dtype not in OUT_DTYPES or o.shape != im.shape or not o.is_contiguous()
                for o, im in zip(outs, images)):
            raise ValueError("outs must be contiguous tensors of the images' shapes and one uint8 / uint16 / "
                             "float32 dtype")
        if not workspace.is_contiguous():
            raise ValueError("workspace must be contiguous")
        if not images:
            return outs
        low, lfmt = None, 0
        if lowres_images is not None:
            lowres_images = _check_images(lowres_images, "lowres_images")
            if len(lowres_images) != len(images):
                raise ValueError("lowres_images must hold one image per image")
            low, lfmt = _lib.image_descs(lowres_images), _PX_FMT[lowres_images[0].dtype]
        with torch.cuda.device(images[0].device):
            rc = _lib.load().hdrnet_model_run_ragged_px(
                self.handle, _lib.image_descs(images, outs), len(images), _PX_FMT[images[0].dtype],
                _PX_FMT[outs[0].dtype], low, lfmt, workspace.data_ptr(),
                workspace.numel() * workspace.element_size(), torch.cuda.current_stream(images[0].device).cuda_stream)
        _lib.check(rc, f"{self.model_name} (frozen, ragged)")
        return outs

    def close(self) -> None:
        """Destroy the C object (waits for work still reading its weights); later calls raise."""
        if self._handle is not None:
            handle, self._handle = self._handle, None
            _lib.check(_lib.load().hdrnet_model_destroy(handle), "destroying the frozen model")

    def __del__(self):
        try:
            self.close()
        except Exception:   # interpreter shutdown: the library may be gone already
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
