"""A frozen model (``checkpoint.freeze_model``) run through the whole-model C-ABI
(``hdrnet_model_*``, include/hdrnet_b200.h): the object a C or C++ caller would hold, owned from
Python.  Its results are bit for bit those of ``models.*.inference_image`` on the same weights, with one
exception: the pyramid from uint8 / uint16 pixels converts the image with the bit-exact img_as_float,
where ``inference_image`` divides through torch (``models.image_to_float``, DESIGN.md row f-11); its
results are bit for bit ``HDRNetGaussianPyrNN.inference`` on the host's img_as_float, then
``quantize_u8`` / ``quantize_u16``.

    model = FrozenModel("frozen_model.hdrnet")            # weights uploaded to the current device
    out = model(image_u8)                                  # [B,H,W,3] uint8 -> uint8, current stream
    model.run(image_u8, out, workspace)                    # caller-lent buffers: CUDA-graph capturable

``__call__`` takes the output and the workspace from torch's caching allocator on the current
stream; ``run`` takes them from the caller and does nothing else on the host, so a
``torch.cuda.CUDAGraph`` can capture it.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from .checkpoint import FROZEN_KINDS
from .models import OUT_DTYPES, _PX_FMT, _check_image, _check_out_dtype


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
        self.model_name = FROZEN_KINDS[kind]

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

    def __call__(self, image: torch.Tensor, lowres_image: torch.Tensor | None = None,
                 out_dtype=torch.uint8) -> torch.Tensor:
        """image [B,H,W,3] uint8 / uint16 / float32 on the model's device -> [B,H,W,3] `out_dtype`
        (uint8, uint16 or float32), as ``inference_image(image, params, lowres_image, out_dtype)``."""
        _check_out_dtype(out_dtype)
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
