"""Python op boundary: drop-in for the reference's ``hdrnet/hdrnet_ops.py``.

The reference binds ``bilateral_slice`` / ``bilateral_slice_apply`` from a TF op library
(hdrnet/hdrnet_ops.py:23-31).  Here the same two names take ``torch.Tensor`` arguments in the
same order, with the same shapes (TF NHWC) and the same ``has_offset`` attribute, and call
the hand-written sm_90a kernels through the C-ABI (include/hdrnet_b200.h):

    bilateral_slice(grid[B,gh,gw,gd,gc], guide[B,H,W])                      -> [B,H,W,gc]
    bilateral_slice_apply(grid, guide, input[B,H,W,n_in], has_offset)        -> [B,H,W,n_out]

* CUDA tensors: asynchronous launch on the current torch stream of the tensors' device.
* CPU tensors: the host-buffer path (row-band pipelined H2D -> kernel -> D2H on the current
  CUDA device), i.e. what feeding numpy arrays to the reference's session does
  (hdrnet/bin/run.py:185).  Pinned tensors overlap copies with compute.

Error convention (hdrnet/ops/bilateral_slice_apply_op.cc:147-193, bilateral_slice_op.cc:
126-133): the conditions the reference rejects with ``InvalidArgument`` raise ``ValueError``
with the reference's message; a failed launch raises ``HdrnetLibraryError`` (the reference's
``Internal("... kernel failed.")``).  There is no CPU fallback of the computation.
"""
from __future__ import annotations

import ctypes
import threading

import torch

from . import _lib

__all__ = ["bilateral_slice", "bilateral_slice_apply", "bilateral_slice_apply_rows", "slice_indices"]

_ctx_lock = threading.Lock()
_host_ctx = {}  # device index -> hdrnet_host_ctx*


def _require_cuda() -> None:
    if not torch.cuda.is_available():
        raise _lib.HdrnetLibraryError(
            "hdrnet_b200 needs a CUDA device (sm_90a); there is no CPU implementation")


def _f32c(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if t.dtype != torch.float32:
        raise TypeError(f"{what} must be float32 (the op is registered for float only), got {t.dtype}")
    return t.contiguous()


def _same_device(*ts: torch.Tensor) -> torch.device:
    dev = ts[0].device
    for t in ts[1:]:
        if t.device != dev:
            raise ValueError(f"all tensors must be on one device, got {dev} and {t.device}")
    return dev


_host_locks = {}  # device index -> lock serialising calls on that device's host context


def _host_call_lock(device_index: int) -> threading.Lock:
    with _ctx_lock:
        return _host_locks.setdefault(device_index, threading.Lock())


def _host_context(device_index: int):
    with _ctx_lock:
        ctx = _host_ctx.get(device_index)
        if ctx is None:
            lib = _lib.load()
            ctx = ctypes.c_void_p()
            with torch.cuda.device(device_index):
                _lib.check(lib.hdrnet_host_ctx_create(ctypes.byref(ctx), 0), "host context")
            _host_ctx[device_index] = ctx
        return ctx


def _workspace(dev: torch.device, nbytes: int) -> torch.Tensor:
    """Slab-row workspace of ONE call, from torch's caching allocator on the current stream (the
    library never allocates).  Per call on purpose: a block cached across calls would be shared by
    calls on different streams / threads, whose pre-passes overwrite each other's slab rows.  The
    allocator hands a freed block back to the same stream only (stream-ordered reuse), so dropping
    the tensor right after the launch is safe."""
    return torch.empty((max(int(nbytes), 16) + 3) // 4, dtype=torch.float32, device=dev)


def _check_slice_args(grid, guide, grid_msg):
    if grid.dim() != 5:
        raise ValueError(grid_msg)
    if guide.dim() != 3:
        raise ValueError("Guide image should be 3D (batch_size, height, width)")
    if guide.shape[0] != grid.shape[0]:
        raise ValueError("Batch sizes should match.")


class _SliceFn(torch.autograd.Function):
    """Gradient registration of BilateralSlice (hdrnet/hdrnet_ops.py:34-38)."""

    @staticmethod
    def forward(ctx, grid, guide):
        ctx.save_for_backward(grid, guide)
        with torch.no_grad():
            return bilateral_slice(grid, guide)

    @staticmethod
    def backward(ctx, grad):
        grid, guide = ctx.saved_tensors
        grad = grad.contiguous()
        B, gh, gw, gd, gc = grid.shape
        _, H, W = guide.shape
        gv, uv = torch.empty_like(grid), torch.empty_like(guide)
        with torch.cuda.device(grid.device):
            rc = _lib.load().hdrnet_slice_grad_f32(
                grid.data_ptr(), guide.data_ptr(), grad.data_ptr(), gv.data_ptr(), uv.data_ptr(),
                B, H, W, gh, gw, gd, gc, torch.cuda.current_stream(grid.device).cuda_stream)
        _lib.check(rc, "BilateralSliceGrad")
        return gv, uv


class _SliceApplyFn(torch.autograd.Function):
    """Gradient registration of BilateralSliceApply (hdrnet/hdrnet_ops.py:41-48)."""

    @staticmethod
    def forward(ctx, grid, guide, input, has_offset):  # noqa: A002
        ctx.save_for_backward(grid, guide, input)
        ctx.has_offset = bool(has_offset)
        with torch.no_grad():
            return bilateral_slice_apply(grid, guide, input, has_offset)

    @staticmethod
    def backward(ctx, grad):
        grid, guide, input = ctx.saved_tensors  # noqa: A001
        grad = grad.contiguous()
        B, gh, gw, gd, gc = grid.shape
        _, H, W, n_in = input.shape
        n_out = gc // (n_in + int(ctx.has_offset))
        gv, uv, iv = torch.empty_like(grid), torch.empty_like(guide), torch.empty_like(input)
        with torch.cuda.device(grid.device):
            rc = _lib.load().hdrnet_slice_apply_grad_f32(
                grid.data_ptr(), guide.data_ptr(), input.data_ptr(), grad.data_ptr(), gv.data_ptr(),
                uv.data_ptr(), iv.data_ptr(), B, H, W, gh, gw, gd, n_in, n_out,
                int(ctx.has_offset), torch.cuda.current_stream(grid.device).cuda_stream)
        _lib.check(rc, "BilateralSliceApplyGrad")
        return gv, uv, iv, None


def _wants_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(t.requires_grad for t in ts)


def bilateral_slice(grid: torch.Tensor, guide: torch.Tensor, name=None, *,
                    variant: int = _lib.VARIANT_AUTO) -> torch.Tensor:
    """Slices a bilateral grid with a guide image (reference op ``BilateralSlice``,
    hdrnet/ops/bilateral_slice_op.cc:120-174, :274-290).  ``variant`` forces a kernel for tests."""
    del name
    lib = _lib.load()
    grid = _f32c(grid, "grid")
    guide = _f32c(guide, "guide")
    _check_slice_args(grid, guide,
                      "Grid should be 5D (batch_size, grid_height, grid_width, grid_depth, "
                      "grid_channels).")
    dev = _same_device(grid, guide)
    B, gh, gw, gd, gc = grid.shape
    _, H, W = guide.shape
    if dev.type == "cuda" and _wants_grad(grid, guide):
        return _SliceFn.apply(grid, guide)
    if dev.type != "cuda":
        raise _lib.HdrnetLibraryError("bilateral_slice: tensors must be CUDA tensors "
                                      "(only bilateral_slice_apply has a host-buffer path)")
    _require_cuda()
    out = torch.empty((B, H, W, gc), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = lib.hdrnet_slice_f32_variant(grid.data_ptr(), guide.data_ptr(), out.data_ptr(), B, H, W,
                                          gh, gw, gd, gc, int(variant), stream)
    _lib.check(rc, "BilateralSlice")
    return out


def bilateral_slice_apply(grid: torch.Tensor, guide: torch.Tensor, input: torch.Tensor,  # noqa: A002
                          has_offset: bool, name=None, *, out: torch.Tensor | None = None,
                          variant: int = _lib.VARIANT_AUTO) -> torch.Tensor:
    """Slices the grid and applies the per-pixel affine transform to ``input`` in one pass
    (reference op ``BilateralSliceApply``, hdrnet/ops/bilateral_slice_apply_op.cc:140-235,
    :382-419).  ``out`` (optional, beyond the reference) reuses a preallocated result buffer;
    ``variant`` forces a kernel variant for tests."""
    del name
    lib = _lib.load()
    grid = _f32c(grid, "grid")
    guide = _f32c(guide, "guide")
    input = _f32c(input, "input")  # noqa: A001
    if grid.dim() != 5:
        raise ValueError("Input grid should be 5D (batch_size, height, width, depth, "
                         "output_channels * input_channels)")
    if guide.dim() != 3:
        raise ValueError("Guide image should be 3D (batch_size, height, width)")
    if input.dim() != 4:
        raise ValueError("Input image should be 4D (batch_size, height, width, input_channels)")
    if tuple(input.shape[:3]) != tuple(guide.shape):
        raise ValueError("Input and guide size should match.")
    if guide.shape[0] != grid.shape[0]:
        raise ValueError("Batch sizes should match.")
    has_offset = bool(has_offset)
    B, gh, gw, gd, gc = grid.shape
    _, H, W, n_in = input.shape
    J = n_in + (1 if has_offset else 0)
    if gc % J != 0:
        if has_offset:
            raise ValueError("Slicing with affine offset, grid should have "
                             "output_channels * (input_channels + 1) channels.")
        raise ValueError("Slicing without affine offset, grid should have "
                         "output_channels * input_channels channels.")
    n_out = gc // J
    dev = _same_device(grid, guide, input)
    _require_cuda()

    shape = (B, H, W, n_out)
    if out is not None:
        if tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != dev \
                or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous float32 tensor of shape {shape} on {dev}")

    if dev.type == "cuda" and out is None and _wants_grad(grid, guide, input):
        return _SliceApplyFn.apply(grid, guide, input, has_offset)

    if dev.type == "cuda":
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            # A workspace from torch's caching allocator (the library never allocates) lets AUTO
            # pick the texture-assisted kernel for large images (>= 2 Mi px, W % 4 == 0).
            ws_ptr, ws_bytes = 0, 0
            explicit_tex = int(variant) in (_lib.VARIANT_TEX, _lib.VARIANT_TEX_ASYNC)
            if (int(variant) == _lib.VARIANT_AUTO or explicit_tex) and n_in == 3 and n_out == 3 \
                    and has_offset and W % 4 == 0 and (explicit_tex or B * H * W >= (1 << 21)):
                ws = _workspace(dev, lib.hdrnet_slice_apply_workspace_bytes(B, H, gw, gd))
                ws_ptr, ws_bytes = ws.data_ptr(), ws.numel() * 4
            rc = lib.hdrnet_slice_apply_f32_ws(
                grid.data_ptr(), guide.data_ptr(), input.data_ptr(), out.data_ptr(), B, H, W, gh,
                gw, gd, n_in, n_out, int(has_offset), int(variant), ws_ptr, ws_bytes, stream)
        _lib.check(rc, "BilateralSliceApply")
        return out

    # Host buffers: pipelined copies + kernels on the current CUDA device.
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, pin_memory=guide.is_pinned())
    device_index = torch.cuda.current_device()
    ctx = _host_context(device_index)
    # one call at a time per context: its staging buffers and streams are the context's own
    # (ctypes releases the GIL, so threads could otherwise interleave inside the library)
    with _host_call_lock(device_index), torch.cuda.device(device_index):
        rc = lib.hdrnet_slice_apply_host_f32(ctx, grid.data_ptr(), guide.data_ptr(),
                                             input.data_ptr(), out.data_ptr(), B, H, W, gh, gw,
                                             gd, n_in, n_out, int(has_offset))
    _lib.check(rc, "BilateralSliceApply(host)")
    return out


def bilateral_slice_apply_rows(grid: torch.Tensor, guide: torch.Tensor, input: torch.Tensor,  # noqa: A002
                               has_offset: bool, y_off: int, height: int, *,
                               out: torch.Tensor | None = None,
                               variant: int = _lib.VARIANT_AUTO) -> torch.Tensor:
    """A ROW BAND of ``bilateral_slice_apply``: ``guide`` [B, rows, W] and ``input`` [B, rows, W, n_in]
    hold image rows ``y_off .. y_off + rows - 1`` of images that are ``height`` rows tall; the grid is
    whole.  The op is pointwise in (x, y) (hdrnet/ops/bilateral_slice_apply.cu.cc:75, :80), so bands
    need no halo and equal the rows of the whole-image call bit for bit (same kernel).  Beyond the
    reference: it is the multi-GPU fallback for fewer images than GPUs (SURVEY.md section 8e,
    ``parallel.slice_apply_sharded``).  Inference only (no gradient registration); CUDA tensors."""
    lib = _lib.load()
    grid = _f32c(grid, "grid")
    guide = _f32c(guide, "guide")
    input = _f32c(input, "input")  # noqa: A001
    if grid.dim() != 5:
        raise ValueError("Input grid should be 5D (batch_size, height, width, depth, "
                         "output_channels * input_channels)")
    if guide.dim() != 3:
        raise ValueError("Guide image should be 3D (batch_size, height, width)")
    if input.dim() != 4:
        raise ValueError("Input image should be 4D (batch_size, height, width, input_channels)")
    if tuple(input.shape[:3]) != tuple(guide.shape):
        raise ValueError("Input and guide size should match.")
    if guide.shape[0] != grid.shape[0]:
        raise ValueError("Batch sizes should match.")
    has_offset = bool(has_offset)
    B, gh, gw, gd, gc = grid.shape
    _, rows, W, n_in = input.shape
    y_off, height = int(y_off), int(height)
    if y_off < 0 or y_off + rows > height:
        raise ValueError(f"row band [{y_off}, {y_off + rows}) does not fit an image of {height} rows")
    J = n_in + (1 if has_offset else 0)
    if gc % J != 0:
        raise ValueError("Slicing with affine offset, grid should have output_channels * (input_channels + 1) "
                         "channels." if has_offset else
                         "Slicing without affine offset, grid should have output_channels * input_channels channels.")
    n_out = gc // J
    dev = _same_device(grid, guide, input)
    _require_cuda()
    if dev.type != "cuda":
        raise _lib.HdrnetLibraryError("bilateral_slice_apply_rows: tensors must be CUDA tensors")
    if _wants_grad(grid, guide, input):
        raise ValueError("bilateral_slice_apply_rows is an inference path: call it under torch.no_grad() "
                         "or use bilateral_slice_apply for gradients")
    shape = (B, rows, W, n_out)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=dev)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != dev or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float32 tensor of shape {shape} on {dev}")
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        ws_ptr, ws_bytes = 0, 0
        explicit_tex = int(variant) in (_lib.VARIANT_TEX, _lib.VARIANT_TEX_ASYNC)
        if (int(variant) == _lib.VARIANT_AUTO or explicit_tex) and n_in == 3 and n_out == 3 \
                and has_offset and W % 4 == 0 and (explicit_tex or B * rows * W >= (1 << 21)):
            ws = _workspace(dev, lib.hdrnet_slice_apply_workspace_bytes(B, rows, gw, gd))
            ws_ptr, ws_bytes = ws.data_ptr(), ws.numel() * 4
        rc = lib.hdrnet_slice_apply_rows_f32_ws(
            grid.data_ptr(), guide.data_ptr(), input.data_ptr(), out.data_ptr(), B, height, W, rows, y_off,
            gh, gw, gd, n_in, n_out, int(has_offset), int(variant), ws_ptr, ws_bytes, stream)
    _lib.check(rc, "BilateralSliceApply(rows)")
    return out


def slice_indices(guide: torch.Tensor, grid_shape) -> torch.Tensor:
    """Debug: unclamped lower cell indices (gx0, gy0, gz0) per pixel, int32 [B,H,W,3], from
    the same device code the slice kernels run (bit-exactness check vs the oracle)."""
    lib = _lib.load()
    _require_cuda()
    guide = _f32c(guide, "guide")
    if guide.dim() != 3 or guide.device.type != "cuda":
        raise ValueError("guide must be a CUDA tensor [B,H,W]")
    gh, gw, gd = (int(v) for v in grid_shape)
    B, H, W = guide.shape
    idx = torch.empty((B, H, W, 3), dtype=torch.int32, device=guide.device)
    with torch.cuda.device(guide.device):
        stream = torch.cuda.current_stream(guide.device).cuda_stream
        rc = lib.hdrnet_slice_indices_i32(guide.data_ptr(), idx.data_ptr(), B, H, W, gh, gw, gd,
                                          stream)
    _lib.check(rc, "slice_indices")
    return idx
