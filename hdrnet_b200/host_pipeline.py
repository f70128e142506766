"""Host-resident images through the model, frame by frame, with the copies hidden.

The reference CLI (hdrnet/bin/run.py:145-190) loads an image on the host, feeds it through
``sess.run`` and saves the uint8 result: per frame, pixels go host -> device, the whole model
runs, the prediction comes back.  ``models.*.inference_image`` is that per-frame path with the
image already on the device; this module is the part around it for a batch / stream of frames
that lives in (pinned) host memory: three CUDA streams -- copy-in, compute, copy-out -- so that
frame i + 1 is uploading and frame i - 1 is downloading while frame i computes.  For 4K uint8
frames the model's GPU time per frame is well below a frame's PCIe time in one direction, so a
pipelined batch approaches the PCIe time of ONE direction instead of the sum of
upload + compute + download.

Device buffers are owned by the pipeline (``depth`` frames in, the model's outputs are held until
their download has finished), one call at a time per pipeline object; results are bitwise those
of ``inference_image`` on the same frames.
"""
from __future__ import annotations

import threading

import torch

from . import _lib


class HostImagePipeline:
    """``pipe = HostImagePipeline(models.HDRNetCurves, params, device); out = pipe(frames)``.

    frames: [N, H, W, 3] uint8 / uint16 / float32 CPU tensor (pinned memory for asynchronous
    copies; pageable memory works but serialises).  Returns / fills ``out`` [N, H, W, 3] uint8 (or
    float32 with ``out_dtype=torch.float32``) on the CPU.  ``frames_per_step`` frames travel and
    run together (1 = lowest latency per frame and the best overlap)."""

    def __init__(self, model_cls, params, device=None, depth: int = 2, frames_per_step: int = 1,
                 out_dtype=torch.uint8):
        if not torch.cuda.is_available():
            raise _lib.HdrnetLibraryError("HostImagePipeline needs a CUDA device: hdrnet_b200 has no CPU path")
        self.model_cls, self.params, self.out_dtype = model_cls, params, out_dtype
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.depth = max(2, int(depth))
        self.step = max(1, int(frames_per_step))
        self._lock = threading.Lock()
        with torch.cuda.device(self.device):
            self.s_in, self.s_run, self.s_out = (torch.cuda.Stream(self.device) for _ in range(3))
        self._in_bufs = None   # depth device tensors [step, H, W, 3], allocated on s_in

    def _buffers(self, shape, dtype):
        key = (tuple(shape), dtype)
        if self._in_bufs is None or self._in_bufs[0] != key:
            with torch.cuda.stream(self.s_in):   # the blocks belong to the stream that writes them
                bufs = [torch.empty(shape, dtype=dtype, device=self.device) for _ in range(self.depth)]
            self._in_bufs = (key, bufs)
        return self._in_bufs[1]

    def __call__(self, frames: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
        if not isinstance(frames, torch.Tensor) or frames.is_cuda:
            raise TypeError("frames must be a CPU tensor (device tensors go to inference_image directly)")
        if frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError(f"frames must be [N,H,W,3], got {tuple(frames.shape)}")
        if frames.dtype not in (torch.uint8, torch.uint16, torch.float32):
            raise TypeError(f"frames must be uint8, uint16 or float32, got {frames.dtype}")
        frames = frames.contiguous()
        N, H, W, _ = frames.shape
        if out is None:
            out = torch.empty((N, H, W, 3), dtype=self.out_dtype, pin_memory=frames.is_pinned())
        elif tuple(out.shape) != (N, H, W, 3) or out.dtype != self.out_dtype or out.is_cuda or not out.is_contiguous():
            raise ValueError("out must be a contiguous CPU tensor [N,H,W,3] of the pipeline's out_dtype")
        if N == 0:
            return out
        with self._lock, torch.cuda.device(self.device):
            bufs = self._buffers((self.step, H, W, 3), frames.dtype)
            caller = torch.cuda.current_stream(self.device)
            for s in (self.s_in, self.s_run, self.s_out):
                s.wait_stream(caller)          # whatever produced `frames` / last used `out` on the caller's stream
            n_steps = (N + self.step - 1) // self.step
            consumed = [None] * n_steps        # event: the model has read input buffer of step i
            results = []                       # device outputs, alive until the final synchronisation
            for i in range(n_steps):
                lo, hi = i * self.step, min(N, (i + 1) * self.step)
                buf = bufs[i % self.depth][: hi - lo]
                with torch.cuda.stream(self.s_in):
                    if i >= self.depth:
                        self.s_in.wait_event(consumed[i - self.depth])   # buffer free again
                    buf.copy_(frames[lo:hi], non_blocking=True)
                    arrived = torch.cuda.Event()
                    arrived.record(self.s_in)
                with torch.cuda.stream(self.s_run):
                    self.s_run.wait_event(arrived)
                    res = self.model_cls.inference_image(buf, self.params, out_dtype=self.out_dtype)
                    consumed[i] = torch.cuda.Event()
                    consumed[i].record(self.s_run)
                    done = consumed[i]
                with torch.cuda.stream(self.s_out):
                    self.s_out.wait_event(done)
                    res.record_stream(self.s_out)
                    out[lo:hi].copy_(res, non_blocking=True)
                results.append(res)
            self.s_out.synchronize()           # the call returns with `out` complete (sess.run semantics)
            self.s_run.synchronize()
        return out
