"""Training data from image pairs, batched on the device: the reference's ``ImageFilesDataPipeline``
(hdrnet/data_pipeline.py:126-240); and from input images alone, ``UnsharpMaskDataPipeline``, whose
targets are unsharp masks of the inputs (this project's definition: its class docstring).

Layout (data_pipeline.py:174-200): ``<data_dir>/filelist.txt`` names one file per line; the pair is
``<data_dir>/input/<name>`` and ``<data_dir>/output/<name>``.  ``path`` may be the directory or the
``filelist.txt`` in it (the reference's CLI is given the latter).

At start-up every pair is decoded on ``nthreads`` host threads (``cv2.imread(IMREAD_UNCHANGED)``;
alpha dropped, BGR -> RGB, grey replicated to 3 channels, as bin/run.py decodes) and kept in its
storage format (uint8, uint16 or float32, chosen per file).  Each batch is ONE kernel
(``hdrnet_train_batch_f32``, csrc/train_batch.cu) that gathers the flipped, rotated and cropped
full-resolution input and target and the nearest-neighbour network input.  Where its sources live
is chosen at start-up from the free device memory (``device_budget``):

* Device tier, when the dataset fits beside ``memory_margin``: every pair is uploaded once into one
  device buffer and the kernel reads the crops straight from it; the host only draws random numbers.
* Streamed tier, otherwise: the decoded pairs stay on the host.  A crop reads only its
  ``source_window``, so host threads copy each sample's input and target windows into one of two
  pinned staging slots, one host-to-device copy per batch moves the slot to one of two device slots
  on a copy stream, and the kernel reads the windows there.  Batches ``step + 1, step + 2`` are
  built ahead while ``step`` trains; the batches are bitwise those of the device tier.

Only when even the two device staging slots do not fit is ``MemoryError`` raised.

Semantics are ``_augment_data`` (data_pipeline.py:126-171): flip left-right, flip up-down (each
with p = 1/2), rot90 by k uniform in 0..3 (counter-clockwise), then a uniform random crop of
``output_resolution`` on the rotated extent -- or the centre crop ``int((H - oh) / 2)`` -- and TF1
``resize_images(NEAREST_NEIGHBOR)`` of the crop to the network input.  Pixels become float32 as
``tf.to_float(x) / 255`` (or 65535).

Deliberate differences:

* The random draws are a pure function of ``(seed, step)`` (numpy's PCG64): a per-epoch
  permutation of the file list, then per-sample flips, rotation and crop origin.  A resumed run gets
  the batches an uninterrupted one would, with no RNG state saved.  TF's random streams (and its
  shuffling queue) cannot be reproduced, so the batches are not the reference's.
* The network input is ``params['net_input_size']``; the reference hard-codes 256
  (data_pipeline.py:166).  They are equal at the default.
* Each file keeps its own pixel format; the reference decides from the first file of each folder.
* No queue runners: a batch is ready when its kernel has run.
* The whole dataset must fit in host memory: it is decoded once at start-up, not on demand.
"""
from __future__ import annotations

import concurrent.futures
import ctypes
import functools
import logging
import os
import threading
import time
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

__all__ = ["ImageFilesDataPipeline", "UnsharpMaskDataPipeline"]

log = logging.getLogger("data_pipeline")

# Device memory the cache leaves free for the training step itself (activations, gradients, Adam
# moments, workspaces): about 3x what a step at the reference's training size uses.
MEMORY_MARGIN = 2 << 30

_FMT = {np.dtype(np.uint8): _lib.PX_U8, np.dtype(np.uint16): _lib.PX_U16, np.dtype(np.float32): _lib.PX_F32}
_TORCH_FMT = {torch.uint8: _lib.PX_U8, torch.uint16: _lib.PX_U16, torch.float32: _lib.PX_F32}


def data_paths(path: str):
    """(data directory, filelist.txt path) of a data directory or of the filelist in it."""
    if os.path.isdir(path):
        return path, os.path.join(path, "filelist.txt")
    return os.path.dirname(os.path.abspath(path)), path


def read_filelist(filelist: str) -> list:
    """The names in ``filelist.txt``, one per non-blank line, surrounding whitespace stripped."""
    if not os.path.isfile(filelist):
        raise ValueError(f"{filelist}: no such file list (expected <data_dir>/filelist.txt)")
    with open(filelist) as f:
        names = [line.strip() for line in f if line.strip()]
    if not names:
        raise ValueError(f"{filelist} names no images")
    return names


def decode_image(path: str) -> np.ndarray:
    """[H, W, 3] RGB in the file's storage format (uint8, uint16 or float32)."""
    import cv2
    im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if im is None:
        raise ValueError(f"{path}: cannot be read as an image")
    if im.ndim == 2:
        im = im[:, :, None]
    if im.shape[2] == 1:
        im = np.repeat(im, 3, axis=2)
    im = im[:, :, :3][:, :, ::-1]                 # drop alpha, BGR -> RGB
    if im.dtype not in _FMT:
        raise ValueError(f"{path}: pixel type {im.dtype} is not uint8, uint16 or float32")
    return np.ascontiguousarray(im)


def load_pairs(path: str, nthreads: int = 1):
    """(names, inputs, targets, data directory): every pair named by the file list, decoded."""
    dirname, filelist = data_paths(path)
    names = read_filelist(filelist)
    files = [os.path.join(dirname, sub, n) for n in names for sub in ("input", "output")]
    with concurrent.futures.ThreadPoolExecutor(max(1, int(nthreads))) as ex:
        ims = list(ex.map(decode_image, files))
    return names, ims[0::2], ims[1::2], dirname


def load_inputs(path: str, nthreads: int = 1):
    """(names, inputs, data directory): every input named by the file list, decoded; ``output/`` is
    not read (UnsharpMaskDataPipeline computes its targets)."""
    dirname, filelist = data_paths(path)
    names = read_filelist(filelist)
    with concurrent.futures.ThreadPoolExecutor(max(1, int(nthreads))) as ex:
        ims = list(ex.map(decode_image, [os.path.join(dirname, "input", n) for n in names]))
    return names, ims, dirname


def check_inputs(names, inputs, dirname, output_resolution, rotate: bool) -> None:
    """ValueError naming the file when an input is smaller than ``output_resolution`` for a rotation
    the flags allow: ``check_pairs`` for a pipeline without target images."""
    check_pairs(names, inputs, inputs, dirname, output_resolution, rotate)


def check_pairs(names, inputs, targets, dirname, output_resolution, rotate: bool) -> None:
    """ValueError naming the file when a pair's images differ in size, or when a pair is smaller
    than ``output_resolution`` for a rotation the flags allow (the reference asserts)."""
    oh, ow = (int(v) for v in output_resolution)
    for name, a, b in zip(names, inputs, targets):
        src = os.path.join(dirname, "input", name)
        if a.shape[:2] != b.shape[:2]:
            raise ValueError(f"{src} is {a.shape[0]}x{a.shape[1]} but {os.path.join(dirname, 'output', name)} "
                             f"is {b.shape[0]}x{b.shape[1]}: an input/output pair must have one size")
        H, W = a.shape[:2]
        extents = [(H, W), (W, H)] if rotate else [(H, W)]
        for rh, rw in extents:
            if oh > rh or ow > rw:
                how = " when rotated" if (rh, rw) != (H, W) else ""
                raise ValueError(f"{src} is {H}x{W}, smaller{how} than the output resolution {oh}x{ow}")


class Draw(NamedTuple):
    """One sample of a batch: which pair, and its augmentation."""
    index: int
    fliplr: bool
    flipud: bool
    rot90: int
    crop_y: int
    crop_x: int


class Sampler:
    """The batches of a run as a pure function of ``(seed, step)``.

    Sample ``p = step * batch_size + i`` of the run is entry ``p mod n`` of epoch ``p // n``'s
    permutation of the n pairs (the identity without ``shuffle``).  Its flips (p = 1/2 each), its
    rotation k (uniform in 0..3) and its crop origin (uniform over the rotated extent, else the
    centre crop ``int((H - oh) / 2)``) come from a PCG64 stream seeded with ``(seed, step)``; the
    draws are made whatever the flags, so enabling one augmentation does not move the others.

    ``shard=(rank, world)`` names the part of each batch one rank of a data-parallel run builds:
    rows ``[rank * B / world, (rank + 1) * B / world)`` of ``draws(step)`` (``shard_draws``);
    ``batch_size`` stays the whole batch's, which ``world`` must divide."""

    def __init__(self, sizes, batch_size, output_resolution, shuffle=False, fliplr=False, flipud=False,
                 rotate=False, random_crop=False, seed=0, shard=(0, 1)):
        self.sizes = [tuple(int(v) for v in s) for s in sizes]
        self.batch_size = int(batch_size)
        self.oh, self.ow = (int(v) for v in output_resolution)
        self.shuffle, self.fliplr, self.flipud = bool(shuffle), bool(fliplr), bool(flipud)
        self.rotate, self.random_crop, self.seed = bool(rotate), bool(random_crop), int(seed)
        self.rank, self.world = check_shard(shard, self.batch_size)
        self.shard_size = self.batch_size // self.world
        if not self.sizes:
            raise ValueError("no samples")

    @functools.lru_cache(maxsize=4)
    def permutation(self, epoch: int) -> np.ndarray:
        n = len(self.sizes)
        if not self.shuffle:
            return np.arange(n)
        return np.random.Generator(np.random.PCG64([self.seed, 0, epoch])).permutation(n)

    def draws(self, step: int) -> list:
        n = len(self.sizes)
        rng = np.random.Generator(np.random.PCG64([self.seed, 1, int(step)]))
        out = []
        for i in range(self.batch_size):
            p = int(step) * self.batch_size + i
            index = int(self.permutation(p // n)[p % n])
            lr, ud = rng.random(2) < 0.5
            k = int(rng.integers(0, 4))
            uy, ux = rng.random(2)
            lr, ud, k = bool(lr) and self.fliplr, bool(ud) and self.flipud, k if self.rotate else 0
            H, W = self.sizes[index]
            rh, rw = (W, H) if k % 2 else (H, W)
            if self.random_crop:
                cy, cx = int(uy * (rh - self.oh + 1)), int(ux * (rw - self.ow + 1))
            else:
                cy, cx = int((rh - self.oh) / 2), int((rw - self.ow) / 2)     # tf.to_int32: truncation
            out.append(Draw(index, lr, ud, k, cy, cx))
        return out

    def shard_draws(self, step: int) -> list:
        """This shard's rows of ``draws(step)``."""
        lo = self.rank * self.shard_size
        return self.draws(step)[lo:lo + self.shard_size]


def check_shard(shard, batch_size: int):
    """``(rank, world)`` of ``shard``; ValueError unless 0 <= rank < world and world divides
    ``batch_size`` (every rank builds an equal part of the batch)."""
    rank, world = (int(v) for v in shard)
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"shard {tuple(shard)}: expected (rank, world) with 0 <= rank < world")
    if int(batch_size) % world:
        raise ValueError(f"the batch size {batch_size} is not a multiple of the world size {world}: every rank "
                         "must build an equal part of the batch")
    return rank, world


def source_window(H: int, W: int, draw: Draw, oh: int, ow: int):
    """``(y0, x0, h, w)``: the rectangle of the un-augmented H x W source that ``draw``'s oh x ow crop
    reads (h x w = oh x ow, or ow x oh when ``rot90`` is odd).

    The crop maps onto the source as ``source_pixel`` in csrc/train_batch.cu does: rotation on the
    flipped source.  Cut out as an image of its own, the window gives the same crop (and so the same
    nearest-neighbour network input) under the same flips and rotation with the crop origin at
    (0, 0)."""
    cy, cx, k = int(draw.crop_y), int(draw.crop_x), int(draw.rot90)
    # the crop's rows [cy, cy + oh) and columns [cx, cx + ow) of the rotated extent, on the flipped
    # source: (first row, rows, first column, columns)
    if k == 0:
        y, h, x, w = cy, oh, cx, ow
    elif k == 1:                                 # y = c, x = W - 1 - r
        y, h, x, w = cx, ow, W - cy - oh, oh
    elif k == 2:                                 # y = H - 1 - r, x = W - 1 - c
        y, h, x, w = H - cy - oh, oh, W - cx - ow, ow
    elif k == 3:                                 # y = H - 1 - c, x = r
        y, h, x, w = H - cx - ow, ow, cy, oh
    else:
        raise ValueError(f"rot90 must be 0..3, got {k}")
    if draw.flipud:
        y = H - y - h
    if draw.fliplr:
        x = W - x - w
    if y < 0 or x < 0 or y + h > H or x + w > W:
        raise ValueError(f"the {oh}x{ow} crop at ({cy}, {cx}) with rot90 {k} lies outside the {H}x{W} source")
    return y, x, h, w


def _check_source(t, what):
    if not isinstance(t, torch.Tensor) or t.dtype not in _TORCH_FMT or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f"{what} must be a [H, W, 3] uint8 / uint16 / float32 tensor")
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{what} must be a contiguous CUDA tensor")


def train_batch(inputs, targets, draws, output_resolution, size: int, out=None):
    """One batch through ``hdrnet_train_batch_f32``: ``inputs[b]`` / ``targets[b]`` are the b-th
    sample's source images ([H, W, 3] CUDA tensors, uint8 / uint16 / float32, any mix), ``draws[b]``
    its augmentation (``Draw``; ``index`` is not used here).  Returns ``(image_input, image_output,
    lowres_input)``: [B, oh, ow, 3], [B, oh, ow, 3], [B, size, size, 3] float32, written into
    ``out`` when given."""
    oh, ow = (int(v) for v in output_resolution)
    B = len(draws)
    if len(inputs) != B or len(targets) != B:
        raise ValueError("one input and one target per draw")
    descs = (_lib.TrainSample * max(B, 1))()
    for b, (x, y, d) in enumerate(zip(inputs, targets, draws)):
        _check_source(x, f"inputs[{b}]")
        _check_source(y, f"targets[{b}]")
        if x.shape != y.shape or x.device != y.device:
            raise ValueError(f"sample {b}: input {tuple(x.shape)} and target {tuple(y.shape)} differ in extent or device")
        descs[b] = _lib.TrainSample(x.data_ptr(), y.data_ptr(), _TORCH_FMT[x.dtype], _TORCH_FMT[y.dtype],
                                    x.shape[0], x.shape[1], int(bool(d.fliplr)), int(bool(d.flipud)), int(d.rot90),
                                    int(d.crop_y), int(d.crop_x))
    device = inputs[0].device if B else torch.device("cuda", torch.cuda.current_device())
    if out is None:
        out = (torch.empty((B, oh, ow, 3), dtype=torch.float32, device=device),
               torch.empty((B, oh, ow, 3), dtype=torch.float32, device=device),
               torch.empty((B, size, size, 3), dtype=torch.float32, device=device))
    for t, shape in zip(out, ((B, oh, ow, 3), (B, oh, ow, 3), (B, size, size, 3))):
        if t.shape != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != device:
            raise ValueError(f"out: expected contiguous float32 {shape} tensors on {device}")
    with torch.cuda.device(device):
        rc = _lib.load().hdrnet_train_batch_f32(
            ctypes.cast(descs, ctypes.c_void_p), B, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
            oh, ow, int(size), torch.cuda.current_stream(device).cuda_stream)
    _lib.check(rc, "train_batch")
    return out


ALIGN = 256           # byte alignment of every image in the device cache and of every staged window
STREAM_SLOTS = 2      # pinned and device staging slots of the streamed tier


def _aligned(nbytes: int) -> int:
    return -(-int(nbytes) // ALIGN) * ALIGN


def cache_bytes(images) -> int:
    """Bytes of the device tier's cache of ``images`` (each starts 256-byte aligned)."""
    return sum(_aligned(im.nbytes) for im in images)


def slot_bytes(formats, batch_size: int, output_resolution) -> int:
    """Bytes of one staging slot of the streamed tier: ``batch_size`` samples of the widest
    (input dtype, target dtype) pair in ``formats``, each window of oh x ow pixels 256-byte aligned."""
    oh, ow = (int(v) for v in output_resolution)
    widest = max(_aligned(oh * ow * 3 * np.dtype(a).itemsize) + _aligned(oh * ow * 3 * np.dtype(b).itemsize)
                 for a, b in formats)
    return int(batch_size) * widest


USM_MAX_SIGMA = 32.0    # radius int(4 * 32 + 0.5) = 128


def check_usm(blur_sigma, sharpen):
    """``(blur_sigma, sharpen)`` as floats; ValueError unless 0 < blur_sigma <= 32 and sharpen is
    finite."""
    try:
        sigma, amount = float(blur_sigma), float(sharpen)
    except (TypeError, ValueError):
        raise ValueError(f"blur_sigma {blur_sigma!r} and sharpen {sharpen!r} must be numbers") from None
    if not 0.0 < sigma <= USM_MAX_SIGMA:
        raise ValueError(f"blur_sigma must be in (0, {USM_MAX_SIGMA:g}] source pixels, got {blur_sigma!r}")
    if not np.isfinite(amount):
        raise ValueError(f"sharpen must be a finite number, got {sharpen!r}")
    return sigma, amount


def usm_radius(blur_sigma) -> int:
    """The Gaussian's radius in source pixels: scipy.ndimage.gaussian_filter1d's ``int(4.0 * sigma + 0.5)``."""
    return int(4.0 * float(blur_sigma) + 0.5)


def grown_window(H: int, W: int, draw: Draw, oh: int, ow: int, radius: int):
    """``(y0, x0, h, w)``: ``source_window`` grown by ``radius`` on each side and clipped to the H x W
    source, the pixels the unsharp-mask target of ``draw``'s crop reads."""
    y, x, h, w = source_window(H, W, draw, oh, ow)
    r = int(radius)
    y0, x0 = max(0, y - r), max(0, x - r)
    return y0, x0, min(H, y + h + r) - y0, min(W, x + w + r) - x0


def usm_slot_bytes(inputs, batch_size: int, output_resolution, radius: int, rotate: bool) -> int:
    """Bytes of one staging slot of UnsharpMaskDataPipeline's streamed tier: ``batch_size`` samples
    of the largest grown window (``grown_window``) any of ``inputs`` can give under the rotations
    ``rotate`` allows, each 256-byte aligned."""
    oh, ow = (int(v) for v in output_resolution)
    r = int(radius)
    widest = 0
    for im in inputs:
        H, W = im.shape[:2]
        for h, w in ((oh, ow), (ow, oh)) if rotate else ((oh, ow),):
            widest = max(widest, _aligned(min(H, h + 2 * r) * min(W, w + 2 * r) * 3 * im.itemsize))
    return int(batch_size) * widest


def usm_batch(inputs, draws, output_resolution, size, blur_sigma, sharpen, windows=None, out=None):
    """One UnsharpMaskDataPipeline batch through ``hdrnet_train_batch_usm_f32``: ``inputs[b]`` is the
    b-th sample's source ([H, W, 3] CUDA tensor, uint8 / uint16 / float32, any mix) or, when
    ``windows[b] = (H, W, y0, x0)`` is given, the window of an H x W source at (y0, x0) that holds
    ``grown_window`` of its crop; ``draws[b]`` is the augmentation on the full source.  Returns
    ``(image_input, image_output, lowres_input)`` as ``train_batch`` does, the target being the
    unsharp mask of the input (``UnsharpMaskDataPipeline``); ``size`` None leaves out the network
    input (returned as None) and ``out`` may then hold None in its place."""
    sigma, amount = check_usm(blur_sigma, sharpen)
    oh, ow = (int(v) for v in output_resolution)
    B = len(draws)
    if len(inputs) != B or (windows is not None and len(windows) != B):
        raise ValueError("one input (and window) per draw")
    descs = (_lib.UsmSample * max(B, 1))()
    for b, (x, d) in enumerate(zip(inputs, draws)):
        _check_source(x, f"inputs[{b}]")
        H, W, y0, x0 = (x.shape[0], x.shape[1], 0, 0) if windows is None else (int(v) for v in windows[b])
        descs[b] = _lib.UsmSample(x.data_ptr(), _TORCH_FMT[x.dtype], H, W, y0, x0, x.shape[0], x.shape[1],
                                  int(bool(d.fliplr)), int(bool(d.flipud)), int(d.rot90), int(d.crop_y),
                                  int(d.crop_x))
    device = inputs[0].device if B else torch.device("cuda", torch.cuda.current_device())
    shapes = ((B, oh, ow, 3), (B, oh, ow, 3), None if size is None else (B, int(size), int(size), 3))
    if out is None:
        out = tuple(None if sh is None else torch.empty(sh, dtype=torch.float32, device=device) for sh in shapes)
    for t, shape in zip(out, shapes):
        if shape is None:
            if t is not None:
                raise ValueError("out: no network input is written without size")
        elif t is None or t.shape != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != device:
            raise ValueError(f"out: expected contiguous float32 {shape} tensors on {device}")
    lib = _lib.load()
    ws_bytes = lib.hdrnet_train_batch_usm_workspace_bytes(ctypes.cast(descs, ctypes.c_void_p), B, oh, ow, sigma)
    with torch.cuda.device(device):
        ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=device)
        rc = lib.hdrnet_train_batch_usm_f32(
            ctypes.cast(descs, ctypes.c_void_p), B, out[0].data_ptr(), out[1].data_ptr(),
            0 if out[2] is None else out[2].data_ptr(), oh, ow, 0 if size is None else int(size), sigma, amount,
            ws.data_ptr(), int(ws_bytes), torch.cuda.current_stream(device).cuda_stream)
    _lib.check(rc, "usm_batch")
    return out


def unsharp_mask(image, blur_sigma, sharpen):
    """The unsharp-mask target of a whole image: ``clip(x + sharpen * (x - G * x), 0, 1)`` with x the
    float32 pixels of ``image`` ([H, W, 3] CUDA tensor, uint8 / uint16 / float32; integers as v / 255
    or v / 65535), G the Gaussian of ``blur_sigma`` source pixels with reflection at the image's edges
    (``UnsharpMaskDataPipeline``).  Returns [H, W, 3] float32: the target the pipeline gives the
    whole-image crop with no flip or rotation, from the same kernel.  Scores ``bin/run.py`` outputs
    against the targets a USM-trained model learned."""
    _check_source(image, "image")
    H, W = int(image.shape[0]), int(image.shape[1])
    fin = torch.empty((1, H, W, 3), dtype=torch.float32, device=image.device)
    fout = torch.empty_like(fin)
    usm_batch([image], [Draw(0, False, False, 0, 0, 0)], (H, W), None, blur_sigma, sharpen,
              out=(fin, fout, None))
    return fout[0]


def device_budget(device) -> int:
    """Free device memory on ``device`` in bytes, as the tier selection sees it."""
    return torch.cuda.mem_get_info(device)[0]


def choose_tier(dataset_bytes: int, staging_bytes: int, device, margin: int = MEMORY_MARGIN) -> str:
    """``"device"`` when the dataset fits in ``device_budget(device) - margin``, else ``"stream"``
    when the staging slots do; MemoryError, naming the byte counts, when neither fits."""
    free = device_budget(device)
    available = free - margin
    if dataset_bytes <= available:
        return "device"
    if staging_bytes <= available:
        return "stream"
    raise MemoryError(
        f"the dataset needs {dataset_bytes} bytes of device memory and streaming it from the host needs "
        f"{staging_bytes} bytes of staging slots; {free} bytes are free and {margin} are kept for training, so "
        f"{max(available, 0)} are available: use a smaller batch or output resolution")


class DeviceCache:
    """Decoded images in one device buffer, each in its own storage format."""

    def __init__(self, images, device):
        offsets, total = [], 0
        for im in images:
            offsets.append(total)
            total += _aligned(im.nbytes)
        self.nbytes = total
        self.buffer = torch.empty(total, dtype=torch.uint8, device=device)
        self.images = []
        for im, off in zip(images, offsets):
            flat = torch.from_numpy(np.ascontiguousarray(im).reshape(-1).view(np.uint8))
            dst = self.buffer[off:off + im.nbytes]
            dst.copy_(flat)
            self.images.append(dst.view(getattr(torch, im.dtype.name)).view(im.shape))


class _Staged(NamedTuple):
    """A batch in device slot ``slot``: each sample's (input, target) window views and its draw with
    the crop at the window's origin; ``uploaded`` is the event of the slot's copy.  Without targets
    (UnsharpMaskDataPipeline) each view is the crop's window grown by the blur radius, ``draws`` keep
    the crop on the full source and ``windows`` holds each view's ``(H, W, y0, x0)``.  ``nbytes``: the
    bytes the slot's copy moved."""
    slot: int
    inputs: list
    targets: list
    draws: list
    uploaded: object
    windows: list = None
    nbytes: int = 0


class HostStream:
    """The streamed tier: decoded pairs on the host, each batch's crop windows staged through
    ``STREAM_SLOTS`` pinned and device slots by a producer thread, packed by ``nthreads`` workers.

    A device slot is reused only after the batch kernel that read it has been enqueued (its
    ``consumed`` event recorded on the consumer's stream; the copy stream waits on it), and a pinned
    slot only after its previous upload has completed (the producer waits on the host)."""

    def __init__(self, inputs, targets, sampler, output_resolution, device, nthreads=1, radius=None):
        self.inputs, self.targets, self.sampler = inputs, targets, sampler
        self.oh, self.ow = (int(v) for v in output_resolution)
        self.device = device
        self.radius = radius        # targets None: stage each crop's window grown by this
        if targets is None:
            self.slot_bytes = usm_slot_bytes(inputs, sampler.shard_size, output_resolution, radius,
                                             sampler.rotate)
        else:
            self.slot_bytes = slot_bytes({(a.dtype, b.dtype) for a, b in zip(inputs, targets)},
                                         sampler.shard_size, output_resolution)
        with torch.cuda.device(device):
            self.copy_stream = torch.cuda.Stream(device)
            with torch.cuda.stream(self.copy_stream):     # the blocks belong to the stream that writes them
                self.dev = [torch.empty(self.slot_bytes, dtype=torch.uint8, device=device)
                            for _ in range(STREAM_SLOTS)]
            self.pinned = [torch.empty(self.slot_bytes, dtype=torch.uint8, pin_memory=True)
                           for _ in range(STREAM_SLOTS)]
            self.uploaded = [torch.cuda.Event() for _ in range(STREAM_SLOTS)]
        self.consumed = [None] * STREAM_SLOTS              # event: the last batch kernel that read the slot
        self.busy = [False] * STREAM_SLOTS                 # the slot holds a batch not yet consumed
        self.ready = {}                                    # step -> _Staged or the exception that built it
        self.filling = None                                # (step, generation) being built
        self.next = None                                   # next step to build; None: idle
        self.generation = 0
        self.closed = False
        self.pack_seconds, self.packed = 0.0, 0            # host time copying windows, batches packed
        self.cond = threading.Condition()
        self.pool = concurrent.futures.ThreadPoolExecutor(max(1, int(nthreads)),
                                                          thread_name_prefix="hdrnet-stream-pack")
        self.thread = threading.Thread(target=self._produce, name="hdrnet-stream", daemon=True)
        self.thread.start()

    # ---- producer ------------------------------------------------------------------------------
    def _pack(self, slot: int, step: int) -> _Staged:
        """Copy batch ``step``'s windows (the sampler's shard of them) into pinned slot ``slot`` and
        upload it to device slot ``slot`` on the copy stream."""
        draws = self.sampler.shard_draws(step)
        if self.targets is None:
            return self._pack_grown(slot, draws)
        layout, off = [], 0
        for d in draws:
            a, b = self.inputs[d.index], self.targets[d.index]
            y0, x0, h, w = source_window(a.shape[0], a.shape[1], d, self.oh, self.ow)
            na, nb = h * w * 3 * a.itemsize, h * w * 3 * b.itemsize
            layout.append((d, (y0, x0, h, w), off, off + _aligned(na)))
            off += _aligned(na) + _aligned(nb)
        self.uploaded[slot].synchronize()                  # the pinned slot's last upload has completed
        host = self.pinned[slot].numpy()

        def copy(item):
            d, (y0, x0, h, w), oa, ob = item
            for src, o in ((self.inputs[d.index], oa), (self.targets[d.index], ob)):
                dst = host[o:o + h * w * 3 * src.itemsize].view(src.dtype).reshape(h, w, 3)
                np.copyto(dst, src[y0:y0 + h, x0:x0 + w])

        t0 = time.perf_counter()
        list(self.pool.map(copy, layout))
        self.pack_seconds += time.perf_counter() - t0
        self.packed += 1
        with torch.cuda.device(self.device), torch.cuda.stream(self.copy_stream):
            if self.consumed[slot] is not None:
                self.copy_stream.wait_event(self.consumed[slot])
            self.dev[slot][:off].copy_(self.pinned[slot][:off], non_blocking=True)
            self.uploaded[slot].record(self.copy_stream)
        dev = self.dev[slot]
        inputs, targets, crops = [], [], []
        for d, (_, _, h, w), oa, ob in layout:
            a, b = self.inputs[d.index], self.targets[d.index]
            inputs.append(dev[oa:oa + h * w * 3 * a.itemsize].view(getattr(torch, a.dtype.name)).view(h, w, 3))
            targets.append(dev[ob:ob + h * w * 3 * b.itemsize].view(getattr(torch, b.dtype.name)).view(h, w, 3))
            crops.append(d._replace(crop_y=0, crop_x=0))
        return _Staged(slot, inputs, targets, crops, self.uploaded[slot], None, off)

    def _pack_grown(self, slot: int, draws) -> _Staged:
        """``_pack`` without targets: each sample's crop window grown by ``radius`` on each side and
        clipped to the source (``grown_window``), the draw unchanged."""
        layout, off = [], 0
        for d in draws:
            a = self.inputs[d.index]
            win = grown_window(a.shape[0], a.shape[1], d, self.oh, self.ow, self.radius)
            layout.append((d, win, off))
            off += _aligned(win[2] * win[3] * 3 * a.itemsize)
        self.uploaded[slot].synchronize()                  # the pinned slot's last upload has completed
        host = self.pinned[slot].numpy()

        def copy(item):
            d, (y0, x0, h, w), o = item
            src = self.inputs[d.index]
            np.copyto(host[o:o + h * w * 3 * src.itemsize].view(src.dtype).reshape(h, w, 3),
                      src[y0:y0 + h, x0:x0 + w])

        t0 = time.perf_counter()
        list(self.pool.map(copy, layout))
        self.pack_seconds += time.perf_counter() - t0
        self.packed += 1
        with torch.cuda.device(self.device), torch.cuda.stream(self.copy_stream):
            if self.consumed[slot] is not None:
                self.copy_stream.wait_event(self.consumed[slot])
            self.dev[slot][:off].copy_(self.pinned[slot][:off], non_blocking=True)
            self.uploaded[slot].record(self.copy_stream)
        dev = self.dev[slot]
        inputs, windows = [], []
        for d, (y0, x0, h, w), o in layout:
            a = self.inputs[d.index]
            inputs.append(dev[o:o + h * w * 3 * a.itemsize].view(getattr(torch, a.dtype.name)).view(h, w, 3))
            windows.append((a.shape[0], a.shape[1], y0, x0))
        return _Staged(slot, inputs, None, list(draws), self.uploaded[slot], windows, off)

    def _produce(self):
        while True:
            with self.cond:
                while not self.closed and (self.next is None or all(self.busy)):
                    self.cond.wait()
                if self.closed:
                    return
                step, gen = self.next, self.generation
                slot = self.busy.index(False)
                self.busy[slot] = True
                self.filling = (step, gen)
                self.next = step + 1
            try:
                item = self._pack(slot, step)
            except BaseException as e:          # handed to the batch() that asks for this step
                item = e
            with self.cond:
                self.filling = None
                if gen != self.generation:
                    self.busy[slot] = False     # built for a sequence that was restarted
                else:
                    self.ready[step] = item
                    if isinstance(item, BaseException):
                        self.busy[slot] = False
                        self.next = None        # stop building ahead after a failure
                self.cond.notify_all()

    # ---- consumer ------------------------------------------------------------------------------
    def _release(self, step):
        item = self.ready.pop(step)
        if isinstance(item, _Staged):
            self.busy[item.slot] = False

    def take(self, step: int) -> _Staged:
        """Batch ``step``'s staged windows, built ahead when ``step`` follows the last request, else
        built now (and building ahead restarts from ``step + 1``)."""
        step = int(step)
        with self.cond:
            if self.closed:
                raise RuntimeError("the data pipeline is closed")
            expected = step in self.ready or (self.filling is not None and self.filling == (step, self.generation))
            for s in [s for s in self.ready if s < step or not expected]:
                self._release(s)
            if not expected:
                self.generation += 1
                self.next = step
            self.cond.notify_all()
            with torch.profiler.record_function("data_pipeline.stream.wait"):
                while step not in self.ready:
                    self.cond.wait()
            item = self.ready[step]
            if isinstance(item, BaseException):
                self.ready.pop(step)
                raise item
            if self.next is None:
                self.next = step + 1
            return item

    def consumed_by(self, item: _Staged, stream) -> None:
        """The batch kernel that reads ``item`` has been enqueued on ``stream``: the slot may be
        refilled once it has run."""
        ev = torch.cuda.Event()
        ev.record(stream)
        self.dev[item.slot].record_stream(stream)
        with self.cond:
            self.consumed[item.slot] = ev
            for s, it in list(self.ready.items()):
                if it is item:
                    self._release(s)
            self.cond.notify_all()

    def close(self) -> None:
        with self.cond:
            if self.closed:
                return
            self.closed = True
            self.cond.notify_all()
        self.thread.join()
        self.pool.shutdown(wait=True)
        self.copy_stream.synchronize()


class ImageFilesDataPipeline:
    """The reference's ImageFilesDataPipeline on the device (keyword names of data_pipeline.py:71-82).

    ``batch(step)`` returns the reference's sample dict for training step ``step``: ``image_input``,
    ``image_output`` [B, oh, ow, 3] and ``lowres_input`` [B, S, S, 3], float32 on ``device``, with
    S = ``params['net_input_size']`` (256 without params).  ``tier`` is ``"device"`` or ``"stream"``
    (module docstring); ``close()`` (or leaving a ``with`` block) stops the streamed tier's threads.

    ``shard=(rank, world)``: one rank of a data-parallel run.  ``batch_size`` is the whole batch, and
    ``batch(step)`` holds only this rank's B / world rows of it (``Sampler.shard_draws``), on either
    tier; the streamed tier packs and uploads only their windows.  ValueError, before any file is
    read, when ``world`` does not divide ``batch_size``."""

    def __init__(self, path, batch_size=32, output_resolution=(1080, 1920), shuffle=False, fliplr=False,
                 flipud=False, rotate=False, random_crop=False, params=None, nthreads=1, seed=0, device=None,
                 memory_margin=MEMORY_MARGIN, shard=(0, 1)):
        check_shard(shard, batch_size)
        self.path = path
        self.batch_size = int(batch_size)
        self.output_resolution = [int(v) for v in output_resolution]
        self.net_input_size = int((params or {}).get("net_input_size", 256))
        names, inputs, targets, dirname = load_pairs(path, nthreads)
        check_pairs(names, inputs, targets, dirname, self.output_resolution, rotate)
        self.names = names
        self.nsamples = len(names)
        self.sampler = Sampler([a.shape[:2] for a in inputs], batch_size, self.output_resolution, shuffle,
                               fliplr, flipud, rotate, random_crop, seed, shard)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        images = [im for pair in zip(inputs, targets) for im in pair]
        self.dataset_bytes = cache_bytes(images)
        self.staging_bytes = STREAM_SLOTS * slot_bytes({(a.dtype, b.dtype) for a, b in zip(inputs, targets)},
                                                       self.sampler.shard_size, self.output_resolution)
        self.tier = choose_tier(self.dataset_bytes, self.staging_bytes, self.device, memory_margin)
        self.stream = None
        if self.tier == "device":
            cache = DeviceCache(images, self.device)
            self.cache = cache
            self.inputs, self.targets = cache.images[0::2], cache.images[1::2]
            log.info("%s: %d pairs, %.1f MB on %s", dirname, self.nsamples, cache.nbytes / 1e6, self.device)
        else:
            self.stream = HostStream(inputs, targets, self.sampler, self.output_resolution, self.device, nthreads)
            log.info("%s: %d pairs, %.1f MB: more than the %.1f MB of %s's free memory less the %.1f MB kept "
                     "for training, so they stay on the host and each batch's crops are streamed through %d "
                     "staging slots of %.1f MB", dirname, self.nsamples, self.dataset_bytes / 1e6,
                     device_budget(self.device) / 1e6, self.device, memory_margin / 1e6, STREAM_SLOTS,
                     self.stream.slot_bytes / 1e6)

    def batch(self, step: int) -> dict:
        if self.stream is None:
            draws = self.sampler.shard_draws(step)
            fin, fout, low = train_batch([self.inputs[d.index] for d in draws],
                                         [self.targets[d.index] for d in draws],
                                         draws, self.output_resolution, self.net_input_size)
            return {"image_input": fin, "image_output": fout, "lowres_input": low}
        item = self.stream.take(step)
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(item.uploaded)
        try:
            fin, fout, low = train_batch(item.inputs, item.targets, item.draws, self.output_resolution,
                                         self.net_input_size)
        finally:
            self.stream.consumed_by(item, stream)
        return {"image_input": fin, "image_output": fout, "lowres_input": low}

    def close(self) -> None:
        """Stop and join the streamed tier's threads (nothing to do on the device tier)."""
        if self.stream is not None:
            self.stream.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class UnsharpMaskDataPipeline(ImageFilesDataPipeline):
    """Training data from input images alone: the target is an unsharp mask of the input.

    The reference's ``scripts/usm/*.sh`` recipes name this pipeline (``--data_pipeline
    UnsharpMaskDataPipeline --blur_sigma S --sharpen A``), but its ``data_pipeline.py`` does not define
    it and its ``train.py`` has neither flag; what follows is this project's definition.  With x the
    float32 input exactly as ``image_input`` holds it (v / 255, v / 65535, or float32 as stored):

    * b = G * x per channel, G the separable Gaussian of standard deviation ``blur_sigma`` source
      pixels: radius r = int(4 sigma + 0.5), weights exp(-k^2 / 2 sigma^2) for |k| <= r normalised to
      sum 1, along source x, then source y, with half-sample symmetric reflection (d c b a | a b c d,
      repeated when r reaches the extent) at the source image's edges: scipy's
      ``ndimage.gaussian_filter1d(..., mode="reflect", truncate=4.0)`` on each axis.
    * target = clip(x + sharpen * (x - b), 0, 1), in the range an image-file target has.
    * The target is a function of the un-augmented source pixel: the crop selects pixels (its edges
      get no boundary effects) and the flips and rot90 move them, so this equals augmenting first.
    * ``image_input`` and ``lowres_input`` are ``ImageFilesDataPipeline``'s for the same input and draw.

    0 < ``blur_sigma`` <= 32 and a finite ``sharpen``, else ValueError before any file is read.
    Takes ``ImageFilesDataPipeline``'s keywords; reads ``filelist.txt`` and ``input/`` only.  The
    device tier caches the inputs alone (``dataset_bytes`` counts them); the streamed tier stages
    each sample's crop window grown by r on each side and clipped to the source, and gives the
    device tier's batches bit for bit.  One kernel, ``hdrnet_train_batch_usm_f32``
    (csrc/usm_batch.cu), builds each batch."""

    def __init__(self, path, batch_size=32, output_resolution=(1080, 1920), shuffle=False, fliplr=False,
                 flipud=False, rotate=False, random_crop=False, params=None, nthreads=1, seed=0, device=None,
                 memory_margin=MEMORY_MARGIN, shard=(0, 1), blur_sigma=None, sharpen=None):
        self.blur_sigma, self.sharpen = check_usm(blur_sigma, sharpen)
        self.radius = usm_radius(self.blur_sigma)
        check_shard(shard, batch_size)
        self.path = path
        self.batch_size = int(batch_size)
        self.output_resolution = [int(v) for v in output_resolution]
        self.net_input_size = int((params or {}).get("net_input_size", 256))
        names, inputs, dirname = load_inputs(path, nthreads)
        check_inputs(names, inputs, dirname, self.output_resolution, rotate)
        self.names = names
        self.nsamples = len(names)
        self.sampler = Sampler([a.shape[:2] for a in inputs], batch_size, self.output_resolution, shuffle,
                               fliplr, flipud, rotate, random_crop, seed, shard)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.dataset_bytes = cache_bytes(inputs)
        self.staging_bytes = STREAM_SLOTS * usm_slot_bytes(inputs, self.sampler.shard_size, self.output_resolution,
                                                           self.radius, rotate)
        self.tier = choose_tier(self.dataset_bytes, self.staging_bytes, self.device, memory_margin)
        self.stream = None
        self.targets = None
        if self.tier == "device":
            self.cache = DeviceCache(inputs, self.device)
            self.inputs = self.cache.images
            log.info("%s: %d inputs, %.1f MB on %s (unsharp-mask targets: sigma %g, sharpen %g)", dirname,
                     self.nsamples, self.cache.nbytes / 1e6, self.device, self.blur_sigma, self.sharpen)
        else:
            self.stream = HostStream(inputs, None, self.sampler, self.output_resolution, self.device, nthreads,
                                     radius=self.radius)
            log.info("%s: %d inputs, %.1f MB: more than the %.1f MB of %s's free memory less the %.1f MB kept "
                     "for training, so they stay on the host and each batch's crops, grown by the blur radius %d, "
                     "are streamed through %d staging slots of %.1f MB", dirname, self.nsamples,
                     self.dataset_bytes / 1e6, device_budget(self.device) / 1e6, self.device, memory_margin / 1e6,
                     self.radius, STREAM_SLOTS, self.stream.slot_bytes / 1e6)

    def batch(self, step: int) -> dict:
        if self.stream is None:
            draws = self.sampler.shard_draws(step)
            fin, fout, low = usm_batch([self.inputs[d.index] for d in draws], draws, self.output_resolution,
                                       self.net_input_size, self.blur_sigma, self.sharpen)
            return {"image_input": fin, "image_output": fout, "lowres_input": low}
        item = self.stream.take(step)
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(item.uploaded)
        try:
            fin, fout, low = usm_batch(item.inputs, item.draws, self.output_resolution, self.net_input_size,
                                       self.blur_sigma, self.sharpen, windows=item.windows)
        finally:
            self.stream.consumed_by(item, stream)
        return {"image_input": fin, "image_output": fout, "lowres_input": low}
