"""Training data from image pairs, kept on the device: the reference's ``ImageFilesDataPipeline``
(hdrnet/data_pipeline.py:126-240).

Layout (data_pipeline.py:174-200): ``<data_dir>/filelist.txt`` names one file per line; the pair is
``<data_dir>/input/<name>`` and ``<data_dir>/output/<name>``.  ``path`` may be the directory or the
``filelist.txt`` in it (the reference's CLI is given the latter).

At start-up every pair is decoded on ``nthreads`` host threads (``cv2.imread(IMREAD_UNCHANGED)``;
alpha dropped, BGR -> RGB, grey replicated to 3 channels, as bin/run.py decodes) and uploaded once,
in its storage format (uint8, uint16 or float32, chosen per file), into one device buffer.  Each
batch is then ONE kernel (``hdrnet_train_batch_f32``, csrc/train_batch.cu) that gathers the flipped,
rotated and cropped full-resolution input and target and the nearest-neighbour network input
straight from that cache; the host only draws random numbers.

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
* The whole dataset must fit in device memory; streaming from the host is not implemented.
"""
from __future__ import annotations

import concurrent.futures
import ctypes
import functools
import logging
import os
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

__all__ = ["ImageFilesDataPipeline"]

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
    draws are made whatever the flags, so enabling one augmentation does not move the others."""

    def __init__(self, sizes, batch_size, output_resolution, shuffle=False, fliplr=False, flipud=False,
                 rotate=False, random_crop=False, seed=0):
        self.sizes = [tuple(int(v) for v in s) for s in sizes]
        self.batch_size = int(batch_size)
        self.oh, self.ow = (int(v) for v in output_resolution)
        self.shuffle, self.fliplr, self.flipud = bool(shuffle), bool(fliplr), bool(flipud)
        self.rotate, self.random_crop, self.seed = bool(rotate), bool(random_crop), int(seed)
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


class DeviceCache:
    """Decoded images in one device buffer, each in its own storage format."""

    ALIGN = 256

    def __init__(self, images, device, margin: int = MEMORY_MARGIN):
        offsets, total = [], 0
        for im in images:
            offsets.append(total)
            total += -(-im.nbytes // self.ALIGN) * self.ALIGN
        free, _ = torch.cuda.mem_get_info(device)
        if total > free - margin:
            raise MemoryError(
                f"the dataset needs {total} bytes of device memory; {free} bytes are free and {margin} are kept "
                f"for training, so {max(free - margin, 0)} are available.  Streaming from the host is not "
                "implemented: use fewer or smaller images")
        self.nbytes = total
        self.buffer = torch.empty(total, dtype=torch.uint8, device=device)
        self.images = []
        for im, off in zip(images, offsets):
            flat = torch.from_numpy(np.ascontiguousarray(im).reshape(-1).view(np.uint8))
            dst = self.buffer[off:off + im.nbytes]
            dst.copy_(flat)
            self.images.append(dst.view(getattr(torch, im.dtype.name)).view(im.shape))


class ImageFilesDataPipeline:
    """The reference's ImageFilesDataPipeline on the device (keyword names of data_pipeline.py:71-82).

    ``batch(step)`` returns the reference's sample dict for training step ``step``: ``image_input``,
    ``image_output`` [B, oh, ow, 3] and ``lowres_input`` [B, S, S, 3], float32 on ``device``, with
    S = ``params['net_input_size']`` (256 without params)."""

    def __init__(self, path, batch_size=32, output_resolution=(1080, 1920), shuffle=False, fliplr=False,
                 flipud=False, rotate=False, random_crop=False, params=None, nthreads=1, seed=0, device=None,
                 memory_margin=MEMORY_MARGIN):
        self.path = path
        self.batch_size = int(batch_size)
        self.output_resolution = [int(v) for v in output_resolution]
        self.net_input_size = int((params or {}).get("net_input_size", 256))
        names, inputs, targets, dirname = load_pairs(path, nthreads)
        check_pairs(names, inputs, targets, dirname, self.output_resolution, rotate)
        self.names = names
        self.nsamples = len(names)
        self.sampler = Sampler([a.shape[:2] for a in inputs], batch_size, self.output_resolution, shuffle,
                               fliplr, flipud, rotate, random_crop, seed)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        cache = DeviceCache([im for pair in zip(inputs, targets) for im in pair], self.device, memory_margin)
        self.cache = cache
        self.inputs, self.targets = cache.images[0::2], cache.images[1::2]
        log.info("%s: %d pairs, %.1f MB on %s", dirname, self.nsamples, cache.nbytes / 1e6, self.device)

    def batch(self, step: int) -> dict:
        draws = self.sampler.draws(step)
        fin, fout, low = train_batch([self.inputs[d.index] for d in draws], [self.targets[d.index] for d in draws],
                                     draws, self.output_resolution, self.net_input_size)
        return {"image_input": fin, "image_output": fout, "lowres_input": low}
