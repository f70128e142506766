"""Multi-GPU plumbing for the batch-sharded path (SURVEY.md section 8e).

The hot path has no per-frame exchange: every output pixel depends only on its own image's
grid / guide / input (hdrnet/ops/bilateral_slice_apply.cu.cc:67-125 -- the batch index only
selects slabs), and the coefficient network is per-image (hdrnet/models.py:63, :95).  So the
design is one process per GPU, images sharded over ranks, and exactly ONE collective: a
broadcast of the flat coefficient-network weight buffer (~1.93 MB) at init over NCCL
(NVLink / NVSwitch); "nccl" on GPUs, "gloo" in the CPU tests.  The reference itself has no
distributed code at all (SURVEY.md section 2b).

Data-parallel training (bin/train.py under torchrun) adds, per step, one all-reduce of the flat
gradient buffer (all_reduce_mean_) and one of a few scalars (sum_over_ranks); the pointwise-NN guide's
training-mode batch norm adds one all-gather of the input moments (moments_over_ranks); the coefficient
network's, with --coefficient_batch_stats, one all-gather of each batch-norm layer's moments in the
forward and of its VJP sums in the backward (bn_moments_over_ranks, bn_sums_over_ranks); and each
checkpoint one all-gather of a digest of the state (check_ranks_agree).
"""
from __future__ import annotations

import hashlib
import os

import numpy as np
import torch
import torch.distributed as dist

__all__ = ["init_distributed", "shard_batch", "shard_rows", "shard_plan", "slice_apply_sharded",
           "broadcast_weights", "max_over_ranks", "finalize", "bind_to_gpu_numa", "gpu_cpu_affinity",
           "world_size", "all_reduce_mean_", "sum_over_ranks", "merge_moments", "moments_over_ranks",
           "bn_moments_over_ranks", "bn_sums_over_ranks", "check_ranks_agree"]


def gpu_cpu_affinity(device_index: int) -> list[int]:
    """CPUs of the NUMA node / root complex GPU `device_index` hangs off (NVML's "ideal CPU
    affinity", what `nvidia-smi topo -m` prints), restricted to the CPUs this process may run on.
    Empty when NVML or the information is not available."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(device_index)
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = [w * 64 + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1]
    except Exception:
        return []
    try:
        allowed = os.sched_getaffinity(0)
    except (AttributeError, OSError):
        allowed = set(range(os.cpu_count() or 1))
    return sorted(c for c in cpus if c in allowed)


def bind_to_gpu_numa(device_index: int) -> list[int]:
    """Pin this process (and the threads it starts later: the host path's copy threads, pinned
    allocations' first touch) to the CPUs local to its GPU.  Call BEFORE allocating pinned host
    memory: with eight ranks feeding 1.9 GB per step each, buffers that land on the other socket
    cross the inter-socket link on every H2D / D2H copy.  Returns the CPU list it bound to ([] = left unbound)."""
    cpus = gpu_cpu_affinity(device_index)
    if not cpus:
        return []
    try:
        os.sched_setaffinity(0, cpus)
    except (AttributeError, OSError):
        return []
    return cpus


def init_distributed(backend: str | None = None):
    """Join the process group described by torchrun's environment (RANK, WORLD_SIZE,
    LOCAL_RANK, MASTER_ADDR, MASTER_PORT).  Returns (rank, world, local_rank).  With
    WORLD_SIZE unset or 1 nothing is initialised."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        kwargs = {}
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
            kwargs["device_id"] = torch.device("cuda", local_rank)
        dist.init_process_group(backend, rank=rank, world_size=world, **kwargs)
    return rank, world, local_rank


def shard_batch(n_images: int, rank: int, world: int):
    """Contiguous, balanced image range [start, end) of rank `rank` (earlier ranks take the
    remainder).  Ranks beyond the image count get an empty range: use shard_rows then."""
    base, rem = divmod(n_images, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard_rows(height: int, rank: int, world: int):
    """Row band [y0, y1) of ONE image for rank `rank`: the fallback when there are fewer
    images than GPUs.  Every band needs the whole (98 KB) grid; no halo is needed because the
    gather is pointwise in x, y (the kernels take the band's y offset and the full height)."""
    return shard_batch(height, rank, world)


def shard_plan(n_images: int, height: int, rank: int, world: int):
    """What rank `rank` of `world` computes of a job of `n_images` images of `height` rows:
    ("batch", lo, hi) -- whole images [lo, hi) -- when every rank gets at least one image, else
    ("rows", y0, y1) -- rows [y0, y1) of EVERY image (SURVEY.md section 8e: fewer images than GPUs).
    The parts of all ranks tile the job exactly; a part may be empty (more ranks than rows)."""
    if n_images >= world:
        return ("batch",) + shard_batch(n_images, rank, world)
    return ("rows",) + shard_rows(height, rank, world)


def slice_apply_sharded(grid, guide, input, has_offset, rank: int, world: int):  # noqa: A002
    """This rank's part of ``hdrnet_ops.bilateral_slice_apply(grid, guide, input, has_offset)`` over
    the whole job's CUDA tensors (replicated or rank-local views): returns (plan, out_part) with
    plan = shard_plan(...) and out_part = out[lo:hi] ("batch") or out[:, y0:y1] ("rows").  No
    communication: the caller places the parts (they tile the output)."""
    from . import hdrnet_ops
    B, H = int(guide.shape[0]), int(guide.shape[1])
    plan = shard_plan(B, H, rank, world)
    kind, lo, hi = plan
    with torch.no_grad():
        if kind == "batch":
            return plan, hdrnet_ops.bilateral_slice_apply(grid[lo:hi], guide[lo:hi], input[lo:hi], has_offset)
        return plan, hdrnet_ops.bilateral_slice_apply_rows(grid, guide[:, lo:hi], input[:, lo:hi], has_offset,
                                                           y_off=lo, height=H)


def broadcast_weights(weights: dict | None, src: int = 0, device=None) -> dict:
    """One collective at init: rank `src` holds the weight dict (reference variable names ->
    numpy arrays); every rank returns an identical dict.  The arrays travel as ONE flat
    float32 buffer (a single broadcast: latency-bound, ~2 MB), preceded by a broadcast of the
    name/shape manifest."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        if weights is None:
            raise ValueError("broadcast_weights: no process group and no weights")
        return weights
    rank = dist.get_rank()
    manifest = [None]
    if rank == src:
        if weights is None:
            raise ValueError("broadcast_weights: the source rank must provide the weights")
        manifest[0] = [(k, tuple(np.asarray(weights[k]).shape)) for k in sorted(weights)]
    dist.broadcast_object_list(manifest, src=src)
    manifest = manifest[0]
    total = int(sum(int(np.prod(s)) for _, s in manifest))
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) \
            if dist.get_backend() == "nccl" else torch.device("cpu")
    flat = torch.empty(total, dtype=torch.float32, device=device)
    if rank == src:
        host = np.concatenate([np.asarray(weights[k], np.float32).reshape(-1) for k, _ in manifest])
        flat.copy_(torch.from_numpy(host))
    dist.broadcast(flat, src=src)
    host = flat.cpu().numpy()
    out, off = {}, 0
    for k, shape in manifest:
        n = int(np.prod(shape))
        out[k] = host[off:off + n].reshape(shape).copy()
        off += n
    return out


def max_over_ranks(value: float, device=None) -> float:
    """Device-side timing aggregation: the job takes as long as its slowest rank."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) \
            if dist.get_backend() == "nccl" else torch.device("cpu")
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def world_size() -> int:
    """Ranks of the default process group; 1 when there is none."""
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _staged(t: torch.Tensor) -> torch.Tensor:
    """The tensor a collective works on: ``t`` itself with NCCL, a host copy with gloo."""
    return t if dist.get_backend() == "nccl" else t.detach().cpu()


def all_reduce_mean_(tensors) -> None:
    """Average ``tensors`` (float32, same shapes on every rank) over the ranks, in place, with ONE
    all-reduce of a single flat float32 buffer: with NCCL on the device, with gloo staged through the
    host.  Every rank is left with the same bits.  Data-parallel training calls it on the gradients
    after ``backward``: each rank's loss is the mean over its equal shard, so their average is the
    gradient of the mean loss over the whole batch."""
    world = world_size()
    if world == 1 or not tensors:
        return
    flat = torch.cat([t.detach().reshape(-1) for t in tensors])
    buf = _staged(flat)
    dist.all_reduce(buf)
    buf.div_(world)
    if buf is not flat:
        flat.copy_(buf)
    off = 0
    with torch.no_grad():
        for t in tensors:
            n = t.numel()
            t.copy_(flat[off:off + n].view_as(t))
            off += n


def sum_over_ranks(values) -> np.ndarray:
    """Sum a short float64 vector over the ranks (one all-reduce); ``values`` itself without a group."""
    v = np.asarray(values, np.float64).reshape(-1)
    if world_size() == 1:
        return v
    device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else "cpu"
    t = torch.from_numpy(v.copy()).to(device)
    dist.all_reduce(t)
    return t.cpu().numpy()


def _all_gather(t: torch.Tensor) -> np.ndarray:
    """[world, *t.shape]: every rank's ``t``, in rank order, as a host array."""
    buf = _staged(t.contiguous())
    parts = [torch.empty_like(buf) for _ in range(world_size())]
    dist.all_gather(parts, buf)
    return torch.stack(parts).cpu().numpy()


def merge_moments(counts, moments) -> np.ndarray:
    """The moments of the union of disjoint pixel sets, in float64: ``counts[r]`` pixels with
    ``moments[r]`` = (the mean of the 3 channels, then their biased covariance c00 c01 c02 c11 c12
    c22), as hdrnet_guide_nn_stats_f32 computes them.  Each set's covariance is taken about the
    union's mean, so a small variance about a large mean keeps its digits."""
    n = np.asarray(counts, np.float64)
    mom = np.asarray(moments, np.float64).reshape(len(n), 9)
    total = n.sum()
    if total == 0:
        return np.zeros(9)
    mean = (n[:, None] * mom[:, :3]).sum(0) / total
    d = mom[:, :3] - mean
    iu = np.triu_indices(3)
    cov = (n[:, None] * (mom[:, 3:] + (d[:, :, None] * d[:, None, :])[:, iu[0], iu[1]])).sum(0) / total
    return np.concatenate([mean, cov])


def moments_over_ranks(moments, npix: int):
    """(moments, pixels) of the whole batch from this rank's ``moments`` over its ``npix`` pixels:
    one all-gather of every rank's (count, moments), merged by ``merge_moments`` in rank order, so
    every rank gets the same bits.  Without a group: ``(moments, npix)`` unchanged."""
    if world_size() == 1:
        return np.asarray(moments, np.float64), int(npix)
    row = torch.from_numpy(np.concatenate([[float(npix)], np.asarray(moments, np.float64).reshape(9)]))
    if dist.get_backend() == "nccl":
        row = row.to(torch.device("cuda", torch.cuda.current_device()))
    rows = _all_gather(row)
    return merge_moments(rows[:, 0], rows[:, 1:]), int(rows[:, 0].sum())


def _all_gather_tensor(t: torch.Tensor) -> torch.Tensor:
    """[world, *t.shape]: every rank's ``t``, in rank order, on ``t``'s device (staged through the host
    with gloo)."""
    buf = _staged(t.contiguous())
    parts = [torch.empty_like(buf) for _ in range(world_size())]
    dist.all_gather(parts, buf)
    return torch.stack(parts).to(t.device)


def bn_moments_over_ranks(moments: torch.Tensor) -> torch.Tensor:
    """The batch-norm moments of the whole batch from this rank's ``moments`` [3, C] (float64 count,
    mean and M2 per channel over its rows, as hdrnet_bn_stats_f32 writes them): one all-gather, then
    the ranks merged in rank order (Chan et al.) in float64, so every rank gets the same bits.  Without
    a group: ``moments`` itself, and nothing leaves the device."""
    if world_size() == 1:
        return moments
    parts = _all_gather_tensor(moments)
    n, mean, m2 = parts[0].unbind(0)
    for nb, mb, m2b in parts[1:]:
        nt = n + nb
        d = mb - mean
        mean = mean + d * (nb / nt)
        m2 = m2 + m2b + d * d * (n * nb / nt)
        n = nt
    return torch.stack([n, mean, m2])


def bn_sums_over_ranks(sums: torch.Tensor) -> torch.Tensor:
    """The batch-norm VJP sums [2, C] (float64 A and B per channel, hdrnet_bn_relu_grad_sums_f32) of
    the whole batch: one all-gather, added in rank order, so every rank gets the same bits.  Without a
    group: ``sums`` itself."""
    if world_size() == 1:
        return sums
    parts = _all_gather_tensor(sums)
    total = parts[0]
    for p in parts[1:]:
        total = total + p
    return total


def check_ranks_agree(arrays, what: str = "the training state") -> None:
    """RuntimeError unless every rank holds the same bytes in ``arrays`` (host arrays, same order on
    every rank): one all-gather of a 64-bit digest of them.  Nothing to do without a group."""
    if world_size() == 1:
        return
    h = hashlib.blake2b(digest_size=8)
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    mine = np.frombuffer(h.digest(), np.int64).copy()
    t = torch.from_numpy(mine)
    if dist.get_backend() == "nccl":
        t = t.to(torch.device("cuda", torch.cuda.current_device()))
    digests = _all_gather(t).reshape(-1)
    if not (digests == digests[0]).all():
        bad = [r for r in range(len(digests)) if digests[r] != digests[0]]
        raise RuntimeError(f"{what} differs between ranks: ranks {bad} disagree with rank 0 (digests "
                           f"{[hex(int(d) & (2 ** 64 - 1)) for d in digests]})")


def finalize():
    if dist.is_initialized():
        dist.destroy_process_group()
