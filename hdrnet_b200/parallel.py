"""Multi-GPU plumbing for the batch-sharded path (SURVEY.md section 8e).

The hot path has no per-frame exchange: every output pixel depends only on its own image's
grid / guide / input (hdrnet/ops/bilateral_slice_apply.cu.cc:67-125 -- the batch index only
selects slabs), and the coefficient network is per-image (hdrnet/models.py:63, :95).  So the
design is one process per GPU, images sharded over ranks, and exactly ONE collective: a
broadcast of the flat coefficient-network weight buffer (~1.93 MB) at init over NCCL
(NVLink / NVSwitch); "nccl" on GPUs, "gloo" in the CPU tests.  The reference itself has no
distributed code at all (SURVEY.md section 2b).
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.distributed as dist

__all__ = ["init_distributed", "shard_batch", "shard_rows", "shard_plan", "slice_apply_sharded",
           "broadcast_weights", "max_over_ranks", "finalize", "bind_to_gpu_numa", "gpu_cpu_affinity"]


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


def finalize():
    if dist.is_initialized():
        dist.destroy_process_group()
