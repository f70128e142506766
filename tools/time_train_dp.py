"""Time data-parallel training steps (hdrnet_b200/bin/train.py under a process group).

For each world size from 1 to the number of visible GPUs, one process per GPU (NCCL), and at two
shapes -- 16 x 512² as the global batch (16 / world images per rank), and one 2048² crop per rank
(global batch = world size, the ``ll`` recipes' crop) -- the steady-state steps per second of the
CLI's step as Trainer.run takes it (train_step, then the loss and PSNR read on the host and, with
several ranks, the per-step scalar all-reduce), on HDRNetCurves with the device tier.  Each rank's
gradient all-reduce (parallel.all_reduce_mean_) is timed with CUDA events around it, every step.
With --shared-gloo, world 2 is also run with both ranks on card 0 over gloo (the all-reduce staged
through the host), the set-up of the equivalence tests: its step rate says nothing about scaling.
The card's name and power limit are read in the same run.  Prints one JSON object; --out also
writes it.

    python tools/time_train_dp.py [--steps 30 --warmup 5 --out tools_out/train_dp.json] [--shared-gloo]
"""
from __future__ import annotations

import argparse
import json
import os
import socket
import sys
import tempfile
import time

import numpy as np
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hdrnet_b200 import parallel  # noqa: E402
from hdrnet_b200.bin import train  # noqa: E402
from time_train_pipeline import synthetic_pairs  # noqa: E402
from time_train_step import gpu_identity  # noqa: E402

# name -> (global batch at world w, crop, source extent, pairs)
SHAPES = {"16x512": (lambda w: 16, 512, (600, 700), 32),
          "2048_per_rank": (lambda w: w, 2048, (2136, 2236), 4)}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank(rank, world, port, backend, data, batch, crop, steps, warmup, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    if world > 1:
        parallel.init_distributed(backend)
    try:
        events = []
        reduce = parallel.all_reduce_mean_

        def timed_reduce(tensors):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            reduce(tensors)
            b.record()
            events.append((a, b))

        parallel.all_reduce_mean_ = timed_reduce
        with tempfile.TemporaryDirectory() as ckpt:
            parser = train.build_parser()
            args = parser.parse_args([ckpt, data, "--fliplr", "--flipud", "--rotate", "--batch_size", str(batch),
                                      "--output_resolution", str(crop), str(crop)])
            t = train.Trainer(args, train.model_params(parser, args))
            grad_bytes = 4 * sum(t.weights[k].numel() for k in t.names)

            def step():
                loss, psnr = t.train_step()
                vals = [float(loss), float(psnr), 0.0, 0.0]
                if world > 1:
                    parallel.sum_over_ranks(vals)

            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            events.clear()
            t0 = time.perf_counter()
            for _ in range(steps):
                step()
            torch.cuda.synchronize()
            elapsed = parallel.max_over_ranks(time.perf_counter() - t0)
            t.close()
        ms = [a.elapsed_time(b) for a, b in events]
        q.put((rank, {"steps_per_s": steps / elapsed, "step_ms": 1e3 * elapsed / steps,
                      "images_per_rank": batch // world, "grad_bytes": grad_bytes,
                      "allreduce_ms_median": float(np.median(ms)) if ms else None,
                      "allreduce_ms_max": float(max(ms)) if ms else None}))
    except BaseException as e:
        q.put((rank, repr(e)))
        raise
    finally:
        parallel.finalize()


def run_world(world, backend, data, batch, crop, steps, warmup):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, world, port, backend, data, batch, crop, steps, warmup, q))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=1800) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shared-gloo", action="store_true", help="also run world 2 on card 0 over gloo")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_dp.py needs a CUDA device")
    ngpu = torch.cuda.device_count()
    res = {"gpu": gpu_identity(), "visible_gpus": ngpu, "model": "HDRNetCurves", "steps": a.steps,
           "warmup": a.warmup}
    runs = [(w, "nccl") for w in range(1, ngpu + 1)] + ([(2, "gloo")] if a.shared_gloo else [])
    for name, (batch_of, crop, (sh, sw), pairs) in SHAPES.items():
        with tempfile.TemporaryDirectory() as tmp:
            data = os.path.join(tmp, "data")
            synthetic_pairs(data, pairs, sh, sw)
            for world, backend in runs:
                key = f"{name}_world{world}_{backend}" + ("_shared_card" if backend == "gloo" else "")
                res[key] = run_world(world, backend, data, batch_of(world), crop, a.steps, a.warmup)
                print(key, json.dumps(res[key]), flush=True)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
