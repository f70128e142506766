"""Time the training CLI's data path and step on the device (hdrnet_b200/bin/train.py).

In one run, with the card's name and power limit read in the same run:
  * CUDA-event time of the batch-assembly kernel (hdrnet_train_batch_f32) at the reference's training
    size -- 16 crops of 512² with flips, rotations and random crops, plus the 256² network input --
    from a cache of uint8 sources and from one of uint16 sources (u8 / u16 / u8 / u16), with the
    bytes the kernel must move and the bandwidth that implies;
  * the CLI's steady-state step (train.Trainer.train_step: batch kernel, forward, L2 loss, PSNR,
    backward, Adam.step) on a synthetic dataset, alternated with tools/time_train_step.py's whole
    step plus Adam.step on fixed tensors (A / B / A / B).
Prints one JSON object; --out also writes it.

    python tools/time_train_pipeline.py [--steps 20 --warmup 5 --reps 5 --out tools_out/train_pipeline.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hdrnet_b200 import data_pipeline as dp, metrics, models  # noqa: E402
from hdrnet_b200.bin import train  # noqa: E402
from time_train_step import gpu_identity, timed  # noqa: E402

B, OH, S = 16, 512, 256
SRC_H, SRC_W, N_SRC = 600, 700, 32


def kernel_record(dtype, steps, warmup, reps):
    rng = np.random.RandomState(0)
    hi = np.iinfo(dtype).max + 1
    srcs = [torch.from_numpy(rng.randint(0, hi, size=(SRC_H, SRC_W, 3)).astype(dtype)).cuda() for _ in range(2 * B)]
    sampler = dp.Sampler([(SRC_H, SRC_W)] * B, B, (OH, OH), shuffle=True, fliplr=True, flipud=True, rotate=True,
                         random_crop=True, seed=0)
    draws = sampler.draws(0)
    out = (torch.empty(B, OH, OH, 3, device="cuda"), torch.empty(B, OH, OH, 3, device="cuda"),
           torch.empty(B, S, S, 3, device="cuda"))

    def call():
        dp.train_batch([srcs[d.index] for d in draws], [srcs[B + d.index] for d in draws], draws, (OH, OH), S, out=out)

    t = timed(call, steps, warmup, reps)
    item = np.dtype(dtype).itemsize
    nbytes = B * (2 * OH * OH * 3 * item + 2 * OH * OH * 3 * 4 + S * S * 3 * (item + 4))
    t.update(bytes=nbytes, tb_per_s=nbytes / (t["ms"] * 1e-3) / 1e12)
    return t


def synthetic_dataset(root, n=N_SRC):
    import cv2
    os.makedirs(os.path.join(root, "input"))
    os.makedirs(os.path.join(root, "output"))
    rng = np.random.RandomState(1)
    names = []
    for i in range(n):
        name = f"{i:03d}.png"
        cv2.imwrite(os.path.join(root, "input", name), rng.randint(0, 256, size=(SRC_H, SRC_W, 3)).astype(np.uint8))
        cv2.imwrite(os.path.join(root, "output", name), rng.randint(0, 65536, size=(SRC_H, SRC_W, 3)).astype(np.uint16))
        names.append(name)
    with open(os.path.join(root, "filelist.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_pipeline.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "batch": B, "crop": OH, "lowres": S, "source": [SRC_H, SRC_W],
           "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    for tag in ("a", "b"):          # alternated: the first window also pays for the clock ramp
        res[f"batch_kernel_u8_{tag}"] = kernel_record(np.uint8, a.steps, a.warmup, a.reps)
        res[f"batch_kernel_u16_{tag}"] = kernel_record(np.uint16, a.steps, a.warmup, a.reps)

    with tempfile.TemporaryDirectory() as tmp:
        synthetic_dataset(os.path.join(tmp, "data"))
        parser = train.build_parser()
        args = parser.parse_args([os.path.join(tmp, "ckpt"), os.path.join(tmp, "data"), "--fliplr", "--flipud", "--rotate"])
        cli = train.Trainer(args, train.model_params(parser, args))

        # tools/time_train_step.py's step on fixed tensors, plus Adam.step
        params = dict(models.DEFAULT_PARAMS)
        rng = np.random.RandomState(0)
        wts = {k: torch.from_numpy(v).cuda().requires_grad_(k.startswith(train.COEFFS))
               for k, v in models.init_weights(params, seed=0).items()}
        p = dict(params, weights=wts)
        low = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
        full = torch.from_numpy(rng.rand(B, OH, OH, 3).astype(np.float32)).cuda()
        target = torch.from_numpy(rng.rand(B, OH, OH, 3).astype(np.float32)).cuda()
        opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-4)

        def fixed_step():
            opt.zero_grad(set_to_none=True)
            metrics.l2_loss(target, models.HDRNetCurves.inference(low, full, p)).backward()
            opt.step()

        for tag in ("a", "b"):
            res[f"cli_step_{tag}"] = timed(cli.train_step, a.steps, a.warmup, a.reps)
            res[f"fixed_step_adam_{tag}"] = timed(fixed_step, a.steps, a.warmup, a.reps)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
