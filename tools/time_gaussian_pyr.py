"""Time HDRNetGaussianPyr (the curves-guide pyramid) against HDRNetGaussianPyrNN, alternated in one run.

CUDA-event times (median over --reps windows of --steps calls each, after --warmup calls, with the
min-max spread), the two models' windows interleaved so that both see the same state of a shared card:
  * ``inference_image`` at 8 x 3840 x 2160 (4K), uint8 in and out, with the synthetic weights of
    ``models.init_weights`` (net input 256, default hyperparameters);
  * the training step of the recipes (the CLI's Trainer.train_step work on one fixed batch: forward,
    L2 loss, backward, Adam) at 1 x 2048² with the guides trained: HDRNetGaussianPyr as
    ``--train_guide`` runs it, HDRNetGaussianPyrNN as ``--train_guide --guide_batch_stats`` does.
Reads the card's name and power limit in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_gaussian_pyr.py [--steps 10 --warmup 3 --reps 5 --out tools_out/gaussian_pyr.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import models  # noqa: E402
from time_train_step import gpu_identity  # noqa: E402

MODELS = ("HDRNetGaussianPyr", "HDRNetGaussianPyrNN")


def make_inference(model_name, B=8, H=2160, W=3840, seed=0):
    params = dict(models.DEFAULT_PARAMS, model_name=model_name)
    p = dict(params, weights=models.init_weights(params, seed=seed, model_name=model_name))
    g = torch.Generator(device="cuda").manual_seed(seed)
    img = torch.randint(0, 256, (B, H, W, 3), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    mdl = getattr(models, model_name)

    def call():
        with torch.no_grad():
            mdl.inference_image(img, p, out_dtype=torch.uint8)
    return call


def make_step(model_name, B=1, S=2048, seed=0):
    params = dict(models.DEFAULT_PARAMS, model_name=model_name)
    init = models.init_weights(params, seed=seed, model_name=model_name)
    wts = {k: torch.from_numpy(v).cuda().requires_grad_("/moving_" not in k) for k, v in init.items()}
    p = dict(params, weights=wts, guide_grad=True)
    training = model_name == "HDRNetGaussianPyrNN"     # its guides' batch norm in training mode
    opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-4)
    rng = np.random.RandomState(seed)
    low = torch.from_numpy(rng.rand(B, 256, 256, 3).astype(np.float32)).cuda()
    full = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
    target = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
    mdl = getattr(models, model_name)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = ((mdl.inference(low, full, p, is_training=training) - target) ** 2).mean()
        loss.backward()
        opt.step()
    return step


def alternated(fns: dict, steps, warmup, reps):
    """{name: median / min / max ms per call}, the names' windows interleaved rep by rep."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    per = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                fn()
            b.record()
            b.synchronize()
            per[k].append(a.elapsed_time(b) / steps)
    return {k: {"ms": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_gaussian_pyr.py needs a CUDA device")
    rec = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    rec["inference_image_8x4k_u8"] = alternated({m: make_inference(m) for m in MODELS}, a.steps, a.warmup, a.reps)
    torch.cuda.empty_cache()
    rec["train_step_1x2048_train_guide"] = alternated({m: make_step(m) for m in MODELS}, a.steps, a.warmup, a.reps)
    print(json.dumps(rec, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
