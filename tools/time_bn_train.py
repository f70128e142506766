"""Time the training CLI's step of HDRNetCurves with and without the coefficient network's batch norm in
training mode (--batch_norm --coefficient_batch_stats) at the reference's training size (batch 16,
256² network input, 512² output): what train.Trainer.train_step runs on a device-resident batch --
inference(..., is_training), L2 loss, backward, Adam.

CUDA-event times (median over --reps windows of --steps steps, after --warmup steps, with the min-max
spread), the two configurations alternated window by window; the training-mode batch-norm kernels
alone (statistics, batch norm + relu, VJP sums, VJP) at every batch-norm layer shape; and the number of
kernel launches per step of each configuration from one torch.profiler record.  Reads the card's name
and power limit in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_bn_train.py [--steps 20 --warmup 5 --reps 7 --out tools_out/bn_train.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import _lib, metrics, models  # noqa: E402

B, S, HW = 16, 256, 512


def gpu_identity():
    rec = {"name": torch.cuda.get_device_name(0)}
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    if q.returncode == 0 and q.stdout.strip():
        rec["power_limit"], rec["sm_max_clock"] = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return rec


def make_step(batch_norm: bool, seed=0):
    params = dict(models.DEFAULT_PARAMS, batch_norm=batch_norm)
    w = {k: torch.from_numpy(v).cuda() for k, v in models.init_weights(params, seed=seed).items()}
    names = sorted(k for k in w if k.startswith("inference/coefficients/") and "/moving_" not in k)
    for k in names:
        w[k].requires_grad_(True)
    opt = torch.optim.Adam([w[k] for k in names], lr=1e-4)
    p = dict(params, weights=w)
    if batch_norm:
        p["coefficient_batch_stats"] = True
    g = torch.Generator(device="cuda").manual_seed(seed)
    low = torch.rand(B, S, S, 3, device="cuda", generator=g)
    full = torch.rand(B, HW, HW, 3, device="cuda", generator=g)
    target = torch.rand(B, HW, HW, 3, device="cuda", generator=g)

    def step():
        opt.zero_grad(set_to_none=True)
        pred = models.HDRNetCurves.inference(low, full, p, is_training=batch_norm)
        loss = metrics.l2_loss(target, pred)
        loss.backward()
        opt.step()
    return step


def window(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def summary(per):
    return {"ms": float(np.median(per)), "min": float(min(per)), "max": float(max(per))}


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def kernel_times(steps, warmup, reps):
    """The four batch-norm calls at each batch-norm layer shape of the default network at batch 16."""
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    shapes = [("splat/conv2", B * 64 * 64, 16), ("splat/conv3", B * 32 * 32, 32), ("splat/conv4", B * 16 * 16, 64),
              ("global/conv1", B * 8 * 8, 64), ("global/conv2", B * 4 * 4, 64), ("global/fc1", B, 256),
              ("global/fc2", B, 128), ("local/conv1", B * 16 * 16, 64)]
    out = {}
    for name, N, C in shapes:
        z, dy, y, dz = (torch.randn(N, C, device="cuda") for _ in range(4))
        beta, mm, mv, dbeta = (torch.zeros(C, device="cuda") for _ in range(4))
        mom = torch.empty(3, C, dtype=torch.float64, device="cuda")
        sums = torch.empty(2, C, dtype=torch.float64, device="cuda")
        nb = lib.hdrnet_bn_stats_workspace_bytes(N, C)
        ws = torch.empty(nb // 8 + 1, dtype=torch.float64, device="cuda")

        def call():
            lib.hdrnet_bn_stats_f32(z.data_ptr(), N, C, mom.data_ptr(), ws.data_ptr(), nb, st)
            lib.hdrnet_bn_relu_f32(z.data_ptr(), N, C, mom.data_ptr(), beta.data_ptr(), y.data_ptr(), mm.data_ptr(),
                                   mv.data_ptr(), st)
            lib.hdrnet_bn_relu_grad_sums_f32(z.data_ptr(), dy.data_ptr(), N, C, mom.data_ptr(), beta.data_ptr(),
                                             sums.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), nb, st)
            lib.hdrnet_bn_relu_grad_f32(z.data_ptr(), dy.data_ptr(), N, C, mom.data_ptr(), beta.data_ptr(),
                                        sums.data_ptr(), dz.data_ptr(), st)
        for _ in range(warmup):
            call()
        out[name] = {"N": N, "C": C, "us_all_four": 1e3 * summary([window(call, steps) for _ in range(reps)])["ms"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_bn_train.py needs a CUDA device")
    steps = {"plain": make_step(False), "batch_norm": make_step(True)}
    for fn in steps.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    per = {k: [] for k in steps}
    for _ in range(a.reps):
        for k, fn in steps.items():
            per[k].append(window(fn, a.steps))
    rec = {"gpu": gpu_identity(), "shape": f"{B} x {S}^2 / {HW}^2",
           "step": {k: summary(v) for k, v in per.items()},
           "launches_per_step": {k: launches(fn) for k, fn in steps.items()},
           "bn_kernels": kernel_times(a.steps, a.warmup, a.reps)}
    rec["bn_step_cost_ms"] = rec["step"]["batch_norm"]["ms"] - rec["step"]["plain"]["ms"]
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
