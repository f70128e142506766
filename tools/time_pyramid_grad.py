"""Time HDRNetGaussianPyrNN's training path: the resize VJP (hdrnet_resize_bilinear_grad_f32) and the
CLI's training step with --train_guide --guide_batch_stats.

CUDA-event times (median over --reps repetitions of --steps calls each, after --warmup calls, with
the min-max spread) of
  * the resize VJP at the pyramid's four shapes for 1 x 2048² (2048² -> 1024² -> 512² in
    _multiscale_input and back up in _output) and for 16 x 512², with the bytes it must move
    (read dout, write din), the achieved bytes/s and their share of the H100 SXM's 3.35 TB/s;
  * Trainer.train_step's work (forward in training mode, L2 loss, backward, Adam) for the pyramid at
    1 x 2048² with channel multiplier 1 and 4, and at 16 x 512², alternated with
    HDRNetPointwiseNNGuide at the same sizes (its guide trained in training mode too);
  * in a separate profiled run, one pyramid step at each size: device time per kernel, grouped
    (coefficients forward and backward, batch statistics, slice-apply forward and VJPs, guide VJPs,
    resize forward and VJPs), and the device-to-host copies and syncs of the three levels' statistics.
Reads the card's name and power limit in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_pyramid_grad.py [--steps 20 --warmup 5 --reps 5 --out tools_out/pyramid_grad.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import _lib, models  # noqa: E402
from time_train_step import gpu_identity, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM5 peak HBM3 bandwidth
SIZES = {"1x2048_cm1": (1, 2048, 1), "1x2048_cm4": (1, 2048, 4), "16x512_cm1": (16, 512, 1)}

# kernel-name substrings -> step phase (first match wins); kernels of torch itself (the loss, Adam,
# slicing copies) fall into the last group
GROUPS = [("resize VJP", ("resize_bilinear_ac_grad",)), ("resize forward", ("resize_bilinear_ac",)),
          ("guide VJP", ("vjp_partial", "vjp_finish", "vjp_dx")), ("batch statistics", ("stats_partial", "stats_reduce")),
          ("slice-apply VJP", ("slice_grad",)), ("guide forward", ("guide_kernel",)),
          ("slice-apply forward", ("slice_apply",)),
          ("coefficients backward", ("conv_dgrad", "wgrad_", "fuse_dglobal", "fuse_dlocal", "fc_grad", "fc_d")),
          ("coefficients forward", ("hdrnet_b200::",)), ("torch (loss, Adam, copies)", ("",))]


def resize_case(B, H, W, OH, OW, steps, warmup, reps):
    """The VJP of a forward resize [B,H,W,3] -> [B,OH,OW,3]: reads dout, writes din."""
    lib = _lib.load()
    dout = torch.randn(B, OH, OW, 3, device="cuda")
    din = torch.empty(B, H, W, 3, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        _lib.check(lib.hdrnet_resize_bilinear_grad_f32(dout.data_ptr(), din.data_ptr(), B, H, W, 3, OH, OW, stream),
                   "resize VJP")
    t = timed(call, steps, warmup, reps)
    nbytes = 4 * (dout.numel() + din.numel())
    t.update(forward=[B, H, W, OH, OW], bytes=nbytes, bytes_per_s=nbytes / (t["ms"] * 1e-3))
    t["hbm_share"] = t["bytes_per_s"] / HBM_BYTES_PER_S
    return t


def make_step(model_name, B, S, cm, seed=0):
    """Trainer.train_step's work on one fixed batch: training-mode forward with every guide trained,
    the L2 loss, backward, Adam."""
    params = dict(models.DEFAULT_PARAMS, model_name=model_name, channel_multiplier=cm)
    init = models.init_weights(params, seed=seed, model_name=model_name)
    wts = {k: torch.from_numpy(v).cuda().requires_grad_("/moving_" not in k) for k, v in init.items()}
    p = dict(params, weights=wts, guide_grad=True)
    opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-4)
    rng = np.random.RandomState(seed)
    low = torch.from_numpy(rng.rand(B, 256, 256, 3).astype(np.float32)).cuda()
    full = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
    target = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
    mdl = getattr(models, model_name)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = ((mdl.inference(low, full, p, is_training=True) - target) ** 2).mean()
        loss.backward()
        opt.step()
    return step


def profile_step(step):
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        step()
        torch.cuda.synchronize()
    groups = {g: {"device_us": 0.0, "kernels": 0} for g, _ in GROUPS}
    kernels = {}
    host = {}
    for e in prof.key_averages():
        dev = getattr(e, "self_device_time_total", 0) or 0
        if e.key in ("cudaMemcpyAsync", "cudaStreamSynchronize", "cudaDeviceSynchronize", "aten::_local_scalar_dense",
                     "aten::_to_copy"):
            host[e.key] = {"count": e.count, "cpu_total_us": e.cpu_time_total}
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA or dev <= 0 or "#" in e.key:
            continue        # record_function ranges (Optimizer.step#...) would count their kernels twice
        kernels[e.key[:90]] = {"count": e.count, "device_us": dev}
        low = e.key
        if "Memcpy" in low or "Memset" in low:
            name = "copies and memsets"
            groups.setdefault(name, {"device_us": 0.0, "kernels": 0})
        else:
            name = next(g for g, subs in GROUPS if any(s in low for s in subs))
        groups[name]["device_us"] += dev
        groups[name]["kernels"] += e.count
    total = sum(g["device_us"] for g in groups.values())
    for g in groups.values():
        g["share"] = g["device_us"] / total if total else 0.0
    top = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["device_us"])[:25])
    return {"device_total_us": total, "groups": groups, "host_syncs_and_copies": host, "top_kernels": top}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_pyramid_grad.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    for B, S in ((1, 2048), (16, 512)):
        res[f"resize_vjp_{B}x{S}"] = [resize_case(B, h, h, oh, oh, a.steps, a.warmup, a.reps)
                                      for h, oh in ((S, S // 2), (S // 2, S // 4), (S // 4, S // 2), (S // 2, S))]
    for key, (B, S, cm) in SIZES.items():
        steps = {"HDRNetGaussianPyrNN": make_step("HDRNetGaussianPyrNN", B, S, cm),
                 "HDRNetPointwiseNNGuide": make_step("HDRNetPointwiseNNGuide", B, S, cm)}
        rec = {}
        for name in ("HDRNetGaussianPyrNN", "HDRNetPointwiseNNGuide") * 2:      # alternated A/B/A/B
            rec.setdefault(name, []).append(timed(steps[name], max(a.steps // 2, 3), a.warmup, a.reps))
        res[f"step_{key}"] = rec
        del steps
        torch.cuda.empty_cache()
    res["profile"] = {}
    for key, (B, S, cm) in SIZES.items():
        res["profile"][key] = profile_step(make_step("HDRNetGaussianPyrNN", B, S, cm))
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
