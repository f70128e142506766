"""Time the training-mode pointwise-NN guide: its batch statistics (hdrnet_guide_nn_stats_f32), its
VJP (hdrnet_guide_nn_grad_f32), and what training the guide in training mode adds to a step.

CUDA-event times (median over --reps repetitions of --steps calls each, after --warmup calls, with
the min-max spread) of
  * the stats kernel, and the VJP with and without dinput, at the training size (16 x 512²) and at
    one 4K frame (3840 x 2160), with the bytes each call moves per pixel and the share of the H100
    SXM's 3.35 TB/s they amount to;
  * the CLI's training step at the training size (batch 16, 256² network input, 512² output:
    forward, L2 loss, backward, Adam) with the guide fixed in its inference form (the default), and
    with --train_guide --guide_batch_stats, alternated A/B/A/B in one run;
  * a torch.profiler trace of one training-mode step: the host time of the device-to-host copy of
    the moments (the fold's sync) and how long the GPU sits idle around it.
Reads the card's name and power limit in the same run.  Prints one JSON object; --out also writes it
(and the trace, as <out>.trace.json).

    python tools/time_nn_guide_grad.py [--steps 20 --warmup 5 --reps 5 --out tools_out/nn_guide_grad.json]
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
G = "inference/guide/"
NN = "HDRNetPointwiseNNGuide"


def kernel_case(wts, B, H, W, steps, warmup, reps):
    lib = _lib.load()
    npix = B * H * W
    x = torch.rand(B, H, W, 3, device="cuda")
    dg = torch.randn(B, H, W, device="cuda")
    dx = torch.empty_like(x)
    host = [np.ascontiguousarray(np.asarray(wts[G + n], np.float32).reshape(-1)) for n in models._NN_GUIDE_VARS]
    F = host[1].size
    dp = torch.empty(5 * F + 1, device="cuda")
    sbytes = lib.hdrnet_guide_nn_stats_workspace_bytes(npix)
    sws = torch.empty(sbytes // 4, device="cuda")
    mom_d = torch.empty(9, dtype=torch.float64, device="cuda")
    nbytes = lib.hdrnet_guide_nn_grad_workspace_bytes(npix, F)
    ws = torch.empty(nbytes // 4, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    out = {"shape": [B, H, W], "feats": F}

    def stats():
        _lib.check(lib.hdrnet_guide_nn_stats_f32(x.data_ptr(), npix, mom_d.data_ptr(), sws.data_ptr(), sbytes,
                                                 stream), "stats")

    t = timed(stats, steps, warmup, reps)
    t["bytes_per_px"] = 12
    t["hbm_share"] = 12 * npix / (t["ms"] * 1e-3) / HBM_BYTES_PER_S
    out["stats"] = t
    mom = np.ascontiguousarray(mom_d.cpu().numpy())
    ptrs = [models._hp(a) for a in host[:3]]
    for name, dxp, px_bytes in (("vjp_with_dinput", dx.data_ptr(), 16 + 28), ("vjp_params_only", None, 16)):
        def call(dxp=dxp):
            _lib.check(lib.hdrnet_guide_nn_grad_f32(x.data_ptr(), dg.data_ptr(), dxp, npix, *ptrs, float(host[3][0]),
                                                    F, models._hp(mom), dp.data_ptr(), ws.data_ptr(), nbytes, stream),
                       "guide VJP")
        t = timed(call, steps, warmup, reps)
        t["bytes_per_px"] = px_bytes
        t["hbm_share"] = px_bytes * npix / (t["ms"] * 1e-3) / HBM_BYTES_PER_S
        out[name] = t
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_nn_guide_grad.py needs a CUDA device")
    params = dict(models.DEFAULT_PARAMS, model_name=NN)
    init = models.init_weights(params, seed=0, model_name=NN)
    rng = np.random.RandomState(0)
    res = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    for F in (16, 32):
        w = models.init_weights(dict(params, guide_complexity=F), seed=0, model_name=NN)
        res[f"train_16x512_F{F}"] = kernel_case(w, 16, 512, 512, a.steps, a.warmup, a.reps)
        res[f"frame_4k_F{F}"] = kernel_case(w, 1, 2160, 3840, a.steps, a.warmup, a.reps)

    low = torch.from_numpy(rng.rand(16, 256, 256, 3).astype(np.float32)).cuda()
    full = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()
    target = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()

    def make_step(train_guide):
        wts = {k: torch.from_numpy(v).cuda().requires_grad_(
            k.startswith("inference/coefficients/") or (train_guide and k.startswith(G) and "/moving_" not in k))
            for k, v in init.items()}
        p = dict(params, weights=wts, guide_grad=train_guide)
        opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            loss = ((models.HDRNetPointwiseNNGuide.inference(low, full, p, is_training=train_guide) - target) ** 2).mean()
            loss.backward()
            opt.step()
        return step

    steps = {}
    for train_guide in (False, True, False, True):          # alternated A/B/A/B
        key = "step_guide_batch_stats_trained" if train_guide else "step_guide_fixed"
        steps.setdefault(key, []).append(timed(make_step(train_guide), a.steps, a.warmup, a.reps))
    res.update(steps)

    step = make_step(True)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    ev = prof.key_averages()
    copies = [e for e in ev if e.key in ("aten::_to_copy", "aten::copy_", "cudaMemcpyAsync", "cudaStreamSynchronize")]
    res["profile_one_step"] = {
        e.key: {"count": e.count, "cpu_total_us": e.cpu_time_total, "device_total_us": getattr(e, "device_time_total", 0)}
        for e in copies}
    res["profile_one_step"]["self_cpu_total_us"] = sum(e.self_cpu_time_total for e in ev)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
        prof.export_chrome_trace(a.out + ".trace.json")


if __name__ == "__main__":
    main()
