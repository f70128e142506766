"""Time the curves-guide VJP (hdrnet_guide_curves_grad_f32) and what training the guide adds to a
fine-tuning step of HDRNetCurves.

CUDA-event times (median over --reps repetitions of --steps calls each, after --warmup calls, with
the min-max spread) of
  * the VJP alone, with and without dinput, at the training size (16 x 512²) and at 8 x 4K
    (3840 x 2160), with the bytes each call moves per pixel and the share of the H100 SXM's
    3.35 TB/s they amount to;
  * the fine-tuning step at the training size (batch 16, 256² network input, 512² output: forward,
    L2 loss, backward, no optimizer) with the guide held fixed and with it trained.
Reads the card's name and power limit in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_guide_grad.py [--steps 20 --warmup 5 --reps 5 --out tools_out/guide_grad.json]
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


def vjp_case(wts, B, H, W, steps, warmup, reps):
    lib = _lib.load()
    npix = B * H * W
    x = torch.rand(B, H, W, 3, device="cuda")
    dg = torch.randn(B, H, W, device="cuda")
    dx = torch.empty_like(x)
    dp = torch.empty(112, device="cuda")
    nbytes = lib.hdrnet_guide_curves_grad_workspace_bytes(npix)
    ws = torch.empty(nbytes // 4, device="cuda")
    host = [np.ascontiguousarray(np.asarray(wts[G + n], np.float32).reshape(-1)) for n in models._CURVES_VARS]
    ptrs = [models._hp(a) for a in host[:5]]
    stream = torch.cuda.current_stream().cuda_stream
    out = {"shape": [B, H, W], "workspace_bytes": int(nbytes)}
    for name, dxp, px_bytes in (("with_dinput", dx.data_ptr(), 28), ("params_only", None, 16)):
        def call(dxp=dxp):
            _lib.check(lib.hdrnet_guide_curves_grad_f32(x.data_ptr(), dg.data_ptr(), dxp, npix, *ptrs,
                                                        float(host[5][0]), dp.data_ptr(), ws.data_ptr(), nbytes,
                                                        stream), "guide VJP")
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
        sys.exit("time_guide_grad.py needs a CUDA device")
    params = dict(models.DEFAULT_PARAMS)
    init = models.init_weights(params, seed=0)
    rng = np.random.RandomState(0)
    res = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    res["vjp_train"] = vjp_case(init, 16, 512, 512, a.steps, a.warmup, a.reps)
    res["vjp_4k_x8"] = vjp_case(init, 8, 2160, 3840, a.steps, a.warmup, a.reps)

    low = torch.from_numpy(rng.rand(16, 256, 256, 3).astype(np.float32)).cuda()
    full = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()
    target = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()
    steps = {}
    for train_guide in (False, True, False):               # alternated A/B/A
        wts = {k: torch.from_numpy(v).cuda().requires_grad_(k.startswith("inference/coefficients/")
                                                             or (train_guide and k.startswith(G)))
               for k, v in init.items()}
        p = dict(params, weights=wts, guide_grad=train_guide)
        train_vars = [v for v in wts.values() if v.requires_grad]

        def step():
            loss = ((models.HDRNetCurves.inference(low, full, p) - target) ** 2).sum()
            torch.autograd.grad(loss, train_vars)

        key = "step_guide_trained" if train_guide else "step_guide_fixed"
        steps[key if key not in steps else key + "_again"] = timed(step, a.steps, a.warmup, a.reps)
    res.update(steps)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
