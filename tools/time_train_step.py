"""Time one fine-tuning step of HDRNetCurves at the reference's training size (hdrnet/bin/train.py:
224-236: batch 16, 256² network input, 512² output): forward, L2 loss, backward, no optimizer.

CUDA-event times (median over --reps repetitions of --steps steps each, after --warmup steps, with
the min-max spread) of
  * the whole step and its forward;
  * the slice-apply VJP (hdrnet_slice_apply_grad_f32) on its own;
  * every coefficient layer's VJP on its own (the autograd Functions of models.py, fed the layer's
    real activations);
  * the coefficient network forward + backward, and the same graph in torch.nn.functional autograd
    (cuDNN, float32, TF32 off) as a yardstick.
Reads the card's name and power limit in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_train_step.py [--steps 20 --warmup 5 --reps 5 --out tools_out/train_step.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import hdrnet_ops, models  # noqa: E402

P = "inference/coefficients"


def gpu_identity():
    rec = {"name": torch.cuda.get_device_name(0)}
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    if q.returncode == 0 and q.stdout.strip():
        rec["power_limit"], rec["sm_max_clock"] = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return rec


def timed(fn, steps, warmup, reps):
    """Median and spread of the per-call time (ms) over `reps` windows of `steps` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) / steps)
    return {"ms": float(np.median(per)), "min": float(min(per)), "max": float(max(per))}


def layer_inputs(low, L, gd):
    """Each layer's (Function, inputs, (weights, bias), extra args) from one real forward; the convs
    get the model's packed weights."""
    out, x = [], low
    n_ds = sum(1 for k in L if "/splat/" in k)

    def conv(s, x, stride, relu):
        w, b, packed = L[s]
        out.append((s, models._ConvFn, x, (w, b), (stride, relu, packed)))
        return models._ConvFn.apply(x, w, b, stride, relu, packed)

    with torch.no_grad():
        for i in range(n_ds):
            x = conv(f"{P}/splat/conv{i + 1}", x, 2, True)
        splat = x
        g = conv(f"{P}/global/conv1", splat, 2, True)
        g = conv(f"{P}/global/conv2", g, 2, True).reshape(low.shape[0], -1)
        for name, relu in (("fc1", True), ("fc2", True), ("fc3", False)):
            s = f"{P}/global/{name}"
            out.append((s, models._FcFn, g, L[s][:2], (relu,)))
            g = models._FcFn.apply(g, *L[s][:2], relu)
        loc = conv(f"{P}/local/conv1", splat, 1, True)
        loc = conv(f"{P}/local/conv2", loc, 1, False)
    s = f"{P}/prediction/conv1"
    out.append((s, "fuse", (loc, g), L[s], (gd, 3, 4)))
    return out


def cudnn_network(x, wts, params):
    """The coefficient graph in torch.nn.functional (NCHW, explicit asymmetric SAME pads)."""
    def conv(t, scope, s, relu=True, bias=True):
        w = wts[scope + "/weights"]
        k = w.shape[0]
        pads = []
        for n in (t.shape[3], t.shape[2]):
            o = -(-n // s)
            tot = max((o - 1) * s + k - n, 0)
            pads += [tot // 2, tot - tot // 2]
        y = F.conv2d(F.pad(t, pads), w.permute(3, 2, 0, 1), wts.get(scope + "/biases") if bias else None, stride=s)
        return F.relu(y) if relu else y

    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    x = x.permute(0, 3, 1, 2)
    for i in range(n_ds):
        x = conv(x, f"{P}/splat/conv{i + 1}", 2)
    splat = x
    g = conv(conv(splat, f"{P}/global/conv1", 2), f"{P}/global/conv2", 2)
    g = g.permute(0, 2, 3, 1).reshape(g.shape[0], -1)
    for name, relu in (("fc1", True), ("fc2", True), ("fc3", False)):
        g = F.linear(g, wts[f"{P}/global/{name}/weights"].t(), wts[f"{P}/global/{name}/biases"])
        g = F.relu(g) if relu else g
    loc = conv(conv(splat, f"{P}/local/conv1", 1), f"{P}/local/conv2", 1, relu=False, bias=False)
    fused = F.relu(loc + g[:, :, None, None])
    return conv(fused, f"{P}/prediction/conv1", 1, relu=False)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_step.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    params = dict(models.DEFAULT_PARAMS)
    gd = params["luma_bins"]
    rng = np.random.RandomState(0)
    wts = {k: torch.from_numpy(v).cuda().requires_grad_(k.startswith(P))
           for k, v in models.init_weights(params, seed=0).items()}
    p = dict(params, weights=wts)
    low = torch.from_numpy(rng.rand(16, 256, 256, 3).astype(np.float32)).cuda()
    full = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()
    target = torch.from_numpy(rng.rand(16, 512, 512, 3).astype(np.float32)).cuda()
    train_vars = [v for v in wts.values() if v.requires_grad]
    res = {"gpu": gpu_identity(), "batch": 16, "lowres": 256, "fullres": 512,
           "steps": a.steps, "warmup": a.warmup, "reps": a.reps}

    def step():
        loss = ((models.HDRNetCurves.inference(low, full, p) - target) ** 2).sum()
        torch.autograd.grad(loss, train_vars)

    def forward():   # the step's forward and loss, recording the tape as the step does
        return ((models.HDRNetCurves.inference(low, full, p) - target) ** 2).sum()

    res["step"] = timed(step, a.steps, a.warmup, a.reps)
    res["forward"] = timed(forward, a.steps, a.warmup, a.reps)

    # slice-apply VJP alone
    grid = models.HDRNetCurves._coefficients(low, p).detach().reshape(16, 16, 16, gd, 12).requires_grad_(True)
    with torch.no_grad():
        guide = models.HDRNetCurves._guide(full, p)
    out = hdrnet_ops.bilateral_slice_apply(grid, guide, full, True)
    ct = torch.randn_like(out)
    res["slice_apply_vjp"] = timed(lambda: torch.autograd.grad(out, grid, ct, retain_graph=True),
                                   a.steps, a.warmup, a.reps)

    # every coefficient layer's VJP alone
    # the model's prepared layers: the variables themselves, and the convs' packed weights
    L = {s: (wb[0][0, 0], wb[1]) if "/prediction/" in s else wb
         for s, wb in models._prepare(wts, params, low.device, False).layers.items()}
    layers = {}
    for scope, fn, x, wb, extra in layer_inputs(low, L, gd):
        if fn == "fuse":
            xs = [t.detach().requires_grad_(True) for t in x]
            y = models._FusePredictFn.apply(*xs, *wb, *extra)
            ins = xs + [t for t in wb if t is not None]
        else:
            xs = x.detach().requires_grad_(not scope.endswith("splat/conv1"))
            y = fn.apply(xs, *wb, *extra)
            ins = ([xs] if xs.requires_grad else []) + [t for t in wb if t is not None]
        dy = torch.randn_like(y)
        layers[scope.replace(P + "/", "")] = timed(lambda y=y, ins=ins, dy=dy: torch.autograd.grad(
            y, ins, dy, retain_graph=True), a.steps, a.warmup, a.reps)
    res["layer_vjps"] = layers
    res["layer_vjps_total_ms"] = sum(v["ms"] for v in layers.values())

    # the coefficient network forward + backward: ours and cuDNN
    dgrid = torch.randn(16, 16, 16, gd, 3, 4, device="cuda")
    lowg = low

    def ours():
        torch.autograd.grad(models.HDRNetCurves._coefficients(lowg, p), train_vars, dgrid)

    cw = {k: v.detach().clone().requires_grad_(True) for k, v in wts.items() if k.startswith(P)}
    dpred = torch.randn(16, gd * 12, 16, 16, device="cuda")

    def cudnn():
        torch.autograd.grad(cudnn_network(lowg, cw, params), list(cw.values()), dpred)

    res["coefficients_fwd_bwd"] = timed(ours, a.steps, a.warmup, a.reps)
    res["cudnn_fwd_bwd"] = timed(cudnn, a.steps, a.warmup, a.reps)
    res["coefficients_fwd_bwd_again"] = timed(ours, a.steps, a.warmup, a.reps)   # alternated A/B/A
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
