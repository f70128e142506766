"""Coefficient network: one-call launch chain vs the per-layer kernels, by batch size."""
import os, sys, statistics, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import models
p = dict(models.DEFAULT_PARAMS)
p["weights"] = models.init_weights(p, seed=0)


def t(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3


for B in (1, 2, 4, 8, 16, 32, 64):
    low = torch.rand(B, 256, 256, 3, device="cuda")
    res = {}
    for label, mb in (("chain", 64), ("per-layer", 0)):
        models.CHAIN_CNN_MAX_BATCH = mb
        f = lambda: models.HDRNetCurves._coefficients(low, p)
        res[label] = statistics.median(t(f) for _ in range(3))
        g = torch.cuda.CUDAGraph()      # launch overhead out: the kernels' own time
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            f(); torch.cuda.synchronize()
            with torch.cuda.graph(g):
                f()
        res[label + " (graph)"] = statistics.median(t(g.replay) for _ in range(3))
    print(f"batch {B}: " + "  ".join(f"{k}: {v:.1f} us" for k, v in res.items()), flush=True)
