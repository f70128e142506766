"""Any-shape row kernel (shapes outside the TMA contract) at 4K x 8: ms and fraction of the HBM roofline."""
import os, sys, json, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import hdrnet_ops
PEAK = json.load(open("MEASURED_PEAKS.json")).get("hbm_gbs", 3350.0) if os.path.exists("MEASURED_PEAKS.json") else 3350.0

def t(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters

B, H = 8, 2160
for label, W, n_in, n_out, off in (("no offset 3->3, W=3840", 3840, 3, 3, False), ("offset 3->3, W=3838", 3838, 3, 3, True),
                                   ("offset 4->9 (pyramid grid), W=3840", 3840, 3, 9, True), ("slice gc=12, W=3838", 3838, 0, 12, None)):
    g = torch.Generator(device="cuda").manual_seed(0)
    guide = torch.rand(B, H, W, device="cuda", generator=g)
    if off is None:
        grid = torch.randn(B, 16, 16, 8, 12, device="cuda", generator=g)
        fn = lambda: hdrnet_ops.bilateral_slice(grid, guide)
        bpp = 4 + 48
    else:
        gc = n_out * (n_in + int(off))
        grid = torch.randn(B, 16, 16, 8, gc, device="cuda", generator=g)
        im = torch.rand(B, H, W, n_in, device="cuda", generator=g)
        fn = lambda: hdrnet_ops.bilateral_slice_apply(grid, guide, im, has_offset=off)
        bpp = 4 + 4 * n_in + 4 * n_out
    ms = t(fn)
    gbs = B * H * W * bpp / ms / 1e6
    print(f"{label}: {ms:.3f} ms  {gbs:.0f} GB/s  {gbs / PEAK:.3f} of {PEAK:.0f}", flush=True)
