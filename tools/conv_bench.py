import os, sys, torch, numpy as np
sys.path.insert(0, ".")
from hdrnet_b200 import models
def t(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3
for B in (1, 8, 64):
    for (H, cin, cout, k, s) in [(16, 64, 64, 3, 1), (32, 32, 64, 3, 2), (64, 16, 32, 3, 2), (16, 64, 96, 1, 1)]:
        x = torch.rand(B, H, H, cin, device="cuda"); w = torch.rand(k, k, cin, cout, device="cuda"); b = torch.rand(cout, device="cuda")
        res = []
        for flag in ("0", "1"):
            os.environ["HDRNET_CONV_TCGEN05"] = flag
            res.append(t(lambda: models._conv(x, (w, b), stride=s)))
        packed = models.pack_conv_weights(w)
        res.append(t(lambda: models._conv(x, (w, b, packed), stride=s)))
        flops = 2 * B * (H // s) ** 2 * cout * k * k * cin
        print(f"B={B} {H}x{H}x{cin}->{cout} k{k}s{s}: cuda-core {res[0]:.1f} us, tensor cores {res[1]:.1f} us, tensor cores pipelined+packed {res[2]:.1f} us ({flops/res[2]/1e6:.2f} TFLOP/s eff.)")
p = dict(models.DEFAULT_PARAMS); p["weights"] = models.init_weights(p, 0)
for B in (1, 8):
    low = torch.rand(B, 256, 256, 3, device="cuda")
    for flag in ("0", "1"):
        os.environ["HDRNET_CONV_TCGEN05"] = flag
        print("coefficient CNN B=%d tensor-core convs=%s: %.1f us" % (B, flag, t(lambda: models.HDRNetCurves._coefficients(low, p))))
