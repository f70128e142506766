"""Times the model path's full-resolution stage (guide + slice + apply in one kernel) at 4K x 8:
    python tools/time_fused.py
HDRNET_LIB_OVERRIDE=path.so times another build of the library instead."""
import os, sys, statistics, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import models, _lib
if os.environ.get("HDRNET_LIB_OVERRIDE"):      # another build of the library, for an A/B
    _lib.LIB_PATH = os.path.abspath(os.environ["HDRNET_LIB_OVERRIDE"])
B, H, W = 8, 2160, 3840
gen = torch.Generator(device="cuda").manual_seed(1)
im8 = torch.randint(0, 256, (B, H, W, 3), device="cuda", generator=gen, dtype=torch.uint8)
imf = models.image_to_float(im8)
out = {}
for kind, name in (("curves", "HDRNetCurves"), ("nn", "HDRNetPointwiseNNGuide")):
    p = dict(models.DEFAULT_PARAMS, model_name=name)
    p["weights"] = models.init_weights(p, seed=0, model_name=name)
    cls = getattr(models, name)
    coeffs = cls._coefficients(models.lowres_from_image(im8, 256), p)
    for px, im, dt in (("f32", imf, torch.float32), ("u8", im8, torch.uint8)):
        f = lambda: cls._fullres(coeffs, im, p, dt)
        ts = []
        for r in range(5):
            for _ in range(2): f()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20): f()
            b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) / 20)
        out[f"{kind} {px}"] = statistics.median(ts)
import hashlib
sha = hashlib.sha1(cls._fullres(coeffs, im8, p, torch.uint8).cpu().numpy().tobytes()).hexdigest()[:10]
print("lib=%s  u8-sha=%s  " % (os.environ.get("HDRNET_LIB_OVERRIDE", "product"), sha) + "  ".join(f"{k}: {v:.4f} ms" for k, v in out.items()))
