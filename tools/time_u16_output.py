"""Time the fused full-resolution call (guide + slice + apply in one kernel, ``_fullres``) with a
uint16 result against the 8-bit result it replaces.

For HDR+ 12 MP x 8 (3024 x 4032) and 4K x 8 (2160 x 3840), with the curves guide and the pointwise-NN
guide, three pixel formats of the same call on the same coefficients:
  * uint16 -> uint16 (6 + 6 = 12 bytes per pixel);
  * uint16 -> uint8  (6 + 3 =  9 bytes per pixel: bench.py's HDR+ record);
  * uint8  -> uint8  (3 + 3 =  6 bytes per pixel).
CUDA-event times: the formats alternate round by round (--rounds rounds of --steps calls each, after
--warmup calls of each); the median and the min-max spread per format, the bytes per second the
pixel stream needs (the formats' bytes per pixel; the grid and the slab rows are not counted) and
their share of the H100 SXM's 3.35 TB/s.  Reads the card's name, power limit and maximum SM clock in
the same run.  Prints one JSON object; --out also writes it.

    python tools/time_u16_output.py [--steps 10 --warmup 3 --rounds 5 --out tools_out/u16_output.json]
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
from time_train_step import gpu_identity, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM5 peak HBM3 bandwidth
SHAPES = {"hdrp_12mp_x8": (8, 3024, 4032), "4k_x8": (8, 2160, 3840)}
GUIDES = ("HDRNetCurves", "HDRNetPointwiseNNGuide")
# name -> (input dtype, output dtype, bytes per pixel)
FORMATS = {"u16->u16": (torch.uint16, torch.uint16, 12), "u16->u8": (torch.uint16, torch.uint8, 9),
           "u8->u8": (torch.uint8, torch.uint8, 6)}


def case(model_name, B, H, W, a):
    p = dict(models.DEFAULT_PARAMS, model_name=model_name)
    p["weights"] = models.init_weights(p, seed=0, model_name=model_name)
    cls = getattr(models, model_name)
    gen = torch.Generator(device="cuda").manual_seed(5)
    codes = torch.randint(0, 65536, (B, H, W, 3), device="cuda", generator=gen, dtype=torch.int32)
    im16, im8 = codes.to(torch.uint16), (codes >> 8).to(torch.uint8)      # uint16 has no CUDA shift
    del codes
    coeffs = cls._coefficients(models.lowres_from_image(im16, p["net_input_size"]), p)
    images = {torch.uint16: im16, torch.uint8: im8}
    calls = {name: (lambda x=images[i], o=o: cls._fullres(coeffs, x, p, o)) for name, (i, o, _) in FORMATS.items()}
    for fn in calls.values():
        timed(fn, 1, a.warmup, 1)
    per = {name: [] for name in FORMATS}
    for _ in range(a.rounds):                                  # interleaved: A B C A B C ...
        for name, fn in calls.items():
            per[name].append(timed(fn, a.steps, 0, 1)["ms"])
    out = {}
    for name, (_, _, bpp) in FORMATS.items():
        ms = float(np.median(per[name]))
        bps = B * H * W * bpp / (ms * 1e-3)
        out[name] = {"ms": ms, "min": min(per[name]), "max": max(per[name]), "bytes_per_px": bpp,
                     "gb_s": bps / 1e9, "hbm_share": bps / HBM_BYTES_PER_S}
    out["u16->u16 over u16->u8"] = out["u16->u16"]["ms"] / out["u16->u8"]["ms"]
    del im16, im8, images
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_u16_output.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds}
    with torch.no_grad():
        for key, (B, H, W) in SHAPES.items():
            res[key] = {name: case(name, B, H, W, a) for name in GUIDES}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
