"""Time a ragged batch (images of different sizes in one call) against a loop of single-image calls.

For each image set, model (curves, pointwise NN) and pixel format (uint8 -> uint8, uint16 -> uint16)
the outputs of every path are first compared with the ragged call's (reported per path: the loops
run the coefficient network at batch 1, the ragged call at batch B), then CUDA-event times are taken round by round,
the paths alternated within each round:
  ragged      models.<Model>.inference_images(images)        (one call)
  loop-py     [inference_image(im[None]) for im in images]   (one call per image)
  loop-c      [FrozenModel(im[None]) for im in images]       (one call per image, C-ABI)
  frozen-rag  FrozenModel(images)                            (one call, C-ABI)
  stacked     inference_image(stack(images))                 (same-size sets only)
Prints one JSON line per case with the median ms of each path, and the card's name and power limit.

    python tools/time_ragged.py [--rounds 15] [--out tools_out/time_ragged.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from hdrnet_b200 import checkpoint, models  # noqa: E402
from hdrnet_b200.frozen import FrozenModel  # noqa: E402


def image_sets(rng):
    mixed = []
    for i in range(16):   # 1-4 MP, odd widths included
        mp = rng.uniform(1.0, 4.0) * 1e6
        w = int(np.sqrt(mp * 4 / 3)) | (1 if i % 3 == 0 else 0)
        h = int(mp / w)
        mixed.append((h, w) if i % 2 else (w, h))
    return {
        "16x12MP-mixed-orientation": [(3024, 4032) if i % 2 else (4032, 3024) for i in range(16)],
        "16x1-4MP-mixed": mixed,
        "8x4K-same": [(2160, 3840)] * 8,
    }


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:   # report, do not fail the measurement
        return f"unknown ({e})"


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = np.random.RandomState(0)
    gpu = card()
    tmp = tempfile.mkdtemp()
    lines = []
    for name in ("HDRNetCurves", "HDRNetPointwiseNNGuide"):
        params = dict(models.DEFAULT_PARAMS, model_name=name)
        params["weights"] = models.init_weights(params, seed=1, model_name=name)
        cls = getattr(models, name)
        path = os.path.join(tmp, name + ".hdrnet")
        checkpoint.freeze_model(params["weights"], params, path)
        frozen = FrozenModel(path)
        for set_name, shapes in image_sets(rng).items():
            for dt in (torch.uint8, torch.uint16):
                top = 256 if dt == torch.uint8 else 65536
                ims = [torch.randint(0, top, (h, w, 3), device="cuda", dtype=torch.int32).to(dt) for h, w in shapes]
                same = len(set(shapes)) == 1
                paths = {
                    "ragged": lambda: cls.inference_images(ims, params, out_dtype=dt),
                    "loop-py": lambda: [cls.inference_image(im[None], params, out_dtype=dt)[0] for im in ims],
                    "loop-c": lambda: [frozen(im[None], out_dtype=dt)[0] for im in ims],
                    "frozen-rag": lambda: frozen(ims, out_dtype=dt),
                }
                if same:
                    stacked = torch.stack(ims)
                    paths["stacked"] = lambda: list(cls.inference_image(stacked, params, out_dtype=dt).unbind(0))
                equal = {}
                with torch.no_grad():
                    ref = paths["ragged"]()
                    for k, f in paths.items():   # outputs compared first (also the warm-up)
                        got = f()
                        equal[k] = all(torch.equal(a, b) for a, b in zip(ref, got))
                    torch.cuda.synchronize()
                    times = {k: [] for k in paths}
                    for _ in range(args.rounds):
                        for k, f in paths.items():
                            times[k].append(event_ms(f))
                rec = {"model": name, "set": set_name, "dtype": str(dt).replace("torch.", ""), "gpu": gpu,
                       "equal_to_ragged": equal, "median_ms": {k: round(float(np.median(v)), 3) for k, v in times.items()},
                       "min_ms": {k: round(float(np.min(v)), 3) for k, v in times.items()}}
                best_loop = min(rec["median_ms"]["loop-py"], rec["median_ms"]["loop-c"])
                rec["ragged_over_best_loop"] = round(min(rec["median_ms"]["ragged"], rec["median_ms"]["frozen-rag"])
                                                     / best_loop, 3)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
                del ims
        frozen.close()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
