"""Time UnsharpMaskDataPipeline's batch call (hdrnet_train_batch_usm_f32, csrc/usm_batch.cu) against
the paired pipeline's (hdrnet_train_batch_f32) on the same shapes, and the training CLI's step with
each pipeline at the shape of the reference's ``scripts/usm/train_std.sh``.

* The batch call at 1 x 2048^2 (a crop of a 2136 x 2236 source) and 16 x 512^2 (crops of 600 x 700
  sources), sigma in {1, 4, 16, 32}, uint8 and uint16 sources, every flip and rotation, with
  ``train_batch`` on paired sources of the same shape in alternate windows.
* ``Trainer.train_step`` of HDRNetCurves (batch 1, 2048^2 crops, --nobatch_norm) with
  UnsharpMaskDataPipeline (sigma 4 and 32, sharpen 1) and with ImageFilesDataPipeline on uint8
  pairs, windows alternated.  The datasets are 4 random uint8 PNGs of 2136 x 2236 written to a
  temporary directory.

CUDA-event times: the median over --reps windows of --iters calls (after --warmup calls), with the
min-max spread.  Reads the card's name and power limit in the same run.  Prints one JSON object;
--out also writes it.

    python tools/time_usm.py [--iters 20 --warmup 5 --reps 7 --out tools_out/usm.json]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import data_pipeline as dp  # noqa: E402
from hdrnet_b200.bin import train  # noqa: E402


def gpu_identity():
    rec = {"name": torch.cuda.get_device_name(0)}
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    if q.returncode == 0 and q.stdout.strip():
        rec["power_limit"], rec["sm_max_clock"] = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return rec


def window_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def alternate(fns: dict, iters, warmup, reps):
    """{name: (median, min, max) ms per call}, the functions timed in alternate windows."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            times[k].append(window_ms(fn, iters))
    return {k: {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v))}
            for k, v in times.items()}


def batch_cases(iters, warmup, reps):
    rng = np.random.default_rng(0)
    out = []
    for B, (H, W), crop in ((1, (2136, 2236), 2048), (16, (600, 700), 512)):
        for dtype in (np.uint8, np.uint16):
            hi = np.iinfo(dtype).max + 1
            srcs = [torch.from_numpy(rng.integers(0, hi, (H, W, 3)).astype(dtype)).cuda() for _ in range(B)]
            tgts = [torch.from_numpy(rng.integers(0, hi, (H, W, 3)).astype(dtype)).cuda() for _ in range(B)]
            draws = []
            for i in range(B):
                k = i % 4
                rh, rw = (W, H) if k % 2 else (H, W)
                draws.append(dp.Draw(0, bool(i & 4), bool(i & 8), k, int(rng.integers(0, rh - crop + 1)),
                                     int(rng.integers(0, rw - crop + 1))))
            fns = {"train_batch": lambda: dp.train_batch(srcs, tgts, draws, (crop, crop), 256)}
            for sigma in (1.0, 4.0, 16.0, 32.0):
                fns[f"usm_sigma{sigma:g}"] = (lambda s=sigma: dp.usm_batch(srcs, draws, (crop, crop), 256, s, 1.0))
            res = alternate(fns, iters, warmup, reps)
            rec = {"case": f"{B} x {crop}^2 from {H} x {W}", "dtype": np.dtype(dtype).name, "ms": res}
            print(json.dumps(rec), flush=True)
            out.append(rec)
            del srcs, tgts
            torch.cuda.empty_cache()
    return out


def step_cases(iters, warmup, reps):
    import cv2
    rng = np.random.default_rng(1)
    with tempfile.TemporaryDirectory() as root:
        for sub in ("input", "output"):
            os.makedirs(os.path.join(root, sub))
        names = []
        for i in range(4):
            for sub in ("input", "output"):
                assert cv2.imwrite(os.path.join(root, sub, f"{i}.png"), rng.integers(0, 256, (2136, 2236, 3), np.uint8))
            names.append(f"{i}.png")
        with open(os.path.join(root, "filelist.txt"), "w") as f:
            f.write("\n".join(names) + "\n")
        common = ["--learning_rate", "1e-4", "--batch_size", "1", "--model_name", "HDRNetCurves", "--nobatch_norm",
                  "--output_resolution", "2048", "2048", "--summary_interval", "0", "--checkpoint_interval", "100000"]
        trainers = {}
        for name, flags in (("paired", []),
                            ("usm_sigma4", ["--data_pipeline", "UnsharpMaskDataPipeline", "--blur_sigma", "4",
                                            "--sharpen", "1"]),
                            ("usm_sigma32", ["--data_pipeline", "UnsharpMaskDataPipeline", "--blur_sigma", "32",
                                             "--sharpen", "1"])):
            parser = train.build_parser()
            args = parser.parse_args([os.path.join(root, "ckpt_" + name), root, *common, *flags])
            train.check_data_flags(parser, args)
            trainers[name] = train.Trainer(args, train.model_params(parser, args))
        try:
            res = alternate({k: t.train_step for k, t in trainers.items()}, iters, warmup, reps)
        finally:
            for t in trainers.values():
                t.close()
    rec = {"case": "Trainer.train_step, HDRNetCurves, batch 1, 2048^2 crops of 2136 x 2236 uint8 (train_std.sh shape)",
           "ms": res}
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_usm.py needs a CUDA device")
    rec = {"gpu": gpu_identity(), "batch": batch_cases(a.iters, a.warmup, a.reps),
           "train_step": step_cases(a.iters, a.warmup, a.reps)}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
