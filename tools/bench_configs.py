#!/usr/bin/env python
"""Secondary measurements for BASELINE.json configs 2, 4 (per-GPU share) and 5, plus the
guide-fused model path.  Prints one JSON object per line; bench.py stays the headline.
    python tools/bench_configs.py [--quick]
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, ROOT)
from hdrnet_b200 import _lib, hdrnet_ops, models  # noqa: E402

PEAK = 3350.0   # H100 SXM data sheet, GB/s
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def timeit(fn, warm=5, iters=50):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters  # ms


def slice_apply_case(name, B, H, W, gh, gw, gd, iters=50, variant=_lib.VARIANT_AUTO):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    grid = torch.rand(B, gh, gw, gd, 12, device="cuda", generator=gen)
    guide = torch.rand(B, H, W, device="cuda", generator=gen)
    inp = torch.rand(B, H, W, 3, device="cuda", generator=gen)
    out = torch.empty_like(inp)
    ms = timeit(lambda: hdrnet_ops.bilateral_slice_apply(grid, guide, inp, True, out=out, variant=variant),
                iters=iters)
    npx = B * H * W
    gbs = (npx * 28 + grid.numel() * 4) / ms / 1e6
    print(json.dumps({"case": name, "shape": [B, H, W], "grid": [gh, gw, gd], "ms": round(ms, 4),
                      "MP/s": round(npx / ms / 1e3, 1), "GB/s": round(gbs, 1),
                      "frac_of_measured_hbm": round(gbs / PEAK, 4)}), flush=True)


def any_shape_case(name, B, H, W, gh, gw, gd, n_in, n_out, has_offset, iters=10):
    """Shapes outside the TMA kernels' contract: AUTO (any-shape row kernel) vs the per-pixel kernel."""
    gen = torch.Generator(device="cuda").manual_seed(1234)
    J = n_in + (1 if has_offset else 0)
    grid = torch.rand(B, gh, gw, gd, n_out * J, device="cuda", generator=gen)
    guide = torch.rand(B, H, W, device="cuda", generator=gen)
    inp = torch.rand(B, H, W, n_in, device="cuda", generator=gen)
    out = torch.empty(B, H, W, n_out, device="cuda")
    npx = B * H * W
    nbytes = npx * 4 * (n_in + 1 + n_out) + grid.numel() * 4
    rec = {"case": name, "shape": [B, H, W], "grid": [gh, gw, gd], "n_in": n_in, "n_out": n_out, "has_offset": has_offset,
           "bytes_per_px": 4 * (n_in + 1 + n_out)}
    for label, v in (("auto_rows_any", _lib.VARIANT_AUTO), ("per_pixel_generic", _lib.VARIANT_GENERIC)):
        ms = timeit(lambda: hdrnet_ops.bilateral_slice_apply(grid, guide, inp, has_offset, out=out, variant=v), iters=iters)
        rec[label] = {"ms": round(ms, 4), "MP/s": round(npx / ms / 1e3, 1), "frac_of_measured_hbm": round(nbytes / ms / 1e6 / PEAK, 4)}
    print(json.dumps(rec), flush=True)


def slice_case(name, B, H, W, gh, gw, gd, iters=30, variant=_lib.VARIANT_AUTO):
    gen = torch.Generator(device="cuda").manual_seed(1234)
    grid = torch.rand(B, gh, gw, gd, 12, device="cuda", generator=gen)
    guide = torch.rand(B, H, W, device="cuda", generator=gen)
    ms = timeit(lambda: hdrnet_ops.bilateral_slice(grid, guide, variant=variant), iters=iters)
    npx = B * H * W
    gbs = (npx * 52 + grid.numel() * 4) / ms / 1e6
    print(json.dumps({"case": name, "shape": [B, H, W], "grid": [gh, gw, gd], "ms": round(ms, 4),
                      "MP/s": round(npx / ms / 1e3, 1), "GB/s_at_52B_per_px": round(gbs, 1),
                      "frac_of_measured_hbm": round(gbs / PEAK, 4)}), flush=True)


def model_case(name, model_name, B, H, W, iters=30):
    p = dict(models.DEFAULT_PARAMS, model_name=model_name)
    wts = models.init_weights(p, seed=0, model_name=model_name)
    rng = np.random.RandomState(1)
    # perturb the guide so depth cells are actually exercised
    p["weights"] = wts
    cls = getattr(models, model_name)
    gen = torch.Generator(device="cuda").manual_seed(1)
    low = torch.rand(B, 256, 256, 3, device="cuda", generator=gen)
    full = torch.rand(B, H, W, 3, device="cuda", generator=gen)
    t_all = timeit(lambda: cls.inference(low, full, p), iters=iters)
    t_cnn = timeit(lambda: cls._coefficients(low, p), iters=iters)
    # CUDA-graph replay of the whole model (launch-latency-bound at small batch)
    static_out = cls.inference(low, full, p)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        cls.inference(low, full, p)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            static_out = cls.inference(low, full, p)
    torch.cuda.synchronize()
    t_graph = timeit(g.replay, iters=iters)
    npx = B * H * W
    print(json.dumps({"case": name, "model": model_name, "shape": [B, H, W],
                      "ms_model_eager_launch": round(t_all, 4), "ms_coefficient_cnn": round(t_cnn, 4),
                      "ms_guide_plus_slice_apply": round(t_all - t_cnn, 4),
                      "ms_model_cuda_graph": round(t_graph, 4),
                      "MP/s_model_graph": round(npx / t_graph / 1e3, 1),
                      "fused_GB/s_at_24B_per_px": round(npx * 24 / max(t_all - t_cnn, 1e-6) / 1e6, 1)}),
          flush=True)


def image_case(name, model_name, B, H, W, iters=20):
    """run.py's per-image path (decode format in, uint8 out): device-resident and end to end from
    pinned host memory, integer pixels (inference_image) against the float32 feed (inference)."""
    p = dict(models.DEFAULT_PARAMS, model_name=model_name)
    p["weights"] = models.init_weights(p, seed=0, model_name=model_name)
    cls = getattr(models, model_name)
    gen = torch.Generator(device="cuda").manual_seed(1)
    im8 = torch.randint(0, 256, (B, H, W, 3), device="cuda", generator=gen, dtype=torch.uint8)
    im8_h = im8.cpu().pin_memory()
    out8_h = torch.empty_like(im8_h).pin_memory()
    imf_h = models.image_to_float(im8).cpu().pin_memory()
    low_h = models.lowres_from_image(im8, 256).cpu().pin_memory()
    outf_h = torch.empty_like(imf_h).pin_memory()

    def e2e_u8():
        out8_h.copy_(cls.inference_image(im8_h.cuda(non_blocking=True), p), non_blocking=True)

    def e2e_f32():   # what a float32 feed costs: 12 B/px up (+ lowres), 12 B/px down
        out = cls.inference(low_h.cuda(non_blocking=True), imf_h.cuda(non_blocking=True), p)
        outf_h.copy_(out, non_blocking=True)

    t_dev = timeit(lambda: cls.inference_image(im8, p), iters=iters)
    imf = models.image_to_float(im8)
    low = models.lowres_from_image(im8, 256)
    t_dev_f32 = timeit(lambda: cls.inference(low, imf, p), iters=iters)
    t_e2e = timeit(e2e_u8, warm=2, iters=max(3, iters // 4))
    t_e2e_f32 = timeit(e2e_f32, warm=2, iters=max(3, iters // 4))
    npx = B * H * W
    print(json.dumps({"case": name, "model": model_name, "shape": [B, H, W],
                      "ms_device_u8_in_u8_out": round(t_dev, 4), "MP/s_device_u8": round(npx / t_dev / 1e3, 1),
                      "ms_device_f32": round(t_dev_f32, 4), "MP/s_device_f32": round(npx / t_dev_f32 / 1e3, 1),
                      "ms_e2e_pinned_u8": round(t_e2e, 3), "MP/s_e2e_u8": round(npx / t_e2e / 1e3, 1),
                      "ms_e2e_pinned_f32": round(t_e2e_f32, 3), "MP/s_e2e_f32": round(npx / t_e2e_f32 / 1e3, 1),
                      "pcie_bytes_per_px": {"u8": 6, "f32": 24}}), flush=True)


def main():
    quick = "--quick" in sys.argv
    torch.cuda.set_device(0)
    slice_apply_case("C3 4K x8 (headline shape)", 8, 2160, 3840, 16, 16, 8)
    slice_apply_case("C3 4K x8 texture-assisted kernel (incl. y-blend pre-pass)", 8, 2160, 3840, 16, 16, 8, variant=_lib.VARIANT_TEX)
    slice_apply_case("C2 1080p x1 texture-assisted", 1, 1080, 1920, 16, 16, 8, variant=_lib.VARIANT_TEX)
    slice_apply_case("C3 4K x8 generic kernel", 8, 2160, 3840, 16, 16, 8, iters=10, variant=_lib.VARIANT_GENERIC)
    slice_apply_case("C2 1080p x1", 1, 1080, 1920, 16, 16, 8)
    slice_apply_case("C4 12MP x8 (one GPU's share of batch 64)", 8, 3024, 4032, 16, 16, 8, iters=20)
    for gh, gw, gd in [(8, 8, 4), (16, 16, 4), (16, 16, 8), (32, 32, 8), (32, 32, 16)]:
        slice_apply_case(f"C5 sweep 4K x8 grid {gh}x{gw}x{gd}", 8, 2160, 3840, gh, gw, gd, iters=20)
    any_shape_case("4K x8 has_offset=False (3 -> 4, gc 12)", 8, 2160, 3840, 16, 16, 8, 3, 4, False)
    any_shape_case("4K x8 odd width 3841 (3 -> 3 + offset)", 8, 2160, 3841, 16, 16, 8, 3, 3, True)
    any_shape_case("4K x4 pyramid grid (3 -> 9 + offset, gc 36)", 4, 2160, 3840, 16, 16, 8, 3, 9, True)
    slice_case("un-fused bilateral_slice 4K x8 (TMA kernel)", 8, 2160, 3840, 16, 16, 8)
    slice_case("un-fused bilateral_slice 4K x8 (generic kernel)", 8, 2160, 3840, 16, 16, 8, iters=5,
               variant=_lib.VARIANT_GENERIC)
    model_case("C2 model 1080p x1", "HDRNetCurves", 1, 1080, 1920)
    model_case("model 4K x8", "HDRNetCurves", 8, 2160, 3840, iters=10)
    image_case("image path 4K x8 (u8 in, u8 out)", "HDRNetCurves", 8, 2160, 3840)
    image_case("image path 1080p x1 (u8 in, u8 out)", "HDRNetCurves", 1, 1080, 1920)
    if not quick:
        model_case("C2 model 1080p x1 (NN guide)", "HDRNetPointwiseNNGuide", 1, 1080, 1920)
        model_case("model 4K x8 (NN guide)", "HDRNetPointwiseNNGuide", 8, 2160, 3840, iters=10)


if __name__ == "__main__":
    if "--image-only" in sys.argv:
        torch.cuda.set_device(0)
        image_case("image path 4K x8 (u8 in, u8 out)", "HDRNetCurves", 8, 2160, 3840)
        image_case("image path 4K x8 (u8 in, u8 out, NN guide)", "HDRNetPointwiseNNGuide", 8, 2160, 3840)
        image_case("image path 1080p x1 (u8 in, u8 out)", "HDRNetCurves", 1, 1080, 1920)
    else:
        main()
