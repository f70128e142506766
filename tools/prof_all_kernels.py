"""Runs every kernel of libhdrnet_b200.so once at a representative shape, for one ncu pass:
    ncu --set full --clock-control none -k regex:'hdrnet_b200' -c 200 -f -o tools_out/r02_all_kernels \
        python tools/prof_all_kernels.py
    ncu -i tools_out/r02_all_kernels.ncu-rep --page raw --csv > tools_out/r02_all_kernels_raw.csv
    python tools/ncu_kernel_table.py tools_out/r02_all_kernels_raw.csv > tools_out/all_kernels_ncu.md
Synthetic inputs, seeded synthetic weights.  No warm-up on purpose (every launch is captured)."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import _lib, hdrnet_ops, models

dev = torch.device("cuda")
gen = torch.Generator(device=dev).manual_seed(0)


def params(name, **kw):
    p = dict(models.DEFAULT_PARAMS, model_name=name, **kw)
    p["weights"] = models.init_weights(p, seed=0, model_name=name)
    return p


# ---- model path at 4K x 8: batch-8 CNN (tensor-core packed convs, fc, fuse_predict), fused-guide slice-apply
im = torch.rand(8, 2160, 3840, 3, device=dev, generator=gen)
for name in ("HDRNetCurves", "HDRNetPointwiseNNGuide"):
    p = params(name, batch_norm=(name != "HDRNetCurves"))
    cls = getattr(models, name)
    low = models.lowres_from_image(im, 256)           # lowres_nearest_kernel (float32 source)
    cls.inference(low, im, p)
    cls.inference(low, im, dict(p, debug=True))       # standalone guide kernel + op-API slice-apply
# ---- integer image path: uint8 / uint16 in, uint8 out
im8 = torch.randint(0, 256, (8, 2160, 3840, 3), device=dev, generator=gen, dtype=torch.uint8)
pc = params("HDRNetCurves")
models.HDRNetCurves.inference_image(im8, pc)
im16 = torch.randint(0, 32768, (2, 3024, 4032, 3), device=dev, generator=gen, dtype=torch.int32).to(torch.uint16)
models.HDRNetCurves.inference_image(im16, pc)
del im8, im16
# ---- one 1080p frame: batch-1 CNN (CUDA-core convs, cluster fc), row kernel without workspace
im1 = torch.rand(1, 1080, 1920, 3, device=dev, generator=gen)
models.HDRNetCurves.inference(models.lowres_from_image(im1, 256), im1, pc)
# ---- pyramid model: bilinear resize (+ fused add), three fused NN-guide slice-applies
pp = params("HDRNetGaussianPyrNN")
models.HDRNetGaussianPyrNN.inference(models.lowres_from_image(im1, 256), im1, pp)
# ---- op API: slice-apply forms, un-fused slice, VJPs
grid = torch.rand(8, 16, 16, 8, 12, device=dev, generator=gen)
guide = torch.rand(8, 2160, 3840, device=dev, generator=gen)
for v in (_lib.VARIANT_AUTO, _lib.VARIANT_TEX, _lib.VARIANT_TMA):
    hdrnet_ops.bilateral_slice_apply(grid, guide, im, True, variant=v)
hdrnet_ops.bilateral_slice_apply(grid[:1], guide[:1, :270], im[:1, :270].contiguous(), True, variant=_lib.VARIANT_GENERIC)
hdrnet_ops.bilateral_slice(grid[:2], guide[:2].contiguous())                 # slice_rows_tma_kernel
hdrnet_ops.bilateral_slice(grid[:1], guide[:1, :270].contiguous(), variant=_lib.VARIANT_GENERIC)
g1 = grid[:1].clone().requires_grad_(True)
u1 = guide[:1, :1080, :1920].contiguous().requires_grad_(True)
i1 = im1.clone().requires_grad_(True)
hdrnet_ops.bilateral_slice_apply(g1, u1, i1, True).sum().backward()          # slice_grad_pixel / _grid kernels
g2 = grid[:1].clone().requires_grad_(True)
hdrnet_ops.bilateral_slice(g2, u1.detach()).sum().backward()
hdrnet_ops.slice_indices(guide[:1, :270].contiguous(), (16, 16, 8))
# ---- standalone guide kernels, any-shape row kernels, per-pixel integer-I/O kernel, plain fc kernel
models.HDRNetCurves._guide(im[:2].contiguous(), pc)
pn = params("HDRNetPointwiseNNGuide", batch_norm=True)
models.HDRNetPointwiseNNGuide._guide(im[:2].contiguous(), pn)
g4 = torch.rand(4, 16, 16, 8, 12, device=dev, generator=gen)
hdrnet_ops.bilateral_slice_apply(g4, guide[:4].contiguous(), im[:4].contiguous(), False)      # 3 -> 4, no offset
g7 = torch.rand(2, 16, 16, 8, 7, device=dev, generator=gen)
hdrnet_ops.bilateral_slice(g7, guide[:2].contiguous())                                        # slice, gc = 7
odd = torch.randint(0, 256, (1, 1080, 1921, 3), device=dev, generator=gen, dtype=torch.uint8)
models.HDRNetCurves.inference_image(odd, pc)                                                  # W % 16 != 0
x = torch.rand(64, 1024, device=dev, generator=gen); w = torch.rand(1024, 256, device=dev, generator=gen)
models._fc(x, (w, torch.zeros(256, device=dev)), relu=True)
torch.cuda.synchronize()
print("done")
