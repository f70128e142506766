"""The VJP kernels (csrc/slice_grad.cu) at the sizes they are used at, against the float64
reference (oracle/slice_f64.py, pinned on the CPU by tests/test_slice_f64.py).

tests/test_grad_gpu.py holds the kernels to the float32 reference loops up to 5 k pixels.  Here the
shapes reach what the kernels only do at scale: the reference's training step (--batch_size 16,
--output_resolution 512 512, hdrnet/bin/train.py:212, :228), 1080p and 4K frames, whose grid-VJP
elements sum 4 k to 130 k pixels; more pixels than the per-pixel kernel's grid has threads; grids
with more than one 8-depth x 12-channel tile of the column kernel; degenerate extents and guides.

Bars, from error analysis (the measured errors are in DESIGN.md section 2):
  * every VJP: max |diff| <= 1e-5 of max |ref64| (the project's bar, BASELINE.json);
  * grid VJP, per element: |diff| <= 4e-6 * sum |terms|.  A column that loses one pixel row at
    512 x 512 (~1.5 % of its footprint), or one pixel of a 4K footprint (1 / 130 k ~ 8e-6 of it),
    misses one of the two;
  * guide VJP, per pixel: |diff| <= 1e-5 * max(max |ref64|, sum |terms|).  Its two depth corners'
    derivatives have opposite signs and cancel below float32 round-off where both clamp to one
    border cell, so there it is held to its terms.
Case ids name the kernels and paths they exercise: "column" is slice_grad_grid_kernel, "ztiles" /
"ctiles" its depth / channel tiles, "pixel-stride" the per-pixel kernel's grid-stride loop.
"""
import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import hdrnet_ops
from oracle import slice_f64
from util import assert_parity

pytestmark = pytest.mark.gpu

RTOL = 1e-5
GRID_ELEM = 4e-6


def cuda(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


class Case:
    """op 'apply' (n_in -> n_out, has_offset) or 'slice' (gc channels); data 'signed' (randn grid
    and tangent, input in [0, 1]) or 'pos' (grid and input in [0, 1], tangent 1: every term of a
    grid-VJP element is >= 0, the worst case for float32 accumulation); guides 'rand' ([0, 1)),
    'const', 'wide' ([-0.5, 1.5]), 'centres' (exact cell centres and their float32 neighbours),
    'ends' (exactly 0 and 1)."""

    def __init__(self, B, H, W, gh, gw, gd, op="apply", n_in=3, n_out=3, ho=True, gc=None,
                 data="signed", guides="rand", seed=0, elem_bar=True):
        self.B, self.H, self.W, self.gh, self.gw, self.gd = B, H, W, gh, gw, gd
        self.op, self.n_in, self.n_out, self.ho, self.data, self.guides = op, n_in, n_out, ho, data, guides
        self.gc = gc if op == "slice" else n_out * (n_in + int(ho))
        self.seed = seed
        self.elem_bar = elem_bar

    def arrays(self):
        rng = np.random.RandomState(self.seed)
        B, H, W = self.B, self.H, self.W
        gshape = (B, self.gh, self.gw, self.gd, self.gc)
        grid = (rng.rand(*gshape) if self.data == "pos" else rng.randn(*gshape)).astype(np.float32)
        g = self.guides
        if g == "rand":
            guide = rng.rand(B, H, W)
        elif g == "const":
            guide = np.full((B, H, W), 0.37)
        elif g == "wide":
            guide = 2.0 * rng.rand(B, H, W) - 0.5
        elif g == "centres":
            c = (np.arange(self.gd) + 0.5).astype(np.float32) / np.float32(self.gd)
            vals = np.concatenate([c, np.nextafter(c, np.float32(0)), np.nextafter(c, np.float32(1))])
            guide = vals[rng.randint(0, len(vals), (B, H, W))]
        else:
            guide = rng.randint(0, 2, (B, H, W))
        guide = guide.astype(np.float32)
        nct = self.n_out if self.op == "apply" else self.gc
        ct = (np.ones((B, H, W, nct)) if self.data == "pos" else rng.randn(B, H, W, nct)).astype(np.float32)
        inp = rng.rand(B, H, W, self.n_in).astype(np.float32) if self.op == "apply" else None
        return grid, guide, inp, ct

    def cuda_grads(self, grid, guide, inp, ct):
        g, u = cuda(grid, True), cuda(guide, True)
        if self.op == "apply":
            i = cuda(inp, True)
            hdrnet_ops.bilateral_slice_apply(g, u, i, self.ho).backward(cuda(ct))
            return [t.grad.cpu().numpy() for t in (g, u, i)]
        hdrnet_ops.bilateral_slice(g, u).backward(cuda(ct))
        return [g.grad.cpu().numpy(), u.grad.cpu().numpy(), None]

    def f64(self, grid, guide, inp, ct):
        if self.op == "apply":
            return slice_f64.bilateral_slice_apply_grad(grid, guide, inp, ct, self.ho)
        return slice_f64.bilateral_slice_grad(grid, guide, ct)

    def loops(self, grid, guide, inp, ct):
        """The float32 reference loops (compiled reference where built, else its C restatement)."""
        if self.op == "apply":
            return list(oracle.best().bilateral_slice_apply_grad(grid, guide, inp, ct, self.ho))
        return list(oracle.best().bilateral_slice_grad(grid, guide, ct)) + [None]


def errors(got, r):
    """Error of (grid, guide, input) VJPs against the float64 reference, in the bars' units."""
    gv, uv, iv = (None if a is None else np.asarray(a, np.float64) for a in got)
    e = {}
    d = np.abs(gv - r.grid)
    e["grid"] = float(d.max()) / max(float(np.abs(r.grid).max()), 1e-30)
    # an element without terms (grid_abs == 0) must be exactly 0
    e["grid_elem"] = float(np.where(r.grid_abs > 0, d / np.maximum(r.grid_abs, 1e-300),
                                    np.where(d > 0, np.inf, 0.0)).max())
    scale = np.maximum(float(np.abs(r.guide).max()), r.guide_abs)
    e["guide"] = float((np.abs(uv - r.guide) / np.maximum(scale, 1e-30)).max())
    if iv is not None:
        e["input"] = float(np.abs(iv - r.input).max()) / max(float(np.abs(r.input).max()), 1e-30)
    return e


def check(e, what, elem_bar=True):
    if not elem_bar:
        e = {k: v for k, v in e.items() if k != "grid_elem"}
    bad = [f"{k} {v:.3e}" for k, v in e.items() if v > (GRID_ELEM if k == "grid_elem" else RTOL)]
    assert not bad, f"{what}: " + ", ".join(bad) + f" (all: {e})"


CASES = {
    # the reference's training step: column kernel with 4 k-pixel footprints, pixel-stride loop
    "train-column-pixel-stride": Case(16, 512, 512, 16, 16, 8),
    "train_pos-column-pixel-stride": Case(16, 512, 512, 16, 16, 8, data="pos", seed=1),
    "hd-column": Case(1, 1080, 1920, 16, 16, 8, seed=2),                 # 67.5 px per cell
    "4k-column": Case(1, 2160, 3840, 16, 16, 8, seed=3),                 # 130 k-pixel footprints
    "gd16-column-ztiles-hd": Case(1, 1080, 1920, 32, 32, 16, data="pos", seed=4),
    "gd16-column-ztiles-b16": Case(16, 256, 256, 16, 16, 16, data="pos", seed=5),
    "gd16-column-ztiles-4k": Case(1, 2160, 3840, 32, 32, 16, data="pos", seed=21),   # 32 k-pixel footprints
    "gc16-column-ctiles": Case(4, 512, 512, 16, 16, 8, n_out=4, data="pos", seed=6),
    "gc36-column-ctiles": Case(1, 512, 512, 16, 16, 8, n_out=9, seed=7),
    "slice-gc12-column": Case(4, 512, 512, 16, 16, 8, op="slice", gc=12, seed=8),
    "slice-gc24-column-ctiles": Case(4, 512, 512, 16, 16, 8, op="slice", gc=24, data="pos", seed=9),
    "slice-gc2-column": Case(4, 512, 512, 16, 16, 8, op="slice", gc=2, seed=10),
    "switch-gd8-column": Case(2, 256, 256, 16, 16, 8, data="pos", seed=11),
    "switch-gd9-column-ztiles": Case(2, 256, 256, 16, 16, 9, data="pos", seed=12),
    "switch-gc12-slice-column": Case(2, 256, 256, 16, 16, 8, op="slice", gc=12, data="pos", seed=13),
    "switch-gc13-slice-column-ctiles": Case(2, 256, 256, 16, 16, 8, op="slice", gc=13, data="pos", seed=14),
    "switch-gd1-column": Case(2, 256, 256, 16, 16, 1, guides="wide", seed=15),
    # 7 x 5 pixels on a 16 x 16 grid: an element sums 1-4 pixels, and a float32 tent weight carries
    # the rounding of its cell coordinate (~1e-6 absolute), which the per-element bar, made for long
    # sums, does not allow for.  Measured 4.6e-6 of sum |terms| on the H100, the same as the
    # reference loops' own; the global bar still applies.
    "switch-small-image-column": Case(3, 7, 5, 16, 16, 8, guides="wide", seed=16, elem_bar=False),
    "guides-const-column": Case(2, 512, 512, 16, 16, 8, guides="const", seed=17),
    "guides-wide-column": Case(2, 512, 512, 16, 16, 8, guides="wide", seed=18),
    "guides-centres-column": Case(2, 512, 512, 16, 16, 8, guides="centres", seed=19),
    "guides-ends-column": Case(2, 512, 512, 16, 16, 8, guides="ends", seed=20),
}


@pytest.mark.parametrize("name", list(CASES))
def test_vjps_match_float64_at_scale(name):
    c = CASES[name]
    grid, guide, inp, ct = c.arrays()
    got = c.cuda_grads(grid, guide, inp, ct)
    check(errors(got, c.f64(grid, guide, inp, ct)), name, c.elem_bar)


def test_train_step_matches_reference_loops_and_is_reproducible():
    """The training step against the float32 reference loops at the bar of tests/test_grad_gpu.py,
    and bitwise identical across two runs (no atomics anywhere in the VJP kernels)."""
    c = CASES["train-column-pixel-stride"]
    grid, guide, inp, ct = c.arrays()
    got = c.cuda_grads(grid, guide, inp, ct)
    for a, b, name in zip(got, c.loops(grid, guide, inp, ct), ("grid", "guide", "input")):
        assert_parity(a, b, rtol=2e-5, what=f"train {name} VJP")
    again = c.cuda_grads(grid, guide, inp, ct)
    for a, b in zip(got, again):
        assert np.array_equal(a, b)


def test_4k_grid_vjp_is_the_adjoint_of_the_forward():
    """<ct, slice_apply(grid)> = <grid_vjp, grid>: the forward as AUTO runs it (the issuer-warp
    kernel) against the VJP's own kernels, summed in float64 on the host.  Guides stay inside
    (0.5, gd - 0.5) / gd, where the grid VJP's border override is inactive and the identity exact."""
    c = CASES["4k-column"]
    grid, _, inp, ct = c.arrays()
    gd = c.gd
    guide = ((0.5 + 0.01 + (gd - 1.02) * np.random.RandomState(30).rand(c.B, c.H, c.W)) / gd).astype(np.float32)
    with torch.no_grad():
        out = hdrnet_ops.bilateral_slice_apply(cuda(grid), cuda(guide), cuda(inp), True).cpu().numpy()
    gv = c.cuda_grads(grid, guide, inp, ct)[0]
    lhs = float((ct.astype(np.float64) * out).sum())
    rhs = float((gv.astype(np.float64) * grid).sum())
    scale = float(np.abs(ct.astype(np.float64) * out).sum())
    assert abs(lhs - rhs) <= 1e-5 * scale, f"<ct, F(grid)> {lhs:.6e} != <grid_vjp, grid> {rhs:.6e}"
