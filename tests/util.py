"""Shared helpers for the parity tests."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# BASELINE.json north_star: "outputs match the repo's jax/bilateral_slice.py reference to
# 1e-5 relative fp32".  Relative means relative to the magnitude of the output tensor:
# a pixel whose terms cancel to ~0 cannot be held to 1e-5 of its own value in float32.
RTOL = 1e-5


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def rel_err(actual, expected):
    actual = np.asarray(actual, np.float64)
    expected = np.asarray(expected, np.float64)
    scale = max(float(np.abs(expected).max()), 1e-30)
    return float(np.abs(actual - expected).max()) / scale


def elem_err(actual, expected, floor=1e-3):
    """Worst PER-ELEMENT relative error, |diff| / max(|ref|, floor * max|ref|): the global metric
    above lets a pixel whose terms cancel be wrong by all of its own value; this one holds every
    element that is not itself below `floor` of the tensor's range to its own magnitude."""
    actual = np.asarray(actual, np.float64)
    expected = np.asarray(expected, np.float64)
    scale = max(float(np.abs(expected).max()), 1e-30)
    return float((np.abs(actual - expected) / np.maximum(np.abs(expected), floor * scale)).max())


# Per-element bar: an output is a sum of ~60 float32 products of magnitude up to max|grid| * max|in|;
# with signed inputs the sum may cancel to `floor` of the range, so its float32 round-off is up to
# ~1e-7 / floor = 1e-4 of ITS OWN value.  2e-3 leaves an order of magnitude and still catches any
# wrong cell, weight or channel (those are errors of order 1).
ELEM_RTOL = 2e-3


def assert_parity(actual, expected, rtol=RTOL, what="", elem_rtol=ELEM_RTOL):
    actual = np.asarray(actual)
    expected = np.asarray(expected)
    assert actual.shape == expected.shape, f"{what}: shape {actual.shape} != {expected.shape}"
    assert np.isfinite(actual).all(), f"{what}: non-finite values"
    err = rel_err(actual, expected)
    per_elem = elem_err(actual, expected)
    assert err <= rtol, (f"{what}: max |diff| / max |ref| = {err:.3e} > {rtol:.1e} "
                         f"(worst per-element {per_elem:.3e})")
    if elem_rtol is not None:
        assert per_elem <= elem_rtol, (f"{what}: worst per-element |diff| / max(|ref|, 1e-3 max|ref|) = "
                                       f"{per_elem:.3e} > {elem_rtol:.1e} (global {err:.3e})")


# VJP test extents shared by tests/test_grad_gpu.py (CUDA vs the reference loops) and
# tests/test_slice_f64.py (the float64 reference vs the same loops).
# (B, H, W, gh, gw, gd, n_in, n_out, has_offset)
APPLY_CASES = [
    (3, 8, 5, 6, 3, 7, 3, 4, True),      # hdrnet_ops_test.py:185-195 (gc=16: two channel tiles)
    (3, 30, 25, 16, 12, 8, 3, 3, True),  # default test extents: one column tile (gd<=8, gc<=12)
    (2, 40, 64, 4, 4, 8, 3, 3, True),    # several pixels per cell, mirror boundary on all sides
    (2, 33, 47, 5, 3, 4, 3, 4, False),   # no offset
    (1, 16, 16, 2, 2, 1, 1, 1, True),    # gd = 1: both depth borders at once
]

# (B, H, W, gh, gw, gd, gc)
SLICE_CASES = [(3, 30, 25, 16, 12, 8, 12), (2, 21, 36, 5, 4, 6, 2), (1, 9, 7, 3, 3, 9, 5)]


def rand_case(seed, B, H, W, gh, gw, gd, n_in=3, n_out=3, has_offset=True, signed=False):
    """Seeded inputs as the reference's tests draw them (np.random.rand; hdrnet_ops_test.py:101)."""
    rng = np.random.RandomState(seed)
    J = n_in + (1 if has_offset else 0)
    draw = (lambda *s: rng.randn(*s)) if signed else (lambda *s: rng.rand(*s))
    grid = draw(B, gh, gw, gd, n_out * J).astype(np.float32)
    guide = rng.rand(B, H, W).astype(np.float32)
    inp = draw(B, H, W, n_in).astype(np.float32)
    return grid, guide, inp


# The reference's convergence-by-SGD tests (hdrnet/test/ops_test.py:189-322): a 1 x 32 image sliced
# from a tiny grid is fitted to one period of a sine by plain gradient descent on sum((target-out)^2)
# (l2_optimizer, :178-186) -- over the grid, over the guide (through a sigmoid), or over both.
# name -> (gh, gw, gd, learning rate, steps, the reference's bound on the final loss, what is trained)
SGD_CASES = {
    "grid": (1, 16, 8, 1e-2, 10000, 0.0085, ("grid",)),          # test_grid_optimize  :189-230
    "guide": (1, 8, 2, 1e-3, 6000, 1e-4, ("guide",)),            # test_guide_optimize :232-278
    "both": (1, 8, 2, 1e-1, 10000, 1e-4, ("grid", "guide")),     # test_optimize_both  :280-322
}


def sgd_case(name):
    """Initial values as the reference test builds them.  The reference draws its random initial
    values unseeded; the seeds here are fixed, and for "both" chosen among those for which the
    reference's own loops (oracle) meet the reference's bound -- they do not for every draw."""
    gh, gw, gd, lr, steps, bound, trained = SGD_CASES[name]
    w = 32
    rng = np.random.RandomState({"grid": 1, "guide": 0, "both": 3}[name])
    target = np.sin(np.linspace(0, 2 * np.pi, w)).astype(np.float32)[None, None, :, None]
    if name == "grid":
        guide = np.linspace(0, 1, w).astype(np.float32)[None, None, :]       # used as is
        grid = rng.rand(1, gh, gw, gd, 1).astype(np.float32)
    elif name == "guide":
        guide = np.linspace(0.5 / gd, 1 - 0.5 / gd, w).astype(np.float32)[None, None, :]   # pre-sigmoid
        grid = np.tile(np.linspace(-1, 1, gd).astype(np.float32)[None, None, None, :, None], [1, gh, gw, 1, 1])
    else:
        guide = rng.rand(1, 1, w).astype(np.float32) * 2.0 - 1.0                # pre-sigmoid
        grid = rng.rand(1, gh, gw, gd, 1).astype(np.float32)
    return dict(grid=grid, guide=guide, target=target, lr=lr, steps=steps, bound=bound, trained=trained,
                sigmoid=(name != "grid"))
