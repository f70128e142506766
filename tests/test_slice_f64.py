"""CPU tests that pin the float64 reference of the slice ops and their VJPs (oracle/slice_f64.py).

It is the yardstick of tests/test_grad_scale_gpu.py, where the float32 reference loops no longer
tell whether a gradient is accurate, so it is pinned three independent ways:
  * against the float32 restatement of the reference loops (oracle.port(), itself bit-exact with
    the compiled reference and pinned to the reference's JAX VJPs in tests/test_oracle.py), at the
    extents of tests/test_grad_gpu.py, the stored JAX VJP fixtures and the degenerate extents;
  * by adjoint identities in float64 (the forward is linear in the grid and in the input);
  * by central differences of its own float64 forward for the guide VJP.
"""
import numpy as np
import pytest

from oracle import slice_f64
from util import APPLY_CASES, SLICE_CASES, load_golden, rand_case

# The float32 loops form the cell coordinate (x + 0.5) * fl(gw / W) in float32: up to ~1 ulp of gw
# in every x / y weight, 1e-6 of the result for a 16-cell-wide grid.  Everything else they do is
# well-conditioned float32 arithmetic over a few dozen terms.
PORT_RTOL = 2e-6


def _bar(got, ref, scale, what, rtol=PORT_RTOL):
    got = np.asarray(got, np.float64)
    err = float(np.abs(got - ref).max()) / max(float(scale), 1e-30)
    assert err <= rtol, f"{what}: max |diff| / scale = {err:.3e} > {rtol:.1e}"


def _guide_bar(got, r, what, rtol=PORT_RTOL):
    """The guide VJP sums two depth corners' derivatives of opposite sign; where both corners clamp
    to one border cell (and everywhere when gd = 1) they cancel to ~1e-8 of the terms, below float32
    round-off.  So each pixel is held to the larger of the tensor's range and its own sum of
    |terms|."""
    scale = np.maximum(np.abs(r.guide).max(), r.guide_abs)
    err = float((np.abs(np.asarray(got, np.float64) - r.guide) / np.maximum(scale, 1e-30)).max())
    assert err <= rtol, f"{what}: max |diff| / max(max |ref|, sum |terms|) = {err:.3e} > {rtol:.1e}"


def _check_apply(grid, guide, inp, ct, ho, port, what):
    r = slice_f64.bilateral_slice_apply_grad(grid, guide, inp, ct, ho)
    want = port.bilateral_slice_apply_grad(grid, guide, inp, ct, ho)
    fwd = slice_f64.bilateral_slice_apply(grid, guide, inp, ho)
    _bar(port.bilateral_slice_apply(grid, guide, inp, ho), fwd, np.abs(fwd).max(), f"{what} forward")
    _bar(want[0], r.grid, np.abs(r.grid).max(), f"{what} grid VJP")
    _guide_bar(want[1], r, f"{what} guide VJP")
    _bar(want[2], r.input, np.abs(r.input).max(), f"{what} input VJP")


def _check_slice(grid, guide, ct, port, what):
    r = slice_f64.bilateral_slice_grad(grid, guide, ct)
    want = port.bilateral_slice_grad(grid, guide, ct)
    fwd = slice_f64.bilateral_slice(grid, guide)
    _bar(port.bilateral_slice(grid, guide), fwd, np.abs(fwd).max(), f"{what} forward")
    _bar(want[0], r.grid, np.abs(r.grid).max(), f"{what} grid VJP")
    _guide_bar(want[1], r, f"{what} guide VJP")


@pytest.mark.parametrize("case", APPLY_CASES, ids=str)
@pytest.mark.parametrize("guides", ["unit", "wide"])
def test_f64_apply_matches_port(oracle_port, case, guides):
    B, H, W, gh, gw, gd, n_in, n_out, ho = case
    grid, guide, inp = rand_case(5, B, H, W, gh, gw, gd, n_in, n_out, ho, signed=True)
    if guides == "wide":
        guide = (2.0 * guide - 0.5).astype(np.float32)     # [-0.5, 1.5]: both border overrides
    ct = np.random.RandomState(6).randn(B, H, W, n_out).astype(np.float32)
    _check_apply(grid, guide, inp, ct, ho, oracle_port, f"{case} {guides}")


@pytest.mark.parametrize("y_off, rows", [(0, 7), (13, 5), (33, 7), (39, 1)])
def test_f64_apply_row_band_is_the_whole_image_rows(y_off, rows):
    """A row band (y_off, height) is, value for value, those rows of the whole-image call: the large
    extents tests hold a few rows of a large image to the reference at the cost of those rows."""
    grid, guide, inp = rand_case(7, 2, 40, 23, 6, 5, 4, signed=True)
    whole = slice_f64.bilateral_slice_apply(grid, guide, inp, True)
    band = slice_f64.bilateral_slice_apply(grid, guide[:, y_off:y_off + rows], inp[:, y_off:y_off + rows], True,
                                           y_off=y_off, height=40)
    assert np.array_equal(band, whole[:, y_off:y_off + rows])
    with pytest.raises(ValueError):
        slice_f64.bilateral_slice_apply(grid, guide[:, :rows], inp[:, :rows], True, y_off=41 - rows, height=40)


@pytest.mark.parametrize("case", SLICE_CASES, ids=str)
def test_f64_slice_matches_port(oracle_port, case):
    B, H, W, gh, gw, gd, gc = case
    rng = np.random.RandomState(7)
    grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
    guide = (2.0 * rng.rand(B, H, W) - 0.5).astype(np.float32)
    ct = rng.randn(B, H, W, gc).astype(np.float32)
    _check_slice(grid, guide, ct, oracle_port, str(case))


@pytest.mark.parametrize("name", ["vjp_0", "vjp_1", "vjp_2", "vjp_3"])
def test_f64_slice_vjps_match_port_on_jax_fixtures(oracle_port, name):
    z = load_golden(name)
    _check_slice(z["grid"], z["guide"], z["codomain_tangent"], oracle_port, name)
    # and the stored JAX VJPs themselves, at the bar the port is held to (tests/test_oracle.py)
    r = slice_f64.bilateral_slice_grad(z["grid"], z["guide"], z["codomain_tangent"])
    _bar(z["grid_vjp"], r.grid, np.abs(r.grid).max(), f"{name} JAX grid VJP", rtol=1e-6)


# (B, H, W, gh, gw, gd): degenerate extents
EDGE_SHAPES = [
    (2, 16, 16, 4, 4, 1),     # gd = 1: every pixel clamps both depth corners
    (2, 5, 7, 9, 11, 4),      # H < gh and W < gw: upsampling
    (1, 3, 7, 16, 16, 8),     # a small image on a large grid
    (2, 1, 37, 3, 5, 4),      # H = 1
    (2, 29, 1, 3, 5, 4),      # W = 1
    (1, 1, 1, 2, 3, 8),       # one pixel
]


@pytest.mark.parametrize("shape", EDGE_SHAPES, ids=str)
def test_f64_matches_port_at_degenerate_extents(oracle_port, shape):
    B, H, W, gh, gw, gd = shape
    grid, guide, inp = rand_case(31, B, H, W, gh, gw, gd, 3, 3, True, signed=True)
    guide = (2.0 * guide - 0.5).astype(np.float32)
    ct = np.random.RandomState(32).randn(B, H, W, 3).astype(np.float32)
    _check_apply(grid, guide, inp, ct, True, oracle_port, str(shape))
    ct12 = np.random.RandomState(33).randn(B, H, W, 12).astype(np.float32)
    _check_slice(grid, guide, ct12, oracle_port, str(shape))


def special_guides(gd, n, seed):
    """n guides: exact cell centres (k + 0.5) / gd and their float32 neighbours, the depth borders
    0.5 / gd and 1 - 0.5 / gd with theirs, exactly 0 and 1, and values outside [0, 1]."""
    vals = [0.0, 1.0, -0.25, 1.25]
    for k in range(gd):
        c = np.float32((k + 0.5) / gd)
        vals += [c, np.nextafter(c, np.float32(0)), np.nextafter(c, np.float32(1))]
    vals = np.array(vals, np.float32)
    rng = np.random.RandomState(seed)
    return vals[rng.randint(0, len(vals), n)]


@pytest.mark.parametrize("gd", [1, 4, 8, 16])
def test_f64_matches_port_at_cell_centres_and_borders(oracle_port, gd):
    """Exact cell centres pick cells k and k + 1 and hit SmoothedLerpWeightGrad at |d| == 1 (where
    the reference takes the gradient path); the neighbours one ulp away pick the other pair."""
    B, H, W, gh, gw = 2, 12, 17, 3, 4
    grid, _, inp = rand_case(41, B, H, W, gh, gw, gd, 3, 3, True, signed=True)
    guide = special_guides(gd, B * H * W, 42).reshape(B, H, W)
    ct = np.random.RandomState(43).randn(B, H, W, 3).astype(np.float32)
    _check_apply(grid, guide, inp, ct, True, oracle_port, f"gd={gd}")


def _interior_guides(rng, shape, gd, margin):
    """Guides whose depth coordinate gd*g stays `margin` inside (0.5, gd - 0.5)."""
    lo, hi = (0.5 + margin) / gd, (gd - 0.5 - margin) / gd
    return (lo + (hi - lo) * rng.rand(*shape)).astype(np.float32)


@pytest.mark.parametrize("shape", [(2, 23, 31, 5, 4, 8), (1, 40, 9, 3, 7, 3), (2, 6, 5, 8, 9, 4)], ids=str)
def test_f64_adjoint_identities(shape):
    """The forward is linear in the grid and in the input, so <ct, F(grid)> = <grid_vjp, grid> and
    <ct, F(input)> = <input_vjp, input>, exactly.  The grid identity holds only where the grid VJP's
    border override is inactive: for gd*g < 0.5 or > gd - 0.5 the override gives the border cell
    weight 1 where the forward sums two smoothed weights to 1 - O(1e-8 / d) (at most 1e-4 off,
    next to gd*g = 0.5 and gd - 0.5).  So the guides here keep gd*g inside (0.5, gd - 0.5)."""
    B, H, W, gh, gw, gd = shape
    rng = np.random.RandomState(51)
    guide = _interior_guides(rng, (B, H, W), gd, 0.01)
    for n_in, n_out, ho in ((3, 3, True), (2, 4, False)):
        J = n_in + ho
        grid = rng.randn(B, gh, gw, gd, n_out * J)
        inp = rng.randn(B, H, W, n_in)
        ct = rng.randn(B, H, W, n_out)
        r = slice_f64.bilateral_slice_apply_grad(grid, guide, inp, ct, ho)
        out = slice_f64.bilateral_slice_apply(grid, guide, inp, ho)
        lhs = float((ct * out).sum())
        scale = float(np.abs(ct * out).sum())
        assert abs(lhs - float((r.grid * grid).sum())) <= 1e-12 * scale, "grid adjoint"
        if not ho:   # linear (not affine) in the input only without the offset
            assert abs(lhs - float((r.input * inp).sum())) <= 1e-12 * scale, "input adjoint"
        cts = rng.randn(B, H, W, grid.shape[-1])
        s = slice_f64.bilateral_slice_grad(grid, guide, cts)
        lhs = float((cts * slice_f64.bilateral_slice(grid, guide)).sum())
        scale = float(np.abs(cts * slice_f64.bilateral_slice(grid, guide)).sum())
        assert abs(lhs - float((s.grid * grid).sum())) <= 1e-12 * scale, "slice grid adjoint"


@pytest.mark.parametrize("gd", [1, 3, 8])
def test_f64_guide_vjp_matches_central_differences(gd):
    """Each pixel's output depends on its own guide only, so one pair of forwards at guide +- h
    differentiates every pixel at once.  Guides avoid the weight's kinks: gd*g - 0.5 stays 0.05 away
    from an integer (there d = 0 for one corner and |d| = 1 for the other).  For gd = 1 the
    clamped corners' derivatives cancel to O(1e-8) and the check is against the terms' scale."""
    B, H, W, gh, gw = 2, 14, 19, 4, 5
    rng = np.random.RandomState(61)
    frac = 0.05 + 0.9 * rng.rand(B, H, W)
    guide = (rng.randint(-1, gd + 1, (B, H, W)) + 0.5 + frac) / gd       # float64, beyond [0, 1] too
    grid, _, inp = rand_case(62, B, H, W, gh, gw, gd, 3, 3, True, signed=True)
    ct = rng.randn(B, H, W, 3)
    r = slice_f64.bilateral_slice_apply_grad(grid, guide, inp, ct, True)
    h = 1e-6
    num = ((slice_f64.bilateral_slice_apply(grid, guide + h, inp, True)
            - slice_f64.bilateral_slice_apply(grid, guide - h, inp, True)) * ct).sum(-1) / (2 * h)
    scale = np.maximum(np.abs(r.guide), 1e-3 * r.guide_abs)
    err = float((np.abs(num - r.guide) / np.maximum(scale, 1e-30)).max())
    assert err <= 1e-6, f"apply guide VJP vs central differences: {err:.3e}"
    cts = rng.randn(B, H, W, grid.shape[-1])
    s = slice_f64.bilateral_slice_grad(grid, guide, cts)
    num = ((slice_f64.bilateral_slice(grid, guide + h) - slice_f64.bilateral_slice(grid, guide - h))
           * cts).sum(-1) / (2 * h)
    scale = np.maximum(np.abs(s.guide), 1e-3 * s.guide_abs)
    err = float((np.abs(num - s.guide) / np.maximum(scale, 1e-30)).max())
    assert err <= 1e-6, f"slice guide VJP vs central differences: {err:.3e}"

