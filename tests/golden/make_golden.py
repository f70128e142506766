"""Generate the golden fixtures in tests/golden/ from the REFERENCE itself.

Needs a google/hdrnet checkout and its compiled loops (oracle/_ref, built by oracle.build()):
    HDRNET_REFERENCE=<checkout> python tests/golden/make_golden.py [vjp | live]

Outputs are produced by the reference's own jax/bilateral_slice.py (:299-380), imported
unmodified under the numpy stand-in for jax (oracle/jax_shim.py), and -- for slice-apply --
the reference's ``apply`` semantics (hdrnet/layers.py:153-198).  Inputs follow the
reference's tests:

  ops_test_extents   hdrnet/hdrnet_ops_test.py:91-113, :267-292 -- np.random.seed(1234),
                     np.random.rand, B=3 H=30 W=25 gh=16 gw=12 gd=8, n_in=3, n_out=3
  jax_tf2_extents    hdrnet/hdrnet_ops_jax_tf2_test.py:28-34 grid 16x12x8x2 (guide reduced
                     from 640x480x4 to 2x96x128 to keep the fixture small)
  interpolate_kat    hdrnet/test/ops_test.py:61-86 (grid value = depth index)
  edge_cases         guide exactly 0 / 1 / out of [0,1], 1-pixel-wide image, gd = 1
  vjp_*              the reference's own VJPs of the slice (jax/bilateral_slice.py:26-108, :257-295) at
                     the extents of its gradient tests (hdrnet_ops_test.py:91-100, :185-195) and on a
                     grid coarser / finer than the image; `python make_golden.py vjp` writes only these
  live_reference     what tests/test_oracle.py compares the port with when the reference is at hand:
                     the JAX file's outputs on a signed case, its grid VJP at an exact cell centre,
                     and SHA-256 digests of the compiled C++ loops' outputs (the port must be
                     bit-exact, so a digest is the whole comparison); `python make_golden.py live`
Each .npz stores inputs, outputs and the reference's cell indices.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.normpath(os.path.join(HERE, "..", "..")))
sys.path.insert(0, os.path.normpath(os.path.join(HERE, "..")))

from oracle import jax_shim  # noqa: E402


def save(name, **arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB", {k: v.shape for k, v in arrays.items()})


def case(grid, guide, inp=None):
    gh, gw, gd = grid.shape[1:4]
    d = dict(grid=grid, guide=guide,
             slice=jax_shim.bilateral_slice(grid, guide),
             indices=jax_shim.slice_indices(guide, gh, gw, gd))
    if inp is not None:
        d["input"] = inp
        n_in = inp.shape[-1]
        if grid.shape[-1] % (n_in + 1) == 0:
            d["apply_offset"] = jax_shim.bilateral_slice_apply(grid, guide, inp, True)
        if grid.shape[-1] % n_in == 0:
            d["apply_nooffset"] = jax_shim.bilateral_slice_apply(grid, guide, inp, False)
    return d


def main():
    # hdrnet_ops_test.py:91-113 / :267-292
    np.random.seed(1234)
    B, H, W, gh, gw, gd, n_in, n_out = 3, 30, 25, 16, 12, 8, 3, 3
    grid = np.random.rand(B, gh, gw, gd, (n_in + 1) * n_out).astype(np.float32)
    guide = np.random.rand(B, H, W).astype(np.float32)
    inp = np.random.rand(B, H, W, n_in).astype(np.float32)
    save("ops_test_extents", **case(grid, guide, inp))

    # hdrnet_ops_jax_tf2_test.py:28-34 (reduced spatial size), unseeded there -> seeded here
    rng = np.random.RandomState(20240)
    grid = rng.rand(2, 16, 12, 8, 2).astype(np.float32)
    guide = rng.rand(2, 96, 128).astype(np.float32)
    save("jax_tf2_extents", **case(grid, guide))

    # hdrnet/test/ops_test.py:61-86: expected output == val (tolerance 5e-4 there)
    for val in range(3):
        grid = np.zeros((3, 3, 4, 3, 1), np.float32)
        grid[:, :, :, 1] = 1.0
        grid[:, :, :, 2] = 2.0
        guide = np.full((3, 10, 9), (val + 0.5) / 3.0, np.float32)
        save(f"interpolate_kat_{val}", **case(grid, guide))

    # Edge cases: guide on / beyond the range ends, W = 4 strip, gd = 1, non-square grid.
    rng = np.random.RandomState(7)
    grid = rng.randn(2, 5, 3, 4, 12).astype(np.float32)
    guide = rng.rand(2, 12, 16).astype(np.float32)
    guide[0, 0, :4] = [0.0, 1.0, -0.25, 1.5]
    guide[1, 3, :4] = [0.125, 0.5, 0.875, 1.0 - 2.0 ** -24]
    inp = rng.randn(2, 12, 16, 3).astype(np.float32)
    save("edge_guides", **case(grid, guide, inp))

    grid = rng.rand(1, 2, 2, 1, 12).astype(np.float32)  # gd = 1: both depth corners clamp to 0
    guide = rng.rand(1, 7, 4).astype(np.float32)
    inp = rng.rand(1, 7, 4, 3).astype(np.float32)
    save("edge_gd1", **case(grid, guide, inp))

    # Wide enough for the TMA row kernel (W % 4 == 0, W >= 128), ragged last segment; 4 rows keep
    # the fixture under 1 MB.
    grid = rng.rand(2, 4, 6, 8, 12).astype(np.float32)
    guide = rng.rand(2, 4, 1100).astype(np.float32)
    inp = rng.rand(2, 4, 1100, 3).astype(np.float32)
    save("wide_rows", **case(grid, guide, inp))


def main_vjp():
    # (B, H, W, gh, gw, gd, gc): default test extents; hdrnet_ops_test.py:185-195; a coarse grid; an
    # image narrower than the grid (cells without a pixel centre).  Guides are generic random values:
    # where guide * gd - 0.5 is EXACTLY an integer the JAX helpers take floor == ceil as two corners
    # (the grid VJP counts the pixel twice, the guide VJP returns 0) while the C++ op -- which the
    # library and the oracle port follow -- uses cells k and k + 1; tests/test_oracle.py pins that corner.
    for k, (B, H, W, gh, gw, gd, gc) in enumerate([(3, 30, 25, 16, 12, 8, 12), (3, 8, 5, 6, 3, 7, 4),
                                                   (2, 21, 36, 5, 4, 6, 2), (1, 9, 7, 3, 12, 9, 5)]):
        rng = np.random.RandomState(900 + k)
        grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
        guide = rng.rand(B, H, W).astype(np.float32)
        ct = rng.randn(B, H, W, gc).astype(np.float32)
        gv, uv = jax_shim.bilateral_slice_vjp(grid, guide, ct)
        save(f"vjp_{k}", grid=grid, guide=guide, codomain_tangent=ct, grid_vjp=gv, guide_vjp=uv)


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main_live():
    """Inputs are regenerated by the tests from tests/util.py rand_case; only outputs are stored."""
    import oracle
    from util import rand_case
    grid, guide, inp = rand_case(11, 2, 40, 36, 8, 6, 5, signed=True)
    d = dict(jax_slice=jax_shim.bilateral_slice(grid, guide),
             jax_apply_offset=jax_shim.bilateral_slice_apply(grid, guide, inp, True),
             jax_indices=jax_shim.slice_indices(guide, 8, 6, 5))
    # grid VJP where guide * gd - 0.5 is an exact integer (tests/test_oracle.py, cell-centre test)
    gh, gw, gd, gc, h, w = 3, 2, 4, 1, 6, 5
    rng = np.random.RandomState(11)
    g = rng.rand(1, h, w).astype(np.float32)
    g[0, 2, 3] = 1.5 / gd
    ct = rng.randn(1, h, w, gc).astype(np.float32)
    d["jax_cell_centre_grid_vjp"], _ = jax_shim.bilateral_slice_vjp(np.zeros((1, gh, gw, gd, gc), np.float32), g, ct)
    ref = oracle.ref()
    for k, shape in enumerate([(3, 30, 25, 16, 12, 8), (2, 64, 48, 3, 5, 4), (1, 8, 5, 6, 3, 7)]):
        grid, guide, inp = rand_case(99, *shape, signed=True)
        digests = [sha256(ref.bilateral_slice_apply(grid, guide, inp, ho))
                   for ho in (True, False) if grid.shape[-1] % (3 + ho) == 0]
        digests.append(sha256(ref.bilateral_slice(grid, guide)))
        d[f"ref_forward_sha256_{k}"] = np.array(digests)
    B, H, W, gh, gw, gd, n_in, n_out = 3, 8, 5, 6, 3, 7, 3, 4
    grid, guide, inp = rand_case(5, B, H, W, gh, gw, gd, n_in, n_out, True)
    rng = np.random.RandomState(6)
    ct = rng.rand(B, H, W, n_out).astype(np.float32)
    digests = [sha256(a) for a in ref.bilateral_slice_apply_grad(grid, guide, inp, ct, True)]
    ct = rng.rand(B, H, W, grid.shape[-1]).astype(np.float32)
    digests += [sha256(a) for a in ref.bilateral_slice_grad(grid, guide, ct)]
    d["ref_vjp_sha256"] = np.array(digests)
    save("live_reference", **d)


if __name__ == "__main__":
    if sys.argv[1:] == ["live"]:
        main_live()
    else:
        if sys.argv[1:] != ["vjp"]:
            main()
        main_vjp()
