"""GPU tests of the VJP kernels (SURVEY 8f rank 1) against the compiled reference loops
(oracle/_ref: hdrnet/ops/bilateral_slice_apply.cc:84-259, bilateral_slice.cc:72-168) or their
bit-exact C restatement, plus the reference's own numeric-vs-analytic criterion through
torch.autograd (hdrnet/hdrnet_ops_test.py:173-180, :361-408)."""
import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import hdrnet_ops
from util import APPLY_CASES, SLICE_CASES, assert_parity, rand_case

pytestmark = pytest.mark.gpu


def cuda(a, grad=False):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t.requires_grad_(grad)



@pytest.mark.parametrize("case", APPLY_CASES, ids=str)
def test_slice_apply_vjps_match_reference(case):
    B, H, W, gh, gw, gd, n_in, n_out, ho = case
    grid, guide, inp = rand_case(5, B, H, W, gh, gw, gd, n_in, n_out, ho, signed=True)
    rng = np.random.RandomState(6)
    ct = rng.randn(B, H, W, n_out).astype(np.float32)
    want = oracle.port().bilateral_slice_apply_grad(grid, guide, inp, ct, ho)
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    out = hdrnet_ops.bilateral_slice_apply(g, u, i, ho)
    out.backward(cuda(ct))
    for got, ref, name in zip((g.grad, u.grad, i.grad), want, ("grid", "guide", "input")):
        if name == "guide" and gd == 1:
            # Degenerate: both depth corners clamp to cell 0, the two derivative terms cancel
            # and the reference's own result is float32 rounding noise (|vjp| ~ 1e-7 of the
            # terms).  Bound it against the scale of the TERMS instead of the cancelled sum.
            scale = float(np.abs(grid).max() * np.abs(ct).max() * np.abs(inp).max() * gd * 4)
            assert np.abs(got.cpu().numpy() - ref).max() <= 1e-6 * scale
            continue
        assert_parity(got.cpu().numpy(), ref, rtol=2e-5, what=f"{case} {name} VJP")


@pytest.mark.parametrize("case", SLICE_CASES, ids=str)
def test_slice_vjps_match_reference(case):
    B, H, W, gh, gw, gd, gc = case
    rng = np.random.RandomState(7)
    grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
    guide = rng.rand(B, H, W).astype(np.float32)
    ct = rng.randn(B, H, W, gc).astype(np.float32)
    want = oracle.port().bilateral_slice_grad(grid, guide, ct)
    g, u = cuda(grid, True), cuda(guide, True)
    hdrnet_ops.bilateral_slice(g, u).backward(cuda(ct))
    assert_parity(g.grad.cpu().numpy(), want[0], rtol=2e-5, what="grid VJP")
    assert_parity(u.grad.cpu().numpy(), want[1], rtol=2e-5, what="guide VJP")


@pytest.mark.parametrize("name", ["vjp_0", "vjp_2"])
def test_slice_vjps_match_reference_jax_golden(name):
    """tests/golden/vjp_*.npz: the reference's own JAX VJP functions (jax/bilateral_slice.py:26-108,
    :257-295; tests/golden/make_golden.py) at the reference's default test extents and on a coarse
    grid -- the same bar as against the C++ loops above."""
    from util import load_golden
    z = load_golden(name)
    g, u = cuda(z["grid"], True), cuda(z["guide"], True)
    hdrnet_ops.bilateral_slice(g, u).backward(cuda(z["codomain_tangent"]))
    # global bar only: the per-element statistic is asserted against the C++ loops above
    assert_parity(g.grad.cpu().numpy(), z["grid_vjp"], rtol=2e-5, what=f"{name} grid VJP", elem_rtol=None)
    assert_parity(u.grad.cpu().numpy(), z["guide_vjp"], rtol=2e-5, what=f"{name} guide VJP", elem_rtol=None)


def test_grad_shapes_follow_reference_contract():
    """hdrnet_ops_test.py:125-135, :304-315 (test_grad_shape)."""
    grid, guide, inp = rand_case(1, 3, 30, 25, 16, 12, 8)
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    hdrnet_ops.bilateral_slice_apply(g, u, i, True).sum().backward()
    assert g.grad.shape == g.shape and u.grad.shape == u.shape and i.grad.shape == i.shape


def test_analytic_vs_numeric_gradient_error():
    """The reference's criterion (compute_gradient_error <= 1e-2, hdrnet_ops_test.py:361-363):
    central differences of the CUDA forward vs the CUDA VJPs, for grid and input (the forward is
    piecewise linear in both, so float32 differences are accurate)."""
    grid, guide, inp = rand_case(3, 1, 12, 10, 3, 3, 4, 3, 3, True)
    guide = (0.1 + 0.8 * guide).astype(np.float32)
    rng = np.random.RandomState(4)
    ct = rng.rand(1, 12, 10, 3).astype(np.float32)
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    hdrnet_ops.bilateral_slice_apply(g, u, i, True).backward(cuda(ct))

    def loss(gg, ii):
        with torch.no_grad():
            o = hdrnet_ops.bilateral_slice_apply(cuda(gg), cuda(guide), cuda(ii), True)
        return float((o.double() * cuda(ct).double()).sum())

    eps = 1e-2
    for arr, grad, which in ((grid, g.grad, 0), (inp, i.grad, 1)):
        gflat = grad.cpu().numpy().reshape(-1)
        for k in rng.choice(arr.size, 10, replace=False):
            hi, lo = arr.copy(), arr.copy()
            hi.reshape(-1)[k] += eps
            lo.reshape(-1)[k] -= eps
            num = (loss(hi, inp) - loss(lo, inp)) / (2 * eps) if which == 0 else \
                  (loss(grid, hi) - loss(grid, lo)) / (2 * eps)
            assert abs(num - gflat[k]) <= 1e-2 * max(1.0, abs(num))


def test_backward_is_deterministic():
    grid, guide, inp = rand_case(9, 2, 64, 96, 8, 8, 8)
    ct = np.random.RandomState(1).rand(2, 64, 96, 3).astype(np.float32)
    grads = []
    for _ in range(2):
        g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
        hdrnet_ops.bilateral_slice_apply(g, u, i, True).backward(cuda(ct))
        grads.append((g.grad.clone(), u.grad.clone(), i.grad.clone()))
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_grid_vjp_is_zero_when_there_are_no_pixels():
    """ADVICE r01: B > 0 with H == 0 (or W == 0): no pixel contributes, the grid VJP is a tensor of
    zeros (the reference's kernels write 0 for every cell) -- not uninitialised memory."""
    for H, W in ((0, 8), (8, 0)):
        grid = torch.randn(2, 4, 4, 8, 12, device="cuda", requires_grad=True)
        guide = torch.rand(2, H, W, device="cuda", requires_grad=True)
        inp = torch.randn(2, H, W, 3, device="cuda", requires_grad=True)
        out = hdrnet_ops.bilateral_slice_apply(grid, guide, inp, True)
        assert out.shape == (2, H, W, 3)
        out.sum().backward()
        assert grid.grad is not None and not grid.grad.any()
        g2 = torch.randn(2, 4, 4, 8, 12, device="cuda", requires_grad=True)
        hdrnet_ops.bilateral_slice(g2, guide.detach()).sum().backward()
        assert not g2.grad.any()


@pytest.mark.parametrize("name", ["grid", "guide", "both"])
def test_sgd_convergence_bounds_of_the_reference_tests(name):
    """hdrnet/test/ops_test.py:189-322 (test_grid_optimize, test_guide_optimize, test_optimize_both):
    plain gradient descent on sum((target - slice(grid, guide))^2) through the CUDA forward and VJP
    kernels (torch.autograd) reaches the loss bounds the reference asserts.  tests/test_oracle.py runs
    the same cases through the reference's own loops."""
    from util import sgd_case
    c = sgd_case(name)
    grid = cuda(c["grid"], "grid" in c["trained"])
    v = cuda(c["guide"], "guide" in c["trained"])
    target = cuda(c["target"])
    params = [t for t in (grid, v) if t.requires_grad]

    def forward():
        return hdrnet_ops.bilateral_slice(grid, torch.sigmoid(v) if c["sigmoid"] else v)

    for _ in range(c["steps"]):
        loss = (target - forward()).square().sum()
        grads = torch.autograd.grad(loss, params)
        with torch.no_grad():
            for p, g in zip(params, grads):
                p -= c["lr"] * g
    with torch.no_grad():
        final = float((target - forward()).square().sum())
    assert final < c["bound"], f"{name}: final loss {final:.3e} >= {c['bound']:.1e}"


# ---- the autograd boundary ------------------------------------------------------------------
def _apply_grads(grid, guide, inp, ct, wants=(True, True, True)):
    g, u, i = cuda(grid, wants[0]), cuda(guide, wants[1]), cuda(inp, wants[2])
    hdrnet_ops.bilateral_slice_apply(g, u, i, True).backward(ct if torch.is_tensor(ct) else cuda(ct))
    torch.cuda.synchronize()
    return [None if t.grad is None else t.grad.clone() for t in (g, u, i)]


def _boundary_case(seed=3, B=2, H=40, W=56):
    grid, guide, inp = rand_case(seed, B, H, W, 5, 7, 8, 3, 3, True, signed=True)
    ct = np.random.RandomState(seed + 1).randn(B, H, W, 3).astype(np.float32)
    return grid, guide, inp, ct


def _equal(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


def test_non_contiguous_upstream_gradients():
    """A channel-reordered or transposed output hands backward a non-contiguous gradient; it must
    give what its contiguous copy gives, bitwise."""
    grid, guide, inp, ct = _boundary_case()
    want = _apply_grads(grid, guide, inp, ct)
    # the gradient arrives as a transposed view of a contiguous [B, W, H, C] tensor
    ct_t = cuda(ct).transpose(1, 2).contiguous().transpose(1, 2)
    assert not ct_t.is_contiguous()
    assert _equal(_apply_grads(grid, guide, inp, ct_t), want)
    # through an index and a transpose in the graph
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    out = hdrnet_ops.bilateral_slice_apply(g, u, i, True)
    (out[..., [2, 1, 0]].transpose(1, 2) * cuda(ct[..., [2, 1, 0]]).transpose(1, 2)).sum().backward()
    torch.cuda.synchronize()
    assert _equal([g.grad, u.grad, i.grad], want)


def test_only_some_inputs_require_grad():
    grid, guide, inp, ct = _boundary_case()
    want = _apply_grads(grid, guide, inp, ct)
    for wants in ((False, True, False), (True, False, False), (False, False, True)):
        got = _apply_grads(grid, guide, inp, ct, wants)
        assert _equal(got, [w if f else None for w, f in zip(want, wants)]), wants
    # bilateral_slice with only the guide, then only the grid
    sct = np.random.RandomState(9).randn(*guide.shape, grid.shape[-1]).astype(np.float32)
    ref = oracle.port().bilateral_slice_grad(grid, guide, sct)
    for k in (0, 1):
        g, u = cuda(grid, k == 0), cuda(guide, k == 1)
        hdrnet_ops.bilateral_slice(g, u).backward(cuda(sct))
        assert (g.grad is None) == (k == 1) and (u.grad is None) == (k == 0)
        assert_parity((g.grad if k == 0 else u.grad).cpu().numpy(), ref[k], rtol=2e-5,
                      what=f"slice VJP {k}", elem_rtol=None)


def test_gradients_accumulate_over_two_backward_calls():
    grid, guide, inp, ct = _boundary_case()
    want = _apply_grads(grid, guide, inp, ct)
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    for _ in range(2):
        hdrnet_ops.bilateral_slice_apply(g, u, i, True).backward(cuda(ct))
    torch.cuda.synchronize()
    assert _equal([g.grad, u.grad, i.grad], [2 * w for w in want])


def test_backward_on_a_side_stream():
    """The VJPs launch on the current stream: forward and backward on a side stream, queued behind
    other work there, give the default stream's gradients, bitwise."""
    grid, guide, inp, ct = _boundary_case()
    want = _apply_grads(grid, guide, inp, ct)
    s = torch.cuda.Stream()
    busy = torch.randn(4096, 4096, device="cuda")
    g, u, i = cuda(grid, True), cuda(guide, True), cuda(inp, True)
    c = cuda(ct)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            busy = busy @ busy.T / 4096.0
        hdrnet_ops.bilateral_slice_apply(g, u, i, True).backward(c)
    torch.cuda.synchronize()
    assert _equal([g.grad, u.grad, i.grad], want)


def test_six_d_grids_through_layers():
    """layers.bilateral_slice_apply takes [B,gh,gw,gd,n_out,n_in+1] (output-major) and
    layers.bilateral_slice [B,gh,gw,gd,n_out,n_in] (packed input-major): their gradients are the
    5-D op's, moved back through the same packing."""
    from hdrnet_b200 import layers
    grid, guide, inp, ct = _boundary_case()
    B, gh, gw, gd, gc = grid.shape
    want = _apply_grads(grid, guide, inp, ct)
    g6 = cuda(grid.reshape(B, gh, gw, gd, 3, 4), True)
    u, i = cuda(guide, True), cuda(inp, True)
    layers.bilateral_slice_apply(g6, u, i, True).backward(cuda(ct))
    torch.cuda.synchronize()
    assert _equal([g6.grad.reshape(grid.shape), u.grad, i.grad], want)

    # slice: 6-D channel (i, j) is 5-D channel j * n_out + i
    grid6 = np.ascontiguousarray(grid.reshape(B, gh, gw, gd, 4, 3).transpose(0, 1, 2, 3, 5, 4))  # n_out=3, n_in=4
    sct6 = np.random.RandomState(5).randn(*guide.shape, 3, 4).astype(np.float32)
    grid5 = grid6.transpose(0, 1, 2, 3, 5, 4).reshape(B, gh, gw, gd, 12)
    sct5 = sct6.transpose(0, 1, 2, 4, 3).reshape(*guide.shape, 12)
    g5, u5 = cuda(grid5, True), cuda(guide, True)
    hdrnet_ops.bilateral_slice(g5, u5).backward(cuda(sct5))
    g6, u6 = cuda(grid6, True), cuda(guide, True)
    layers.bilateral_slice(g6, u6).backward(cuda(sct6))
    torch.cuda.synchronize()
    back = g5.grad.reshape(B, gh, gw, gd, 4, 3).permute(0, 1, 2, 3, 5, 4)
    assert torch.equal(g6.grad, back) and torch.equal(u6.grad, u5.grad)


def test_permuting_the_batch_permutes_every_gradient():
    grid, guide, inp, ct = _boundary_case(B=4)
    perm = np.array([2, 0, 3, 1])
    want = _apply_grads(grid, guide, inp, ct)
    got = _apply_grads(grid[perm], guide[perm], inp[perm], ct[perm])
    idx = torch.from_numpy(perm).cuda()
    assert _equal(got, [w[idx] for w in want])
