"""CPU tests of the float64 align-corners resize and its scattered VJP (oracle/resize_f64.py), the
reference the resize VJP kernel is held to: the adjoint identity, central differences, torch
float64 autograd through F.interpolate(align_corners=True) where the scale is exact in binary, and
hand-computed answers, degenerate shapes included."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_np, resize_f64 as R

SHAPES = [(2, 5, 7, 3, 3, 4), (1, 33, 50, 3, 16, 25), (1, 16, 25, 3, 33, 50), (2, 8, 8, 2, 4, 4),
          (1, 1, 1, 3, 16, 24), (1, 5, 7, 3, 1, 1), (1, 1, 6, 2, 5, 3), (1, 4, 1, 1, 2, 9), (1, 2, 3, 1, 40, 70)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_adjoint_identity(shape):
    B, H, W, C, oh, ow = shape
    rng = np.random.RandomState(sum(shape))
    x, y = rng.randn(B, H, W, C), rng.randn(B, oh, ow, C)
    lhs = float((R.resize(x, oh, ow) * y).sum())
    vjp = R.resize_vjp(y, H, W)
    rhs = float((x * vjp.din).sum())
    assert abs(lhs - rhs) <= 1e-12 * max(float((np.abs(x) * vjp.din_abs).sum()), 1.0)
    assert np.all(vjp.din_abs >= np.abs(vjp.din))


@pytest.mark.parametrize("shape", SHAPES[:4], ids=lambda s: "x".join(map(str, s)))
def test_forward_is_the_models_resize(shape):
    B, H, W, C, oh, ow = shape
    x = np.random.RandomState(1).rand(B, H, W, C).astype(np.float32)
    assert np.abs(R.resize(x, oh, ow) - model_np.resize_bilinear_ac(x, oh, ow)).max() <= 1e-6


def test_central_differences():
    rng = np.random.RandomState(3)
    B, H, W, C, oh, ow = 1, 6, 9, 2, 11, 4
    x, y = rng.randn(B, H, W, C), rng.randn(B, oh, ow, C)
    din = R.resize_vjp(y, H, W).din
    h = 1e-4
    for _ in range(20):
        i = tuple(rng.randint(n) for n in x.shape)
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        fd = ((R.resize(xp, oh, ow) - R.resize(xm, oh, ow)) * y).sum() / (2 * h)
        assert abs(fd - din[i]) <= 1e-8 * max(1.0, abs(din[i]))


@pytest.mark.parametrize("hw,ohw", [((5, 5), (3, 3)), ((9, 5), (5, 3)), ((17, 9), (33, 17)), ((3, 3), (2, 2)),
                                    ((5, 9), (9, 17))])
def test_torch_float64_autograd_where_the_scale_is_exact(hw, ohw):
    rng = np.random.RandomState(hw[0] + ohw[0])
    x, y = rng.randn(2, *hw, 3), rng.randn(2, *ohw, 3)
    tx = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
    out = F.interpolate(tx, size=ohw, mode="bilinear", align_corners=True)
    assert np.abs(out.detach().permute(0, 2, 3, 1).numpy() - R.resize(x, *ohw)).max() <= 1e-13
    (out * torch.from_numpy(y).permute(0, 3, 1, 2)).sum().backward()
    want = tx.grad.permute(0, 2, 3, 1).numpy()
    assert np.abs(R.resize_vjp(y, *hw).din - want).max() <= 1e-13


def test_hand_computed_answers():
    # 2x2 -> 3x3: taps (0, 1, 0), (0, 1, 0.5), (1, 1, 0); din = Wyᵀ D Wx with Wy = Wx = [[1, 0], [.5, .5], [0, 1]]
    d = np.arange(9.0).reshape(1, 3, 3, 1)
    assert R.resize_vjp(d, 2, 2).din[0, :, :, 0].tolist() == [[3.0, 6.0], [12.0, 15.0]]
    x = np.array([1.0, 2.0, 3.0, 4.0]).reshape(1, 2, 2, 1)
    assert R.resize(x, 3, 3)[0, :, :, 0].tolist() == [[1.0, 1.5, 2.0], [2.0, 2.5, 3.0], [3.0, 3.5, 4.0]]
    # 3x3 -> 2x2: s = 2, the outputs read the corners only (the hi taps have weight 0)
    d = np.array([1.0, 2.0, 3.0, 4.0]).reshape(1, 2, 2, 1)
    assert R.resize_vjp(d, 3, 3).din[0, :, :, 0].tolist() == [[1, 0, 2], [0, 0, 0], [3, 0, 4]]
    # 1x1 -> 4x4: s = 0, lo == hi == 0 on both axes, both weights land on the one pixel
    d = np.arange(16.0).reshape(1, 4, 4, 1)
    v = R.resize_vjp(d, 1, 1)
    assert v.din.reshape(-1).tolist() == [120.0] and v.din_abs.reshape(-1).tolist() == [120.0]
    # 4x5 -> 1x1: the one output reads pixel (0, 0)
    din = R.resize_vjp(np.full((1, 1, 1, 2), 7.0), 4, 5).din
    assert din[0, 0, 0].tolist() == [7.0, 7.0] and np.count_nonzero(din) == 2
