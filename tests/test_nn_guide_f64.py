"""CPU tests of the float64 training-mode pointwise-NN guide (tests/nn_guide_f64.py): its forward, its
moving-average update and its VJP against torch float64 autograd through F.conv2d -> F.batch_norm
(training=True) -> relu -> conv -> sigmoid, against central differences, and against hand-computed
answers at relu ties and at N = 1 and N = 5."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import nn_guide_f64 as O

G = "inference/guide"


def weights(rng, feats=16):
    return {f"{G}/conv1/weights": rng.randn(1, 1, 3, feats) * 0.8,
            f"{G}/conv1/BatchNorm/beta": rng.randn(feats) * 0.5,
            f"{G}/conv2/weights": rng.randn(1, 1, feats, 1) * 0.5,
            f"{G}/conv2/biases": rng.randn(1) * 0.1}


def torch_guide(x, v):
    """x [B, H, W, 3] float64; the reference's training graph in torch float64."""
    F = v["conv1/BatchNorm/beta"].shape[0]
    z = Fn.conv2d(x.permute(0, 3, 1, 2), v["conv1/weights"].reshape(3, F).t().reshape(F, 3, 1, 1))
    y = Fn.batch_norm(z, None, None, weight=None, bias=v["conv1/BatchNorm/beta"], training=True, eps=1e-3)
    o = Fn.conv2d(torch.relu(y), v["conv2/weights"].reshape(1, F, 1, 1), v["conv2/biases"])
    return torch.sigmoid(o)[:, 0]


@pytest.mark.parametrize("feats", [16, 7])
def test_forward_and_vjp_match_torch_float64_autograd(feats):
    rng = np.random.RandomState(feats)
    w = weights(rng, feats)
    x = rng.rand(3, 11, 13, 3) * 1.2 - 0.1
    g = rng.randn(3, 11, 13)
    v = {n: torch.tensor(np.asarray(w[f"{G}/{n}"], np.float64), requires_grad=True) for n in O.NAMES}
    xt = torch.tensor(x, requires_grad=True)
    out = torch_guide(xt, v)
    (out * torch.tensor(g)).sum().backward()
    assert np.abs(O.guide(x, w) - out.detach().numpy()).max() <= 1e-12
    got = O.vjp(x, g, w)
    assert np.abs(got.dinput - xt.grad.numpy()).max() <= 1e-12 * np.abs(xt.grad.numpy()).max()
    for n in O.NAMES:
        ref = v[n].grad.numpy()
        assert got.dparams[n].shape == ref.shape, n
        assert np.abs(got.dparams[n] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30), n
        assert np.all(got.dparams_abs[n] >= np.abs(got.dparams[n]) * (1 - 1e-12)), n


def test_batch_stats_match_torch_batch_norm_and_the_input_moments():
    rng = np.random.RandomState(3)
    w = weights(rng)
    x = rng.rand(2, 9, 5, 3)
    mu, var = O.batch_stats(x, w)
    xs = x.reshape(-1, 3)
    w1 = w[f"{G}/conv1/weights"].reshape(3, -1)
    C = np.cov(xs.T, bias=True)
    assert np.allclose(mu, xs.mean(0) @ w1, rtol=1e-13, atol=1e-15)
    assert np.allclose(var, np.einsum("if,ij,jf->f", w1, C, w1), rtol=1e-12, atol=1e-15)


def test_vjp_matches_central_differences_away_from_kinks():
    rng = np.random.RandomState(2)
    w = weights(rng, 6)
    x = rng.rand(60, 3)
    g = rng.randn(60)
    got = O.vjp(x, g, w)
    h = 1e-6

    def loss(wts, xx=x):
        return float((O.guide(xx, wts) * g).sum())

    for n in O.NAMES:
        base = np.asarray(w[f"{G}/{n}"], np.float64)
        num = np.empty(base.size)
        for i in range(base.size):
            vals = []
            for sgn in (1, -1):
                pert = base.copy().reshape(-1)
                pert[i] += sgn * h
                vals.append(loss(dict(w, **{f"{G}/{n}": pert.reshape(base.shape)})))
            num[i] = (vals[0] - vals[1]) / (2 * h)
        ref = got.dparams[n].reshape(-1)
        assert np.abs(num - ref).max() <= 1e-6 * max(np.abs(ref).max(), 1.0), n
    num = np.empty_like(x)
    for p in range(x.shape[0]):
        for i in range(3):
            xp, xm = x.copy(), x.copy()
            xp[p, i] += h
            xm[p, i] -= h
            num[p, i] = (loss(w, xp) - loss(w, xm)) / (2 * h)
    assert np.abs(num - got.dinput).max() <= 1e-6 * max(np.abs(got.dinput).max(), 1.0)


def test_known_answer_relu_tie_passes_no_gradient():
    """One feature, beta = 0: x-hat of the pixel at the batch mean is exactly 0, so y = 0 there.  TF's
    ReluGrad (y > 0) gives that pixel no dy; the other two pixels (y = +-sqrt(3/2) / sqrt(1 + 1.5e-3))
    are one active, one not."""
    w = {f"{G}/conv1/weights": np.array([1.0, 0.0, 0.0]).reshape(1, 1, 3, 1),
         f"{G}/conv1/BatchNorm/beta": np.zeros(1),
         f"{G}/conv2/weights": np.array([2.0]).reshape(1, 1, 1, 1),
         f"{G}/conv2/biases": np.zeros(1)}
    x = np.array([[0.0, 0.3, 0.1], [1.0, 0.2, 0.5], [2.0, 0.9, 0.4]])
    g = np.array([1.0, 1.0, 1.0])
    mu, var = O.batch_stats(x, w)
    assert mu[0] == 1.0 and var[0] == 2.0 / 3.0
    s = 1.0 / np.sqrt(2.0 / 3.0 + 1e-3)
    y = (x[:, 0] - 1.0) * s
    assert y[1] == 0.0
    got = O.vjp(x, g, w)
    sg = 1.0 / (1.0 + np.exp(-2.0 * np.maximum(y, 0.0)))
    do = sg * (1 - sg)
    dy = np.array([0.0, 0.0, do[2] * 2.0])                 # only pixel 2 is active; pixel 1 sits on the tie
    assert got.dparams["conv1/BatchNorm/beta"][0] == pytest.approx(dy.sum(), rel=1e-15)
    assert got.dparams["conv2/biases"][0] == pytest.approx(do.sum(), rel=1e-15)
    assert got.dparams["conv2/weights"].reshape(-1)[0] == pytest.approx(do[2] * y[2], rel=1e-14)
    A, B = dy.sum(), (dy * y).sum()
    dz = s * (dy - A / 3 - y * B / 3)
    assert np.allclose(got.dinput[:, 0], dz, rtol=0, atol=1e-15)
    assert not got.dinput[:, 1:].any()
    assert np.allclose(got.dparams["conv1/weights"].reshape(3), x.T @ dz, rtol=0, atol=1e-15)


def test_moving_averages_at_n5_use_the_bessel_corrected_variance():
    rng = np.random.RandomState(5)
    w = weights(rng, 4)
    x = rng.rand(1, 1, 5, 3)
    mu, var = O.batch_stats(x, w)
    mm, mv = O.moving_average_update(np.zeros(4), np.ones(4), x, w)
    assert np.allclose(mm, 1e-3 * mu, rtol=1e-12)
    assert np.allclose(mv, 1.0 - 1e-3 * (1.0 - var * 5.0 / 4.0), rtol=1e-12)
    # the biased variance would be visibly different at N = 5
    assert np.abs(mv - (1.0 - 1e-3 * (1.0 - var))).min() > 1e-5 * var.min()


def test_moving_averages_at_n1_are_defined():
    rng = np.random.RandomState(6)
    w = weights(rng, 4)
    x = rng.rand(1, 1, 1, 3)
    mu, var = O.batch_stats(x, w)
    assert not var.any()
    with np.errstate(all="raise"):
        mm, mv = O.moving_average_update(np.full(4, 0.5), np.full(4, 2.0), x, w)
    assert np.allclose(mm, 0.5 - 1e-3 * (0.5 - mu), rtol=1e-12)
    assert np.allclose(mv, 2.0 - 1e-3 * 2.0, rtol=1e-12)


def test_flat_order_is_the_librarys():
    rng = np.random.RandomState(7)
    w = weights(rng, 5)
    r = O.vjp(rng.rand(10, 3), rng.randn(10), w)
    f = O.flat(r.dparams)
    assert f.shape == (26,)
    assert np.array_equal(f[:15], r.dparams["conv1/weights"].reshape(-1))
    assert np.array_equal(f[15:20], r.dparams["conv1/BatchNorm/beta"])
    assert f[25] == r.dparams["conv2/biases"][0]
