"""CPU pins of the float64 reference for the coefficient network with its batch norm in training mode
(oracle/bn_train_f64.py): against torch float64 autograd through F.batch_norm(training=True), against
central differences, and against cases worked by hand."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from hdrnet_b200 import models
from oracle import bn_train_f64 as BN
from oracle import cnn_grad_f64 as G

TINY_BN = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4, batch_norm=True)


def bn_case(seed=0, B=3, params=TINY_BN):
    rng = np.random.RandomState(seed)
    wts = models.init_weights(params, seed=seed)
    for k in BN.variable_names(params):       # non-zero biases and betas, so that their gradients matter
        if k.endswith(("/biases", "/beta")):
            wts[k] = (0.1 * rng.randn(*wts[k].shape)).astype(np.float32)
    S = params["net_input_size"]
    return wts, rng.rand(B, S, S, 3), rng


def torch_network(wts, params, low, dtype=torch.float64, n_out=3):
    """The same network through F.batch_norm(training=True, eps=1e-3) and torch autograd, in `dtype`."""
    names = BN.variable_names(params)
    v = {k: torch.tensor(np.asarray(wts[k]), dtype=dtype, requires_grad=True) for k in names}
    bn = set(BN.batch_norm_scopes(params))
    specs = {s[0]: s for s in G.layer_specs(params)}
    x0 = torch.tensor(low, dtype=dtype, requires_grad=True)

    def layer(scope, x):
        _, kind, stride, relu, bias = specs[scope]
        z = G.conv_same(x, v[scope + "/weights"], stride) if kind == "conv" else x @ v[scope + "/weights"]
        if scope in bn:
            C = z.shape[-1]
            y = Fn.batch_norm(z.reshape(-1, C), None, None, weight=None, bias=v[scope + "/BatchNorm/beta"],
                              training=True, eps=1e-3)
            return Fn.relu(y).reshape(z.shape)
        z = z + v[scope + "/biases"] if bias else z
        return Fn.relu(z) if relu else z

    P = G.P
    n_ds = int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    x = x0
    for i in range(n_ds):
        x = layer(f"{P}/splat/conv{i + 1}", x)
    g = layer(f"{P}/global/conv2", layer(f"{P}/global/conv1", x))
    g = g.reshape(g.shape[0], -1)
    g = layer(f"{P}/global/fc3", layer(f"{P}/global/fc2", layer(f"{P}/global/fc1", g)))
    loc = layer(f"{P}/local/conv2", layer(f"{P}/local/conv1", x))
    s = f"{P}/prediction/conv1"
    grid = G.fuse_predict(loc, g, v[s + "/weights"][0, 0], v[s + "/biases"], params["luma_bins"], n_out, 4)
    return grid, v, x0


@pytest.mark.parametrize("params", [TINY_BN, dict(TINY_BN, channel_multiplier=2, luma_bins=2)], ids=["tiny", "cm2"])
def test_network_matches_torch_batch_norm_autograd(params):
    wts, low, rng = bn_case(params=params)
    net = BN.TrainingNetwork(wts, params)
    grid = net.forward(low)
    tgrid, v, x0 = torch_network(wts, params, low)
    want = tgrid.detach().numpy()
    assert np.abs(grid - want).max() <= 1e-12 * np.abs(want).max()
    dgrid = rng.randn(*grid.shape)
    got = net.backward(dgrid)
    names = BN.variable_names(params)
    tg = torch.autograd.grad(tgrid, [v[k] for k in names] + [x0], torch.from_numpy(dgrid))
    for k, t in zip(names + ["lowres_input"], tg):
        t = t.numpy()
        assert got[k].shape == t.shape, k
        assert np.abs(got[k] - t).max() <= 1e-12 * max(np.abs(t).max(), 1e-30), k


def test_network_backward_matches_central_differences():
    wts, low, rng = bn_case(seed=1, B=2)
    net = BN.TrainingNetwork(wts, TINY_BN)
    grid = net.forward(low)
    dgrid = rng.randn(*grid.shape)
    grads = net.backward(dgrid)
    names = BN.variable_names(TINY_BN)
    dirs = {k: rng.randn(*np.shape(wts[k])) for k in names}
    dirs["lowres_input"] = rng.randn(*low.shape)
    eps = 1e-6

    def f(sign):
        w = {k: np.asarray(wts[k], np.float64) + sign * eps * dirs[k] for k in names}
        return float((BN.TrainingNetwork(w, TINY_BN).forward(low + sign * eps * dirs["lowres_input"]) * dgrid).sum())

    numeric = (f(1) - f(-1)) / (2 * eps)
    analytic = sum(float((grads[k] * dirs[k]).sum()) for k in dirs)
    assert abs(numeric - analytic) <= 1e-6 * abs(analytic)
    # and one variable alone: a beta of an fc layer, a beta of a conv layer
    for k in (f"{G.P}/global/fc1/BatchNorm/beta", f"{G.P}/splat/conv2/BatchNorm/beta"):
        d = {n: np.zeros_like(np.asarray(wts[n], np.float64)) for n in names}
        d[k] = rng.randn(*d[k].shape)

        def g(sign):
            w = {n: np.asarray(wts[n], np.float64) + sign * eps * d[n] for n in names}
            return float((BN.TrainingNetwork(w, TINY_BN).forward(low) * dgrid).sum())

        num = (g(1) - g(-1)) / (2 * eps)
        assert abs(num - float((grads[k] * d[k]).sum())) <= 1e-6 * max(abs(num), 1e-3), k


def test_fc_at_batch_one_is_relu_of_beta_with_zero_dz():
    rng = np.random.RandomState(3)
    z, beta = rng.randn(1, 7), np.array([0.5, -0.25, 0.0, 1.0, -2.0, 0.125, 3.0])
    y, mean, var = BN.bn_relu(z, beta)
    assert np.array_equal(mean, z[0]) and np.array_equal(var, np.zeros(7))
    assert np.array_equal(y[0], np.maximum(beta, 0.0))
    v = BN.bn_relu_vjp(z, beta, rng.randn(1, 7))
    assert np.array_equal(v.dz, np.zeros((1, 7)))
    assert np.array_equal(v.dbeta != 0, beta > 0)


def test_two_row_channel_by_hand():
    z, beta = np.array([[1.0], [3.0]]), np.array([0.0])
    y, mean, var = BN.bn_relu(z, beta)
    s = 1.0 / np.sqrt(1.0 + 1e-3)                           # mean 2, biased variance 1
    assert mean[0] == 2.0 and var[0] == 1.0
    assert np.allclose(y[:, 0], [0.0, s], rtol=1e-15, atol=0)
    v = BN.bn_relu_vjp(z, beta, np.array([[5.0], [2.0]]))
    # dyh = [0, 2]; A = 2, B = 2 s; dz = s (dyh - A / 2 - zh B / 2) with zh = [-s, s]
    zh = np.array([-s, s])
    want = s * (np.array([0.0, 2.0]) - 1.0 - zh * s)
    assert v.dbeta[0] == 2.0 and np.allclose(v.b[0], 2 * s, rtol=1e-15)
    assert np.allclose(v.dz[:, 0], want, rtol=1e-14, atol=1e-15)


def test_moving_average_update_by_hand():
    # N = 5: the batch variance is Bessel-corrected by 5 / 4
    z = np.array([[1.0], [2.0], [3.0], [4.0], [10.0]])
    _, mean, var = BN.bn_relu(z, np.zeros(1))
    assert mean[0] == 4.0 and var[0] == 10.0
    mm, mv = BN.moving_update(np.array([0.0]), np.array([1.0]), mean, var, 5)
    assert np.isclose(mm[0], 0.001 * 4.0, rtol=1e-12) and np.isclose(mv[0], 1.0 - 0.001 * (1.0 - 12.5), rtol=1e-12)
    # N = 1 feeds a variance of 0
    mm, mv = BN.moving_update(np.array([2.0]), np.array([3.0]), np.array([7.0]), np.array([0.0]), 1)
    assert np.isclose(mm[0], 2.0 - 0.001 * (2.0 - 7.0), rtol=1e-12) and np.isclose(mv[0], 3.0 - 0.001 * 3.0, rtol=1e-12)


def test_the_plain_network_keeps_refusing_batch_norm():
    with pytest.raises(NotImplementedError):
        G.Network({}, TINY_BN)
    with pytest.raises(ValueError):
        BN.TrainingNetwork({}, dict(TINY_BN, batch_norm=False))
