"""CPU pins of the float64 gradient reference for the coefficient network (oracle/cnn_grad_f64.py):
central differences in float64, chaining its per-layer VJPs into its whole-network backward, and its
forward against oracle/model_torch.coefficients."""
import numpy as np
import pytest

from hdrnet_b200 import models
from oracle import cnn_grad_f64 as G
from oracle import model_torch

TINY = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)


def tiny_case(seed=0, B=2, params=TINY):
    rng = np.random.RandomState(seed)
    wts = models.init_weights(params, seed=seed)
    for k in G.variable_names(params):        # non-zero biases, so that their gradients matter
        if k.endswith("/biases"):
            wts[k] = (0.05 * rng.randn(*wts[k].shape)).astype(np.float32)
    S = params["net_input_size"]
    low = rng.rand(B, S, S, 3).astype(np.float32)
    return wts, low, rng


def test_network_backward_matches_central_differences():
    wts, low, rng = tiny_case()
    net = G.Network(wts, TINY)
    grid = net.forward(low)
    dgrid = rng.randn(*grid.shape)
    grads = net.backward(dgrid)
    names = G.variable_names(TINY)
    dirs = {k: rng.randn(*np.shape(wts[k])) for k in names}
    dirs["lowres_input"] = rng.randn(*low.shape)
    eps = 1e-6

    def f(sign):
        w = {k: np.asarray(wts[k], np.float64) + sign * eps * dirs[k] for k in names}
        n = G.Network(w, TINY)
        return float((n.forward(low.astype(np.float64) + sign * eps * dirs["lowres_input"]) * dgrid).sum())

    fd = (f(1) - f(-1)) / (2 * eps)
    an = sum(float((grads[k] * dirs[k]).sum()) for k in dirs)
    assert abs(fd - an) <= 1e-6 * abs(an), (fd, an)
    # and per variable: each gradient alone against its own directional difference
    for k in names[::3] + ["lowres_input"]:
        def g(sign):
            w = {n: np.asarray(wts[n], np.float64) for n in names}
            x = low.astype(np.float64)
            if k == "lowres_input":
                x = x + sign * eps * dirs[k]
            else:
                w[k] = w[k] + sign * eps * dirs[k]
            return float((G.Network(w, TINY).forward(x) * dgrid).sum())
        fd = (g(1) - g(-1)) / (2 * eps)
        an = float((grads[k] * dirs[k]).sum())
        assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-3), (k, fd, an)


@pytest.mark.parametrize("shape", [(2, 9, 7, 3, 5, 3, 2), (1, 8, 10, 4, 6, 3, 1), (2, 7, 6, 5, 4, 1, 2),
                                   (1, 6, 5, 2, 3, 1, 1)])
def test_conv_vjp_matches_central_differences(shape):
    """Odd and even extents at stride 1 and 2, k = 3 and 1: the asymmetric SAME geometry."""
    B, H, W, cin, cout, k, s = shape
    rng = np.random.RandomState(1)
    x, w, dy = rng.randn(B, H, W, cin), rng.randn(k, k, cin, cout), None
    out = G.conv_same(G._t(x), G._t(w), s).numpy()
    dy = rng.randn(*out.shape)
    v = G.conv_vjp(x, w, out, dy, s, relu=False)
    vx, vw = rng.randn(*x.shape), rng.randn(*w.shape)
    eps = 1e-6

    def f(sign):
        return float((G.conv_same(G._t(x + sign * eps * vx), G._t(w + sign * eps * vw), s).numpy() * dy).sum())

    fd = (f(1) - f(-1)) / (2 * eps)
    an = float((v.dx * vx).sum() + (v.dw * vw).sum())
    assert abs(fd - an) <= 1e-7 * abs(an)
    assert np.allclose(v.db, dy.sum((0, 1, 2)), rtol=1e-13)
    # Σ|terms| bounds the gradient and equals it when every term is >= 0
    assert (np.abs(v.dw) <= v.dw_abs * (1 + 1e-12)).all()
    pos = G.conv_vjp(np.abs(x), w, out, np.abs(dy), s, relu=False)
    assert np.allclose(pos.dw, pos.dw_abs, rtol=1e-12)


def test_per_layer_vjps_chain_into_the_network_backward():
    """The per-layer VJPs fed the network's own activations and chained by hand give the
    whole-network backward: the two forms pin each other."""
    wts, low, rng = tiny_case(seed=3)
    net = G.Network(wts, TINY)
    grid = net.forward(low)
    dgrid = rng.randn(*grid.shape)
    want = net.backward(dgrid)
    a = {k: v.detach().numpy() for k, v in net.acts.items()}
    w = {k: np.asarray(v, np.float64) for k, v in wts.items()}
    P = G.P
    gd = TINY["luma_bins"]
    n_ds = 2
    got = {}

    def put(scope, v, bias=True):
        got[scope + "/weights"] = v.dw
        if bias:
            got[scope + "/biases"] = v.db

    splat = a[f"{P}/splat/conv{n_ds}"]
    loc, g = a[f"{P}/local/conv2"], a[f"{P}/global/fc3"]
    fv = G.fuse_predict_vjp(loc, g, w[f"{P}/prediction/conv1/weights"][0, 0], dgrid, gd, 3, 4)
    got[f"{P}/prediction/conv1/weights"] = fv.dw[None, None]
    got[f"{P}/prediction/conv1/biases"] = fv.db
    v = G.conv_vjp(a[f"{P}/local/conv1"], w[f"{P}/local/conv2/weights"], loc, fv.dlocal, 1, False)
    put(f"{P}/local/conv2", v, bias=False)
    v = G.conv_vjp(splat, w[f"{P}/local/conv1/weights"], a[f"{P}/local/conv1"], v.dx, 1, True)
    put(f"{P}/local/conv1", v)
    d_splat = v.dx
    dy = fv.dglobal
    for name, relu in (("fc3", False), ("fc2", True), ("fc1", True)):
        prev = {"fc3": "fc2", "fc2": "fc1", "fc1": "conv2"}[name]
        xin = a[f"{P}/global/{prev}"].reshape(len(low), -1)
        v = G.fc_vjp(xin, w[f"{P}/global/{name}/weights"], a[f"{P}/global/{name}"], dy, relu)
        put(f"{P}/global/{name}", v)
        dy = v.dx
    dy = dy.reshape(a[f"{P}/global/conv2"].shape)
    v = G.conv_vjp(a[f"{P}/global/conv1"], w[f"{P}/global/conv2/weights"], a[f"{P}/global/conv2"], dy, 2, True)
    put(f"{P}/global/conv2", v)
    v = G.conv_vjp(splat, w[f"{P}/global/conv1/weights"], a[f"{P}/global/conv1"], v.dx, 2, True)
    put(f"{P}/global/conv1", v)
    dy = d_splat + v.dx
    for i in range(n_ds, 0, -1):
        xin = low if i == 1 else a[f"{P}/splat/conv{i - 1}"]
        v = G.conv_vjp(xin, w[f"{P}/splat/conv{i}/weights"], a[f"{P}/splat/conv{i}"], dy, 2, True)
        put(f"{P}/splat/conv{i}", v)
        dy = v.dx
    got["lowres_input"] = dy
    assert sorted(got) == sorted(want)
    for k in want:
        scale = np.abs(want[k]).max()
        assert np.abs(got[k] - want[k]).max() <= 1e-12 * scale, k


@pytest.mark.parametrize("params", [TINY, dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8,
                                                luma_bins=8, channel_multiplier=1),
                                    dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=16,
                                         luma_bins=4, channel_multiplier=2)], ids=["tiny", "sb8", "cm2"])
def test_forward_matches_model_torch(params):
    wts, low, _ = tiny_case(seed=5, params=params)
    want = model_torch.coefficients(low, wts, params)
    got = G.Network(wts, params).forward(low)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def test_batch_norm_is_not_restated():
    with pytest.raises(NotImplementedError):
        G.Network({}, dict(TINY, batch_norm=True))


def test_fuse_predict_vjp_sum_of_terms():
    rng = np.random.RandomState(2)
    B, gh, gw, C, gd = 2, 3, 4, 8, 4
    local, glob, w = rng.randn(B, gh, gw, C), rng.randn(B, C), rng.randn(C, gd * 12)
    dgrid = rng.randn(B, gh, gw, gd, 3, 4)
    v = G.fuse_predict_vjp(local, glob, w, dgrid, gd, 3, 4)
    assert (np.abs(v.dw) <= v.dw_abs * (1 + 1e-12)).all() and (np.abs(v.db) <= v.db_abs * (1 + 1e-12)).all()
    # dglobal is the per-image sum of dlocal
    assert np.allclose(v.dglobal, v.dlocal.sum((1, 2)), rtol=1e-12, atol=1e-12)
