"""CPU tests of the float64 curves-guide VJP (oracle/guide_f64.py): against torch float64 autograd
of the same graph, against central differences away from the kinks, and against hand-computed
known answers at the ties (a relu exactly at a knot, the clip exactly at 0 and at 1, and outside)."""
import numpy as np
import pytest
import torch

from oracle import guide_f64, model_torch

G = "inference/guide"


def weights(rng, spread=0.3):
    """Curves-guide variables in the model's shapes, away from the identity-like initial curve."""
    return {f"{G}/ccm": np.eye(3) + spread * rng.randn(3, 3),
            f"{G}/ccm_bias": 0.1 * rng.randn(3),
            f"{G}/shifts": np.sort(rng.rand(1, 1, 3, 16), axis=-1),
            f"{G}/slopes": rng.randn(1, 1, 1, 3, 16) * 0.5,
            f"{G}/channel_mixing/weights": rng.rand(1, 1, 3, 1) * 0.6,
            f"{G}/channel_mixing/biases": np.array([0.1])}


def torch_guide(x, v):
    """The graph of model_torch.guide_curves in float64 torch without its float32 roundings."""
    t = x @ v["ccm"] + v["ccm_bias"]
    u = (v["slopes"].reshape(3, 16) * torch.relu(t[..., None] - v["shifts"].reshape(3, 16))).sum(-1)
    a = u @ v["channel_mixing/weights"].reshape(3) + v["channel_mixing/biases"].reshape(())
    return torch.clamp(a, 0.0, 1.0)


def test_forward_is_model_torchs_guide():
    rng = np.random.RandomState(0)
    w = weights(rng)
    x = rng.rand(2, 5, 7, 3).astype(np.float32)
    want = model_torch.guide_curves(x, w)
    assert np.abs(guide_f64.guide(x, w) - want).max() <= 1e-6


def test_vjp_matches_torch_float64_autograd():
    rng = np.random.RandomState(1)
    w = weights(rng)
    x = rng.rand(3, 17, 19, 3) * 1.2 - 0.1
    g = rng.randn(3, 17, 19)
    v = {n: torch.tensor(np.asarray(w[f"{G}/{n}"], np.float64), requires_grad=True) for n in guide_f64.NAMES}
    xt = torch.tensor(x, requires_grad=True)
    (torch_guide(xt, v) * torch.tensor(g)).sum().backward()
    got = guide_f64.vjp(x, g, w)
    clipped = guide_f64.preclip(x, w)[0]
    assert 0.05 < np.mean((clipped < 0) | (clipped > 1)) < 0.95      # both sides of the clip are covered
    scale = np.abs(xt.grad.numpy()).max()
    assert np.abs(got.dinput - xt.grad.numpy()).max() <= 1e-12 * scale
    for n in guide_f64.NAMES:
        ref = v[n].grad.numpy()
        assert got.dparams[n].shape == ref.shape, n
        assert np.abs(got.dparams[n] - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30), n
        assert np.all(got.dparams_abs[n] >= np.abs(got.dparams[n]) * (1 - 1e-12)), n


def test_vjp_matches_central_differences_away_from_kinks():
    rng = np.random.RandomState(2)
    w = weights(rng)
    x = rng.rand(400, 3)
    a, t = guide_f64.preclip(x, w)
    s = np.asarray(w[f"{G}/shifts"]).reshape(3, 16)
    far = (np.abs(t[:, :, None] - s).min(axis=(1, 2)) > 1e-3) & (np.abs(a) > 1e-3) & (np.abs(a - 1) > 1e-3)
    x = x[far]
    assert len(x) > 100
    g = rng.randn(len(x))
    got = guide_f64.vjp(x, g, w)
    h = 1e-7

    def loss(wts, xx=x):
        return float((guide_f64.guide(xx, wts) * g).sum())

    for n in guide_f64.NAMES:
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
    for i in range(3):
        e = np.zeros(3)
        e[i] = h
        num = (guide_f64.guide(x + e, w) - guide_f64.guide(x - e, w)) * g / (2 * h)
        assert np.abs(num - got.dinput[:, i]).max() <= 1e-6 * max(np.abs(got.dinput).max(), 1.0)


def tie_weights(slopes, mix_bias=0.0):
    return {f"{G}/ccm": np.eye(3), f"{G}/ccm_bias": np.zeros(3),
            f"{G}/shifts": np.tile(np.arange(16) / 16.0, (1, 1, 3, 1)),
            f"{G}/slopes": np.asarray(slopes, np.float64).reshape(1, 1, 1, 3, 16),
            f"{G}/channel_mixing/weights": np.array([1.0, 0.0, 0.0]).reshape(1, 1, 3, 1),
            f"{G}/channel_mixing/biases": np.array([mix_bias])}


def test_known_answer_pixel_exactly_on_a_knot():
    """Identity ccm, all slopes 1, mix (1, 0, 0): t = x and x_0 = 0.25 = s_4 exactly.  The relu at
    knot 4 is 0 and so is its gradient; knots 0..3 are active."""
    w = tie_weights(np.ones(48))
    x = np.array([[0.25, 0.5, 0.7]])
    g = np.array([2.0])
    r = guide_f64.vjp(x, g, w)
    assert guide_f64.guide(x, w)[0] == 0.625                          # .25 + .1875 + .125 + .0625
    d = r.dparams
    want_shift = np.zeros((3, 16))
    want_shift[0, :4] = -2.0
    assert np.array_equal(d["shifts"].reshape(3, 16), want_shift)
    want_slope = np.zeros((3, 16))
    want_slope[0, :4] = 2.0 * np.array([0.25, 0.1875, 0.125, 0.0625])
    assert np.array_equal(d["slopes"].reshape(3, 16), want_slope)
    assert np.array_equal(d["ccm_bias"], [8.0, 0.0, 0.0])              # g * mix_0 * u'_0 = 2 * 4
    assert np.array_equal(d["ccm"], [[2.0, 0, 0], [4.0, 0, 0], [5.6, 0, 0]])
    assert np.allclose(d["channel_mixing/weights"].reshape(3), [1.25, 4.5, 8.55], rtol=0, atol=1e-14)
    assert np.array_equal(d["channel_mixing/biases"], [2.0])
    assert np.array_equal(r.dinput, [[8.0, 0.0, 0.0]])


@pytest.mark.parametrize("x0,mix_bias,inside", [(0.0, 0.0, True), (1.0, 0.0, True), (0.25, -0.5, False),
                                                (1.5, 0.0, False)])
def test_known_answers_at_and_beyond_the_clip(x0, mix_bias, inside):
    """Slope 1 on knot 0 (s = 0), mix (1, 0, 0): a = relu(x_0) + mix_bias.  a = 0 and a = 1 pass the
    gradient (clip_by_value at equality); a < 0 and a > 1 do not."""
    slopes = np.zeros(48)
    slopes[0] = 1.0
    w = tie_weights(slopes, mix_bias)
    x = np.array([[x0, 0.3, 0.6]])
    r = guide_f64.vjp(x, np.array([3.0]), w)
    d = {n: v.reshape(-1) for n, v in r.dparams.items()}
    if not inside:
        assert all(not v.any() for v in d.values()) and not r.dinput.any()
        return
    active = x0 > 0.0                       # relu(t - 0) at t = 0 has gradient 0
    assert np.array_equal(d["channel_mixing/biases"], [3.0])
    assert np.array_equal(d["channel_mixing/weights"], [3.0 * x0, 0, 0])     # u_1 = u_2 = 0: no slopes
    # every knot of channel 0 gets g mix_0 relu(x_0 - k / 16), whatever its slope
    assert np.array_equal(d["slopes"][:16], 3.0 * np.maximum(x0 - np.arange(16) / 16.0, 0.0))
    assert not d["slopes"][16:].any()
    assert d["shifts"][0] == (-3.0 if active else 0.0) and not d["shifts"][1:].any()
    assert np.array_equal(d["ccm_bias"], [3.0 if active else 0.0, 0, 0])
    assert np.array_equal(r.dinput, [[3.0 if active else 0.0, 0, 0]])
    assert np.array_equal(d["ccm"], np.array([x0, 0, 0, 0.3, 0, 0, 0.6, 0, 0]) * (3.0 if active else 0.0))


def test_flat_order_is_the_librarys():
    rng = np.random.RandomState(3)
    r = guide_f64.vjp(rng.rand(10, 3), rng.randn(10), weights(rng))
    f = guide_f64.flat(r.dparams)
    assert f.shape == (112,)
    assert np.array_equal(f[12:60], r.dparams["shifts"].reshape(-1))
    assert f[111] == r.dparams["channel_mixing/biases"][0]
