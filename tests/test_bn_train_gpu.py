"""The coefficient network's batch norm in training mode on an H100 (csrc/bn_train.cu): the kernels at
every batch-norm layer shape of the default network at 16 x 256^2 and at other shapes against the
float64 reference (oracle/bn_train_f64.py), their buffer contract, and the model paths
(_coefficients and inference with is_training=True and params['coefficient_batch_stats']) against the
float64 network."""

import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, models
from oracle import bn_train_f64 as BN

pytestmark = pytest.mark.gpu

P = "inference/coefficients"


def layer_shapes(params, B):
    """(scope, N, C) of every batch-norm layer of the network at batch B."""
    S, sb, gd, cm = params["net_input_size"], params["spatial_bin"], params["luma_bins"], params["channel_multiplier"]
    n_ds = int(np.log2(S / sb))
    out = []
    for i in range(1, n_ds):
        h = S >> (i + 1)
        out.append((f"splat/conv{i + 1}", B * h * h, cm * (2 ** i) * gd))
    c8, h = 8 * cm * gd, sb
    out += [("global/conv1", B * (h // 2) ** 2, c8), ("global/conv2", B * (h // 4) ** 2, c8),
            ("global/fc1", B, 32 * cm * gd), ("global/fc2", B, 16 * cm * gd), ("local/conv1", B * h * h, c8)]
    return out


DEFAULT = dict(models.DEFAULT_PARAMS, batch_norm=True)
SHAPES = ([(f"default/{s}", n, c) for s, n, c in layer_shapes(DEFAULT, 16)] +
          [(f"cm2/{s}", n, c) for s, n, c in layer_shapes(dict(DEFAULT, channel_multiplier=2), 4)] +
          [(f"gd16/{s}", n, c) for s, n, c in layer_shapes(dict(DEFAULT, luma_bins=16), 2)] +
          [("cm4gd16/global/fc1", 16, 2048), ("B1/fc1", 1, 256), ("B1/conv", 64, 64), ("7x5", 35, 64),
           ("C3", 1000, 3), ("C37", 4099, 37), ("C45", 333, 45), ("C100", 777, 100)])


def dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def stream():
    return torch.cuda.current_stream().cuda_stream


class Run:
    """One layer through the four kernels; every output a fresh buffer filled with `fill`."""

    def __init__(self, z, beta, dy, mm, mv, fill=float("nan"), ws_bytes=None):
        lib = _lib.load()
        N, C = z.shape
        need = lib.hdrnet_bn_stats_workspace_bytes(N, C)
        nb = need if ws_bytes is None else ws_bytes
        ws = torch.empty((need + 8) // 8, dtype=torch.float64, device="cuda")
        self.moments = torch.full((3, C), fill, dtype=torch.float64, device="cuda")
        self.rc = [lib.hdrnet_bn_stats_f32(z.data_ptr(), N, C, self.moments.data_ptr(), ws.data_ptr(), nb, stream())]
        self.y = torch.full_like(z, fill)
        self.mm, self.mv = mm.clone(), mv.clone()
        self.rc.append(lib.hdrnet_bn_relu_f32(z.data_ptr(), N, C, self.moments.data_ptr(), beta.data_ptr(),
                                              self.y.data_ptr(), self.mm.data_ptr(), self.mv.data_ptr(), stream()))
        self.sums = torch.full((2, C), fill, dtype=torch.float64, device="cuda")
        self.dbeta = torch.full((C,), fill, dtype=torch.float32, device="cuda")
        self.rc.append(lib.hdrnet_bn_relu_grad_sums_f32(z.data_ptr(), dy.data_ptr(), N, C, self.moments.data_ptr(),
                                                        beta.data_ptr(), self.sums.data_ptr(), self.dbeta.data_ptr(),
                                                        ws.data_ptr(), nb, stream()))
        self.dz = torch.full_like(z, fill)
        self.rc.append(lib.hdrnet_bn_relu_grad_f32(z.data_ptr(), dy.data_ptr(), N, C, self.moments.data_ptr(),
                                                   beta.data_ptr(), self.sums.data_ptr(), self.dz.data_ptr(), stream()))
        torch.cuda.synchronize()

    def host(self):
        return {k: getattr(self, k).cpu().numpy() for k in ("moments", "y", "mm", "mv", "sums", "dbeta", "dz")}


def layer_case(N, C, seed=0):
    rng = np.random.RandomState(seed)
    z = (rng.randn(N, C) * rng.uniform(0.1, 3.0, C) + rng.randn(C)).astype(np.float32)
    z[:, 0] = (0.9 + 1e-3 * rng.randn(N)).astype(np.float32)     # a small spread about a large mean
    beta = (0.5 * rng.randn(C)).astype(np.float32)
    dy = rng.randn(N, C).astype(np.float32)
    mm = rng.randn(C).astype(np.float32)
    mv = rng.uniform(0.5, 2.0, C).astype(np.float32)
    return z, beta, dy, mm, mv


@pytest.mark.parametrize("name,N,C", SHAPES, ids=[s[0] for s in SHAPES])
def test_kernels_match_float64(name, N, C):
    z, beta, dy, mm, mv = layer_case(N, C)
    r = Run(dev(z), dev(beta), dev(dy), dev(mm), dev(mv))
    assert r.rc == [0, 0, 0, 0]
    got = r.host()
    y64, mean, var = BN.bn_relu(z, beta)
    assert np.array_equal(got["moments"][0], np.full(C, float(N)))
    assert (np.abs(got["moments"][1] - mean) <= 1e-6 * np.maximum(np.abs(mean), np.sqrt(var) + 1e-30)).all()
    assert (np.abs(got["moments"][2] / N - var) <= 1e-6 * var + 1e-300).all()
    rng_y = max(float(np.ptp(y64)), 1e-30)
    assert np.abs(got["y"] - y64).max() <= 2e-6 * rng_y
    v = BN.bn_relu_vjp(z, beta, dy, mask=got["y"] > 0)       # the CUDA forward's relu mask
    rng_dz = max(float(np.ptp(v.dz)), 1e-30)
    assert np.abs(got["dz"] - v.dz).max() <= 1e-5 * rng_dz, name
    assert (np.abs(got["dbeta"] - v.dbeta) <= 4e-6 * v.dbeta_abs + 1e-30).all()
    assert np.allclose(got["sums"][0], v.dbeta, rtol=1e-9, atol=1e-9 * v.dbeta_abs.max())
    wm, wv = BN.moving_update(mm, mv, mean, var, N)
    assert np.abs(got["mm"] - wm).max() <= 1e-6 * max(np.abs(wm).max(), 1.0)
    assert np.abs(got["mv"] - wv).max() <= 1e-6 * max(np.abs(wv).max(), 1.0)
    # the same bits again, over outputs filled with something else
    again = Run(dev(z), dev(beta), dev(dy), dev(mm), dev(mv), fill=0.0).host()
    for k in got:
        assert np.array_equal(got[k].view(np.uint8), again[k].view(np.uint8)), k


def test_buffer_contract():
    lib = _lib.load()
    N, C = 3000, 37
    z, beta, dy, mm, mv = layer_case(N, C, seed=4)
    need = lib.hdrnet_bn_stats_workspace_bytes(N, C)
    assert need > 0 and lib.hdrnet_bn_stats_workspace_bytes(0, C) == 0
    assert lib.hdrnet_bn_stats_workspace_bytes(N, 9000) == 0
    g = 64   # NaN guard bands around every output
    zb, dyb, betab = dev(z), dev(dy), dev(beta)

    def banded(n, dtype):
        return torch.full((n + 2 * g,), float("nan"), dtype=dtype, device="cuda")

    mom, y, sums, dbeta, dz = (banded(3 * C, torch.float64), banded(N * C, torch.float32),
                               banded(2 * C, torch.float64), banded(C, torch.float32), banded(N * C, torch.float32))
    mmb, mvb = banded(C, torch.float32), banded(C, torch.float32)
    mmb[g:g + C], mvb[g:g + C] = dev(mm), dev(mv)
    ws = torch.empty(need // 8, dtype=torch.float64, device="cuda")        # lent at exactly its size
    p = lambda t: t[g:].data_ptr()                                          # noqa: E731
    assert lib.hdrnet_bn_stats_f32(zb.data_ptr(), N, C, p(mom), ws.data_ptr(), need, stream()) == 0
    assert lib.hdrnet_bn_relu_f32(zb.data_ptr(), N, C, p(mom), betab.data_ptr(), p(y), p(mmb), p(mvb), stream()) == 0
    assert lib.hdrnet_bn_relu_grad_sums_f32(zb.data_ptr(), dyb.data_ptr(), N, C, p(mom), betab.data_ptr(), p(sums),
                                            p(dbeta), ws.data_ptr(), need, stream()) == 0
    assert lib.hdrnet_bn_relu_grad_f32(zb.data_ptr(), dyb.data_ptr(), N, C, p(mom), betab.data_ptr(), p(sums), p(dz),
                                       stream()) == 0
    torch.cuda.synchronize()
    for t, n in ((mom, 3 * C), (y, N * C), (sums, 2 * C), (dbeta, C), (dz, N * C), (mmb, C), (mvb, C)):
        assert torch.isnan(t[:g]).all() and torch.isnan(t[g + n:]).all()
        assert not torch.isnan(t[g:g + n]).any()
    want = Run(zb.reshape(N, C), betab, dyb.reshape(N, C), dev(mm), dev(mv)).host()
    assert np.array_equal(y[g:g + N * C].cpu().numpy(), want["y"].reshape(-1))
    assert np.array_equal(dz[g:g + N * C].cpu().numpy(), want["dz"].reshape(-1))
    # one byte short: refused before anything is written
    out = torch.full((3 * C,), 7.0, dtype=torch.float64, device="cuda")
    s2 = torch.full((2 * C,), 7.0, dtype=torch.float64, device="cuda")
    assert lib.hdrnet_bn_stats_f32(zb.data_ptr(), N, C, out.data_ptr(), ws.data_ptr(), need - 1, stream()) \
        == _lib.E_BAD_SHAPE
    assert lib.hdrnet_bn_relu_grad_sums_f32(zb.data_ptr(), dyb.data_ptr(), N, C, p(mom), betab.data_ptr(),
                                            s2.data_ptr(), None, ws.data_ptr(), need - 1, stream()) == _lib.E_BAD_SHAPE
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (s2 == 7.0).all()
    # every other error before any launch
    assert lib.hdrnet_bn_stats_f32(zb.data_ptr(), 0, C, out.data_ptr(), ws.data_ptr(), need, stream()) == _lib.E_BAD_SHAPE
    assert lib.hdrnet_bn_stats_f32(zb.data_ptr(), N, 9000, out.data_ptr(), ws.data_ptr(), 1 << 30, stream()) \
        == _lib.E_UNSUPPORTED
    assert lib.hdrnet_bn_relu_f32(zb.data_ptr(), N, C, p(mom), betab.data_ptr(), p(y), p(mmb), None, stream()) \
        == _lib.E_NULL_POINTER
    assert lib.hdrnet_bn_relu_grad_f32(zb.data_ptr(), dyb.data_ptr(), N, C, p(mom), None, p(sums), p(dz), stream()) \
        == _lib.E_NULL_POINTER
    assert lib.hdrnet_bn_stats_f32(zb.data_ptr(), N, C, out.data_ptr() + 4, ws.data_ptr(), need, stream()) \
        == _lib.E_BAD_SHAPE
    torch.cuda.synchronize()
    assert (out == 7.0).all()


# ---- the model paths --------------------------------------------------------------------------------
def tensor_weights(params, model_name="HDRNetCurves", seed=0, grad=True):
    rng = np.random.RandomState(seed + 100)
    w = models.init_weights(params, seed=seed, model_name=model_name)
    for k in w:
        if k.endswith(("/beta", "/biases")) and k.startswith(P):
            w[k] = (0.1 * rng.randn(*w[k].shape)).astype(np.float32)
    t = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    for k in BN.variable_names(params):
        t[k].requires_grad_(grad)
    return w, t


def float32_errors(w, params, low, dgrid, want, n_out=3):
    """What a float32 implementation reaches: the same network in torch float32 on the CPU
    (F.batch_norm training=True), each gradient's error against the float64 network over its scale."""
    from test_bn_train_f64 import torch_network
    names = BN.variable_names(params)
    grid, v, x0 = torch_network(w, params, low, dtype=torch.float32, n_out=n_out)
    grads = torch.autograd.grad(grid, [v[k] for k in names] + [x0], torch.from_numpy(dgrid).float())
    return {k: np.abs(g.double().numpy() - want[k]).max() / max(np.ptp(want[k]), np.abs(want[k]).max(), 1e-30)
            for k, g in zip(names + ["lowres_input"], grads)}


def bound(e32):
    """A gradient is held to 1e-5 of its scale, or to three times what float32 on the CPU reaches (two
    float32 sums in different orders differ by a small factor; on an H100 the widest was 2.1x, the
    pyramid's splat/conv1/biases)."""
    return max(1e-5, 3.0 * e32)


def coefficient_check(params, B, n_out, seed=0):
    """_coefficients(is_training=True): the grid, every variable's and lowres_input's gradient and the
    moving averages against the float64 network; the worst error over each quantity's range, and
    (key "float32") the same errors of a float32 implementation."""
    w, t = tensor_weights(params, model_name=params.get("model_name", "HDRNetCurves"), seed=seed)
    rng = np.random.RandomState(seed)
    S = params["net_input_size"]
    low = rng.rand(B, S, S, 3).astype(np.float32)
    x = dev(low).requires_grad_(True)
    cls = models.HDRNetGaussianPyrNN if n_out == 9 else models.HDRNetCurves
    p = dict(params, weights=t, coefficient_batch_stats=True)
    grid = cls._coefficients(x, p, is_training=True)
    dgrid = rng.randn(*grid.shape).astype(np.float32)
    names = BN.variable_names(params)
    grads = torch.autograd.grad(grid, [t[k] for k in names] + [x], dev(dgrid))
    net = BN.TrainingNetwork(w, params, n_out=n_out)
    want = net.forward(low)
    wg = net.backward(dgrid.astype(np.float64))
    errs = {"grid": np.abs(grid.detach().cpu().numpy() - want).max() / np.ptp(want)}
    for k, g in zip(names + ["lowres_input"], grads):
        ref = wg[k]
        errs[k] = np.abs(g.cpu().numpy() - ref).max() / max(np.ptp(ref), np.abs(ref).max(), 1e-30)
    for scope in BN.batch_norm_scopes(params):
        mean, var, n = net.stats[scope]
        wm, wv = BN.moving_update(w[scope + "/BatchNorm/moving_mean"], w[scope + "/BatchNorm/moving_variance"],
                                  mean, var, n)
        errs[scope + "/moving_mean"] = np.abs(t[scope + "/BatchNorm/moving_mean"].cpu().numpy() - wm).max()
        errs[scope + "/moving_variance"] = np.abs(t[scope + "/BatchNorm/moving_variance"].cpu().numpy() - wv).max()
    # F.batch_norm refuses one row per channel (fc at B = 1): there the bound is 1e-5
    errs["float32"] = float32_errors(w, params, low, dgrid.astype(np.float64), wg, n_out) if B > 1 else {}
    return errs


@pytest.mark.parametrize("case", ["curves_16x256", "pyramid_cm4_4x256", "gd16_B1"])
def test_coefficients_training_match_float64(case):
    params, B, n_out = {"curves_16x256": (DEFAULT, 16, 3),
                        "pyramid_cm4_4x256": (dict(DEFAULT, channel_multiplier=4, model_name="HDRNetGaussianPyrNN"),
                                              4, 9),
                        "gd16_B1": (dict(DEFAULT, luma_bins=16, net_input_size=64, spatial_bin=8), 1, 3)}[case]
    errs = coefficient_check(params, B, n_out)
    e32 = errs.pop("float32")
    worst = max(errs, key=errs.get)
    print(f"MEASURE bn-train {case}: worst {worst} {errs[worst]:.3g}; float32 on the CPU: worst "
          f"{max(e32, key=e32.get, default=None)} {max(e32.values(), default=0.0):.3g}")
    for k, e in errs.items():
        assert e <= (1e-6 if "/moving_" in k else bound(e32.get(k, 0.0))), f"{k}: {e:.3g} (float32 {e32.get(k)})"


# Whole-network float32 against float64, the float64 network on its own forward.  Batch norm divides
# a conv's rounding error by the channel's spread, so the training path runs its convs on the CUDA
# cores (float32 rounded to nearest); with the 3xTF32 tensor-core form the worst gradient at
# 16 x 256^2 was 1.0e-2 of range (DESIGN.md row f-14).  Each gradient is held to bound(): 1e-5, or
# three times the error of the same network in torch float32, where float32 itself does not reach 1e-5.


def test_moving_averages_over_four_calls():
    params = dict(DEFAULT, net_input_size=64, spatial_bin=8)
    w, t = tensor_weights(params, grad=False)
    rng = np.random.RandomState(9)
    p = dict(params, weights=t, coefficient_batch_stats=True)
    want = {k: np.asarray(v, np.float64) for k, v in w.items() if "/moving_" in k}
    for _ in range(4):
        low = rng.rand(3, 64, 64, 3).astype(np.float32)
        with torch.no_grad():
            models.HDRNetCurves._coefficients(dev(low), p, is_training=True)
        net = BN.TrainingNetwork(w, params)
        net.forward(low)
        for scope in BN.batch_norm_scopes(params):
            mean, var, n = net.stats[scope]
            mk, vk = scope + "/BatchNorm/moving_mean", scope + "/BatchNorm/moving_variance"
            want[mk], want[vk] = BN.moving_update(want[mk], want[vk], mean, var, n)
    for k, v in want.items():
        assert np.abs(t[k].cpu().numpy() - v).max() <= 1e-6 * max(np.abs(v).max(), 1.0), k


def test_training_path_never_synchronises():
    params = dict(DEFAULT, net_input_size=64, spatial_bin=8)
    _, t = tensor_weights(params)
    x = torch.rand(4, 64, 64, 3, device="cuda", requires_grad=True)
    p = dict(params, weights=t, coefficient_batch_stats=True)
    models.HDRNetCurves._coefficients(x, p, is_training=True)       # warm-up: module loads, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        grid = models.HDRNetCurves._coefficients(x, p, is_training=True)
        grid.backward(torch.ones_like(grid))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert all(t[k].grad is not None for k in BN.variable_names(params))


def test_nn_guide_model_trains_both_batch_norms():
    params = dict(DEFAULT, net_input_size=64, spatial_bin=8, model_name="HDRNetPointwiseNNGuide")
    w, t = tensor_weights(params, model_name="HDRNetPointwiseNNGuide")
    for k in ("inference/guide/conv1/weights", "inference/guide/conv1/BatchNorm/beta"):
        t[k].requires_grad_(True)
    before = {k: v.clone() for k, v in t.items() if "/moving_" in k}
    low, full = torch.rand(2, 64, 64, 3, device="cuda"), torch.rand(2, 40, 64, 3, device="cuda")
    out = models.HDRNetPointwiseNNGuide.inference(low, full, dict(params, weights=t, coefficient_batch_stats=True,
                                                                  guide_grad=True), is_training=True)
    out.square().mean().backward()
    for k in BN.variable_names(params) + ["inference/guide/conv1/weights"]:
        assert t[k].grad is not None and torch.isfinite(t[k].grad).all(), k
    assert all(not torch.equal(before[k], t[k]) for k in before)     # guide and coefficient moving averages


def test_teacher_student_fit_converges():
    params = dict(DEFAULT, net_input_size=64, spatial_bin=8)
    _, teacher = tensor_weights(params, seed=1, grad=False)
    _, student = tensor_weights(params, seed=2)
    rng = np.random.RandomState(5)
    names = BN.variable_names(params)
    opt = torch.optim.Adam([student[k] for k in names], lr=1e-3)
    ps, pt = (dict(params, weights=w, coefficient_batch_stats=True) for w in (student, teacher))
    losses = []
    for step in range(300):
        low = dev(rng.rand(8, 64, 64, 3))
        with torch.no_grad():
            target = models.HDRNetCurves._coefficients(low, pt, is_training=True)
        opt.zero_grad()
        loss = (models.HDRNetCurves._coefficients(low, ps, is_training=True) - target).square().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    first, last = float(np.mean(losses[:5])), float(np.mean(losses[-10:]))
    print(f"MEASURE bn-train teacher-student: first {first:.4g} last {last:.4g} factor {first / last:.1f}")
    # 3.1x over 300 steps on an H100; the CLI student (test_train_bn_cli_gpu.py) holds the 10x bar
    assert np.isfinite(losses).all() and first / last >= 2.0


def test_nn_model_with_guide_grad_matches_the_float64_chain():
    """HDRNetPointwiseNNGuide.inference(is_training=True) with both batch norms in training mode and
    guide_grad, L2 loss at 4 x 256^2 (network input and image): every coefficient variable against
    the float64 network (bn_train_f64) chained from the float64 slice-apply VJP, every guide variable
    and fullres_input against nn_guide_f64 and slice_f64, within 1e-5 of their scale."""
    import nn_guide_f64 as O
    from oracle import slice_f64
    from test_nn_guide_grad_gpu import guide_weights, near_ties
    NN = models.HDRNetPointwiseNNGuide
    params = dict(DEFAULT, model_name="HDRNetPointwiseNNGuide")
    w, t = tensor_weights(params, model_name="HDRNetPointwiseNNGuide", seed=3)
    rng = np.random.RandomState(4)
    for k, v in guide_weights(rng).items():
        w[k] = v
        t[k] = torch.from_numpy(v).cuda().requires_grad_("/moving_" not in k)
    low = rng.rand(4, 256, 256, 3).astype(np.float32)
    full = rng.rand(4, 256, 256, 3).astype(np.float32)
    p = dict(params, weights=t, guide_grad=True, coefficient_batch_stats=True)
    tf = dev(full).requires_grad_(True)
    out = NN.inference(dev(low), tf, p, is_training=True)
    wn = {k: v.detach().cpu().numpy() for k, v in t.items()}
    keep = np.where(near_ties(full, wn), 0.0, 1.0).astype(np.float32)
    target = rng.rand(*full.shape).astype(np.float32)
    (((out - dev(target)) * dev(keep[..., None])) ** 2).sum().backward()
    with torch.no_grad():
        guide = NN._guide(dev(full), dict(p), is_training=True).cpu().numpy()
    net = BN.TrainingNetwork(w, params)
    grid = net.forward(low)
    ctn = 2.0 * (out.detach().cpu().numpy().astype(np.float64) - target) * keep[..., None] ** 2
    sv = slice_f64.bilateral_slice_apply_grad(grid.reshape(4, 16, 16, 8, 12), guide, full, ctn, True)
    want = net.backward(sv.grid.reshape(grid.shape))
    gv = O.vjp(full, sv.guide, wn)
    errs = {}

    def rel(got, ref):
        return float(np.abs(np.asarray(got, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))

    e32 = float32_errors(w, params, low, sv.grid.reshape(grid.shape), want)
    for k in BN.variable_names(params):
        errs[k] = rel(t[k].grad.cpu().numpy(), want[k])
    for n in O.NAMES:
        errs["guide/" + n] = rel(t[f"inference/guide/{n}"].grad.cpu().numpy(), gv.dparams[n])
    errs["fullres_input"] = rel(tf.grad.cpu().numpy(), sv.input + gv.dinput)
    worst = max(errs, key=errs.get)
    print(f"MEASURE bn-train nn guide_grad 4x256: worst {worst} {errs[worst]:.3g}; float32 on the CPU: worst "
          f"{max(e32, key=e32.get)} {max(e32.values()):.3g}")
    for k, e in errs.items():
        assert e <= bound(e32.get(k, 0.0)), f"{k}: {e:.3g} (float32 {e32.get(k)})"
