"""GPU tests of the coefficient network's backward (csrc/cnn_grad.cu, models._ConvFn / _FcFn /
_FusePredictFn) against the float64 reference (oracle/cnn_grad_f64.py): per-layer VJPs at every
shape of the networks the models build, the whole network and the model end to end at the
reference's training size, the autograd boundary, no stale weights, and a teacher-student fit."""
import time

import numpy as np
import pytest
import torch

from hdrnet_b200 import layers, models
from oracle import cnn_grad_f64 as G
from oracle import slice_f64

pytestmark = pytest.mark.gpu

BAR = 1e-5         # every gradient: max |diff| / max |ref|; weight / bias grads: per element / Σ|terms|
P = G.P
TRAIN = dict(models.DEFAULT_PARAMS)          # 256² network input, 16 x 16 x 8 grid (train.py:224-236)
SMALL = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, luma_bins=4)


def report(what, **errs):
    print("MEASURE", what, " ".join(f"{k}={v:.2e}" for k, v in errs.items()), flush=True)


def rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def per_elem(got, ref, terms):
    d = np.abs(np.asarray(got, np.float64) - ref)
    return float((d / np.maximum(terms, 1e-30)).max())


def check_wgrad(what, got, v_d, v_abs):
    g, e = rel(got, v_d), per_elem(got, v_d, v_abs)
    assert g <= BAR, f"{what}: {g:.3e} of max |ref|"
    assert e <= BAR, f"{what}: {e:.3e} of Σ|terms|"
    return g, e


def cuda(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32))).cuda().requires_grad_(grad)


def np_(t):
    return t.detach().cpu().numpy()


def net_layer_shapes(params, B, n_out=3):
    """(kind, B, H, W, cin, cout, k, stride, relu, bias) of every layer of the network."""
    S, sb, gd, cm = params["net_input_size"], params["spatial_bin"], params["luma_bins"], params["channel_multiplier"]
    shapes, H, cin = [], S, 3
    n_ds = int(np.log2(S / sb))
    for i in range(n_ds):
        shapes.append(("conv", B, H, H, cin, cm * 2 ** i * gd, 3, 2, True, True))
        H, cin = H // 2, cm * 2 ** i * gd
    c8 = 8 * cm * gd
    g1 = (sb + 1) // 2
    shapes += [("conv", B, sb, sb, cin, c8, 3, 2, True, True), ("conv", B, g1, g1, c8, c8, 3, 2, True, True)]
    flat = ((g1 + 1) // 2) ** 2 * c8
    shapes += [("fc", B, 1, 1, flat, 32 * cm * gd, 1, 1, True, True), ("fc", B, 1, 1, 32 * cm * gd, 16 * cm * gd, 1, 1, True, True),
               ("fc", B, 1, 1, 16 * cm * gd, c8, 1, 1, False, True)]
    shapes += [("conv", B, sb, sb, cin, c8, 3, 1, True, True), ("conv", B, sb, sb, c8, c8, 3, 1, False, False)]
    shapes += [("fuse", B, sb, sb, c8, gd, n_out, 4, False, True)]
    return shapes


EXTRA = [("conv", 2, 33, 50, 5, 12, 3, 1, True, True), ("conv", 2, 33, 50, 5, 12, 3, 2, True, True),
         ("conv", 1, 33, 50, 8, 16, 1, 2, False, False), ("conv", 1, 17, 9, 16, 8, 1, 1, True, False),
         ("conv", 1, 64, 64, 3, 8, 3, 2, False, True), ("fc", 1, 1, 1, 300, 70, 1, 1, True, True),
         ("fc", 5, 1, 1, 64, 40, 1, 1, False, False), ("fuse", 1, 5, 7, 24, 3, 3, 4, False, True)]

CASES = ([("train",) + s for s in net_layer_shapes(TRAIN, 16)] +
         [("bn_small",) + s for s in net_layer_shapes(SMALL, 2)] +
         [("cm2",) + s for s in net_layer_shapes(dict(models.DEFAULT_PARAMS, channel_multiplier=2,
                                                       net_input_size=128), 2)] +
         [("pyramid",) + s for s in net_layer_shapes(dict(models.DEFAULT_PARAMS, net_input_size=128), 2, n_out=9)
          if s[0] == "fuse"] +
         [("b1",) + s for s in net_layer_shapes(TRAIN, 1)] +
         [("extra",) + s for s in EXTRA])


def layer_vjps(kind, B, H, W, cin, cout, k, s, relu, bias, seed=0):
    """The CUDA layer forward + backward through the autograd Functions, and the float64 VJPs of the
    same layer fed the CUDA forward's own output (for the ReLU mask)."""
    rng = np.random.RandomState(seed)
    if kind == "fuse":
        C, gd, n_out, n_in = cin, cout, k, s
        O = gd * n_out * n_in
        loc, glob = rng.randn(B, H, W, C), rng.randn(B, C)
        w, b = rng.randn(1, 1, C, O) / np.sqrt(C), rng.randn(O) * 0.1
        tl, tg, tw, tb = cuda(loc, True), cuda(glob, True), cuda(w, True), cuda(b, True)
        grid = models._FusePredictFn.apply(tl, tg, tw[0, 0], tb, gd, n_out, n_in)
        dgrid = rng.randn(*grid.shape).astype(np.float32)
        grid.backward(cuda(dgrid))
        v = G.fuse_predict_vjp(np_(tl), np_(tg), np_(tw)[0, 0], dgrid, gd, n_out, n_in)
        return ([("dlocal", tl.grad, v.dlocal, None), ("dglobal", tg.grad, v.dglobal, None),
                 ("dw", tw.grad[0, 0], v.dw, v.dw_abs), ("db", tb.grad, v.db, v.db_abs)])
    x = np.maximum(rng.randn(B, H, W, cin), 0) if kind == "conv" else np.maximum(rng.randn(B, cin), 0)
    wshape = (k, k, cin, cout) if kind == "conv" else (cin, cout)
    w = rng.randn(*wshape) / np.sqrt(k * k * cin)
    b = rng.randn(cout) * 0.1
    tx, tw = cuda(x, True), cuda(w, True)
    tb = cuda(b, True) if bias else None
    if kind == "conv":
        out = models._ConvFn.apply(tx, tw, tb, s, relu)
    else:
        out = models._FcFn.apply(tx, tw, tb, relu)
    dy = rng.randn(*out.shape).astype(np.float32)
    out.backward(cuda(dy))
    o = np_(out)
    v = G.conv_vjp(np_(tx), np_(tw), o, dy, s, relu) if kind == "conv" else G.fc_vjp(np_(tx), np_(tw), o, dy, relu)
    res = [("dx", tx.grad, v.dx, None), ("dw", tw.grad, v.dw, v.dw_abs)]
    if bias:
        res.append(("db", tb.grad, v.db, v.db_abs))
    return res


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(v) for v in c))
def test_layer_vjps_match_float64(case):
    name, kind, *shape = case
    errs = {}
    for what, got, ref, terms in layer_vjps(kind, *shape):
        got = np_(got)
        assert got.shape == ref.shape and np.isfinite(got).all()
        if terms is None:
            errs[what] = rel(got, ref)
            assert errs[what] <= BAR, f"{case} {what}: {errs[what]:.3e}"
        else:
            errs[what], errs[what + "_elem"] = check_wgrad(f"{case} {what}", got, ref, terms)
    report(f"layer {name} {kind} {shape}", **errs)


def tensor_weights(params, seed=0, grad=True, model_name=None):
    w = models.init_weights(params, seed=seed, model_name=model_name)
    rng = np.random.RandomState(seed + 100)
    out = {}
    for k, v in w.items():
        if k.endswith("/biases") and k.startswith(P):
            v = (0.05 * rng.randn(*v.shape)).astype(np.float32)     # non-zero, so their gradients matter
        t = torch.from_numpy(v).cuda()
        out[k] = t.requires_grad_(grad and k.startswith(P))
    return out


def test_whole_network_at_training_size():
    """_coefficients(...).backward(dgrid) at 16 x 256² against the float64 network's own forward and
    backward: a ReLU mask may flip between the two forwards, so the global bar only."""
    torch.manual_seed(0)
    wts = tensor_weights(TRAIN)
    rng = np.random.RandomState(1)
    low = rng.rand(16, 256, 256, 3).astype(np.float32)
    tl = cuda(low, True)
    t0 = time.time()
    grid = models.HDRNetCurves._coefficients(tl, dict(TRAIN, weights=wts))
    dgrid = rng.randn(*grid.shape).astype(np.float32)
    grid.backward(cuda(dgrid))
    net = G.Network({k: np_(v) for k, v in wts.items()}, TRAIN)
    want_grid = net.forward(low)
    assert rel(np_(grid), want_grid) <= 1e-5
    want = net.backward(dgrid)
    errs = {}
    for k, ref in want.items():
        got = np_(tl.grad if k == "lowres_input" else wts[k].grad)
        errs[k.replace(P + "/", "")] = e = rel(got, ref)
        assert e <= BAR, f"{k}: {e:.3e}"
    report("whole network 16x256^2", **errs)
    print(f"whole network: {time.time() - t0:.1f} s", flush=True)


def test_end_to_end_l2_loss_at_training_size():
    """L2 loss of HDRNetCurves.inference at 16 x 512² (256² network input) against a target, back to
    every coefficient variable; float64: slice_f64's grid VJP, with the CUDA guide, feeds the float64
    network backward."""
    wts = tensor_weights(TRAIN, seed=2)
    rng = np.random.RandomState(3)
    low = rng.rand(16, 256, 256, 3).astype(np.float32)
    full = rng.rand(16, 512, 512, 3).astype(np.float32)
    target = rng.rand(16, 512, 512, 3).astype(np.float32)
    params = dict(TRAIN, weights=wts)
    tf = cuda(full)
    out = models.HDRNetCurves.inference(cuda(low), tf, params)
    loss = ((out - cuda(target)) ** 2).sum()
    loss.backward()
    with torch.no_grad():
        fused = models.HDRNetCurves.inference(cuda(low), tf, params)
        guide = np_(models.HDRNetCurves._guide(tf, params))
    fwd_err = rel(np_(out), np_(fused))
    ct = 2.0 * (np_(out).astype(np.float64) - target)
    gv = slice_f64.bilateral_slice_apply_grad(np.zeros((16, 16, 16, 8, 12)), guide, full, ct, True)[0]
    net = G.Network({k: np_(v) for k, v in wts.items()}, TRAIN)
    net.forward(low)
    want = net.backward(gv.reshape(16, 16, 16, 8, 3, 4))
    errs = {}
    for k in G.variable_names(TRAIN):
        errs[k.replace(P + "/", "")] = e = rel(np_(wts[k].grad), want[k])
        assert e <= BAR, f"{k}: {e:.3e}"
    report("end to end 16x512^2", autograd_vs_fused_forward=fwd_err, **errs)
    assert fwd_err <= 1e-6


def small_setup(seed=0, B=2):
    rng = np.random.RandomState(seed)
    low = cuda(rng.rand(B, 64, 64, 3))
    full = cuda(rng.rand(B, 48, 160, 3))
    return rng, low, full


def grads_of(wts):
    return {k: v.grad.clone() for k, v in wts.items() if v.grad is not None}


def test_backward_is_bitwise_reproducible_and_accumulates():
    wts = tensor_weights(TRAIN)
    rng = np.random.RandomState(4)
    low = cuda(rng.rand(16, 256, 256, 3), True)
    params = dict(TRAIN, weights=wts)
    dgrid = cuda(rng.randn(16, 16, 16, 8, 3, 4))
    models.HDRNetCurves._coefficients(low, params).backward(dgrid)
    first = grads_of(wts)
    first["x"] = low.grad.clone()
    for v in list(wts.values()) + [low]:
        v.grad = None
    models.HDRNetCurves._coefficients(low, params).backward(dgrid)
    for k, v in first.items():
        got = low.grad if k == "x" else wts[k].grad
        assert torch.equal(got, v), k
    models.HDRNetCurves._coefficients(low, params).backward(dgrid)      # accumulates
    for k, v in first.items():
        got = low.grad if k == "x" else wts[k].grad
        assert torch.equal(got, v + v), k


def test_non_contiguous_upstream_gradient_and_side_stream():
    wts = tensor_weights(SMALL)
    _, low, _ = small_setup()
    params = dict(SMALL, weights=wts)
    grid = models.HDRNetCurves._coefficients(low, params)
    dense = torch.randn(grid.shape[::-1], device="cuda")
    nc = dense.permute(5, 4, 3, 2, 1, 0)
    assert not nc.is_contiguous()
    grid.backward(nc)
    want = grads_of(wts)
    for v in wts.values():
        v.grad = None
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g2 = models.HDRNetCurves._coefficients(low, params)
        g2.backward(nc.contiguous())
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for k, v in want.items():
        assert torch.equal(wts[k].grad, v), k


def test_partial_requires_grad():
    rng, low, _ = small_setup()
    full = tensor_weights(SMALL)
    params = dict(SMALL, weights=full)
    dgrid = cuda(rng.randn(2, 8, 8, 4, 3, 4))
    models.HDRNetCurves._coefficients(low, params).backward(dgrid)
    want = grads_of(full)
    # only the local branch and the prediction
    part = {k: v.detach().clone().requires_grad_("/local/" in k or "/prediction/" in k) for k, v in full.items()}
    models.HDRNetCurves._coefficients(low, dict(SMALL, weights=part)).backward(dgrid)
    for k, v in part.items():
        if v.requires_grad:
            assert torch.equal(v.grad, want[k]), k
        else:
            assert v.grad is None
    # only the input
    frozen = {k: v.detach() for k, v in full.items()}
    x = low.clone().requires_grad_(True)
    models.HDRNetCurves._coefficients(x, dict(SMALL, weights=frozen)).backward(dgrid)
    x2 = low.clone().requires_grad_(True)
    models.HDRNetCurves._coefficients(x2, params).backward(dgrid)
    assert torch.equal(x.grad, x2.grad)


def test_layers_conv_and_fc_with_tensor_variables():
    rng = np.random.RandomState(5)
    s = "inference/coefficients/local/conv1"
    f = "inference/coefficients/global/fc1"
    w = {s + "/weights": cuda(rng.randn(3, 3, 8, 16) * 0.2, True), s + "/biases": cuda(rng.randn(16) * 0.1, True),
         f + "/weights": cuda(rng.randn(64, 32) * 0.2, True), f + "/biases": cuda(rng.randn(32) * 0.1, True)}
    x = cuda(rng.rand(2, 11, 13, 8), True)
    y = layers.conv(x, 16, 3, stride=2, scope=s, weights=w)
    dy = rng.randn(*y.shape).astype(np.float32)
    y.backward(cuda(dy))
    v = G.conv_vjp(np_(x), np_(w[s + "/weights"]), np_(y), dy, 2, True)
    assert rel(np_(x.grad), v.dx) <= BAR
    check_wgrad("layers.conv dw", np_(w[s + "/weights"].grad), v.dw, v.dw_abs)
    check_wgrad("layers.conv db", np_(w[s + "/biases"].grad), v.db, v.db_abs)
    with torch.no_grad():
        assert torch.equal(layers.conv(x, 16, 3, stride=2, scope=s, weights=w), y)
    xf = cuda(rng.rand(3, 64), True)
    yf = layers.fc(xf, 32, scope=f, weights=w, activation_fn=None)
    dyf = rng.randn(3, 32).astype(np.float32)
    yf.backward(cuda(dyf))
    v = G.fc_vjp(np_(xf), np_(w[f + "/weights"]), np_(yf), dyf, False)
    assert rel(np_(xf.grad), v.dx) <= BAR
    check_wgrad("layers.fc dw", np_(w[f + "/weights"].grad), v.dw, v.dw_abs)
    # numpy weights next to a bias tensor that requires grad: the bias is used as it is and gets its gradient
    mixed = {k: np_(t) if k.endswith("/weights") else cuda(np_(t), True) for k, t in w.items()}
    y = layers.conv(x.detach(), 16, 3, stride=2, scope=s, weights=mixed)
    y.backward(cuda(dy))
    v = G.conv_vjp(np_(x), mixed[s + "/weights"], np_(y), dy, 2, True)
    check_wgrad("layers.conv db, numpy weights", np_(mixed[s + "/biases"].grad), v.db, v.db_abs)
    yf = layers.fc(xf.detach(), 32, scope=f, weights=mixed, activation_fn=None)
    yf.backward(cuda(dyf))
    v = G.fc_vjp(np_(xf), mixed[f + "/weights"], np_(yf), dyf, False)
    check_wgrad("layers.fc db, numpy weights", np_(mixed[f + "/biases"].grad), v.db, v.db_abs)


@pytest.mark.parametrize("model", [models.HDRNetCurves, models.HDRNetPointwiseNNGuide])
def test_nothing_stale_and_inference_equals_the_differentiable_forward(model, monkeypatch):
    params = dict(SMALL, model_name=model.__name__)
    wts = tensor_weights(params, model_name=model.__name__)
    _, low, full = small_setup(B=3)
    monkeypatch.setattr(models, "CHAIN_CNN_MAX_BATCH", 0)        # the per-layer inference path
    # output pixels per image of every conv layer (SAME padding halves the extent at stride 2)
    S, n_ds = params["net_input_size"], int(np.log2(params["net_input_size"] / params["spatial_bin"]))
    side = {f"{P}/splat/conv{i + 1}": S >> (i + 1) for i in range(n_ds)}
    side.update({f"{P}/global/conv1": S >> (n_ds + 1), f"{P}/global/conv2": S >> (n_ds + 2),
                 f"{P}/local/conv1": S >> n_ds, f"{P}/local/conv2": S >> n_ds})
    px = {s: n * n for s, n in side.items()}
    packable = [s for s in px if models.pack_conv_weights(wts[s + "/weights"].detach()) is not None]
    packed_px = models.PACKED_CONV_MIN_TILES * 128                # tiles of 128 output pixels
    assert 3 * max(px.values()) < packed_px                       # batch 3: CUDA-core convs only
    packed_batch = -(-packed_px // max(px[s] for s in packable))  # the largest packable layer runs packed
    for B in (3, packed_batch):
        low_b = small_setup(B=B)[1]
        grid = model._coefficients(low_b, dict(params, weights=wts))
        assert grid.requires_grad
        with torch.no_grad():
            assert torch.equal(model._coefficients(low_b, dict(params, weights=wts)), grid)
    with torch.no_grad():
        before = model.inference(low, full, dict(params, weights=wts)).clone()
    opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-2)
    out = model.inference(low, full, dict(params, weights=wts))
    assert rel(np_(out), np_(before)) <= 1e-6
    out.square().sum().backward()
    opt.step()
    with torch.no_grad():
        after = model.inference(low, full, dict(params, weights=wts))
        fresh = model.inference(low, full, dict(params, weights={k: v.detach().clone() for k, v in wts.items()}))
    assert not torch.equal(after, before)
    assert torch.equal(after, fresh)
    # the guide variables are read on every call too
    g = "inference/guide/ccm" if model is models.HDRNetCurves else "inference/guide/conv2/biases"
    with torch.no_grad():
        wts[g].add_(0.05)
        moved = model.inference(low, full, dict(params, weights=wts))
        fresh = model.inference(low, full, dict(params, weights={k: v.detach().clone() for k, v in wts.items()}))
    assert torch.equal(moved, fresh) and not torch.equal(moved, after)


def test_pyramid_coefficients_are_differentiable():
    params = dict(SMALL, model_name="HDRNetGaussianPyrNN")
    wts = tensor_weights(params, model_name="HDRNetGaussianPyrNN")
    rng, low, _ = small_setup()
    grid = models.HDRNetGaussianPyrNN._coefficients(low, dict(params, weights=wts))
    assert grid.shape[-2:] == (9, 4)
    dgrid = rng.randn(*grid.shape).astype(np.float32)
    grid.backward(cuda(dgrid))
    net = G.Network({k: np_(v) for k, v in wts.items()}, params, n_out=9)
    net.forward(np_(low))
    want = net.backward(dgrid)
    for k in G.variable_names(params):
        assert rel(np_(wts[k].grad), want[k]) <= BAR, k


def test_teacher_student_fit_converges():
    """Same architecture; teacher weights init_weights(seed=1), student seed 0, the guide fixed
    (the teacher's); Adam at train.py's learning rate 1e-4 (hdrnet/bin/train.py:199), 300 steps on
    one batch of 4 at 64² network input, 128² output."""
    params = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8)
    teacher = {k: torch.from_numpy(v).cuda() for k, v in models.init_weights(params, seed=1).items()}
    student = {k: (torch.from_numpy(v).cuda() if k.startswith(P) else teacher[k]).requires_grad_(k.startswith(P))
               for k, v in models.init_weights(params, seed=0).items()}
    rng = np.random.RandomState(6)
    full = cuda(rng.rand(4, 128, 128, 3))
    low = cuda(np_(full)[:, ::2, ::2])
    with torch.no_grad():
        target = models.HDRNetCurves.inference(low, full, dict(params, weights=teacher))
    opt = torch.optim.Adam([v for v in student.values() if v.requires_grad], lr=1e-4)
    losses = []
    for _ in range(300):
        opt.zero_grad()
        loss = ((models.HDRNetCurves.inference(low, full, dict(params, weights=student)) - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    report("teacher-student", first=losses[0], at100=losses[99], at200=losses[199], last=losses[-1],
           factor=losses[0] / losses[-1])
    # measured on an H100: 10.9 -> 1.01 (step 100) -> 0.50 (200) -> 0.325 (300), a factor of 34;
    # the bar asks for 10
    assert np.isfinite(losses).all()
    assert losses[-1] <= losses[0] / 10.0
