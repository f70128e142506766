"""Model-side tests (coefficient CNN, guides, HDRNet* graphs).

CPU part: host logic only (weight naming / shapes / batch-norm folding / error paths).
GPU part (-m gpu): the CUDA layers and the full models against oracle/model_np.py, the
float64-accumulated numpy restatement of hdrnet/models.py + layers.py, which is pinned by an
independent torch restatement and hand-computed known answers (tests/test_model_kats.py; the
reference has no test or golden vector for models.py and TF cannot run here).

How the 1e-5 bar of BASELINE.json is applied to a whole model: stage by stage.
  * coefficient CNN vs oracle: 2e-5 of range (9-11 float32 layers deep);
  * guide vs oracle: 2e-6 absolute on [0, 1];
  * full-resolution stage: the CUDA output against the pinned SLICE oracle (the compiled reference
    loops) fed the CUDA stage's own coefficients and guide -- 1e-5, the bar itself.  This separates
    the kernel's error from the sensitivity of the op to its inputs (a guide that differs by 1e-7
    moves a pixel's depth coordinate by gd * 1e-7, which alone can exceed 1e-5 of the output);
  * end to end vs the all-oracle pipeline: 1e-4, as a sanity bound on that sensitivity.
"""
import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import _lib, models
from oracle import model_np as M
from util import assert_parity, rel_err

PARAM_SETS = {
    "default": dict(M.DEFAULT_PARAMS),
    "bn_small": dict(M.DEFAULT_PARAMS, batch_norm=True, net_input_size=64, spatial_bin=8, luma_bins=4),
    "cm2": dict(M.DEFAULT_PARAMS, channel_multiplier=2, net_input_size=128, spatial_bin=16),
    "nn_guide": dict(M.DEFAULT_PARAMS, model_name="HDRNetPointwiseNNGuide", batch_norm=True,
                     net_input_size=128, spatial_bin=16),
    "pyramid": dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=128,
                    spatial_bin=16),
}


# ---- CPU: host logic ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_init_weights_has_reference_variable_names_and_shapes(name):
    p = PARAM_SETS[name]
    ours = models.init_weights(p, seed=0)
    ref = M.make_weights(p, seed=0)
    assert sorted(ours) == sorted(ref)
    for k in ref:
        assert np.asarray(ours[k]).shape == np.asarray(ref[k]).shape, k
    assert "inference/coefficients/splat/conv1/weights" in ours       # run.py:92 scope
    n = sum(np.asarray(v).size for v in ours.values())
    if name == "default":
        assert n == 482080                                            # SURVEY 2b: ~482 k params


def test_model_surface_mirrors_reference():
    assert models.HDRNetGaussianPyrNN.n_out() == 9 and models.HDRNetGaussianPyrNN.n_scales() == 3
    for cls in (models.HDRNetCurves, models.HDRNetPointwiseNNGuide):     # models.py:23-27
        assert cls.n_out() == 3 and cls.n_in() == 4
        for m in ("inference", "_coefficients", "_guide", "_output"):
            assert callable(getattr(cls, m))
    assert getattr(models, "HDRNetCurves") is models.HDRNetCurves      # run.py:82-85 lookup


def test_batch_norm_fold_matches_inference_formula():
    rng = np.random.RandomState(0)
    wts = {"s/weights": rng.randn(3, 3, 4, 5).astype(np.float32),
           "s/BatchNorm/beta": rng.randn(5).astype(np.float32),
           "s/BatchNorm/moving_mean": rng.randn(5).astype(np.float32),
           "s/BatchNorm/moving_variance": (0.5 + rng.rand(5)).astype(np.float32)}
    w, b = models._fold(wts, "s", True, False)
    x = rng.randn(2, 6, 6, 4).astype(np.float32)
    direct = M.batch_norm_inference(M.conv2d_same(x, wts["s/weights"]), wts["s/BatchNorm/beta"],
                                    wts["s/BatchNorm/moving_mean"], wts["s/BatchNorm/moving_variance"])
    folded = M.conv2d_same(x, w) + b
    assert np.abs(direct - folded).max() < 1e-5


def test_inference_without_weights_or_gpu_fails_loudly():
    p = dict(M.DEFAULT_PARAMS)
    models._weights = None
    x = torch.zeros(1, 256, 256, 3)
    with pytest.raises((ValueError, _lib.HdrnetLibraryError)):
        models.HDRNetCurves.inference(x, x, p)
    with pytest.raises(NotImplementedError):
        models.HDRNetCurves.inference(x, x, p, is_training=True)


# ---- GPU -----------------------------------------------------------------------------------------
def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,cin,cout,k,stride,relu,bias", [
    (2, 256, 256, 3, 8, 3, 2, True, True),     # splat conv1 (models.py:69-82)
    (2, 32, 32, 32, 64, 3, 2, True, True),     # splat conv4
    (3, 16, 16, 64, 64, 3, 1, False, False),   # local conv2: no bias, no activation (:116-117)
    (2, 16, 16, 64, 96, 1, 1, False, True),    # 1x1 prediction
    (1, 7, 5, 5, 3, 3, 2, True, True),         # odd extents: SAME pad 1 before / 1 after
    (1, 9, 6, 130, 70, 3, 1, True, True),      # Cin > chunk, Cout not a multiple of the tile
])
def test_conv2d_matches_tf_same_semantics(B, H, W, cin, cout, k, stride, relu, bias):
    rng = np.random.RandomState(1)
    x = rng.randn(B, H, W, cin).astype(np.float32)
    w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.randn(cout).astype(np.float32) if bias else None
    ref = M.conv2d_same(x, w, stride) + (0 if b is None else b)
    if relu:
        ref = np.maximum(ref, 0)
    got = models._conv(cuda(x), (cuda(w), None if b is None else cuda(b)), stride=stride, relu=relu)
    assert_parity(got.cpu().numpy(), ref.astype(np.float32), rtol=2e-6)  # fp32 sum over <= 1170 terms


@pytest.mark.gpu
@pytest.mark.parametrize("B,I,O,relu", [(8, 1024, 256, True), (3, 256, 128, True), (1, 128, 64, False),
                                        (11, 70, 37, True)])
def test_fc_matches(B, I, O, relu):
    rng = np.random.RandomState(2)
    x = rng.randn(B, I).astype(np.float32)
    w = (rng.randn(I, O) / np.sqrt(I)).astype(np.float32)
    b = rng.randn(O).astype(np.float32)
    ref = x.astype(np.float64) @ w.astype(np.float64) + b
    if relu:
        ref = np.maximum(ref, 0)
    got = models._fc(cuda(x), (cuda(w), cuda(b)), relu=relu)
    assert_parity(got.cpu().numpy(), ref.astype(np.float32), rtol=2e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_norm,use_bias,stride,act", [(False, True, 2, "relu"), (True, True, 1, "relu"),
                                                            (False, False, 1, None), (False, True, 1, "tanh")])
def test_layers_conv_and_fc_follow_the_reference_constructors(batch_norm, use_bias, stride, act):
    """hdrnet/layers.py:25-93 through the public layers.conv / layers.fc: variables found under
    `scope` by the reference's names, batch norm (center, no scale) instead of the bias, SAME
    padding, fused relu / no activation / an arbitrary activation applied on the output."""
    from hdrnet_b200 import layers
    rng = np.random.RandomState(5)
    wts = {"net/c/weights": (rng.randn(3, 3, 6, 12) / 7).astype(np.float32),
           "net/c/biases": rng.randn(12).astype(np.float32),
           "net/c/BatchNorm/beta": rng.randn(12).astype(np.float32),
           "net/c/BatchNorm/moving_mean": rng.randn(12).astype(np.float32),
           "net/c/BatchNorm/moving_variance": (0.5 + rng.rand(12)).astype(np.float32),
           "net/f/weights": (rng.randn(40, 10) / 6).astype(np.float32),
           "net/f/biases": rng.randn(10).astype(np.float32),
           "net/f/BatchNorm/beta": rng.randn(10).astype(np.float32),
           "net/f/BatchNorm/moving_mean": rng.randn(10).astype(np.float32),
           "net/f/BatchNorm/moving_variance": (0.5 + rng.rand(10)).astype(np.float32)}
    fn = {"relu": layers.relu, None: None, "tanh": torch.tanh}[act]
    post = (lambda a: a) if act != "tanh" else np.tanh
    x = rng.randn(2, 9, 14, 6).astype(np.float32)
    got = layers.conv(cuda(x), 12, 3, stride=stride, use_bias=use_bias, batch_norm=batch_norm,
                      activation_fn=fn, scope="net/c", weights=wts)
    ref = post(M.conv(x, wts, "net/c", stride=stride, use_bias=use_bias, batch_norm=batch_norm, relu=act == "relu"))
    assert_parity(got.cpu().numpy(), ref.astype(np.float32), rtol=2e-6)
    v = rng.randn(5, 40).astype(np.float32)
    got = layers.fc(cuda(v), 10, use_bias=use_bias, batch_norm=batch_norm, activation_fn=fn, scope="net/f", weights=wts)
    ref = post(M.fc(v, wts, "net/f", use_bias=use_bias, batch_norm=batch_norm, relu=act == "relu"))
    assert_parity(got.cpu().numpy(), ref.astype(np.float32), rtol=2e-6)
    with pytest.raises(ValueError):
        layers.conv(cuda(x), 16, 3, scope="net/c", weights=wts)          # num_outputs does not match the variables
    with pytest.raises(NotImplementedError):
        layers.conv(cuda(x), 12, 3, scope="net/c", weights=wts, is_training=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_coefficients_match_oracle(name):
    p = PARAM_SETS[name]
    wts = M.make_weights(p, seed=3)
    rng = np.random.RandomState(4)
    S = p["net_input_size"]
    low = rng.rand(3, S, S, 3).astype(np.float32)
    cls = getattr(models, p["model_name"])
    ref = M.coefficients(low, wts, p, n_out=cls.n_out())
    got = cls._coefficients(cuda(low), dict(p, weights=wts)).cpu().numpy()
    assert got.shape == ref.shape == (3, p["spatial_bin"], p["spatial_bin"], p["luma_bins"], cls.n_out(), 4)
    # 9-11 float32 layers deep; the oracle rounds each activation to float32 once
    assert_parity(got, ref, rtol=2e-5, what=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PARAM_SETS))
@pytest.mark.parametrize("B", [1, 4])
def test_coefficients_chain_and_per_layer_paths_agree(name, B, monkeypatch):
    """Small batches run the whole network behind one library call (hdrnet_coefficients_f32: launch
    chain with paired branches and the fc cluster chain), larger ones layer by layer: both against
    the oracle, and against each other (float32 round-off: the reductions are split differently)."""
    p = PARAM_SETS[name]
    wts = M.make_weights(p, seed=3)
    S = p["net_input_size"]
    low = np.random.RandomState(40 + B).rand(B, S, S, 3).astype(np.float32)
    cls = getattr(models, p["model_name"])
    ref = M.coefficients(low, wts, p, n_out=cls.n_out())
    lib = _lib.load()
    assert lib.hdrnet_coefficients_scratch_bytes(B, S, p["spatial_bin"], p["luma_bins"], p["channel_multiplier"],
                                                 cls.n_out(), cls.n_in()) > 0
    monkeypatch.setattr(models, "CHAIN_CNN_MAX_BATCH", 64)
    one = cls._coefficients(cuda(low), dict(p, weights=wts)).cpu().numpy()
    monkeypatch.setattr(models, "CHAIN_CNN_MAX_BATCH", 0)
    many = cls._coefficients(cuda(low), dict(p, weights=wts)).cpu().numpy()
    assert_parity(one, ref, rtol=2e-5, what=f"{name} chain", elem_rtol=None)
    assert_parity(many, ref, rtol=2e-5, what=f"{name} per layer", elem_rtol=None)
    assert_parity(one, many, rtol=5e-6, what=f"{name} chain vs per layer", elem_rtol=None)


@pytest.mark.gpu
def test_coefficient_chain_argument_checks_and_odd_channel_counts(monkeypatch):
    lib = _lib.load()
    assert lib.hdrnet_coefficients_scratch_bytes(1, 240, 16, 8, 1, 3, 4) == 0      # 240 / 16 not a power of two
    assert lib.hdrnet_coefficients_scratch_bytes(0, 256, 16, 8, 1, 3, 4) == 0
    assert lib.hdrnet_coefficients_scratch_bytes(1, 256, 16, 8, 1, 3, 4) > 0
    z = torch.zeros(64, device="cuda")
    import ctypes
    arr = (ctypes.c_void_p * 12)(*([z.data_ptr()] * 12))
    rc = lib.hdrnet_coefficients_f32(z.data_ptr(), z.data_ptr(), arr, arr, 12, z.data_ptr(), 256, 1, 240, 16, 8, 1, 3, 4, 0)
    assert rc == _lib.E_UNSUPPORTED
    rc = lib.hdrnet_coefficients_f32(z.data_ptr(), z.data_ptr(), arr, arr, 11, z.data_ptr(), 1 << 30, 1, 256, 16, 8, 1, 3, 4, 0)
    assert rc == _lib.E_BAD_SHAPE                                                  # n_layers must be n_ds + 8
    rc = lib.hdrnet_coefficients_f32(z.data_ptr(), z.data_ptr(), arr, arr, 12, z.data_ptr(), 256, 1, 256, 16, 8, 1, 3, 4, 0)
    assert rc == _lib.E_BAD_SHAPE                                                  # scratch too small
    # 6 depth bins: channel counts 6 / 12 / 24 / 48 -- not multiples of 4 early on, fc widths not
    # powers of two: the chain falls back layer by layer to the general kernels, same result
    p = dict(M.DEFAULT_PARAMS, luma_bins=6, net_input_size=64, spatial_bin=16)
    wts = M.make_weights(p, seed=1)
    low = np.random.RandomState(2).rand(1, 64, 64, 3).astype(np.float32)
    for mb in (64, 0):
        monkeypatch.setattr(models, "CHAIN_CNN_MAX_BATCH", mb)
        got = models.HDRNetCurves._coefficients(cuda(low), dict(p, weights=wts)).cpu().numpy()
        assert_parity(got, M.coefficients(low, wts, p), rtol=2e-5, elem_rtol=None, what=f"chain max batch {mb}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,cin,cout,stride,relu,bias", [
    (1, 16, 64, 64, 1, True, True),      # local conv1 at batch 1: 4 output channels per CTA
    (2, 16, 64, 64, 1, False, False),    # local conv2 at batch 2: 8 per CTA
    (1, 16, 64, 64, 2, True, True),      # global conv1
    (1, 8, 64, 64, 2, True, True),       # global conv2: 16 pixels, half a tile
    (1, 128, 8, 16, 2, True, True),      # splat conv2: 2 chunks per tap
    (3, 9, 12, 20, 2, True, True),       # odd extents (asymmetric SAME pads), 3 chunks per tap, Cout % 8 != 0
    (1, 7, 4, 4, 1, False, True),        # one chunk per tap, one channel group
])
def test_small_conv_layers_patch_form_against_oracle(B, H, cin, cout, stride, relu, bias):
    """conv2d_patch_kernel (the shared-memory patch form AUTO takes for small layers, csrc/cnn.cu)
    against the float64-accumulating oracle conv (hdrnet/layers.py:25-59 semantics)."""
    rng = np.random.RandomState(B * 100 + H)
    x = rng.randn(B, H, H, cin).astype(np.float32)
    w = (rng.randn(3, 3, cin, cout) * 0.2).astype(np.float32)
    b = rng.randn(cout).astype(np.float32) if bias else None
    ref = M.conv2d_same(x, w, stride) + (0 if b is None else b)
    if relu:
        ref = np.maximum(ref, 0)
    got = models._conv(cuda(x), (cuda(w), None if b is None else cuda(b)), stride=stride, relu=relu).cpu().numpy()
    assert_parity(got, ref.astype(np.float32), rtol=5e-6, elem_rtol=None)


@pytest.mark.gpu
def test_guides_match_oracle():
    rng = np.random.RandomState(5)
    full = rng.rand(2, 37, 53, 3).astype(np.float32)        # odd size: scalar tail path too
    p = PARAM_SETS["default"]
    wts = M.make_weights(p, seed=6)
    g = models.HDRNetCurves._guide(cuda(full), dict(p, weights=wts)).cpu().numpy()
    assert np.abs(g - M.guide_curves(full, wts)).max() < 2e-6
    p = PARAM_SETS["nn_guide"]
    wts = M.make_weights(p, seed=7)
    g = models.HDRNetPointwiseNNGuide._guide(cuda(full), dict(p, weights=wts)).cpu().numpy()
    assert np.abs(g - M.guide_nn(full, wts)).max() < 2e-6
    full = rng.rand(1, 64, 256, 3).astype(np.float32)       # vector path
    g = models.HDRNetPointwiseNNGuide._guide(cuda(full), dict(p, weights=wts)).cpu().numpy()
    assert np.abs(g - M.guide_nn(full, wts)).max() < 2e-6


@pytest.mark.gpu
@pytest.mark.parametrize("name,H,W", [("default", 270, 480), ("nn_guide", 96, 256), ("bn_small", 33, 50),
                                      ("default", 64, 1920)])
def test_full_inference_matches_oracle(name, H, W):
    """models.py:43-59 end to end: lowres -> coefficients, fullres -> guide -> fused slice-apply
    (guide never materialised when W suits the fused kernel), vs the numpy oracle + the slice
    oracle.  1e-4 relative: the guide is recomputed in float32 inside the kernel, and a guide
    difference of 1e-7 moves a pixel's depth coordinate by gd * 1e-7."""
    p = PARAM_SETS[name]
    wts = M.make_weights(p, seed=8)
    rng = np.random.RandomState(9)
    S = p["net_input_size"]
    low = rng.rand(2, S, S, 3).astype(np.float32)
    full = rng.rand(2, H, W, 3).astype(np.float32)
    ref, ref_coeffs, ref_guide = M.inference(low, full, wts, p, oracle.best().bilateral_slice_apply)
    cls = getattr(models, p["model_name"])
    got = cls.inference(cuda(low), cuda(full), dict(p, weights=wts, debug=True))
    assert_parity(got.cpu().numpy(), ref, rtol=1e-4, what=f"{name} output", elem_rtol=None)
    dbg = cls.last_debug
    assert_parity(dbg["bilateral_coefficients"].cpu().numpy(), ref_coeffs, rtol=2e-5, elem_rtol=None)
    assert np.abs(dbg["guide"].cpu().numpy() - ref_guide).max() < 2e-6
    # the full-resolution stage itself, at the bar: pinned slice oracle on the CUDA stage's inputs
    c = dbg["bilateral_coefficients"].cpu().numpy()
    stage = oracle.best().bilateral_slice_apply(np.ascontiguousarray(c.reshape(c.shape[:4] + (12,))),
                                                dbg["guide"].cpu().numpy(), full, True)
    assert_parity(got.cpu().numpy(), stage, rtol=1e-5, what=f"{name} full-resolution stage")
    # same call without the debug dump takes the guide-fused kernel when W allows it
    got2 = cls.inference(cuda(low), cuda(full), dict(p, weights=wts))
    assert torch.equal(got2, got)


# ---- run.py pre/post (row a11) -----------------------------------------------------------------
def test_run_py_host_preprocessing():
    from hdrnet_b200.bin import run
    u8 = np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3)
    assert run.img_as_float(u8).dtype == np.float32 and run.img_as_float(u8).max() == np.float32(17 / 255)
    assert run.img_as_float(np.array([[65535]], np.uint16))[0, 0] == 1.0
    im = np.arange(8 * 6 * 3, dtype=np.float32).reshape(8, 6, 3)
    low = run.nearest_resize(im, 4)
    assert low.shape == (4, 4, 3)
    assert np.array_equal(low[:, :, 0], im[[1, 3, 5, 7]][:, [0, 2, 3, 5], 0])   # centres of 2x1.5 boxes


@pytest.mark.gpu
def test_run_py_identity_sample_plumbing(tmp_path):
    """BASELINE.json config 1 (plumbing): default-initialised model on a 256x256 image through
    the CLI's process(): checkpoint round trip, u8 -> float, nearest lowres, model, u8 out; and
    the float output equals the oracle's."""
    from hdrnet_b200.bin import run
    p = dict(M.DEFAULT_PARAMS)
    wts = models.init_weights(p, seed=0)
    run.save_checkpoint(str(tmp_path), p, wts)
    params, loaded = run.load_checkpoint(str(tmp_path))
    assert sorted(loaded) == sorted(wts) and params["model_name"] == "HDRNetCurves"
    rng = np.random.RandomState(0)
    im8 = rng.randint(0, 256, size=(256, 256, 3)).astype(np.uint8)
    out8, _ = run.process(models.HDRNetCurves, params, im8)
    assert out8.shape == (256, 256, 3) and out8.dtype == np.uint8
    out = models.HDRNetCurves.inference_image(torch.from_numpy(im8[None]).cuda(), params,
                                              out_dtype=torch.float32)
    im = run.img_as_float(im8)[None]
    low = run.nearest_resize(im[0], 256)[None]
    ref, _, _ = M.inference(low, im, loaded, params, oracle.best().bilateral_slice_apply)
    assert_parity(out.cpu().numpy(), ref, rtol=1e-4, elem_rtol=None)
    ref8 = (255.0 * np.clip(ref, 0, 1)).astype(np.uint8)[0]
    assert np.abs(out8.astype(int) - ref8.astype(int)).max() <= 1


# ---- tensor-core (wgmma, 3xTF32) forms of the conv layers --------------------------------------
def conv_case(rng, B, H, W, cin, cout, k, stride, relu, bias):
    x = rng.randn(B, H, W, cin).astype(np.float32)
    w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.randn(cout).astype(np.float32) if bias else None
    ref = M.conv2d_same(x, w, stride) + (0 if b is None else b)
    return x, w, b, (np.maximum(ref, 0) if relu else ref).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,cin,cout,k,stride,relu,bias", [
    (8, 16, 16, 64, 64, 3, 1, True, True),     # local conv1 (models.py:109-113)
    (1, 16, 16, 64, 64, 3, 1, False, False),   # local conv2 at batch 1: 2 tiles
    (2, 32, 32, 32, 64, 3, 2, True, True),     # splat conv4, stride 2, SAME pad 0/1
    (1, 16, 16, 64, 64, 3, 2, True, True),     # global conv1: half a tile
    (1, 8, 8, 64, 64, 3, 2, True, True),       # global conv2: 16 px
    (3, 16, 16, 64, 96, 1, 1, False, True),    # 1x1 prediction, N = 96
    (1, 9, 7, 8, 16, 3, 1, True, True),        # ragged tile (63 px), K = 72 (partial last chunk)
    (1, 16, 16, 64, 192, 3, 1, True, True),    # Cout > 128: two launches over columns 0-127, 128-191
    (2, 12, 12, 32, 144, 3, 2, False, True),   # Cout = 128 + 16, stride 2
])
def test_conv2d_wgmma_matches_oracle(B, H, W, cin, cout, k, stride, relu, bias):
    """3xTF32 on the tensor cores keeps float32-grade accuracy: 1e-5 of the tensor's range (a plain
    TF32 product would be ~1e-3).  The packed form (pre-packed hi/lo weight tiles, 3-stage ring, one
    TMA copy per chunk) through its entry point at the case's own shape; the unpacked form, which
    hdrnet_conv2d_nhwc_f32 takes from 96 tiles of 128 output pixels, at the batch that reaches them."""
    lib = _lib.load()
    rng = np.random.RandomState(11)
    oh, ow = -(-H // stride), -(-W // stride)
    if cout <= 128:
        x, w, b, ref = conv_case(rng, B, H, W, cin, cout, k, stride, relu, bias)
        wd, bd, xd = cuda(w), None if b is None else cuda(b), cuda(x)
        packed = models.pack_conv_weights(wd)
        assert packed is not None
        out = torch.empty((B, oh, ow, cout), device="cuda")
        _lib.check(lib.hdrnet_conv2d_nhwc_tc_f32(xd.data_ptr(), packed.data_ptr(), 0 if bd is None else bd.data_ptr(),
                                                 out.data_ptr(), B, H, W, cin, cout, k, stride, int(relu),
                                                 torch.cuda.current_stream().cuda_stream), "conv2d (packed)")
        assert_parity(out.cpu().numpy(), ref, rtol=1e-5, what="packed")
    nb = max(B, -(-96 * 128 // (oh * ow)))
    if (B * oh * ow) % 128 and not (nb * oh * ow) % 128:
        nb += 1                                                      # a ragged last tile stays ragged
    x, w, b, ref = conv_case(rng, nb, H, W, cin, cout, k, stride, relu, bias)
    got = models._conv(cuda(x), (cuda(w), None if b is None else cuda(b)), stride=stride, relu=relu)
    assert_parity(got.cpu().numpy(), ref, rtol=1e-5, what=f"unpacked at batch {nb}")


@pytest.mark.gpu
def test_coefficients_with_wgmma_convs():
    """Layer by layer at batch 32: every packable layer of the default network but the two global
    convs (test_conv2d_wgmma_matches_oracle has their shapes) has >= 64 tiles, so runs packed."""
    B = 32
    assert B > models.CHAIN_CNN_MAX_BATCH
    p = PARAM_SETS["default"]
    wts = M.make_weights(p, seed=3)
    low = np.random.RandomState(4).rand(B, 256, 256, 3).astype(np.float32)
    ref = M.coefficients(low, wts, p)
    got = models.HDRNetCurves._coefficients(cuda(low), dict(p, weights=wts)).cpu().numpy()
    assert_parity(got, ref, rtol=5e-5, what="coefficients via tensor-core convs")


# ---- HDRNetGaussianPyrNN (row f-2) -------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,oh,ow", [(2, 64, 96, 32, 48), (1, 33, 50, 16, 25), (1, 16, 24, 33, 50),
                                         (1, 5, 7, 1, 1)])
def test_resize_bilinear_align_corners(B, H, W, oh, ow):
    x = np.random.RandomState(0).rand(B, H, W, 3).astype(np.float32)
    got = models._resize(cuda(x), oh, ow).cpu().numpy()
    assert np.abs(got - M.resize_bilinear_ac(x, oh, ow)).max() < 2e-6
    add = np.random.RandomState(1).rand(B, oh, ow, 3).astype(np.float32)
    got = models._resize(cuda(x), oh, ow, add=cuda(add)).cpu().numpy()
    assert np.abs(got - (M.resize_bilinear_ac(x, oh, ow) + add)).max() < 2e-6


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(256, 512), (70, 90)])
def test_gaussian_pyramid_model_matches_oracle(H, W):
    """models.py:213-289: pyramid, per-level NN guides, per-level slice-apply on rows
    il*3..il*3+2 of the 9-row grid (coarsest first), upsample-add."""
    p = PARAM_SETS["pyramid"]
    wts = M.make_weights(p, seed=12)
    rng = np.random.RandomState(13)
    low = rng.rand(2, p["net_input_size"], p["net_input_size"], 3).astype(np.float32)
    full = rng.rand(2, H, W, 3).astype(np.float32)
    ref, ref_coeffs, ref_guides = M.gaussian_pyr_inference(low, full, wts, p,
                                                           oracle.best().bilateral_slice_apply)
    got = models.HDRNetGaussianPyrNN.inference(cuda(low), cuda(full), dict(p, weights=wts, debug=True))
    assert_parity(got.cpu().numpy(), ref, rtol=1e-4, what="pyramid output", elem_rtol=None)
    dbg = models.HDRNetGaussianPyrNN.last_debug
    assert_parity(dbg["bilateral_coefficients"].cpu().numpy(), ref_coeffs, rtol=2e-5, elem_rtol=None)
    for g, r in zip(dbg["guide"], ref_guides):
        assert np.abs(g.cpu().numpy() - r).max() < 2e-6
    fast = models.HDRNetGaussianPyrNN.inference(cuda(low), cuda(full), dict(p, weights=wts))
    assert_parity(fast.cpu().numpy(), ref, rtol=1e-4, what="pyramid output (guide-fused)", elem_rtol=None)
    # the full-resolution stages at the bar: the oracle's own pyramid / upsample-add around the
    # pinned slice oracle, fed the CUDA stage's coefficients and per-level guides
    c = dbg["bilateral_coefficients"].cpu().numpy()
    lvls = [full]
    for _ in range(2):
        lvls.append(M.resize_bilinear_ac(lvls[-1], lvls[-1].shape[1] // 2, lvls[-1].shape[2] // 2))
    cur = None
    for il in range(3):
        src = 2 - il
        ci = np.ascontiguousarray(c[:, :, :, :, il * 3:(il + 1) * 3, :]).reshape(c.shape[:4] + (12,))
        o = oracle.best().bilateral_slice_apply(ci, dbg["guide"][src].cpu().numpy(), lvls[src], True)
        cur = o if il == 0 else M.resize_bilinear_ac(cur, o.shape[1], o.shape[2]) + o
    assert_parity(got.cpu().numpy(), cur, rtol=1e-5, what="pyramid full-resolution stages", elem_rtol=None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["default", "nn_guide"])
def test_full_inference_large_image_takes_texture_assisted_kernel(name):
    """>= 2 Mi pixels: models.inference lends a workspace and the library runs the
    texture-assisted guide-fused kernel; same oracle, same tolerance."""
    p = PARAM_SETS[name]
    wts = M.make_weights(p, seed=21)
    rng = np.random.RandomState(22)
    S = p["net_input_size"]
    low = rng.rand(1, S, S, 3).astype(np.float32)
    full = rng.rand(1, 1024, 2048, 3).astype(np.float32)
    ref, _, _ = M.inference(low, full, wts, p, oracle.best().bilateral_slice_apply)
    cls = getattr(models, p["model_name"])
    got = cls.inference(cuda(low), cuda(full), dict(p, weights=wts))
    assert_parity(got.cpu().numpy(), ref, rtol=1e-4, what=f"{name} 2 MP output", elem_rtol=None)


@pytest.mark.gpu
def test_fuse_predict_with_weights_larger_than_shared_memory():
    """ADVICE r01: HDRNetGaussianPyrNN at channel_multiplier 4 (scripts/*/train_gpyrnn_cm4.sh) has
    a 256 x 288 prediction conv (295 KB): the fused fusion + prediction + unroll kernel must read
    the weights through the cache instead of refusing the model."""
    rng = np.random.RandomState(3)
    B, gh, gw, C, gd, n_out, n_in = 2, 4, 4, 256, 8, 9, 4
    O = gd * n_out * n_in
    loc = rng.randn(B, gh, gw, C).astype(np.float32)
    glob = rng.randn(B, C).astype(np.float32)
    w = (rng.randn(C, O) / np.sqrt(C)).astype(np.float32)
    b = rng.randn(O).astype(np.float32)
    out = torch.empty(B, gh, gw, gd, n_out, n_in, device="cuda")
    d_loc, d_glob, d_w, d_b = cuda(loc), cuda(glob), cuda(w), cuda(b)     # keep the device buffers alive
    rc = _lib.load().hdrnet_fuse_predict_f32(d_loc.data_ptr(), d_glob.data_ptr(), d_w.data_ptr(),
                                             d_b.data_ptr(), out.data_ptr(), B, gh, gw, C, gd, n_out, n_in,
                                             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0
    f = np.maximum(loc + glob[:, None, None, :], 0).astype(np.float64)
    pred = f @ w.astype(np.float64) + b                                   # [B, gh, gw, O], o = (j*n_out + i)*gd + z
    ref = pred.reshape(B, gh, gw, n_in, n_out, gd).transpose(0, 1, 2, 5, 4, 3)
    assert_parity(out.cpu().numpy(), ref.astype(np.float32), rtol=2e-6)
